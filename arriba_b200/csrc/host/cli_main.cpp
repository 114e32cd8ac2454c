// cli_main.cpp -- the `arriba` command line of arriba-b200: same option letters, defaults and error texts as the reference
// (options.cpp:270-485, usage options.cpp:109-268), driving the pipeline through the public C ABI only.
// Not supported (fail loudly): -G.
#include <getopt.h>
#include <unistd.h>
#include <sys/resource.h>
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <climits>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <iomanip>
#include <iostream>
#include <map>
#include <sstream>
#include <string>
#include <thread>
#include "../../../include/arriba_b200.h"

static void crash(bool condition, const std::string& message) { if (condition) { std::cerr << "ERROR: " << message << std::endl; exit(1); } }
static std::string stamp() { time_t now = time(0); char b[100]; strftime(b, sizeof(b), "[%Y-%m-%dT%X]", localtime(&now)); return b; }

static bool to_int(const char* s, long& v) { char* e; v = strtol(s, &e, 10); return *s != ' ' && e != s && *e == '\0' && v != LONG_MAX && v != LONG_MIN; }
static bool to_float(const char* s, float& v) { char* e; v = strtof(s, &e); return *s != ' ' && e != s && *e == '\0' && v != HUGE_VALF && v != -HUGE_VALF; }
static bool int_in(const char* s, long lo, long hi, long& v) { return to_int(s, v) && v >= lo && v <= hi; }
static bool float_in(const char* s, float lo, float hi, float& v) { return to_float(s, v) && v >= lo && v <= hi; }

static const char* FILTERS[] = {"", "duplicates", "inconsistently_clipped", "homopolymer", "read_through", "same_gene", "small_insert_size", "long_gap", "hairpin", "multimappers",
	"mismatches", "mismappers", "relative_support", "intronic", "non_coding_neighbors", "intragenic_exonic", "internal_tandem_duplication", "min_support", "known_fusions", "spliced",
	"blacklist", "end_to_end", "in_vitro", "merge_adjacent", "select_best", "marginal_read_through", "short_anchor", "no_coverage", "many_spliced", "no_genomic_support",
	"uninteresting_contigs", "viral_contigs", "top_expressed_viral_contigs", "low_coverage_viral_contigs", "genomic_support", "isoforms", "low_entropy", "homologs"};

static void usage() {
	std::cout << "arriba-b200: H100-native implementation of Arriba's post-alignment path (reference version 2.5.1 semantics)\n\n"
	          << "Usage: arriba [-c Chimeric.out.sam] -x Aligned.out.bam -g annotation.gtf -a assembly.fa -o fusions.tsv [-O fusions.discarded.tsv] [OPTIONS]\n\n"
	          << " -x FILE  BAM or SAM (plain or BGZF) with main and chimeric alignments (STAR --chimOutType WithinBAM); a pipe is read as it arrives:\n"
	          << "          STAR ... --outStd BAM_Unsorted --outBAMcompression 0 | arriba -x /dev/stdin ...\n"
	          << " -c FILE  chimeric alignments in a separate file (STAR --chimOutType SeparateSAMold: Chimeric.out.sam; SAM, BGZF SAM or BAM; a file or a pipe), read before -x\n"
	          << " -g FILE  gene annotation (GTF)\n -a FILE  assembly (FastA)\n"
	          << " -o FILE  output file   -O FILE  discarded candidates\n -f LIST  disable filters (comma/space separated)\n -s MODE  strandedness auto|yes|no|reverse\n"
	          << " -i/-v contig lists, -E e-value cutoff, -S min support, -m/-L/-H/-R/-A/-M/-K/-V/-F/-U/-Q/-e/-l/-z/-Z thresholds as in the reference\n"
	          << " -b FILE  blacklist (optionally .gz; required unless '-f blacklist')\n"
	          << " -k FILE  known fusions (optionally .gz)   -t FILE  tags (optionally .gz)\n"
	          << " -p FILE  protein domains (GFF3, optionally .gz)\n"
	          << " -d FILE  genomic breakpoints from whole-genome sequencing (four-column or VCF, optionally .gz)\n -D N     maximum genomic breakpoint distance (default 100000)\n"
	          << " -@ N     host threads for decoding and annotation   -u external duplicate marking   -X extra info for discarded candidates\n"
	          << " -I       fill gaps in the fusion_transcript column with the exons of the chosen transcripts (in the discarded file only with -X)\n";
}

int main(int argc, char** argv) {
	time_t start_time; time(&start_time);
	std::cout << stamp() << " Launching Arriba (arriba-b200, reference semantics 2.5.1)" << std::endl;
	arb_run_options o; arb_default_run_options(&o);
	o.echo_progress = 1;
	o.threads = (int) std::max(1u, std::min(32u, std::thread::hardware_concurrency()));
	crash(argc > 1 && (std::string(argv[1]).empty() || argv[1][0] != '-'), std::string("cannot interpret the first argument: ") + argv[1]);
	std::string bam, gtf, fasta, out, discarded, interesting, viral, blacklist, genomic, known_fusions, tags, protein_domains, chimeric;
	opterr = 0;
	const std::string valid = "c:x:d:g:G:o:O:t:p:a:b:k:s:i:v:f:E:S:m:L:H:D:R:A:M:K:V:F:U:Q:e:T:C:l:z:Z:@:uXIh";
	std::map<char, unsigned> seen; int c; long iv; bool threads_given = false;
	while ((c = getopt(argc, argv, valid.c_str())) != -1) {
		crash(++seen[(char) c] > 1, std::string("option -") + (char) c + " specified too often");
		const std::string opt = std::string("-") + (char) c;
		switch (c) {
			case 'x': bam = optarg; crash(access(optarg, R_OK), "file not found/readable: " + bam); break;
			case 'g': gtf = optarg; crash(access(optarg, R_OK), "file not found/readable: " + gtf); break;
			case 'a': fasta = optarg; crash(access(optarg, R_OK), "file not found/readable: " + fasta); break;
			case 'o': out = optarg; break;
			case 'O': discarded = optarg; break;
			case 'b': blacklist = optarg; crash(access(optarg, R_OK), "file not found/readable: " + blacklist); break;
			case 'd': genomic = optarg; crash(access(optarg, R_OK), "file not found/readable: " + genomic); break;
			case 'D': crash(!int_in(optarg, 0, INT_MAX, iv), "invalid argument to " + opt); o.max_genomic_breakpoint_distance = (uint32_t) iv; break;
			case 'k': known_fusions = optarg; crash(access(optarg, R_OK), "file not found/readable: " + known_fusions); break;
			case 't': tags = optarg; crash(access(optarg, R_OK), "file not found/readable: " + tags); break;
			case 'p': protein_domains = optarg; crash(access(optarg, R_OK), "file not found/readable: " + protein_domains); break;
			case 'c': {
				chimeric = optarg; crash(access(optarg, R_OK), "file not found/readable: " + chimeric);
				const std::string junction_suffix = ".junction"; // options.cpp:280, 293-296
				if (chimeric.size() >= junction_suffix.size() && chimeric.compare(chimeric.size() - junction_suffix.size(), junction_suffix.size(), junction_suffix) == 0)
					std::cerr << "WARNING: it seems you passed the chimeric junction file ('Chimeric.out.junction') to the parameter -c, but this parameter takes the chimeric alignments file ('Chimeric.out.sam') as input" << std::endl;
				break;
			}
			case 'I': o.fill_sequence_gaps = 1; break;
			case 'G':
				crash(true, "option " + opt + " is not supported by arriba-b200 (see DESIGN.md, out of scope)"); break;
			case 's': { const std::string m = optarg; o.strandedness = m == "auto" ? 3 : m == "yes" ? 1 : m == "no" ? 0 : m == "reverse" ? 2 : -1; crash(o.strandedness < 0, "invalid type of strandedness: " + m); break; }
			case 'i': interesting = optarg; std::replace(interesting.begin(), interesting.end(), ',', ' '); break;
			case 'v': viral = optarg; std::replace(viral.begin(), viral.end(), ',', ' '); break;
			case 'f': {
				std::string list = optarg; std::replace(list.begin(), list.end(), ',', ' ');
				std::istringstream ss(list); std::string name;
				while (ss >> name) { int id = -1; for (int k = 1; k < ARB_N_FILTERS; ++k) if (name == FILTERS[k]) id = k; crash(id < 0, "invalid argument to option -f: " + name); o.params.filter_mask &= ~((uint64_t) 1 << id); }
				break;
			}
			case 'E': crash(!float_in(optarg, 0, FLT_MAX, o.params.evalue_cutoff), "argument to " + opt + " must be greater than 0"); break;
			case 'S': crash(!int_in(optarg, 0, INT_MAX, iv), "invalid argument to " + opt); o.min_support = (int32_t) iv; break;
			case 'm': crash(!float_in(optarg, 0, 1, o.params.max_mismapper_fraction), "argument to " + opt + " must be between 0 and 1"); break;
			case 'L': crash(!float_in(optarg, 0, 1, o.params.max_homolog_identity), "argument to " + opt + " must be between 0 and 1"); break;
			case 'H': crash(!int_in(optarg, 2, INT_MAX, iv), "argument to " + opt + " must be greater than 1"); o.params.homopolymer_length = (uint32_t) iv; break;
			case 'R': crash(!int_in(optarg, 0, INT_MAX, iv), "invalid argument to " + opt); o.params.min_read_through_distance = (int32_t) iv; break;
			case 'A': crash(!int_in(optarg, 0, INT_MAX, iv), "invalid argument to " + opt); o.min_anchor_length = (uint32_t) iv; break;
			case 'M': crash(!int_in(optarg, 0, INT_MAX, iv), "invalid argument to " + opt); o.min_spliced_events = (uint32_t) iv; break;
			case 'K': crash(!float_in(optarg, 0, 1, o.params.max_kmer_content), "argument to " + opt + " must be between 0 and 1"); break;
			case 'V': crash(!float_in(optarg, 0, 1, o.params.mismatch_pvalue_cutoff), "argument to " + opt + " must be between 0 and 1"); break;
			case 'F': crash(!int_in(optarg, 1, INT_MAX, iv), "argument to " + opt + " must be an integer greater than 0"); o.fragment_length = (uint32_t) iv; break;
			case 'U': crash(!int_in(optarg, 1, SHRT_MAX, iv), "argument to " + opt + " must be an integer between 1 and " + std::to_string(SHRT_MAX)); o.params.subsampling_threshold = (uint32_t) iv; break;
			case 'Q': crash(!float_in(optarg, 0, 1, o.high_expression_quantile), "argument to " + opt + " must be between 0 and 1"); break;
			case 'e': crash(!float_in(optarg, 0, 1, o.exonic_fraction), "argument to " + opt + " must be between 0 and 1"); break;
			case 'l': crash(!int_in(optarg, 1, INT_MAX, iv), "argument to " + opt + " must be an integer greater than 0"); o.params.max_itd_length = (uint32_t) iv; break;
			case 'z': crash(!float_in(optarg, 0, 1, o.min_itd_allele_fraction), "argument to " + opt + " must be between 0 and 1"); break;
			case 'Z': crash(!int_in(optarg, 1, INT_MAX, iv), "argument to " + opt + " must be an integer greater than 0"); o.min_itd_support = (uint32_t) iv; break;
			case 'T': crash(!int_in(optarg, 1, INT_MAX, iv), "invalid argument to " + opt); o.top_viral_contigs = (uint32_t) iv; break; // options.cpp:432
			case 'C': crash(!float_in(optarg, 0, 1, o.viral_contig_min_covered_fraction), "argument to " + opt + " must be between 0 and 1"); break; // options.cpp:435
			case '@': crash(!int_in(optarg, 1, INT_MAX, iv), "argument to " + opt + " must be an integer greater than 0"); o.threads = (int32_t) iv; threads_given = true; break;
			case 'u': o.params.external_duplicate_marking = 1; break;
			case 'X': o.print_extra_info_for_discarded_fusions = 1; break;
			case 'h': usage(); return 0;
			default:
				crash(valid.find(std::string(1, (char) optopt) + ":") != std::string::npos, std::string("option -") + (char) optopt + " requires an argument");
				crash(true, std::string("unknown option: -") + (char) optopt);
		}
		crash(optind < argc && (std::string(argv[optind]).empty() || argv[optind][0] != '-'), "option " + opt + " has too many arguments (arguments with blanks must be wrapped in quotes)");
	}
	(void) threads_given;
	if (argc == 1) { usage(); crash(true, "no arguments given"); }
	crash(bam.empty(), "missing mandatory option -x");
	crash(gtf.empty(), "missing mandatory option -g");
	crash(out.empty(), "missing mandatory option -o");
	crash(fasta.empty(), "missing mandatory option -a");
	const bool blacklist_on = o.params.filter_mask >> 20 & 1;
	crash(blacklist_on && blacklist.empty(), "filter 'blacklist' enabled, but missing option -b (use '-f blacklist' if you want to disable the blacklist)");
	o.bam_file = bam.c_str(); o.gtf_file = gtf.c_str(); o.assembly_file = fasta.c_str(); o.output_file = out.c_str();
	o.discarded_output_file = discarded.empty() ? NULL : discarded.c_str();
	o.interesting_contigs = interesting.empty() ? NULL : interesting.c_str(); o.viral_contigs = viral.empty() ? NULL : viral.c_str();
	o.genomic_breakpoints_file = genomic.empty() ? NULL : genomic.c_str();
	o.blacklist_file = blacklist.empty() ? NULL : blacklist.c_str();
	o.known_fusions_file = known_fusions.empty() ? NULL : known_fusions.c_str(); o.tags_file = tags.empty() ? NULL : tags.c_str();
	o.protein_domains_file = protein_domains.empty() ? NULL : protein_domains.c_str();
	o.chimeric_file = chimeric.empty() ? NULL : chimeric.c_str();

	arb_pipeline* p = NULL;
	crash(arb_pipeline_create(&p, &o) != 0, arb_pipeline_error(NULL));
	std::cout << stamp() << " Loading assembly from '" << fasta << "' " << std::endl;
	std::cout << stamp() << " Loading annotation from '" << gtf << "' " << std::endl;
	if (arb_pipeline_run(p) != 0) { std::string m = arb_pipeline_error(p); arb_pipeline_destroy(p); crash(true, m); }
	std::cout << stamp() << " Freeing resources" << std::endl;
	arb_pipeline_destroy(p);
	time_t end_time; time(&end_time);
	struct rusage ru; getrusage(RUSAGE_SELF, &ru);
	auto hhmmss = [](unsigned long long s) { std::ostringstream x; x << std::setfill('0') << std::setw(2) << s / 3600 << ":" << std::setw(2) << s % 3600 / 60 << ":" << std::setw(2) << s % 60; return x.str(); };
	std::cout << stamp() << " Done (elapsed time=" << hhmmss((unsigned long long) difftime(end_time, start_time)) << ", CPU time=" << hhmmss(ru.ru_utime.tv_sec + ru.ru_stime.tv_sec)
	          << ", peak memory=" << std::setprecision(3) << (ru.ru_maxrss / (1024.0 * 1024)) << "gb)" << std::endl;
	return 0;
}
