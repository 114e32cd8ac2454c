// tools/synth.cpp -- deterministic synthetic world + chimeric BAM generator (test/bench infrastructure).
//
// Emits the inputs the `arriba` CLI consumes (SURVEY.md section 8d; shapes required by the reference's
// ingest are listed in SURVEY.md Appendix B, i.e. read_chimeric_alignments.cpp:611-748):
//   <prefix>.fa   assembly (contigs 1..22,X,Y; lengths proportional to hg38 * --scale)
//   <prefix>.gtf  gene annotation (multi-exon genes, overlapping/antisense genes, CDS, paralogs)
//   <prefix>.bam  STAR-WithinBAM-style records: split reads (primary+SA, mate, 0x800 supplementary),
//                 discordant mates, duplicates, multimappers (HI tag), normal / read-through pairs
// Everything derives from one 64-bit seed. No code or data of the reference is used.
#include <zlib.h>
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <unordered_set>
#include <vector>

using namespace std;

// ---------------------------------------------------------------------------------- rng
struct rng_t {
	uint64_t s;
	explicit rng_t(uint64_t seed): s(seed) {}
	uint64_t next() { // splitmix64
		uint64_t z = (s += 0x9E3779B97F4A7C15ULL);
		z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
		z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
		return z ^ (z >> 31);
	}
	uint32_t below(uint32_t n) { return n == 0 ? 0 : (uint32_t) ((next() >> 11) % n); }
	int range(int lo, int hi) { return lo + (int) below((uint32_t) (hi - lo + 1)); } // inclusive
	double unif() { return (next() >> 11) * (1.0 / 9007199254740992.0); }
	bool chance(double p) { return unif() < p; }
	int poisson(double lambda) {
		if (lambda > 30) { // normal approximation
			double u1 = unif(), u2 = unif();
			double z = sqrt(-2 * log(u1 + 1e-300)) * cos(2 * M_PI * u2);
			int v = (int) floor(lambda + sqrt(lambda) * z + 0.5);
			return v < 0 ? 0 : v;
		}
		double l = exp(-lambda), p = 1; int k = 0;
		do { ++k; p *= unif(); } while (p > l);
		return k - 1;
	}
};

static const char BASES[4] = {'A', 'C', 'G', 'T'};
static inline char comp(char c) {
	switch (c) { case 'A': return 'T'; case 'C': return 'G'; case 'G': return 'C'; case 'T': return 'A'; default: return c; }
}

// ---------------------------------------------------------------------------------- world
struct exon_t { int start, end; }; // 0-based inclusive
struct transcript_t { vector<int> exons; }; // indices into gene.exons (ascending coordinate)
struct gene_t {
	int contig, start, end; bool plus;
	vector<exon_t> exons; // ascending
	vector<transcript_t> transcripts;
	bool coding; int cds_start, cds_end;
	int paralog_of; // -1 or gene index
	string id, name;
};
struct breakpoint_t {
	int gene1, gene2; int contig1, contig2; int pos1, pos2;
	bool down1, down2; // true = DOWNSTREAM (retained sequence is left of the breakpoint)
	int tr1, tr2; // transcript used to walk, -1 = contiguous genome
	bool mismapper; // clipped segment is also alignable next to the breakpoint in the donor gene
	int depth;
};
struct world_t {
	vector<string> contig_names;
	vector<string> seq;
	vector<gene_t> genes;
	vector<vector<int> > genes_by_contig;
	vector<breakpoint_t> bps;
};

static const double HG38_MB[24] = {248.96, 242.19, 198.30, 190.21, 181.54, 170.81, 159.35, 145.14, 138.39, 133.80, 135.09, 133.28,
                                   114.36, 107.04, 101.99, 90.34, 83.26, 80.37, 58.62, 64.44, 46.71, 50.82, 156.04, 57.23};

struct params_t {
	string prefix = "synth";
	uint64_t seed = 0xA881BA;
	double scale = 0.001;
	int n_genes = 400;
	int n_breakpoints = 200;
	long n_fragments = 20000;
	int read_length = 101;
	double normal_frac = 0.10;
	double split_frac = 0.65;
	double dup_frac = 0.05;
	double multimap_frac = 0.02;
	double subst_rate = 0.01;
	double indel_frac = 0.02; // fraction of fragments with one indel
	double nbase_frac = 0.05; // fraction of reads with a few N bases
	double spliced_frac = 0.6; // fraction of breakpoint ends at exon boundaries
	double mismapper_frac = 0.03; // fraction of breakpoints whose clipped segment is alignable in the donor
	double paralog_frac = 0.05;
	double satellite_frac = 0.25; // fraction of breakpoints with shifted "satellite" breakpoints (merge_adjacent)
	double softclip_supp_frac = 0.2; // supplementary with soft instead of hard clip
	double nonproper_split_frac = 0.3;
	double deep_frac = 0.01; int deep_depth = 2000; int depth_cap = 280;
	bool shuffle = false;
	bool varnames = false;
	int compress = 0;
	bool chr_prefix = false;
	bool write_world = true, write_reads = true;
	int emit_breakpoints = -1; // emit reads of the first K breakpoints only (bounded samples of the same world)
};

static void make_genome(world_t& w, const params_t& P, rng_t& rng) {
	static const char* names[24] = {"1","2","3","4","5","6","7","8","9","10","11","12","13","14","15","16","17","18","19","20","21","22","X","Y"};
	for (int c = 0; c < 24; ++c) {
		w.contig_names.push_back(string(P.chr_prefix ? "chr" : "") + names[c]);
		size_t len = (size_t) (HG38_MB[c] * 1e6 * P.scale);
		if (len < 20000) len = 20000;
		string s(len, 'A');
		for (size_t i = 0; i < len; i += 32) {
			uint64_t r = rng.next();
			for (size_t j = i; j < i + 32 && j < len; ++j, r >>= 2) s[j] = BASES[r & 3];
		}
		// ~1% of the contig in N runs
		size_t n_runs = len / 100000 + 1;
		for (size_t k = 0; k < n_runs; ++k) {
			size_t run = 200 + rng.below(1800);
			if (run * 2 >= len) continue;
			size_t at = rng.below((uint32_t) (len - run));
			for (size_t j = at; j < at + run; ++j) s[j] = 'N';
		}
		w.seq.push_back(s);
	}
}

static void make_genes(world_t& w, const params_t& P, rng_t& rng) {
	double total = 0;
	for (size_t c = 0; c < w.seq.size(); ++c) total += w.seq[c].size();
	w.genes_by_contig.resize(w.seq.size());
	int gid = 0;
	for (size_t c = 0; c < w.seq.size(); ++c) {
		int n = max(2, (int) floor(P.n_genes * (w.seq[c].size() / total) + 0.5));
		int slot = (int) (w.seq[c].size() / (n + 1));
		if (slot < 3000) { n = max(2, (int) (w.seq[c].size() / 3000) - 1); slot = (int) (w.seq[c].size() / (n + 1)); }
		int prev_start = -1, prev_end = -1; bool prev_plus = true;
		for (int g = 0; g < n; ++g) {
			gene_t G;
			G.contig = (int) c; G.paralog_of = -1;
			int glen = min(200000, max(1500, (int) (slot * (0.3 + 0.5 * rng.unif()))));
			int start = slot / 2 + g * slot + rng.below((uint32_t) max(1, slot - glen - 1));
			G.plus = rng.chance(0.5);
			if (prev_start >= 0 && rng.chance(0.10)) { // overlapping gene, often antisense
				start = prev_start + (prev_end - prev_start) / 3 + rng.below((uint32_t) max(1, (prev_end - prev_start) / 3));
				G.plus = rng.chance(0.5) ? !prev_plus : prev_plus;
			}
			int end = start + glen - 1;
			if (end >= (int) w.seq[c].size() - 2000) continue;
			G.start = start; G.end = end;
			// exons
			int n_exons = 3 + rng.below(10);
			while (n_exons > 1 && n_exons * 450 > glen) --n_exons;
			vector<int> cuts;
			int pos = start;
			for (int e = 0; e < n_exons; ++e) {
				int elen = 80 + rng.below(320);
				int remaining_exons = n_exons - e - 1;
				int max_end = end - remaining_exons * 450;
				exon_t E; E.start = pos; E.end = min(pos + elen - 1, max_end);
				if (e == n_exons - 1) E.end = end;
				if (E.end - E.start > 1500) E.start = E.end - 300 - rng.below(400); // keep the last exon reasonably short
				G.exons.push_back(E);
				if (remaining_exons > 0) {
					int room = (end - remaining_exons * 450) - E.end;
					int intron = 50 + (room > 100 ? rng.below((uint32_t) (room / remaining_exons)) : 0);
					pos = E.end + 1 + intron;
				}
			}
			if (G.exons.front().start != start) G.start = G.exons.front().start;
			transcript_t T;
			for (size_t e = 0; e < G.exons.size(); ++e) T.exons.push_back((int) e);
			G.transcripts.push_back(T);
			if (G.exons.size() >= 4 && rng.chance(0.3)) {
				transcript_t T2; int skip = 1 + rng.below((uint32_t) G.exons.size() - 2);
				for (size_t e = 0; e < G.exons.size(); ++e) if ((int) e != skip) T2.exons.push_back((int) e);
				G.transcripts.push_back(T2);
			}
			G.coding = rng.chance(0.7);
			if (G.coding) {
				const exon_t& first = G.exons[G.exons.size() > 2 ? (G.plus ? 0 : 0) : 0];
				const exon_t& last = G.exons.back();
				G.cds_start = first.start + rng.below((uint32_t) max(1, (first.end - first.start) / 2));
				G.cds_end = last.end - rng.below((uint32_t) max(1, (last.end - last.start) / 2));
				if (rng.chance(0.2)) G.cds_start = first.start; // first base of the first exon coding (incomplete annotation case)
			} else { G.cds_start = G.cds_end = -1; }
			char buf[64];
			snprintf(buf, sizeof(buf), "ENSG%08d.%d", gid + 1, 1 + (int) rng.below(9)); G.id = buf;
			snprintf(buf, sizeof(buf), "GENE%d", gid + 1); G.name = buf;
			++gid;
			w.genes_by_contig[c].push_back((int) w.genes.size());
			w.genes.push_back(G);
			prev_start = G.start; prev_end = G.end; prev_plus = G.plus;
		}
	}
	// microsatellite tracts inside ~3% of exons (exercise low_entropy / homopolymer on matching reads)
	for (size_t g = 0; g < w.genes.size(); ++g)
		for (size_t e = 0; e < w.genes[g].exons.size(); ++e)
			if (rng.chance(0.03)) {
				const exon_t& E = w.genes[g].exons[e];
				int len = E.end - E.start + 1;
				int tract = min(len, 40 + (int) rng.below(120));
				int at = E.start + rng.below((uint32_t) (len - tract + 1));
				int period = 1 + rng.below(3);
				char unit[3] = {BASES[rng.below(4)], BASES[rng.below(4)], BASES[rng.below(4)]};
				string& s = w.seq[w.genes[g].contig];
				for (int i = 0; i < tract; ++i) s[at + i] = unit[i % period];
			}
	// paralogs: copy the sequence of another gene (same structure) with 2% divergence
	int n_par = (int) (w.genes.size() * P.paralog_frac);
	for (int k = 0; k < n_par; ++k) {
		int src = rng.below((uint32_t) w.genes.size());
		const gene_t S = w.genes[src];
		if (S.paralog_of >= 0) continue;
		// find a gene-free destination: replace another gene entirely (the victim takes the source's structure)
		int dst = rng.below((uint32_t) w.genes.size());
		gene_t& D = w.genes[dst];
		if (dst == src || D.paralog_of >= 0) continue;
		int slen = S.end - S.start + 1;
		// destination window must be free of other genes: require the next gene on the contig to start after the copy
		const vector<int>& on_contig = w.genes_by_contig[D.contig];
		bool ok = D.start + slen + 500 < (int) w.seq[D.contig].size();
		for (size_t j = 0; j < on_contig.size() && ok; ++j) {
			const gene_t& O = w.genes[on_contig[j]];
			if (on_contig[j] != dst && !(O.end < D.start - 200 || O.start > D.start + slen + 200)) ok = false;
		}
		bool used_as_source = false;
		for (size_t j = 0; j < w.genes.size(); ++j) if (w.genes[j].paralog_of == dst) used_as_source = true;
		if (!ok || used_as_source) continue;
		int shift = D.start - S.start;
		D.end = D.start + slen - 1; D.plus = S.plus; D.exons = S.exons; D.transcripts = S.transcripts;
		for (size_t e = 0; e < D.exons.size(); ++e) { D.exons[e].start += shift; D.exons[e].end += shift; }
		D.coding = S.coding; D.cds_start = S.cds_start < 0 ? -1 : S.cds_start + shift; D.cds_end = S.cds_end < 0 ? -1 : S.cds_end + shift;
		D.paralog_of = src;
		const string& ss = w.seq[S.contig]; string& ds = w.seq[D.contig];
		for (int i = 0; i < slen; ++i) {
			char b = ss[S.start + i];
			if (b != 'N' && rng.chance(0.02)) b = BASES[rng.below(4)];
			ds[D.start + i] = b;
		}
	}
}

// pick a breakpoint position inside/near a gene; returns position and the transcript to walk (-1 = none)
static void pick_end(const world_t& w, const params_t& P, rng_t& rng, int g, bool down, int& pos, int& tr) {
	const gene_t& G = w.genes[g];
	double r = rng.unif();
	tr = (int) rng.below((uint32_t) G.transcripts.size());
	const transcript_t& T = G.transcripts[tr];
	if (r < P.spliced_frac) { // exon boundary: retained side ends at a splice site
		int e = T.exons[rng.below((uint32_t) T.exons.size())];
		pos = down ? G.exons[e].end : G.exons[e].start;
	} else if (r < P.spliced_frac + 0.25) { // exon interior
		int e = T.exons[rng.below((uint32_t) T.exons.size())];
		pos = G.exons[e].start + rng.below((uint32_t) (G.exons[e].end - G.exons[e].start + 1));
	} else if (r < P.spliced_frac + 0.35) { // intronic
		pos = G.start + rng.below((uint32_t) (G.end - G.start + 1));
		tr = -1;
	} else { // intergenic, within 30 kb of the gene
		int off = 500 + rng.below(30000);
		pos = rng.chance(0.5) ? G.start - off : G.end + off;
		tr = -1;
		int clen = (int) w.seq[G.contig].size();
		if (pos < 2000 || pos > clen - 2000) { pos = G.start + 10; }
	}
}

static void make_breakpoints(world_t& w, const params_t& P, rng_t& rng) {
	int ng = (int) w.genes.size();
	double mean_depth = (double) P.n_fragments / max(1, P.n_breakpoints);
	for (int b = 0; b < P.n_breakpoints; ++b) {
		breakpoint_t B;
		B.mismapper = false;
		double r = rng.unif();
		int g1 = rng.below((uint32_t) ng), g2 = g1;
		bool consistent = rng.chance(0.8);
		if (r < 0.70) { // inter-chromosomal
			do { g2 = rng.below((uint32_t) ng); } while (w.genes[g2].contig == w.genes[g1].contig);
		} else if (r < 0.90) { // intra-chromosomal, distant
			const vector<int>& L = w.genes_by_contig[w.genes[g1].contig];
			for (int t = 0; t < 20; ++t) {
				g2 = L[rng.below((uint32_t) L.size())];
				if (abs(w.genes[g2].start - w.genes[g1].start) > min(1000000, (int) w.seq[w.genes[g1].contig].size() / 4)) break;
			}
		} else if (r < 0.94) { // read-through: neighbouring gene downstream
			const vector<int>& L = w.genes_by_contig[w.genes[g1].contig];
			size_t i = find(L.begin(), L.end(), g1) - L.begin();
			g2 = L[min(i + 1, L.size() - 1)];
		} else if (r < 0.97) { // paralog partner, if any
			for (int t = 0; t < ng; ++t) { int c = rng.below((uint32_t) ng); if (w.genes[c].paralog_of >= 0) { g1 = w.genes[c].paralog_of; g2 = c; break; } }
		} // else: intragenic (duplication / inversion / ITD-shaped), g2 == g1
		B.gene1 = g1; B.gene2 = g2;
		const gene_t& G1 = w.genes[g1]; const gene_t& G2 = w.genes[g2];
		B.contig1 = G1.contig; B.contig2 = G2.contig;
		// directions: a transcriptionally consistent fusion keeps the 5' part of gene1 and the 3' part of gene2
		B.down1 = consistent ? G1.plus : rng.chance(0.5);
		B.down2 = consistent ? !G2.plus : rng.chance(0.5);
		pick_end(w, P, rng, g1, B.down1, B.pos1, B.tr1);
		pick_end(w, P, rng, g2, B.down2, B.pos2, B.tr2);
		if (g1 == g2) {
			double q = rng.unif();
			if (q < 0.4) { // ITD-shaped: UPSTREAM at the lower, DOWNSTREAM at the higher coordinate, < 100 bp apart, inside one exon
				int e = G1.transcripts[0].exons[rng.below((uint32_t) G1.transcripts[0].exons.size())];
				int elen = G1.exons[e].end - G1.exons[e].start + 1;
				if (elen > 60) {
					int d = 12 + rng.below((uint32_t) min(80, elen - 20));
					int a = G1.exons[e].start + rng.below((uint32_t) (elen - d));
					B.pos1 = a + d; B.down1 = true;  // retained left of a+d
					B.pos2 = a; B.down2 = false;     // continues right of a  => duplication of [a, a+d]
					B.tr1 = B.tr2 = 0;
				}
			} else if (q < 0.7) { // inversion
				B.down2 = B.down1;
			} else { // duplication / deletion-like
				B.down2 = !B.down1;
			}
		}
		if (B.contig1 == B.contig2 && B.pos1 == B.pos2) B.pos2 += 37;
		B.depth = rng.chance(P.deep_frac) ? P.deep_depth : min(P.depth_cap, rng.poisson(mean_depth));
		if (b < P.n_breakpoints * P.mismapper_frac && g1 != g2) {
			// mismapper: the acceptor locus around pos2 becomes a diverged copy of the donor locus around pos1 (homologous partner), so the
			// clipped segment of every split read is also alignable next to the breakpoint in the other gene
			B.down1 = true; B.down2 = false;
			string& s1 = w.seq[B.contig1]; string& s2 = w.seq[B.contig2];
			const int n = 170;
			if (B.pos1 - n > 0 && B.pos1 + 1 + n < (int) s1.size() && B.pos2 - n > 0 && B.pos2 + n < (int) s2.size()) {
				const double divergence = rng.chance(0.5) ? 0.02 : 0.12; // some copies are too diverged to re-align
				for (int i = -n; i < n; ++i) {
					char c = s1[B.pos1 + 1 + i];
					if (c == 'N') c = 'A';
					if (rng.chance(divergence)) c = BASES[rng.below(4)];
					s2[B.pos2 + i] = c;
				}
				B.tr1 = -1; B.tr2 = -1; // walk contiguously so that the copied stretch is what reads see
				B.mismapper = true;
			}
		}
		w.bps.push_back(B);
		if (rng.chance(P.satellite_frac) && !B.mismapper) { // alternative alignments of the same junction: a few reads at a breakpoint shifted by <= 5 bp on both ends
			const int n_sat = 1 + rng.below(2);
			for (int k = 0; k < n_sat; ++k) {
				breakpoint_t S = B;
				int delta = 1 + rng.below(5); if (rng.chance(0.5)) delta = -delta;
				S.pos1 = B.pos1 + delta;
				S.pos2 = B.pos2 + delta * ((B.down1 == B.down2) ? -1 : +1); // keeps the pair mergeable (merge_adjacent_fusions.cpp:48,63)
				if (rng.chance(0.15)) S.pos2 += 1; // ... or not
				S.depth = 1 + rng.below(6);
				if (S.pos1 > 1000 && S.pos2 > 1000 && S.pos1 < (int) w.seq[S.contig1].size() - 1000 && S.pos2 < (int) w.seq[S.contig2].size() - 1000) w.bps.push_back(S);
			}
		}
	}
}

// ---------------------------------------------------------------------------------- output: FASTA / GTF
static void write_fasta(const world_t& w, const string& path) {
	FILE* f = fopen(path.c_str(), "wb");
	if (!f) { perror(path.c_str()); exit(1); }
	static char buf[1 << 16];
	setvbuf(f, buf, _IOFBF, sizeof(buf));
	for (size_t c = 0; c < w.seq.size(); ++c) {
		fprintf(f, ">%s synthetic\n", w.contig_names[c].c_str());
		const string& s = w.seq[c];
		for (size_t i = 0; i < s.size(); i += 80) {
			size_t n = min((size_t) 80, s.size() - i);
			fwrite(s.data() + i, 1, n, f);
			fputc('\n', f);
		}
	}
	fclose(f);
}

static void write_gtf(const world_t& w, const string& path) {
	FILE* f = fopen(path.c_str(), "wb");
	if (!f) { perror(path.c_str()); exit(1); }
	fprintf(f, "##description: synthetic annotation\n");
	for (size_t g = 0; g < w.genes.size(); ++g) {
		const gene_t& G = w.genes[g];
		const char* contig = w.contig_names[G.contig].c_str();
		char strand = G.plus ? '+' : '-';
		fprintf(f, "%s\tsynth\tgene\t%d\t%d\t.\t%c\t.\tgene_id \"%s\"; gene_name \"%s\";\n", contig, G.start + 1, G.end + 1, strand, G.id.c_str(), G.name.c_str());
		for (size_t t = 0; t < G.transcripts.size(); ++t) {
			char tid[64]; snprintf(tid, sizeof(tid), "ENST%08d%02d.%d", (int) g + 1, (int) t + 1, 1 + (int) (g % 5));
			const transcript_t& T = G.transcripts[t];
			for (size_t k = 0; k < T.exons.size(); ++k) {
				const exon_t& E = G.exons[G.plus ? T.exons[k] : T.exons[T.exons.size() - 1 - k]];
				fprintf(f, "%s\tsynth\texon\t%d\t%d\t.\t%c\t.\tgene_id \"%s\"; transcript_id \"%s\"; gene_name \"%s\"; exon_number \"%d\";\n",
				        contig, E.start + 1, E.end + 1, strand, G.id.c_str(), tid, G.name.c_str(), (int) k + 1);
				if (G.coding && E.end >= G.cds_start && E.start <= G.cds_end)
					fprintf(f, "%s\tsynth\tCDS\t%d\t%d\t.\t%c\t0\tgene_id \"%s\"; transcript_id \"%s\"; gene_name \"%s\";\n",
					        contig, max(E.start, G.cds_start) + 1, min(E.end, G.cds_end) + 1, strand, G.id.c_str(), tid, G.name.c_str());
			}
		}
	}
	fclose(f);
}

// ---------------------------------------------------------------------------------- BAM writer
struct bam_writer_t {
	FILE* f; int level;
	vector<unsigned char> buf;
	vector<unsigned char> zbuf;
	bam_writer_t(): f(NULL), level(0) {}
	void open(const string& path, int lvl) {
		f = fopen(path.c_str(), "wb");
		if (!f) { perror(path.c_str()); exit(1); }
		level = lvl; zbuf.resize(1 << 17);
	}
	void flush_block(const unsigned char* data, size_t n) {
		// one BGZF block = gzip member with BC extra field (SAMv1 4.1)
		z_stream zs; memset(&zs, 0, sizeof(zs));
		deflateInit2(&zs, level, Z_DEFLATED, -15, 8, Z_DEFAULT_STRATEGY);
		zs.next_in = (Bytef*) data; zs.avail_in = n;
		zs.next_out = &zbuf[18]; zs.avail_out = zbuf.size() - 26;
		deflate(&zs, Z_FINISH);
		size_t clen = zs.total_out;
		deflateEnd(&zs);
		unsigned char* h = &zbuf[0];
		static const unsigned char hdr[12] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0};
		memcpy(h, hdr, 12); h[12] = 'B'; h[13] = 'C'; h[14] = 2; h[15] = 0;
		size_t bsize = clen + 25;
		h[16] = bsize & 0xff; h[17] = bsize >> 8;
		uint32_t crc = crc32(crc32(0, NULL, 0), data, n);
		unsigned char* t = &zbuf[18 + clen];
		for (int i = 0; i < 4; ++i) t[i] = crc >> (8 * i);
		for (int i = 0; i < 4; ++i) t[4 + i] = ((uint32_t) n) >> (8 * i);
		fwrite(h, 1, clen + 26, f);
	}
	void write(const void* p, size_t n) {
		const unsigned char* c = (const unsigned char*) p;
		buf.insert(buf.end(), c, c + n);
		while (buf.size() >= 0xff00) {
			flush_block(&buf[0], 0xff00);
			buf.erase(buf.begin(), buf.begin() + 0xff00);
		}
	}
	void close() {
		if (!buf.empty()) flush_block(&buf[0], buf.size());
		buf.clear();
		flush_block(NULL, 0); // EOF marker block
		fclose(f);
	}
};

struct record_t { // one BAM alignment record, host representation
	string qname; int flag; int tid; int pos; vector<uint32_t> cigar; string seq; int mtid, mpos;
	int hi, nh; string sa;
};

static void put32(vector<unsigned char>& v, uint32_t x) { for (int i = 0; i < 4; ++i) v.push_back(x >> (8 * i)); }
static void put16(vector<unsigned char>& v, uint32_t x) { v.push_back(x & 0xff); v.push_back(x >> 8); }

static int nt16(char c) {
	switch (c) { case 'A': return 1; case 'C': return 2; case 'G': return 4; case 'T': return 8; case 'N': return 15; default: return 15; }
}

static void encode_record(const record_t& r, vector<unsigned char>& out) {
	vector<unsigned char> v;
	put32(v, (uint32_t) r.tid); put32(v, (uint32_t) r.pos);
	v.push_back((unsigned char) (r.qname.size() + 1)); v.push_back(255);
	put16(v, 4680); // bin (unused by consumers here)
	put16(v, (uint32_t) r.cigar.size()); put16(v, (uint32_t) r.flag);
	put32(v, (uint32_t) r.seq.size());
	put32(v, (uint32_t) r.mtid); put32(v, (uint32_t) r.mpos); put32(v, 0);
	v.insert(v.end(), r.qname.begin(), r.qname.end()); v.push_back(0);
	for (size_t i = 0; i < r.cigar.size(); ++i) put32(v, r.cigar[i]);
	for (size_t i = 0; i < r.seq.size(); i += 2) {
		int hi = nt16(r.seq[i]), lo = i + 1 < r.seq.size() ? nt16(r.seq[i + 1]) : 0;
		v.push_back((unsigned char) (hi << 4 | lo));
	}
	for (size_t i = 0; i < r.seq.size(); ++i) v.push_back(30);
	v.push_back('N'); v.push_back('H'); v.push_back('C'); v.push_back((unsigned char) r.nh);
	if (r.hi > 0) { v.push_back('H'); v.push_back('I'); v.push_back('C'); v.push_back((unsigned char) r.hi); }
	if (!r.sa.empty()) { v.push_back('S'); v.push_back('A'); v.push_back('Z'); v.insert(v.end(), r.sa.begin(), r.sa.end()); v.push_back(0); }
	put32(out, (uint32_t) v.size());
	out.insert(out.end(), v.begin(), v.end());
}

// ---------------------------------------------------------------------------------- fragments
struct col_t { int gpos; unsigned char seg; unsigned char ins; }; // one base of the sequenced molecule

// positions of a segment, outward from the breakpoint; k = 0 is the breakpoint base itself
static void walk_segment(const world_t& w, int contig, int pos, bool down, int gene, int tr, int need, vector<int>& gpos) {
	gpos.clear();
	int clen = (int) w.seq[contig].size();
	int dir = down ? -1 : +1;
	if (tr < 0) {
		for (int k = 0; k < need; ++k) { int p = pos + dir * k; if (p < 0 || p >= clen) break; gpos.push_back(p); }
		return;
	}
	const gene_t& G = w.genes[gene];
	const transcript_t& T = G.transcripts[tr];
	// locate exon containing pos
	int at = -1;
	for (size_t i = 0; i < T.exons.size(); ++i) if (G.exons[T.exons[i]].start <= pos && pos <= G.exons[T.exons[i]].end) at = (int) i;
	if (at < 0) { walk_segment(w, contig, pos, down, gene, -1, need, gpos); return; }
	int p = pos;
	while ((int) gpos.size() < need) {
		const exon_t& E = G.exons[T.exons[at]];
		int stop = down ? E.start : E.end;
		for (; (int) gpos.size() < need && (down ? p >= stop : p <= stop); p += dir) gpos.push_back(p);
		if ((int) gpos.size() >= need) break;
		int next = at + (down ? -1 : +1);
		if (next < 0 || next >= (int) T.exons.size()) { // ran out of exons: continue into flanking genome
			for (; (int) gpos.size() < need && p >= 0 && p < clen; p += dir) gpos.push_back(p);
			break;
		}
		at = next;
		p = down ? G.exons[T.exons[at]].end : G.exons[T.exons[at]].start;
	}
}

struct aln_t { int contig, start; bool reverse; vector<uint32_t> cigar; int clip_front_q, clip_back_q; };

static inline void push_op(vector<uint32_t>& c, uint32_t len, uint32_t op) {
	if (len == 0) return;
	if (!c.empty() && (c.back() & 0xf) == op) c.back() += len << 4; else c.push_back(len << 4 | op);
}

// build an alignment for columns [x,y) (molecule order), all inside one segment; forward = molecule runs along the genome's forward strand
static bool build_alignment(const vector<col_t>& cols, int x, int y, bool forward, int del_at, aln_t& A) {
	A.cigar.clear();
	int prev = -1; bool first = true; int start = -1;
	int n = y - x;
	for (int i = 0; i < n; ++i) {
		int idx = forward ? x + i : y - 1 - i;
		const col_t& c = cols[idx];
		if (c.ins) { if (first) return false; push_op(A.cigar, 1, 1); continue; }
		if (first) { start = c.gpos; first = false; }
		else {
			int gap = c.gpos - prev - 1;
			if (gap < 0) return false;
			if (gap > 0) {
				// deletion iff the two molecule columns straddle del_at
				int lo = forward ? idx - 1 : idx, hi = forward ? idx : idx + 1;
				(void) lo;
				bool is_del = del_at >= 0 && hi == del_at;
				// inserted columns between them do not matter: deletions and insertions are never adjacent
				push_op(A.cigar, (uint32_t) gap, is_del ? 2 : 3);
			}
		}
		push_op(A.cigar, 1, 0);
		prev = c.gpos;
	}
	if (first) return false;
	if ((A.cigar.back() & 0xf) != 0 || (A.cigar.front() & 0xf) != 0) return false;
	A.start = start;
	return true;
}

static string cigar_to_string(const vector<uint32_t>& c) {
	string s; char b[16];
	for (size_t i = 0; i < c.size(); ++i) { snprintf(b, sizeof(b), "%u%c", c[i] >> 4, "MIDNSHP=XB"[c[i] & 0xf]); s += b; }
	return s;
}

struct generator_t {
	const world_t& w; const params_t& P; rng_t rng;
	vector<vector<unsigned char> > chunks; // encoded fragments (for shuffling)
	bam_writer_t out;
	long name_counter; long name_mod;
	long n_emitted_fragments;
	generator_t(const world_t& w_, const params_t& P_): w(w_), P(P_), rng(P_.seed ^ 0x5EEDF00DULL), name_counter(0), n_emitted_fragments(0) {
		name_mod = 1000003; while (name_mod < (long) (P.n_fragments * 2 + 1000)) name_mod = name_mod * 2 + 1;
		while (true) { bool prime = true; for (long d = 3; d * d <= name_mod; d += 2) if (name_mod % d == 0) { prime = false; break; } if (prime) break; name_mod += 2; }
	}
	string next_name() {
		long id = (long) (((__int128) (name_counter + 1) * 7368787) % name_mod);
		++name_counter;
		char b[48];
		if (P.varnames) snprintf(b, sizeof(b), (id % 3 == 0) ? "r%ld" : (id % 3 == 1 ? "read_%ld/x" : "R%ld"), id);
		else snprintf(b, sizeof(b), "r%010ld", id);
		return b;
	}
	char base_at(const col_t& c, bool forward, int contig) const { char b = w.seq[contig][c.gpos]; return forward ? b : comp(b); }

	void emit(const vector<record_t>& recs) {
		vector<unsigned char> enc;
		for (size_t i = 0; i < recs.size(); ++i) encode_record(recs[i], enc);
		if (P.shuffle) chunks.push_back(enc); else out.write(&enc[0], enc.size());
	}
	void mutate(string& s) {
		for (size_t i = 0; i < s.size(); ++i) if (s[i] != 'N' && rng.chance(P.subst_rate)) s[i] = BASES[rng.below(4)];
		if (rng.chance(P.nbase_frac)) { int n = 1 + rng.below(3); for (int k = 0; k < n; ++k) s[rng.below((uint32_t) s.size())] = 'N'; }
	}
	static string revcomp(const string& s) { string r(s.rbegin(), s.rend()); for (size_t i = 0; i < r.size(); ++i) r[i] = comp(r[i]); return r; }

	// generate one chimeric fragment of breakpoint B (optionally relocated onto a paralog for multimapping hits)
	bool make_fragment(const breakpoint_t& B, const vector<int>& g1, const vector<int>& g2, bool want_split, const string& qname, int hi, int nh,
	                   vector<record_t>& recs, uint64_t frag_seed) {
		rng_t r(frag_seed);
		const int L = P.read_length;
		int I = max(L + 20, (int) (2 * L + 60 + 40 * (r.unif() + r.unif() + r.unif() - 1.5))); // insert size
		int J; // molecule index (within fragment) of the first base of segment 2
		if (want_split) {
			int a = 14 + r.below((uint32_t) (L - 28)); // junction inside a read, both parts >= 14
			J = r.chance(0.5) ? a : I - L + a;
		} else {
			if (I < 2 * L + 8) I = 2 * L + 8;
			J = L + 2 + r.below((uint32_t) (I - 2 * L - 3)); // junction in the unsequenced middle
		}
		int len1 = J, len2 = I - J;
		if (len1 > (int) g1.size() || len2 > (int) g2.size()) return false;
		// columns of the sequenced molecule
		vector<col_t> cols(I);
		for (int m = 0; m < I; ++m) {
			if (m < J) { cols[m].gpos = g1[J - 1 - m]; cols[m].seg = 0; }
			else { cols[m].gpos = g2[m - J]; cols[m].seg = 1; }
			cols[m].ins = 0;
		}
		bool fwd[2] = {B.down1, !B.down2};
		int contig[2] = {B.contig1, B.contig2};
		string F(I, 'A');
		for (int m = 0; m < I; ++m) F[m] = base_at(cols[m], fwd[cols[m].seg], contig[cols[m].seg]);
		// optional indel, away from all boundaries
		int del_at = -1;
		if (r.chance(P.indel_frac)) {
			int at = 16 + r.below((uint32_t) max(1, I - 32));
			int bounds[4] = {J, L, I - L, I};
			bool ok = true;
			for (int k = 0; k < 4; ++k) if (abs(at - bounds[k]) < 16) ok = false;
			if (at < 16 || at > I - 16) ok = false;
			// both neighbours must be contiguous in the genome (not at an exon junction)
			if (ok && abs(cols[at].gpos - cols[at - 1].gpos) != 1) ok = false;
			if (ok && abs(cols[at + 2].gpos - cols[at - 3].gpos) != 5) ok = false;
			if (ok) {
				if (r.chance(0.5)) { // insertion of 2 bases: columns at, at+1 become inserted bases
					cols[at].ins = cols[at + 1].ins = 1;
					F[at] = BASES[r.below(4)]; F[at + 1] = BASES[r.below(4)];
				} else { // deletion of 3 genome bases: shift the rest of this segment by 3 outward
					int seg = cols[at].seg;
					int dir = (cols[at].gpos > cols[at - 1].gpos) ? 1 : -1;
					bool contiguous = true;
					if (seg == 0) { // segment 1 lies left of J in the molecule: shift columns [0,at) outward
						for (int m = 1; m < at && contiguous; ++m) if (cols[m].gpos - cols[m - 1].gpos != dir) contiguous = false;
						if (contiguous) { for (int m = 0; m < at; ++m) { cols[m].gpos -= 3 * dir; F[m] = base_at(cols[m], fwd[0], contig[0]); } del_at = at; }
					} else {
						for (int m = at + 1; m < I && contiguous; ++m) if (cols[m].gpos - cols[m - 1].gpos != dir) contiguous = false;
						if (contiguous) { for (int m = at; m < I; ++m) { cols[m].gpos += 3 * dir; F[m] = base_at(cols[m], fwd[1], contig[1]); } del_at = at; }
					}
					for (int m = 0; m < I; ++m) if (cols[m].gpos < 0 || cols[m].gpos >= (int) w.seq[contig[cols[m].seg]].size()) return false;
				}
			}
		}
		string readA = F.substr(0, L), readB = revcomp(F.substr(I - L, L));
		mutate(readA); mutate(readB);
		bool a_is_read1 = r.chance(0.5);
		int flagA = a_is_read1 ? 0x40 : 0x80, flagB = a_is_read1 ? 0x80 : 0x40;
		int secondary = hi > 1 ? 0x100 : 0;

		// alignments. Read A covers molecule [0,L), forward w.r.t. the molecule; read B covers [I-L,I), reverse.
		recs.clear();
		if (!want_split) {
			aln_t A, Bn;
			if (!build_alignment(cols, 0, L, fwd[0], del_at, A)) return false;
			if (!build_alignment(cols, I - L, I, fwd[1], del_at, Bn)) return false;
			bool revA = !fwd[0], revB = fwd[1];
			record_t ra, rb;
			ra.qname = rb.qname = qname; ra.hi = rb.hi = hi; ra.nh = rb.nh = nh;
			ra.tid = contig[0]; ra.pos = A.start; ra.cigar = A.cigar; ra.seq = revA ? revcomp(readA) : readA;
			rb.tid = contig[1]; rb.pos = Bn.start; rb.cigar = Bn.cigar; rb.seq = revB ? revcomp(readB) : readB;
			ra.flag = 0x1 | flagA | (revA ? 0x10 : 0) | (revB ? 0x20 : 0) | secondary;
			rb.flag = 0x1 | flagB | (revB ? 0x10 : 0) | (revA ? 0x20 : 0) | secondary;
			ra.mtid = rb.tid; ra.mpos = rb.pos; rb.mtid = ra.tid; rb.mpos = ra.pos;
			if (r.chance(0.5)) { recs.push_back(ra); recs.push_back(rb); } else { recs.push_back(rb); recs.push_back(ra); }
			return true;
		}
		// split read
		bool in_A = J < L;
		aln_t prim, supp, mate;
		bool soft_supp = r.chance(P.softclip_supp_frac);
		record_t rp, rs, rm; // primary (with SA), supplementary, mate
		rp.qname = rs.qname = rm.qname = qname; rp.hi = rs.hi = rm.hi = hi; rp.nh = rs.nh = rm.nh = nh;
		bool proper = !r.chance(P.nonproper_split_frac);
		if (in_A) {
			// read A = [0,J) in segment 1 (outer part -> supplementary) + [J,L) in segment 2 (inner part, with mate B)
			if (!build_alignment(cols, J, L, fwd[1], del_at, prim)) return false;
			if (!build_alignment(cols, 0, J, fwd[0], del_at, supp)) return false;
			if (!build_alignment(cols, I - L, I, fwd[1], del_at, mate)) return false;
			bool rev_prim = !fwd[1], rev_supp = !fwd[0], rev_mate = fwd[1];
			// read-order CIGARs: primary = S(J) + ops ; supplementary = ops + H(L-J)
			vector<uint32_t> cp, cs;
			if (!rev_prim) { push_op(cp, J, 4); cp.insert(cp.end(), prim.cigar.begin(), prim.cigar.end()); }
			else { cp = prim.cigar; cp.push_back((uint32_t) J << 4 | 4); }
			uint32_t clip_op = soft_supp ? 4 : 5;
			if (!rev_supp) { cs = supp.cigar; cs.push_back((uint32_t) (L - J) << 4 | clip_op); }
			else { cs.push_back((uint32_t) (L - J) << 4 | clip_op); cs.insert(cs.end(), supp.cigar.begin(), supp.cigar.end()); }
			rp.tid = contig[1]; rp.pos = prim.start; rp.cigar = cp; rp.seq = rev_prim ? revcomp(readA) : readA;
			string supp_read = soft_supp ? readA : readA.substr(0, J);
			rs.tid = contig[0]; rs.pos = supp.start; rs.cigar = cs; rs.seq = rev_supp ? revcomp(supp_read) : supp_read;
			rm.tid = contig[1]; rm.pos = mate.start; rm.cigar = mate.cigar; rm.seq = rev_mate ? revcomp(readB) : readB;
			rp.flag = 0x1 | (proper ? 0x2 : 0) | flagA | (rev_prim ? 0x10 : 0) | (rev_mate ? 0x20 : 0) | secondary;
			rs.flag = 0x800 | 0x1 | flagA | (rev_supp ? 0x10 : 0) | (rev_mate ? 0x20 : 0) | secondary;
			rm.flag = 0x1 | (proper ? 0x2 : 0) | flagB | (rev_mate ? 0x10 : 0) | (rev_prim ? 0x20 : 0) | secondary;
		} else {
			// read B covers [I-L,I): [I-L,J) in segment 1 (inner part, with mate A) + [J,I) in segment 2 (outer part -> supplementary)
			int n2 = I - J; // bases of read B in segment 2 = its 5' end
			if (!build_alignment(cols, I - L, J, fwd[0], del_at, prim)) return false;
			if (!build_alignment(cols, J, I, fwd[1], del_at, supp)) return false;
			if (!build_alignment(cols, 0, L, fwd[0], del_at, mate)) return false;
			bool rev_prim = fwd[0], rev_supp = fwd[1], rev_mate = !fwd[0];
			vector<uint32_t> cp, cs;
			// genome-order CIGAR: for a reverse-strand alignment the read's 5' end is at the right
			if (rev_prim) { cp = prim.cigar; cp.push_back((uint32_t) n2 << 4 | 4); }
			else { push_op(cp, n2, 4); cp.insert(cp.end(), prim.cigar.begin(), prim.cigar.end()); }
			uint32_t clip_op = soft_supp ? 4 : 5;
			if (rev_supp) { cs.push_back((uint32_t) (L - n2) << 4 | clip_op); cs.insert(cs.end(), supp.cigar.begin(), supp.cigar.end()); }
			else { cs = supp.cigar; cs.push_back((uint32_t) (L - n2) << 4 | clip_op); }
			rp.tid = contig[0]; rp.pos = prim.start; rp.cigar = cp; rp.seq = rev_prim ? revcomp(readB) : readB;
			string supp_read = soft_supp ? readB : readB.substr(0, n2);
			rs.tid = contig[1]; rs.pos = supp.start; rs.cigar = cs; rs.seq = rev_supp ? revcomp(supp_read) : supp_read;
			rm.tid = contig[0]; rm.pos = mate.start; rm.cigar = mate.cigar; rm.seq = rev_mate ? revcomp(readA) : readA;
			rp.flag = 0x1 | (proper ? 0x2 : 0) | flagB | (rev_prim ? 0x10 : 0) | (rev_mate ? 0x20 : 0) | secondary;
			rs.flag = 0x800 | 0x1 | flagB | (rev_supp ? 0x10 : 0) | (rev_mate ? 0x20 : 0) | secondary;
			rm.flag = 0x1 | (proper ? 0x2 : 0) | flagA | (rev_mate ? 0x10 : 0) | (rev_prim ? 0x20 : 0) | secondary;
		}
		rp.mtid = rm.tid; rp.mpos = rm.pos; rm.mtid = rp.tid; rm.mpos = rp.pos; rs.mtid = rm.tid; rs.mpos = rm.pos;
		rp.sa = w.contig_names[rs.tid] + "," + to_string(rs.pos + 1) + "," + ((rs.flag & 0x10) ? "-" : "+") + "," + cigar_to_string(rs.cigar) + ",255,0;";
		rs.sa = w.contig_names[rp.tid] + "," + to_string(rp.pos + 1) + "," + ((rp.flag & 0x10) ? "-" : "+") + "," + cigar_to_string(rp.cigar) + ",255,0;";
		int order = r.below(3);
		if (order == 0) { recs.push_back(rm); recs.push_back(rp); recs.push_back(rs); }
		else if (order == 1) { recs.push_back(rp); recs.push_back(rs); recs.push_back(rm); }
		else { recs.push_back(rs); recs.push_back(rp); recs.push_back(rm); }
		return true;
	}

	// normal (non-chimeric) proper pair from a transcript; some cross into the neighbouring gene (read-through shape), some are soft-clipped
	bool make_normal(const string& qname, vector<record_t>& recs) {
		const int L = P.read_length;
		int g = rng.below((uint32_t) w.genes.size());
		const gene_t& G = w.genes[g];
		int tr = rng.below((uint32_t) G.transcripts.size());
		const transcript_t& T = G.transcripts[tr];
		int e = T.exons[rng.below((uint32_t) T.exons.size())];
		int pos = G.exons[e].start;
		vector<int> gp;
		int I = 2 * L + 20 + rng.below(120);
		bool read_through = rng.chance(0.08);
		walk_segment(w, G.contig, pos, false, g, tr, I + 8, gp);
		if ((int) gp.size() < I) return false;
		if (read_through) {
			// splice from the end of this gene's last exon into the first exon of the next gene on the contig
			const vector<int>& Lc = w.genes_by_contig[G.contig];
			size_t i = find(Lc.begin(), Lc.end(), g) - Lc.begin();
			if (i + 1 >= Lc.size()) return false;
			const gene_t& N = w.genes[Lc[i + 1]];
			if (N.start <= G.end + 50) return false;
			gp.clear();
			int take = 30 + rng.below((uint32_t) (2 * L - 40));
			const exon_t& last = G.exons[T.exons.back()];
			for (int p = max(last.start, last.end - take + 1); p <= last.end; ++p) gp.push_back(p);
			vector<int> rest;
			walk_segment(w, N.contig, N.exons[0].start, false, Lc[i + 1], 0, I, rest);
			gp.insert(gp.end(), rest.begin(), rest.end());
			if ((int) gp.size() < I) return false;
		}
		vector<col_t> cols(I);
		for (int m = 0; m < I; ++m) { cols[m].gpos = gp[m]; cols[m].seg = 0; cols[m].ins = 0; }
		string F(I, 'A');
		for (int m = 0; m < I; ++m) F[m] = w.seq[G.contig][gp[m]];
		aln_t A, B;
		int clipA = 0, clipB = 0;
		if (rng.chance(0.05)) clipA = 12 + rng.below(20); // 5' soft clip of read A (ITD detection path)
		if (rng.chance(0.05)) clipB = 12 + rng.below(20);
		if (!build_alignment(cols, clipA, L, true, -1, A)) return false;
		if (!build_alignment(cols, I - L, I - clipB, true, -1, B)) return false;
		string readA = F.substr(0, L), readB = F.substr(I - L, L); // both stored in genome-forward orientation
		for (int i = 0; i < clipA; ++i) readA[i] = BASES[rng.below(4)];
		for (int i = 0; i < clipB; ++i) readB[L - 1 - i] = BASES[rng.below(4)];
		mutate(readA); mutate(readB);
		record_t ra, rb;
		ra.qname = rb.qname = qname; ra.hi = rb.hi = 1; ra.nh = rb.nh = 1;
		ra.tid = rb.tid = G.contig; ra.pos = A.start; rb.pos = B.start;
		if (clipA) ra.cigar.push_back((uint32_t) clipA << 4 | 4);
		ra.cigar.insert(ra.cigar.end(), A.cigar.begin(), A.cigar.end());
		rb.cigar = B.cigar;
		if (clipB) rb.cigar.push_back((uint32_t) clipB << 4 | 4);
		ra.seq = readA; rb.seq = readB;
		bool a1 = rng.chance(0.5);
		ra.flag = 0x1 | 0x2 | 0x20 | (a1 ? 0x40 : 0x80);
		rb.flag = 0x1 | 0x2 | 0x10 | (a1 ? 0x80 : 0x40);
		ra.mtid = rb.tid; ra.mpos = rb.pos; rb.mtid = ra.tid; rb.mpos = ra.pos;
		recs.clear();
		if (rng.chance(0.5)) { recs.push_back(ra); recs.push_back(rb); } else { recs.push_back(rb); recs.push_back(ra); }
		return true;
	}

	void run(const string& path) {
		out.open(path, P.compress);
		// header
		vector<unsigned char> h;
		string text = "@HD\tVN:1.4\tSO:unsorted\n";
		for (size_t c = 0; c < w.seq.size(); ++c) text += "@SQ\tSN:" + w.contig_names[c] + "\tLN:" + to_string(w.seq[c].size()) + "\n";
		text += "@PG\tID:synth\tPN:arriba-b200-synth\n";
		h.push_back('B'); h.push_back('A'); h.push_back('M'); h.push_back(1);
		put32(h, (uint32_t) text.size()); h.insert(h.end(), text.begin(), text.end());
		put32(h, (uint32_t) w.seq.size());
		for (size_t c = 0; c < w.seq.size(); ++c) {
			put32(h, (uint32_t) w.contig_names[c].size() + 1);
			h.insert(h.end(), w.contig_names[c].begin(), w.contig_names[c].end()); h.push_back(0);
			put32(h, (uint32_t) w.seq[c].size());
		}
		out.write(&h[0], h.size());

		const int need = 2 * P.read_length + 400;
		vector<int> g1, g2, p1, p2;
		vector<record_t> recs;
		long normal_every = P.normal_frac > 0 ? max(1L, (long) (1.0 / P.normal_frac)) : 0;
		long since_normal = 0;
		for (size_t b = 0; b < w.bps.size(); ++b) {
			if (P.emit_breakpoints >= 0 && (int) b >= P.emit_breakpoints) break;
			const breakpoint_t& B = w.bps[b];
			walk_segment(w, B.contig1, B.pos1, B.down1, B.gene1, B.tr1, need, g1);
			walk_segment(w, B.contig2, B.pos2, B.down2, B.gene2, B.tr2, need, g2);
			// paralog relocation of end 2 for multimapping hits
			bool has_paralog = false; breakpoint_t B2 = B;
			for (size_t g = 0; g < w.genes.size() && !has_paralog; ++g)
				if (w.genes[g].paralog_of == B.gene2 && B.gene2 != B.gene1 && B.tr2 >= 0) {
					int shift = w.genes[g].start - w.genes[B.gene2].start;
					B2.gene2 = (int) g; B2.contig2 = w.genes[g].contig; B2.pos2 = B.pos2 + shift;
					has_paralog = B2.pos2 >= w.genes[g].start && B2.pos2 <= w.genes[g].end;
				}
			if (has_paralog) walk_segment(w, B2.contig2, B2.pos2, B2.down2, B2.gene2, B2.tr2, need, p2);
			for (int d = 0; d < B.depth; ++d) {
				bool want_split = rng.chance(P.split_frac);
				uint64_t fs = rng.next();
				string qname = next_name();
				bool multi = has_paralog && rng.chance(P.multimap_frac * 10);
				int nh = multi ? 2 : 1;
				if (!make_fragment(B, g1, g2, want_split, qname, 1, nh, recs, fs)) continue;
				emit(recs); ++n_emitted_fragments;
				if (multi && make_fragment(B2, g1, p2, want_split, qname, 2, nh, recs, fs)) emit(recs);
				if (rng.chance(P.dup_frac)) { // PCR duplicate: identical coordinates, new name
					string dn = next_name();
					if (make_fragment(B, g1, g2, want_split, dn, 1, 1, recs, fs)) { emit(recs); ++n_emitted_fragments; }
				}
				if (normal_every && ++since_normal >= normal_every) {
					since_normal = 0;
					for (int t = 0; t < 4; ++t) if (make_normal(next_name(), recs)) { emit(recs); break; }
				}
			}
		}
		if (P.shuffle) {
			// shuffle whole-record order: split fragments into single records first
			vector<vector<unsigned char> > single;
			for (size_t i = 0; i < chunks.size(); ++i) {
				size_t off = 0;
				while (off < chunks[i].size()) {
					uint32_t bs = chunks[i][off] | chunks[i][off + 1] << 8 | chunks[i][off + 2] << 16 | (uint32_t) chunks[i][off + 3] << 24;
					single.push_back(vector<unsigned char>(chunks[i].begin() + off, chunks[i].begin() + off + 4 + bs));
					off += 4 + bs;
				}
			}
			for (size_t i = single.size(); i > 1; --i) swap(single[i - 1], single[rng.below((uint32_t) i)]);
			for (size_t i = 0; i < single.size(); ++i) out.write(&single[i][0], single[i].size());
		}
		out.close();
	}
};

// ---------------------------------------------------------------------------------- the same records as SAM text (SAMv1 1.4), plain or BGZF
static void write_sam(const string& bam_path, const string& sam_path, int bgzf_level /* < 0: plain text */) {
	gzFile in = gzopen(bam_path.c_str(), "rb"); // reads every BGZF member
	if (!in) { perror(bam_path.c_str()); exit(1); }
	auto need = [&](void* p, unsigned n) { if (gzread(in, p, n) != (int) n) { fprintf(stderr, "synth: truncated BAM %s\n", bam_path.c_str()); exit(1); } };
	auto rd32 = [&]() { uint32_t v; need(&v, 4); return v; };
	char magic[4]; need(magic, 4);
	string text(rd32(), '\0'); if (!text.empty()) need(&text[0], text.size());
	vector<string> names(rd32());
	for (size_t k = 0; k < names.size(); ++k) { string n(rd32(), '\0'); need(&n[0], n.size()); names[k] = n.c_str(); rd32(); }
	FILE* plain = NULL; bam_writer_t z;
	if (bgzf_level < 0) { plain = fopen(sam_path.c_str(), "wb"); if (!plain) { perror(sam_path.c_str()); exit(1); } } else z.open(sam_path, bgzf_level);
	auto put = [&](const string& t) { if (plain) fwrite(t.data(), 1, t.size(), plain); else z.write(t.data(), t.size()); };
	put(text.c_str());
	static const char ops[] = "MIDNSHP=X", bases[] = "=ACMGRSVTWYHKDBN";
	vector<unsigned char> b; string line;
	uint32_t bs;
	while (gzread(in, &bs, 4) == 4) {
		b.resize(bs); need(b.data(), bs);
		auto u32 = [&](size_t at) { uint32_t v; memcpy(&v, &b[at], 4); return v; };
		auto u16 = [&](size_t at) { return (uint32_t) b[at] | (uint32_t) b[at + 1] << 8; };
		const int32_t tid = (int32_t) u32(0), pos = (int32_t) u32(4), mtid = (int32_t) u32(20), mpos = (int32_t) u32(24), tlen = (int32_t) u32(28);
		const uint32_t lq = b[8], mapq = b[9], nc = u16(12), flag = u16(14), ls = u32(16);
		size_t at = 32;
		line.assign((const char*) &b[at]); at += lq;
		line += "\t" + to_string(flag) + "\t" + (tid < 0 ? string("*") : names[tid]) + "\t" + to_string(pos + 1) + "\t" + to_string(mapq) + "\t";
		for (uint32_t k = 0; k < nc; ++k) { const uint32_t c = u32(at + 4 * k); line += to_string(c >> 4); line += ops[c & 15]; }
		if (nc == 0) line += "*";
		at += 4 * nc;
		line += "\t" + (mtid < 0 ? string("*") : mtid == tid ? string("=") : names[mtid]) + "\t" + to_string(mpos + 1) + "\t" + to_string(tlen) + "\t";
		for (uint32_t i = 0; i < ls; ++i) line += bases[(b[at + i / 2] >> (i & 1 ? 0 : 4)) & 15];
		if (ls == 0) line += "*";
		at += (ls + 1) / 2;
		line += "\t";
		for (uint32_t i = 0; i < ls; ++i) line += (char) (b[at + i] + 33);
		if (ls == 0) line += "*";
		at += ls;
		while (at + 3 <= b.size()) { // the tags synth writes: C (integers) and Z
			line += "\t"; line += (char) b[at]; line += (char) b[at + 1];
			if (b[at + 2] == 'C') { line += ":i:" + to_string(b[at + 3]); at += 4; }
			else { const string v((const char*) &b[at + 3]); line += ":Z:" + v; at += 3 + v.size() + 1; }
		}
		line += "\n";
		put(line);
	}
	gzclose(in);
	if (plain) fclose(plain); else z.close();
}

// ---------------------------------------------------------------------------------- the same records as STAR's --chimOutType SeparateSAMold pair
// A read's records under one key (name and HI) are chimeric when one of them is supplementary (0x800), a discordant mate or carries an SA tag. The chimeric
// records of keys with HI 1 go to <out>.Chimeric.out.sam (SAM text, as STAR writes it) with 0x800 turned into 0x100 and without their HI and SA tags; every
// other record goes to <out>.Aligned.out.bam, unchanged (BGZF at `level`). Both files carry the BAM's header.
static void write_separate_chimeric(const string& bam_path, const string& out, int level) {
	auto open_in = [&]() { gzFile in = gzopen(bam_path.c_str(), "rb"); if (!in) { perror(bam_path.c_str()); exit(1); } return in; };
	struct record_t { vector<unsigned char> b; string key; bool chimeric; int hit; };
	// every record as (body, "<qname>,<HI>", chimeric on its own, HI)
	auto each = [&](gzFile in, string& header_raw, vector<string>& names, vector<uint32_t>& lengths, auto f) {
		auto need = [&](void* p, unsigned n) { if (gzread(in, p, n) != (int) n) { fprintf(stderr, "synth: truncated BAM %s\n", bam_path.c_str()); exit(1); } };
		auto rd32 = [&]() { uint32_t v; need(&v, 4); return v; };
		char magic[4]; need(magic, 4);
		string text(rd32(), '\0'); if (!text.empty()) need(&text[0], text.size());
		header_raw.assign(magic, 4); uint32_t l = (uint32_t) text.size(); header_raw.append((const char*) &l, 4); header_raw += text;
		const uint32_t n_ref = rd32(); header_raw.append((const char*) &n_ref, 4);
		names.assign(n_ref, string()); lengths.assign(n_ref, 0);
		for (uint32_t k = 0; k < n_ref; ++k) {
			const uint32_t ln = rd32(); string n(ln, '\0'); need(&n[0], ln); const uint32_t len = rd32();
			header_raw.append((const char*) &ln, 4); header_raw += n; header_raw.append((const char*) &len, 4); names[k] = n.c_str(); lengths[k] = len;
		}
		record_t r; uint32_t bs;
		while (gzread(in, &bs, 4) == 4) {
			r.b.resize(bs); need(r.b.data(), bs);
			const unsigned char* b = r.b.data();
			uint32_t flag = (uint32_t) b[14] | (uint32_t) b[15] << 8, nc = (uint32_t) b[12] | (uint32_t) b[13] << 8, ls; memcpy(&ls, b + 16, 4);
			size_t at = 32 + b[8] + 4 * (size_t) nc + (ls + 1) / 2 + ls;
			bool sa = false; r.hit = 1;
			while (at + 3 <= bs) { // the tags synth writes: C (integers) and Z
				if (b[at] == 'S' && b[at + 1] == 'A') sa = true;
				if (b[at + 2] == 'C') { if (b[at] == 'H' && b[at + 1] == 'I') r.hit = b[at + 3]; at += 4; }
				else { at += 3; while (at < bs && b[at]) ++at; ++at; }
			}
			r.key = string((const char*) b + 32) + "," + to_string(r.hit);
			r.chimeric = (flag & 2048) || ((flag & 1) && !(flag & 2)) || sa;
			f(r);
		}
	};
	string header_raw; vector<string> names; vector<uint32_t> lengths;
	unordered_set<string> chimeric;
	{ gzFile in = open_in(); each(in, header_raw, names, lengths, [&](const record_t& r) { if (r.chimeric && r.hit == 1) chimeric.insert(r.key); }); gzclose(in); }
	bam_writer_t x; x.open(out + ".Aligned.out.bam", level); x.write(header_raw.data(), header_raw.size());
	FILE* c = fopen((out + ".Chimeric.out.sam").c_str(), "wb"); if (!c) { perror(out.c_str()); exit(1); }
	for (size_t k = 0; k < names.size(); ++k) fprintf(c, "@SQ\tSN:%s\tLN:%u\n", names[k].c_str(), lengths[k]);
	static const char ops[] = "MIDNSHP=X", bases[] = "=ACMGRSVTWYHKDBN";
	string line;
	gzFile in = open_in();
	each(in, header_raw, names, lengths, [&](const record_t& r) {
		if (!chimeric.count(r.key)) { const uint32_t bs = (uint32_t) r.b.size(); x.write(&bs, 4); x.write(r.b.data(), bs); return; }
		const unsigned char* b = r.b.data(); const size_t bs = r.b.size();
		auto u32 = [&](size_t at) { uint32_t v; memcpy(&v, b + at, 4); return v; };
		const int32_t tid = (int32_t) u32(0), pos = (int32_t) u32(4), mtid = (int32_t) u32(20), mpos = (int32_t) u32(24), tlen = (int32_t) u32(28);
		uint32_t flag = (uint32_t) b[14] | (uint32_t) b[15] << 8; const uint32_t nc = (uint32_t) b[12] | (uint32_t) b[13] << 8, ls = u32(16);
		if (flag & 2048) flag = (flag & ~2048u) | 256u;
		size_t at = 32;
		line.assign((const char*) b + at); at += b[8];
		line += "\t" + to_string(flag) + "\t" + (tid < 0 ? string("*") : names[tid]) + "\t" + to_string(pos + 1) + "\t" + to_string(b[9]) + "\t";
		for (uint32_t k = 0; k < nc; ++k) { const uint32_t op = u32(at + 4 * k); line += to_string(op >> 4); line += ops[op & 15]; }
		if (nc == 0) line += "*";
		at += 4 * nc;
		line += "\t" + (mtid < 0 ? string("*") : mtid == tid ? string("=") : names[mtid]) + "\t" + to_string(mpos + 1) + "\t" + to_string(tlen) + "\t";
		for (uint32_t i = 0; i < ls; ++i) line += bases[(b[at + i / 2] >> (i & 1 ? 0 : 4)) & 15];
		if (ls == 0) line += "*";
		at += (ls + 1) / 2;
		line += "\t";
		for (uint32_t i = 0; i < ls; ++i) line += (char) (b[at + i] + 33);
		if (ls == 0) line += "*";
		at += ls;
		while (at + 3 <= bs) {
			const bool drop = (b[at] == 'H' && b[at + 1] == 'I') || (b[at] == 'S' && b[at + 1] == 'A');
			string field; field += (char) b[at]; field += (char) b[at + 1];
			if (b[at + 2] == 'C') { field += ":i:" + to_string(b[at + 3]); at += 4; }
			else { const string v((const char*) b + at + 3); field += ":Z:" + v; at += 3 + v.size() + 1; }
			if (!drop) line += "\t" + field;
		}
		line += "\n";
		fwrite(line.data(), 1, line.size(), c);
	});
	gzclose(in); fclose(c); x.close();
}

static void usage() {
	fprintf(stderr,
		"usage: synth --prefix P [--seed S] [--scale F] [--genes G] [--breakpoints B] [--fragments N] [--read-length L]\n"
		"             [--normal-frac F] [--split-frac F] [--dup-frac F] [--multimap-frac F] [--mismapper-frac F] [--paralog-frac F]\n"
		"             [--deep-frac F] [--deep-depth D] [--shuffle] [--varnames] [--compress LEVEL] [--chr] [--reads-only]\n"
		"             [--sam] [--sam-bgzf LEVEL] [--sam-only] [--separate-chimeric] [--separate-chimeric-only]\n"
		"  --sam: also write P.sam, the records of P.bam as SAM text (--sam-bgzf: BGZF-compressed at LEVEL); --sam-only: convert an existing P.bam\n"
		"  --separate-chimeric: also write P.bam as STAR's --chimOutType SeparateSAMold pair, P.Chimeric.out.sam and P.Aligned.out.bam;\n"
		"                       --separate-chimeric-only: convert an existing P.bam\n");
	exit(1);
}

int main(int argc, char** argv) {
	params_t P;
	bool sam = false, sam_only = false, separate = false, separate_only = false; int sam_level = -1;
	for (int i = 1; i < argc; ++i) {
		string a = argv[i];
		#define NEXT (i + 1 < argc ? argv[++i] : (usage(), (char*) NULL))
		if (a == "--prefix") P.prefix = NEXT;
		else if (a == "--seed") P.seed = strtoull(NEXT, NULL, 0);
		else if (a == "--scale") P.scale = atof(NEXT);
		else if (a == "--genes") P.n_genes = atoi(NEXT);
		else if (a == "--breakpoints") P.n_breakpoints = atoi(NEXT);
		else if (a == "--fragments") P.n_fragments = atol(NEXT);
		else if (a == "--read-length") P.read_length = atoi(NEXT);
		else if (a == "--normal-frac") P.normal_frac = atof(NEXT);
		else if (a == "--split-frac") P.split_frac = atof(NEXT);
		else if (a == "--dup-frac") P.dup_frac = atof(NEXT);
		else if (a == "--multimap-frac") P.multimap_frac = atof(NEXT);
		else if (a == "--mismapper-frac") P.mismapper_frac = atof(NEXT);
		else if (a == "--paralog-frac") P.paralog_frac = atof(NEXT);
		else if (a == "--satellite-frac") P.satellite_frac = atof(NEXT);
		else if (a == "--subst-rate") P.subst_rate = atof(NEXT);
		else if (a == "--indel-frac") P.indel_frac = atof(NEXT);
		else if (a == "--deep-frac") P.deep_frac = atof(NEXT);
		else if (a == "--deep-depth") P.deep_depth = atoi(NEXT);
		else if (a == "--shuffle") P.shuffle = true;
		else if (a == "--varnames") P.varnames = true;
		else if (a == "--compress") P.compress = atoi(NEXT);
		else if (a == "--chr") P.chr_prefix = true;
		else if (a == "--reads-only") P.write_world = false;
		else if (a == "--emit-breakpoints") P.emit_breakpoints = atoi(NEXT);
		else if (a == "--sam") sam = true;
		else if (a == "--sam-bgzf") { sam = true; sam_level = atoi(NEXT); }
		else if (a == "--sam-only") { sam = true; sam_only = true; }
		else if (a == "--separate-chimeric") separate = true;
		else if (a == "--separate-chimeric-only") { separate = true; separate_only = true; }
		else usage();
	}
	if (sam_only || separate_only) {
		if (sam_only) write_sam(P.prefix + ".bam", P.prefix + ".sam", sam_level);
		if (separate_only) write_separate_chimeric(P.prefix + ".bam", P.prefix, P.compress);
		return 0;
	}
	rng_t rng(P.seed);
	world_t w;
	make_genome(w, P, rng);
	make_genes(w, P, rng);
	make_breakpoints(w, P, rng);
	if (P.write_world) {
		write_fasta(w, P.prefix + ".fa");
		write_gtf(w, P.prefix + ".gtf");
	}
	generator_t gen(w, P);
	gen.run(P.prefix + ".bam");
	if (sam) write_sam(P.prefix + ".bam", P.prefix + ".sam", sam_level);
	if (separate) write_separate_chimeric(P.prefix + ".bam", P.prefix, P.compress);
	size_t total = 0; for (size_t c = 0; c < w.seq.size(); ++c) total += w.seq[c].size();
	fprintf(stderr, "synth: genome=%zu bp, genes=%zu, breakpoints=%zu, chimeric fragments=%ld\n", total, w.genes.size(), w.bps.size(), gen.n_emitted_fragments);
	return 0;
}
