// refdata.cpp -- see refdata.h for the behavioural contract and reference citations.
#include "refdata.h"
#include "../annot_hd.h"
#include <zlib.h>
#include <algorithm>
#include <cstring>
#include <iostream>
#include <set>
#include <sstream>
#include <stdexcept>
#include <tuple>
#include <climits>
#include <cstdlib>

namespace arb { namespace host {

static void fail(const std::string& msg) { throw std::runtime_error(msg); }

bool next_line(const std::string& text, size_t& at, std::string& line) {
	if (at >= text.size()) return false;
	size_t nl = text.find('\n', at);
	if (nl == std::string::npos) nl = text.size();
	line.assign(text, at, nl - at);
	at = nl + 1;
	if (!line.empty() && line[line.size() - 1] == '\r') line.resize(line.size() - 1);
	return true;
}

bool str_to_int(const std::string& text, i32& v) {
	const char* s = text.c_str(); char* e;
	const long r = strtol(s, &e, 10);
	v = (i32) r;
	return *s != ' ' && e != s && *e == '\0' && r != LONG_MAX && r != LONG_MIN;
}

// ------------------------------------------------------------------------------------------- contig names and patterns
std::string remove_chr(std::string contig) { // common.hpp:74-80
	if (contig.compare(0, 3, "chr") == 0) contig.erase(0, 3);
	if (contig == "M") contig = "MT";
	return contig;
}

// Wildcard test of the reference (common.hpp:82-107): the pattern list is whitespace separated; within a pattern '*' splits
// literal pieces that must occur left to right (each at its FIRST occurrence after the previous piece); the first piece is
// anchored at the start unless the pattern begins with '*'; the match must end at the end of the name unless the pattern
// ends with '*'.
bool contig_matches(std::string contig, const std::string& patterns) {
	contig = remove_chr(contig);
	std::istringstream list(patterns);
	std::string pattern;
	while (list >> pattern) {
		pattern = remove_chr(pattern);
		if (pattern.empty()) continue;
		const bool open_end = pattern[pattern.size() - 1] == '*', open_start = pattern[0] == '*';
		std::vector<std::string> pieces;
		size_t p = 0;
		while (p <= pattern.size()) {
			size_t q = pattern.find('*', p);
			if (q == std::string::npos) q = pattern.size();
			if (q > p) pieces.push_back(pattern.substr(p, q - p));
			p = q + 1;
		}
		size_t pos = 0; bool ok = true;
		for (size_t k = 0; k < pieces.size() && ok; ++k) {
			if (pos == 0 && !open_start && contig.compare(0, pieces[k].size(), pieces[k]) != 0) { ok = false; break; }
			pos = contig.find(pieces[k], pos);
			if (pos == std::string::npos) { ok = false; break; }
			pos += pieces[k].size();
		}
		if (ok && (pos == contig.size() || open_end)) return true;
	}
	return false;
}

u16 refdata::contig_id(const std::string& name) {
	std::map<std::string, u16>::iterator it = contig_ids.find(name);
	if (it != contig_ids.end()) return it->second;
	if (contig_ids.size() >= USHRT_MAX - 2) fail("too many contigs");
	u16 id = (u16) contig_ids.size();
	contig_ids[name] = id;
	if (original_names.size() < contig_ids.size()) original_names.resize(contig_ids.size());
	if (seq_off.size() < contig_ids.size()) { seq_off.resize(contig_ids.size(), 0); seq_len.resize(contig_ids.size(), 0); }
	return id;
}

// ------------------------------------------------------------------------------------------- file reading
void read_whole_file(const std::string& path, std::string& out) { // autodecompress_file_t (read_compressed_file.cpp:10-45): .gz is inflated whole (gzip and BGZF members)
	const bool gz = path.size() >= 3 && path.compare(path.size() - 3, 3, ".gz") == 0;
	out.clear();
	if (gz) {
		gzFile f = gzopen(path.c_str(), "rb");
		if (!f) fail("failed to open/decompress file: " + path);
		gzbuffer(f, 1 << 20);
		std::vector<char> buf(1 << 22);
		int n;
		while ((n = gzread(f, buf.data(), (unsigned) buf.size())) > 0) out.append(buf.data(), n);
		if (n < 0) { gzclose(f); fail("failed to decompress file: " + path); }
		gzclose(f);
	} else {
		FILE* f = fopen(path.c_str(), "rb");
		if (!f) fail("failed to open file: " + path);
		fseek(f, 0, SEEK_END); long sz = ftell(f); fseek(f, 0, SEEK_SET);
		out.resize(sz);
		if (sz > 0 && fread(&out[0], 1, sz, f) != (size_t) sz) { fclose(f); fail("failed to load file into memory: " + path); }
		fclose(f);
	}
}

// ------------------------------------------------------------------------------------------- assembly
void refdata::load_assembly(const std::string& fasta_path, const std::string& interesting_contigs) {
	std::string text;
	read_whole_file(fasta_path, text);
	assembly.clear();
	assembly.reserve(text.size() + 64 * 1024);
	const char* p = text.data(); const char* endp = p + text.size();
	int current = -1; // contig being filled, -1 = skip
	while (p < endp) {
		const char* nl = (const char*) memchr(p, '\n', endp - p);
		const char* e = nl ? nl : endp;
		const char* le = e;
		if (le > p && le[-1] == '\r') --le; // DOS line breaks
		if (le > p) {
			if (*p == '>') {
				// name = first whitespace-delimited token after '>'
				const char* s = p + 1; while (s < le && (*s == ' ' || *s == '\t')) ++s;
				const char* t = s; while (t < le && !isspace((unsigned char) *t)) ++t;
				const std::string name(s, t);
				const u16 id = contig_id(remove_chr(name));
				original_names[id] = name;
				if (contig_matches(name, interesting_contigs)) {
					current = id;
					if (seq_len[id] == 0) { // start of a new sequence: align to 64 bytes
						while (assembly.size() % 64) assembly.push_back('\0');
						seq_off[id] = assembly.size();
					} else if (seq_off[id] + seq_len[id] != assembly.size()) {
						fail("contig '" + name + "' appears in several non-adjacent FASTA records");
					}
				} else current = -1;
			} else if (current >= 0) {
				const size_t old = assembly.size();
				assembly.resize(old + (le - p));
				char* dst = &assembly[old];
				for (const char* c = p; c < le; ++c) *dst++ = (char) toupper((unsigned char) *c);
				seq_len[current] += (u32) (le - p);
			}
		}
		p = nl ? nl + 1 : endp;
	}
	for (int k = 0; k < 64; ++k) assembly.push_back('\0');
}

// ------------------------------------------------------------------------------------------- GTF
static bool parse_int_strict(const std::string& s, int& out) { // common.hpp:316-321
	if (s.empty() || s[0] == ' ') return false;
	char* endp; long v = strtol(s.c_str(), &endp, 10);
	out = (int) v;
	return endp != s.c_str() && *endp == '\0' && v != LONG_MAX && v != LONG_MIN;
}

static bool gtf_attribute(const std::string& attributes, const std::vector<std::string>& names, std::string& value) { // annotation.cpp:109-146
	size_t start = std::string::npos;
	for (size_t k = 0; k < names.size() && start >= attributes.size(); ++k) start = attributes.find(names[k] + " \"");
	if (start < attributes.size()) start = attributes.find('"', start);
	size_t end = std::string::npos;
	if (start < attributes.size()) { ++start; end = attributes.find('"', start); }
	if (start >= attributes.size() || end >= attributes.size()) {
		std::string joined;
		for (size_t k = 0; k < names.size(); ++k) joined += (k ? "|" : "") + names[k];
		std::cerr << "WARNING: failed to extract " << joined << " from line in GTF file: " << attributes << std::endl;
		return false;
	}
	value = attributes.substr(start, end - start);
	return true;
}

static std::string strip_ensembl_version(const std::string& id) { // annotation.hpp:29-35
	size_t dot;
	if (id.compare(0, 3, "ENS") == 0 && (dot = id.find_last_of('.')) < id.size()) return id.substr(0, dot);
	return id;
}

void refdata::load_gtf(const std::string& gtf_path) {
	std::string text;
	read_whole_file(gtf_path, text);
	typedef std::tuple<std::string, u16, bool> key_t;
	std::map<key_t, int> transcript_by_id, gene_by_id;
	std::map<key_t, std::vector<u32> > exons_by_transcript; // key uses the FULL transcript id (annotation.cpp:259)
	struct cds_t { bool forward; u16 contig; i32 start, end; std::string transcript_id; };
	std::vector<cds_t> coding_regions;
	const int max_gene_size = 3000000;
	std::set<u32> malformed_genes; std::vector<key_t> malformed_transcripts; std::set<std::string> reported;
	const std::vector<std::string> name_attr = {"gene_name", "gene_id"}, id_attr = {"gene_id"}, tr_attr = {"transcript_id"};
	u32 new_id = 0;
	std::vector<bool> gene_removed, exon_removed;

	size_t p = 0;
	std::string line, fields[9];
	while (p < text.size()) {
		size_t nl = text.find('\n', p);
		if (nl == std::string::npos) nl = text.size();
		size_t le = nl;
		if (le > p && text[le - 1] == '\r') --le;
		line.assign(text, p, le - p);
		p = nl + 1;
		if (line.empty() || line[0] == '#') continue;
		// nine tab-separated fields; fewer, or non-numeric coordinates, make the line unparsable
		size_t q = 0; int nf = 0; bool bad = false;
		for (; nf < 9; ++nf) {
			if (q >= line.size()) { bad = true; break; }
			size_t t = line.find('\t', q);
			fields[nf] = line.substr(q, t == std::string::npos ? std::string::npos : t - q);
			q = t == std::string::npos ? line.size() : t + 1;
		}
		int start = 0, end = 0;
		if (!bad && (!parse_int_strict(fields[3], start) || !parse_int_strict(fields[4], end))) bad = true;
		if (bad || fields[0].empty() || fields[2].empty() || fields[6].empty()) { std::cerr << "WARNING: failed to parse line in GTF file: " << line << std::endl; continue; }
		const std::string& attributes = fields[8];
		std::string gene_name, gene_id;
		if (!gtf_attribute(attributes, name_attr, gene_name) || !gtf_attribute(attributes, id_attr, gene_id)) continue;
		const std::string short_gene_id = strip_ensembl_version(gene_id);
		const u16 contig = contig_id(remove_chr(fields[0]));
		original_names[contig] = fields[0];
		--start; --end; // GTF is one-based
		const bool forward = fields[6][0] == '+';
		const std::string& feature = fields[2];

		if (feature == "exon") {
			std::string transcript_id;
			if (!gtf_attribute(attributes, tr_attr, transcript_id)) continue;
			const std::string short_transcript_id = strip_ensembl_version(transcript_id);
			std::pair<std::map<key_t, int>::iterator, bool> tr = transcript_by_id.insert(std::make_pair(key_t(short_transcript_id, contig, forward), -1));
			if (tr.second) {
				transcript_rec t; t.id = new_id++; t.name = transcript_id; t.first_exon = -1; t.last_exon = -1; t.coding_length = 0;
				tr.first->second = (int) transcripts.size(); transcripts.push_back(t);
			}
			std::pair<std::map<key_t, int>::iterator, bool> ge = gene_by_id.insert(std::make_pair(key_t(short_gene_id, contig, forward), -1));
			u32 g;
			if (ge.second) {
				gene_rec r; r.contig = contig; r.start = start; r.end = end; r.forward = forward; r.gene_id = gene_id; r.name = gene_name;
				r.exonic_length = 0; r.is_dummy = false; r.is_protein_coding = false;
				++new_id;
				g = (u32) genes.size(); ge.first->second = (int) g; genes.push_back(r); gene_removed.push_back(false);
			} else {
				g = (u32) ge.first->second;
				gene_rec& r = genes[g];
				if (r.start > start) r.start = start;
				if (r.end < end) r.end = end;
				if (r.end - r.start > max_gene_size) {
					if (reported.insert(gene_id).second) std::cerr << "WARNING: gene ID '" << gene_id << "' appears to be non-unique and will be ignored" << std::endl;
					malformed_genes.insert(g);
				}
			}
			if (has_sequence(genes[g].contig) && (u32) genes[g].end >= seq_len[genes[g].contig]) {
				if (reported.insert(gene_id).second) std::cerr << "WARNING: gene with ID '" << gene_id << "' extends beyond end of contig and will be ignored" << std::endl;
				malformed_genes.insert(g);
			}
			exon_rec e; e.contig = contig; e.start = start; e.end = end; e.forward = forward; e.gene = g; e.transcript = (u32) tr.first->second;
			e.prev = -1; e.next = -1; e.cds_start = -1; e.cds_end = -1;
			exons_by_transcript[key_t(transcript_id, contig, forward)].push_back((u32) exons.size());
			exons.push_back(e); exon_removed.push_back(false);
		} else if (feature == "CDS") {
			cds_t c; c.forward = forward; c.contig = contig; c.start = start; c.end = end;
			if (!gtf_attribute(attributes, tr_attr, c.transcript_id)) continue;
			coding_regions.push_back(c);
		}
	}
	if (genes.empty()) fail("failed to parse GTF file, please consider using -G");

	// coding regions -> exons of the same transcript (annotation.cpp:279-300)
	for (size_t k = 0; k < coding_regions.size(); ++k) {
		const cds_t& c = coding_regions[k];
		std::map<key_t, std::vector<u32> >::iterator tr = exons_by_transcript.find(key_t(c.transcript_id, c.contig, c.forward));
		if (tr == exons_by_transcript.end()) { std::cerr << "WARNING: CDS record has unknown transcript ID: " << c.transcript_id << std::endl; continue; }
		for (size_t j = 0; j < tr->second.size(); ++j) {
			exon_rec& e = exons[tr->second[j]];
			if ((e.start <= c.start && e.end >= c.start) || (e.start <= c.end && e.end >= c.end) || (e.start >= c.start && e.end <= c.end)) {
				e.cds_start = std::max(c.start, e.start); e.cds_end = std::min(c.end, e.end);
				genes[e.gene].is_protein_coding = true;
			}
		}
	}
	// order exons within each transcript by (contig, end, start) and link neighbours (annotation.cpp:303-309, common.hpp:116-120)
	for (std::map<key_t, std::vector<u32> >::iterator tr = exons_by_transcript.begin(); tr != exons_by_transcript.end(); ++tr) {
		std::vector<u32>& v = tr->second;
		std::sort(v.begin(), v.end(), [this](u32 a, u32 b) {
			const exon_rec& x = exons[a]; const exon_rec& y = exons[b];
			if (x.contig != y.contig) return x.contig < y.contig;
			if (x.end != y.end) return x.end < y.end;
			return x.start < y.start;
		});
		for (size_t j = 0; j < v.size(); ++j) { exons[v[j]].prev = j > 0 ? (i32) v[j - 1] : -1; exons[v[j]].next = j + 1 < v.size() ? (i32) v[j + 1] : -1; }
	}
	for (size_t e = 0; e < exons.size(); ++e) {
		transcript_rec& t = transcripts[exons[e].transcript];
		if (t.first_exon < 0 || exons[e].start < exons[t.first_exon].start) t.first_exon = (i32) e;
		if (t.last_exon < 0 || exons[e].end > exons[t.last_exon].end) t.last_exon = (i32) e;
	}
	for (size_t e = 0; e < exons.size(); ++e)
		if (exons[e].cds_start != -1 && exons[e].cds_end != -1) transcripts[exons[e].transcript].coding_length += exons[e].cds_end - exons[e].cds_start + 1;

	// transcripts the reference removes unconditionally (annotation.cpp:323-336) and unreasonably large ones
	struct fix_t { const char* contig; const char* id; bool forward; };
	static const fix_t fixes[] = {{"4", "ENST00000507166", true}, {"6", "ENST00000467125", false}, {"9", "ENST00000404796", true},
	                              {"9", "ENST00000577563", true}, {"9", "ENST00000580900", true}, {"7", "ENSMUST00000124096", false}};
	for (size_t k = 0; k < sizeof(fixes) / sizeof(fixes[0]); ++k)
		if (contig_ids.count(fixes[k].contig)) malformed_transcripts.push_back(key_t(fixes[k].id, contig_ids[fixes[k].contig], fixes[k].forward));
	for (std::map<key_t, int>::iterator tr = transcript_by_id.begin(); tr != transcript_by_id.end(); ++tr) {
		const transcript_rec& t = transcripts[tr->second];
		if (exons[t.last_exon].end - exons[t.first_exon].start > max_gene_size) {
			malformed_transcripts.push_back(tr->first);
			std::cerr << "WARNING: transcript ID '" << std::get<0>(tr->first) << "' appears to be non-unique and will be ignored" << std::endl;
		}
	}
	auto remove_gene = [&](u32 g) { for (size_t e = 0; e < exons.size(); ++e) if (!exon_removed[e] && exons[e].gene == g) exon_removed[e] = true; gene_removed[g] = true; };
	for (size_t k = 0; k < malformed_transcripts.size(); ++k) {
		std::map<key_t, int>::iterator tr = transcript_by_id.find(malformed_transcripts[k]);
		if (tr == transcript_by_id.end()) continue;
		int g = -1;
		for (size_t e = 0; e < exons.size(); ++e) if (!exon_removed[e] && (int) exons[e].transcript == tr->second) { g = (int) exons[e].gene; exon_removed[e] = true; }
		if (g < 0) continue;
		i32 ns = -1, ne = -1;
		for (size_t e = 0; e < exons.size(); ++e) if (!exon_removed[e] && (int) exons[e].gene == g) {
			if (ns == -1 || ns > exons[e].start) ns = exons[e].start;
			if (ne == -1 || ne < exons[e].end) ne = exons[e].end;
		}
		if (ns == -1) remove_gene((u32) g); else { genes[g].start = ns; genes[g].end = ne; }
	}
	for (std::set<u32>::iterator g = malformed_genes.begin(); g != malformed_genes.end(); ++g) if (!gene_removed[*g]) remove_gene(*g);

	// compact (ids = creation order of the survivors)
	std::vector<i32> gene_map(genes.size(), -1), exon_map(exons.size(), -1);
	std::vector<gene_rec> g2; std::vector<exon_rec> e2;
	for (size_t g = 0; g < genes.size(); ++g) if (!gene_removed[g]) { gene_map[g] = (i32) g2.size(); g2.push_back(genes[g]); }
	for (size_t e = 0; e < exons.size(); ++e) if (!exon_removed[e]) { exon_map[e] = (i32) e2.size(); e2.push_back(exons[e]); }
	for (size_t e = 0; e < e2.size(); ++e) {
		e2[e].gene = (u32) gene_map[e2[e].gene];
		// links into removed exons stay "present" in the reference (dangling pointers are only tested for NULL): keep the flag, drop the target
		e2[e].prev = e2[e].prev < 0 ? -1 : (exon_map[e2[e].prev] >= 0 ? exon_map[e2[e].prev] : -2);
		e2[e].next = e2[e].next < 0 ? -1 : (exon_map[e2[e].next] >= 0 ? exon_map[e2[e].next] : -2);
	}
	for (size_t t = 0; t < transcripts.size(); ++t) {
		transcripts[t].first_exon = transcripts[t].first_exon >= 0 ? exon_map[transcripts[t].first_exon] : -1;
		transcripts[t].last_exon = transcripts[t].last_exon >= 0 ? exon_map[transcripts[t].last_exon] : -1;
	}
	genes.swap(g2); exons.swap(e2);
	for (size_t g = 0; g < genes.size(); ++g) gene_by_name[genes[g].name] = (u32) g; // last one wins, like annotation.cpp:373-375
}

// ------------------------------------------------------------------------------------------- disjoint-region indices
template <class REC> static void build_index(const std::vector<REC>& recs, size_t n_contigs, region_index& ix) {
	std::vector<std::vector<i32> > keys(n_contigs);
	for (size_t k = 0; k < recs.size(); ++k) { keys[recs[k].contig].push_back(recs[k].end); keys[recs[k].contig].push_back(recs[k].start - 1); }
	ix.begin.assign(n_contigs + 1, 0); ix.end.clear(); ix.off.assign(1, 0); ix.items.clear();
	for (size_t c = 0; c < n_contigs; ++c) {
		std::sort(keys[c].begin(), keys[c].end());
		keys[c].erase(std::unique(keys[c].begin(), keys[c].end()), keys[c].end());
		ix.begin[c] = (u32) ix.end.size();
		ix.end.insert(ix.end.end(), keys[c].begin(), keys[c].end());
	}
	ix.begin[n_contigs] = (u32) ix.end.size();
	// region with end key k lists every record with start <= k <= end (ids ascending because records are visited in id order)
	std::vector<std::vector<u32> > lists(ix.end.size());
	for (size_t k = 0; k < recs.size(); ++k) {
		const u32 lo = ix.begin[recs[k].contig], hi = ix.begin[recs[k].contig + 1];
		u32 r = (u32) (std::lower_bound(ix.end.begin() + lo, ix.end.begin() + hi, recs[k].start) - ix.end.begin());
		for (; r < hi && ix.end[r] <= recs[k].end; ++r) lists[r].push_back((u32) k);
	}
	for (size_t r = 0; r < lists.size(); ++r) { ix.items.insert(ix.items.end(), lists[r].begin(), lists[r].end()); ix.off.push_back((u32) ix.items.size()); }
	if (ix.items.empty()) ix.items.push_back(0);
	// search grid: per contig, for every 4,096-base bin the first region that ends at or after the bin's first position
	ix.grid.clear(); ix.grid_begin.assign(n_contigs + 1, 0);
	for (size_t c = 0; c < n_contigs; ++c) {
		ix.grid_begin[c] = (u32) ix.grid.size();
		const u32 lo = ix.begin[c], hi = ix.begin[c + 1];
		const u32 bins = (hi > lo && ix.end[hi - 1] >= 0 ? ((u32) ix.end[hi - 1] >> REGION_GRID_SHIFT) : 0u) + 1;
		u32 r = lo;
		for (u32 b = 0; b < bins; ++b) { const i64 first_pos = (i64) b << REGION_GRID_SHIFT; while (r < hi && ix.end[r] < first_pos) ++r; ix.grid.push_back(r); }
		ix.grid.push_back(hi);
	}
	ix.grid_begin[n_contigs] = (u32) ix.grid.size();
	if (ix.end.empty()) ix.end.push_back(0);
}

void refdata::build_exon_index() { build_index(exons, contig_ids.size(), exon_index); }
void refdata::build_gene_index() { build_index(genes, contig_ids.size(), gene_index); }

// arriba.cpp:166-184: a region's length is credited to every gene that has an exon in it (once per run of equal genes in set order)
void refdata::compute_exonic_lengths() {
	for (size_t g = 0; g < genes.size(); ++g) if (!genes[g].is_dummy) genes[g].exonic_length = 0;
	const size_t n_contigs = contig_ids.size();
	for (size_t c = 0; c < n_contigs; ++c) {
		i32 region_start = 0;
		for (u32 r = exon_index.begin[c]; r < exon_index.begin[c + 1]; ++r) {
			i32 previous = -1;
			for (u32 k = exon_index.off[r]; k < exon_index.off[r + 1]; ++k) {
				const i32 g = (i32) exons[exon_index.items[k]].gene;
				if (g != previous) { genes[g].exonic_length += exon_index.end[r] - region_start; previous = g; }
			}
			region_start = exon_index.end[r];
		}
	}
	for (size_t g = 0; g < genes.size(); ++g) if (genes[g].exonic_length == 0) genes[g].exonic_length = genes[g].end - genes[g].start;
}

void refdata::set_contig_flags(const std::string& interesting, const std::string& viral) {
	contig_flags.assign(contig_ids.size(), 0);
	for (std::map<std::string, u16>::iterator c = contig_ids.begin(); c != contig_ids.end(); ++c)
		contig_flags[c->second] = (contig_matches(c->first, interesting) ? CF_INTERESTING : 0) | (contig_matches(c->first, viral) ? CF_VIRAL : 0);
}

void refdata::flatten() {
	const size_t ng = genes.size(), ne = exons.size();
	f_gene_contig.resize(ng); f_gene_start.resize(ng); f_gene_end.resize(ng); f_gene_exonic_length.resize(ng); f_gene_strand.resize(ng); f_gene_flags.resize(ng);
	for (size_t g = 0; g < ng; ++g) {
		f_gene_contig[g] = genes[g].contig; f_gene_start[g] = genes[g].start; f_gene_end[g] = genes[g].end; f_gene_exonic_length[g] = genes[g].exonic_length;
		f_gene_strand[g] = genes[g].forward; f_gene_flags[g] = (genes[g].is_dummy ? GF_DUMMY : 0) | (genes[g].is_protein_coding ? GF_CODING : 0);
	}
	f_exon_gene.resize(ne); f_exon_start.resize(ne); f_exon_end.resize(ne); f_exon_cds_start.resize(ne); f_exon_cds_end.resize(ne); f_exon_next_start.resize(ne); f_exon_flags.resize(ne);
	for (size_t e = 0; e < ne; ++e) {
		f_exon_gene[e] = exons[e].gene; f_exon_start[e] = exons[e].start; f_exon_end[e] = exons[e].end; f_exon_cds_start[e] = exons[e].cds_start; f_exon_cds_end[e] = exons[e].cds_end;
		f_exon_next_start[e] = exons[e].next >= 0 ? exons[exons[e].next].start : -1;
		f_exon_flags[e] = (exons[e].prev != -1 ? EF_HAS_PREV : 0) | (exons[e].next != -1 ? EF_HAS_NEXT : 0);
	}
	f_seq_off.assign(seq_off.begin(), seq_off.end());
	f_seq_off.resize(contig_ids.size(), 0); seq_len.resize(contig_ids.size(), 0); contig_flags.resize(contig_ids.size(), 0);
}

annot_view refdata::host_view() {
	annot_view v;
	v.n_genes = (u32) genes.size(); v.gene_contig = f_gene_contig.data(); v.gene_start = f_gene_start.data(); v.gene_end = f_gene_end.data();
	v.gene_strand = f_gene_strand.data(); v.gene_exonic_length = f_gene_exonic_length.data(); v.gene_flags = f_gene_flags.data();
	v.n_exons = (u32) exons.size(); v.exon_gene = f_exon_gene.data(); v.exon_start = f_exon_start.data(); v.exon_end = f_exon_end.data();
	v.exon_cds_start = f_exon_cds_start.data(); v.exon_cds_end = f_exon_cds_end.data(); v.exon_next_start = f_exon_next_start.data(); v.exon_flags = f_exon_flags.data();
	v.n_contigs = (u32) contig_ids.size();
	v.exon_region_begin = exon_index.begin.data(); v.exon_region_end = exon_index.end.data(); v.exon_region_off = exon_index.off.data(); v.exon_region_items = exon_index.items.data();
	v.gene_region_begin = gene_index.begin.data(); v.gene_region_end = gene_index.end.data(); v.gene_region_off = gene_index.off.data(); v.gene_region_items = gene_index.items.data();
	v.exon_grid = exon_index.grid.data(); v.exon_grid_begin = exon_index.grid_begin.data(); v.gene_grid = gene_index.grid.data(); v.gene_grid_begin = gene_index.grid_begin.data();
	v.contig_flags = contig_flags.data(); v.contig_seq_off = f_seq_off.data(); v.contig_len = seq_len.data(); v.assembly = assembly.data();
	return v;
}

}} // namespace
