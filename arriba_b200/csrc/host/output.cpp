// output.cpp -- writer of fusions.tsv / fusions.discarded.tsv.
// Behavioural contract: write_fusions_to_file and helpers (output_fusions.cpp:25-1261; the gap filling of -I on the device, fill_gaps_hd.h),
// get_fusion_peptide_sequence / is_in_frame / get_reading_frame / translate_reference_protein (annotate_protein_domains.cpp:164-446).
// Tags (-t) and protein domains (-p) need database files that are not part of the reference repository; their columns are ".".
#include "pipeline.h"
#include "../annot_hd.h"
#include "index_query.h"
#include <algorithm>
#include <charconv>
#include <atomic>
#include <fcntl.h>
#include <sys/stat.h>
#include <sys/uio.h>
#include <unistd.h>
#include <chrono>
#include <cmath>
#include <cstring>
#include <deque>
#include <fstream>
#include <iostream>
#include <map>
#include <memory_resource>
#include <sstream>
#include <stdexcept>
#include <thread>
#include <tuple>
#include <unordered_map>

namespace arb { namespace host {

namespace {
static thread_local std::string* warning_sink = NULL;
struct output_laps { // ARB_TRACE=1: wall time of the parts of the writer, on stderr
	bool on; double last;
	static double now() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
	output_laps(): on(getenv("ARB_TRACE") != NULL), last(now()) {}
	void lap(const char* file, const char* what) { if (!on) return; const double t = now(); fprintf(stderr, "[laps] output %-10s %-34s %8.1f ms\n", file, what, (t - last) * 1e3); last = t; }
};
static int filters_by_name[38]; // filter ids in alphabetical order of their names (the reference keeps them in a std::map<string, ...>)
static void sort_filters_by_name() { for (int f = 0; f < 38; ++f) filters_by_name[f] = f; std::sort(filters_by_name, filters_by_name + 38, [](int a, int b) { return strcmp(FILTER_NAMES[a], FILTER_NAMES[b]) < 0; }); } // set by the formatting threads of writer::write

// Pileup column: what the reads show at one reference position -- a base, "-" (deleted), "_" / ">" / "<" (inside / start / end of an intron) or, for
// an insertion, the inserted bases plus the following one. The reference keeps a map<string, count> per position (output_fusions.cpp:22); almost all keys are
// single characters of a small alphabet, which get counters in an array; everything else goes to the map. entries() restores the map's iteration order.
struct pile_column {
	static const char* symbols() { return "-<=>ABCDGHKMNRSTVWY_"; } // ascending ASCII
	enum { N_SYMBOLS = 20 };
	unsigned int single[N_SYMBOLS]; std::map<std::string, unsigned int> other;
	pile_column() { for (int k = 0; k < N_SYMBOLS; ++k) single[k] = 0; }
	struct symbol_table { signed char at[256]; symbol_table() { for (int k = 0; k < 256; ++k) at[k] = -1; for (int k = 0; k < N_SYMBOLS; ++k) at[(unsigned char) symbols()[k]] = (signed char) k; } };
	static int index_of(char c) { static const symbol_table table; return table.at[(unsigned char) c]; } // a local static: initialised once, also when several threads arrive together
	void add(char c, unsigned int n = 1) { const int x = index_of(c); if (x >= 0) single[x] += n; else other[std::string(1, c)] += n; }
	void add(const std::string& s, unsigned int n = 1) { if (s.size() == 1) add(s[0], n); else other[s] += n; }
	unsigned int total() const { unsigned int t = 0; for (int k = 0; k < N_SYMBOLS; ++k) t += single[k]; for (std::map<std::string, unsigned int>::const_iterator it = other.begin(); it != other.end(); ++it) t += it->second; return t; }
	void entries(std::vector<std::pair<std::string, unsigned int> >& out) const { // ascending by key, like the reference's map
		out.clear();
		std::map<std::string, unsigned int>::const_iterator it = other.begin();
		for (int k = 0; k < N_SYMBOLS; ++k) {
			if (single[k] == 0) continue;
			const std::string key(1, symbols()[k]);
			while (it != other.end() && it->first < key) { out.push_back(*it); ++it; }
			out.push_back(std::make_pair(key, single[k]));
		}
		for (; it != other.end(); ++it) out.push_back(*it);
	}
};
// A pileup under construction. Per position only counters: 16-bit, one per symbol of pile_column (a candidate has at most a few hundred reads); positions
// within WINDOW bases of the breakpoint sit in a flat array (nearly all bases), the rest -- the inside of introns, filled position by position like the
// reference does -- in an open-addressing table; multi-base insertion strings are rare and kept aside. flatten() hands the columns over in ascending
// position as pile_column objects, which is all the consensus needs (the reference keeps a map of maps per pileup, output_fusions.cpp:22).
struct pile_cell { u16 n[pile_column::N_SYMBOLS]; };
struct column_ref { // one position of a finished pileup: the counters and, rarely, the multi-base keys; same iteration order as the reference's map
	const pile_cell* c; const std::map<std::string, unsigned int>* other;
	unsigned int total() const { unsigned int t = 0; for (int k = 0; k < pile_column::N_SYMBOLS; ++k) t += c->n[k]; if (other) for (std::map<std::string, unsigned int>::const_iterator it = other->begin(); it != other->end(); ++it) t += it->second; return t; }
	void entries(std::vector<std::pair<std::string, unsigned int> >& out) const {
		out.clear();
		static const std::map<std::string, unsigned int> none;
		const std::map<std::string, unsigned int>& o = other ? *other : none;
		std::map<std::string, unsigned int>::const_iterator it = o.begin();
		for (int k = 0; k < pile_column::N_SYMBOLS; ++k) {
			if (c->n[k] == 0) continue;
			const std::string key(1, pile_column::symbols()[k]);
			while (it != o.end() && it->first < key) { out.push_back(*it); ++it; }
			out.push_back(std::make_pair(key, (unsigned int) c->n[k]));
		}
		for (; it != o.end(); ++it) out.push_back(*it);
	}
};
typedef std::vector<std::pair<i32, column_ref> > pileup_t;
struct pile_builder {
	enum { WINDOW = 2048 };
	typedef pile_cell cell;
	i32 lo; std::vector<cell> dense; std::vector<u8> used; std::vector<u32> used_list;
	std::vector<i32> far_pos; std::vector<cell> far_cell; std::vector<u32> far_slot; // far_slot: open addressing, index + 1 into far_pos / far_cell, 0 = empty
	std::map<i32, std::map<std::string, unsigned int> > other;
	pile_builder(): lo(0), dense(2 * WINDOW), used(2 * WINDOW, 0), far_slot(1 << 12, 0) { memset(dense.data(), 0, dense.size() * sizeof(cell)); }
	void reset(i32 breakpoint) { // only what the previous pileup touched is cleaned
		for (size_t k = 0; k < used_list.size(); ++k) { memset(&dense[used_list[k]], 0, sizeof(cell)); used[used_list[k]] = 0; }
		used_list.clear(); other.clear(); lo = breakpoint - WINDOW;
		if (!far_pos.empty()) { if (far_slot.size() > (1u << 16)) far_slot.assign(1 << 12, 0); else std::fill(far_slot.begin(), far_slot.end(), 0u); far_pos.clear(); far_cell.clear(); }
	}
	cell& at(i32 pos) {
		const i64 x = (i64) pos - lo;
		if (x >= 0 && x < 2 * WINDOW) { if (!used[x]) { used[x] = 1; used_list.push_back((u32) x); } return dense[x]; }
		if ((far_pos.size() + 1) * 2 > far_slot.size()) { // grow and re-insert
			std::vector<u32> bigger(far_slot.size() * 2, 0); const size_t mask = bigger.size() - 1;
			for (size_t k = 0; k < far_pos.size(); ++k) { size_t h = ((u32) far_pos[k] * 2654435761u) & mask; while (bigger[h]) h = (h + 1) & mask; bigger[h] = (u32) k + 1; }
			far_slot.swap(bigger);
		}
		const size_t mask = far_slot.size() - 1; size_t h = ((u32) pos * 2654435761u) & mask;
		for (; far_slot[h]; h = (h + 1) & mask) if (far_pos[far_slot[h] - 1] == pos) return far_cell[far_slot[h] - 1];
		far_pos.push_back(pos); cell c; memset(&c, 0, sizeof(c)); far_cell.push_back(c); far_slot[h] = (u32) far_pos.size();
		return far_cell.back();
	}
	void add(i32 pos, char symbol, unsigned int n = 1) { const int x = pile_column::index_of(symbol); if (x >= 0) at(pos).n[x] = (u16) (at(pos).n[x] + n); else other[pos][std::string(1, symbol)] += n; }
	void add(i32 pos, const std::string& s) { if (s.size() == 1) add(pos, s[0]); else { at(pos); other[pos][s] += 1; } }
	void flatten(pileup_t& out) { // views into this builder, valid until the next reset()
		out.clear();
		std::vector<std::pair<i32, u32> > far; far.reserve(far_pos.size());
		for (size_t k = 0; k < far_pos.size(); ++k) far.push_back(std::make_pair(far_pos[k], (u32) k));
		std::sort(far.begin(), far.end());
		std::sort(used_list.begin(), used_list.end());
		auto column_of = [&](i32 pos, const cell& c) {
			column_ref r; r.c = &c; r.other = NULL;
			if (!other.empty()) { std::map<i32, std::map<std::string, unsigned int> >::const_iterator o = other.find(pos); if (o != other.end()) r.other = &o->second; }
			return std::make_pair(pos, r);
		};
		size_t k = 0;
		for (; k < far.size() && far[k].first < lo; ++k) out.push_back(column_of(far[k].first, far_cell[far[k].second]));
		for (size_t x = 0; x < used_list.size(); ++x) out.push_back(column_of(lo + (i32) used_list[x], dense[used_list[x]]));
		for (; k < far.size(); ++k) out.push_back(column_of(far[k].first, far_cell[far[k].second]));
	}
};

// The text of a slice of rows: what the writer needs of an output stream (operator<< for strings, characters and integers, write()), appending to one string.
// A std::ostringstream spends more time in its sentries and locale facets than the rows' own logic does (millions of discarded rows are pure formatting).
struct row_buffer {
	std::string s;
	row_buffer& operator<<(const char* x) { s.append(x); return *this; }
	row_buffer& operator<<(const std::string& x) { s.append(x); return *this; }
	row_buffer& operator<<(char c) { s.push_back(c); return *this; }
	row_buffer& operator<<(int v) { return number((long long) v); }
	row_buffer& operator<<(unsigned int v) { return number((unsigned long long) v); }
	row_buffer& operator<<(long v) { return number((long long) v); }
	row_buffer& operator<<(unsigned long v) { return number((unsigned long long) v); }
	row_buffer& operator<<(long long v) { return number(v); }
	row_buffer& operator<<(unsigned long long v) { return number(v); }
	void write(const char* p, size_t n) { s.append(p, n); }
private:
	template <class I> row_buffer& number(I v) { char b[24]; const std::to_chars_result r = std::to_chars(b, b + sizeof(b), v); s.append(b, (size_t) (r.ptr - b)); return *this; }
};

char comp_char(char c) { // assembly.hpp:9-22
	switch (c) {
		case 'a': return 't'; case 't': return 'a'; case 'c': return 'g'; case 'g': return 'c';
		case 'A': return 'T'; case 'T': return 'A'; case 'C': return 'G'; case 'G': return 'C';
		case '[': return ']'; case ']': return '['; default: return c;
	}
}
std::string revcomp(const std::string& s) { std::string r; r.reserve(s.size()); for (size_t i = s.size(); i-- > 0;) r += comp_char(s[i]); return r; }

struct writer {
	pipeline& p; const event_table& e; const refdata& ref; const frag_view f; const u32 N;
	explicit writer(pipeline& pl): p(pl), e(pl.ev), ref(pl.ref), f(pl.frags.view()), N(pl.frags.n) {}

	std::string read_sequence(u32 frag, u32 slot) const {
		const u32 a = f.idx(frag, slot); std::string s(f.seq_len[a], 'N'); const u8* q = f.sq(a);
		for (u32 i = 0; i < f.seq_len[a]; ++i) s[i] = nt16_char(nt16_at(q, i));
		return s;
	}
	bool has_assembly(u32 contig) const { return ref.has_sequence(contig); }

	// ---- pileup of the supporting reads around one breakpoint (output_fusions.cpp:25-107)
	void pileup_reads(const column<u32>& list, u32 lo, u32 hi, u32 mate, bool reverse_complement, u32 direction, i32 breakpoint, pile_builder& pileup) const {
		std::map<std::pair<i32, i32>, unsigned int> introns;
		for (u32 x = lo; x < hi; ++x) {
			// the supporting fragments of a candidate lie all over the fragment table: the columns of the ones a few steps ahead are requested early, then
			// (once the offsets have arrived) their CIGAR and sequence
			if (x + 8 < hi) {
				const u32 g = list[x + 8], ga = f.idx(g, mate), gs = f.idx(g, mate == SUPPLEMENTARY ? SPLIT_READ : mate);
				__builtin_prefetch(&p.labels[g]); __builtin_prefetch(&f.n_aln[g]); __builtin_prefetch(&f.start[ga]); __builtin_prefetch(&f.end[ga]); __builtin_prefetch(&f.aflags[ga]);
				__builtin_prefetch(&f.cigar_off[ga]); __builtin_prefetch(&f.cigar_cnt[ga]); __builtin_prefetch(&f.seq_off[gs]); __builtin_prefetch(&f.seq_len[gs]);
			}
			if (x + 4 < hi) {
				const u32 g = list[x + 4], ga = f.idx(g, mate), gs = f.idx(g, mate == SUPPLEMENTARY ? SPLIT_READ : mate);
				__builtin_prefetch(f.cig(ga)); __builtin_prefetch(f.sq(gs)); __builtin_prefetch(f.sq(gs) + 48);
			}
			const u32 frag = list[x];
			if (p.labels[frag] == F_duplicates) continue;
			const u32 a = f.idx(frag, mate);
			const bool fwd = f.fwd(a);
			if (f.n_aln[frag] == 2 && !((direction == DOWNSTREAM && fwd && f.end[a] <= breakpoint + 2 && f.end[a] >= breakpoint - 200) || (direction == UPSTREAM && !fwd && f.start[a] >= breakpoint - 2 && f.start[a] <= breakpoint + 200))) continue;
			if (f.n_aln[frag] == 3 && (mate == SPLIT_READ || mate == SUPPLEMENTARY) && f.start[a] != breakpoint && f.end[a] != breakpoint) continue;
			// bases are decoded on the fly (reverse-complemented when the supplementary lies on the other strand): no per-read strings
			const u32 sa = f.idx(frag, mate == SUPPLEMENTARY ? SPLIT_READ : mate);
			const u8* const packed = f.sq(sa); const size_t seq_size = f.seq_len[sa];
			static const struct symbol_table { u8 v[32]; symbol_table() { for (u32 c = 0; c < 16; ++c) { v[c] = (u8) pile_column::index_of(nt16_char(c)); v[16 + c] = (u8) pile_column::index_of(comp_char(nt16_char(c))); } } } symbols;
			const u8* const symbol_of_code = symbols.v; // counter index of a base code, as read (0-15) and reverse-complemented (16-31)
			auto base_at = [&](size_t off) { return reverse_complement ? comp_char(nt16_char(nt16_at(packed, (u32) (seq_size - 1 - off)))) : nt16_char(nt16_at(packed, (u32) off)); };
			i32 read_off = 0, ref_off = f.start[a]; int carry = 0; // carry: one base was already consumed by a preceding insertion
			const u32* c = f.cig(a); const u32 nc = f.cigar_cnt[a];
			auto piece = [&](i32 off, size_t n) { std::string s; if ((size_t) off <= seq_size) for (size_t x = (size_t) off; x < seq_size && x < (size_t) off + n; ++x) s += base_at(x); return s; };
			for (u32 k = 0; k < nc; ++k) {
				const u32 op = cig_op(c[k]); const i32 len = (i32) cig_len(c[k]);
				bool as_match = false;
				switch (op) {
					case C_I: pileup.add(ref_off, piece(read_off, len + 1)); read_off += len + 1; ++ref_off; carry = 1; break;
					case C_N: { const i32 s0 = ref_off; ref_off += len - carry; ++introns[std::make_pair(s0, ref_off - 1)]; carry = 0; break; }
					case C_D: for (i32 b = 0; b < len - carry; ++b, ++ref_off) pileup.add(ref_off, '-'); carry = 0; break;
					case C_H: if (mate == SUPPLEMENTARY) read_off += len; break;
					case C_S:
						if (f.n_aln[frag] == 3 && mate == SPLIT_READ && ((k == 0 && fwd) || (k == nc - 1 && !fwd))) { if (k == 0 && fwd) ref_off -= len; as_match = true; } // clipped segment joins the pileup (non-template bases)
						else read_off += len - carry;
						break;
					case C_M: case C_EQ: case C_X: as_match = true; break;
					default: break;
				}
				if (as_match) {
					const i32 run = len - carry;
					const i64 x0 = (i64) ref_off - pileup.lo;
					if (run > 0 && read_off >= 0 && (size_t) read_off + (size_t) run <= seq_size && x0 >= 0 && x0 + run <= 2 * pile_builder::WINDOW) {
						// the whole block lies in the flat window and inside the read: claim the cells once, then one counter per base without any checks
						for (i32 b = 0; b < run; ++b) if (!pileup.used[x0 + b]) { pileup.used[x0 + b] = 1; pileup.used_list.push_back((u32) (x0 + b)); }
						pile_builder::cell* const cells = &pileup.dense[x0];
						if (reverse_complement) for (i32 b = 0; b < run; ++b) ++cells[b].n[symbol_of_code[16 + nt16_at(packed, (u32) (seq_size - 1 - (size_t) (read_off + b)))]];
						else for (i32 b = 0; b < run; ++b) ++cells[b].n[symbol_of_code[nt16_at(packed, (u32) (read_off + b))]];
						read_off += run; ref_off += run;
					} else
					for (i32 b = 0; b < len - carry; ++b, ++read_off, ++ref_off) { // the hot loop of the writer: one counter per base
						if ((size_t) read_off < seq_size) ++pileup.at(ref_off).n[symbol_of_code[reverse_complement ? nt16_at(packed, (u32) (seq_size - 1 - read_off)) + 16 : nt16_at(packed, (u32) read_off)]];
						else pileup.add(ref_off, std::string());
					}
					carry = 0;
				}
			}
		}
		for (std::map<std::pair<i32, i32>, unsigned int>::iterator it = introns.begin(); it != introns.end(); ++it) {
			pileup.add(it->first.first, '>', it->second); pileup.add(it->first.second, '<', it->second);
			const int inside = pile_column::index_of('_');
			for (i32 i = it->first.first + 1; i < it->first.second; ++i) { u16& n = pileup.at(i).n[inside]; n = (u16) (n + it->second); }
		}
	}

	// ---- consensus of a pileup (output_fusions.cpp:109-240)
	void consensus(const pileup_t& pileup, i32 breakpoint, u32 direction, u32 gene, std::string& sequence, std::vector<i32>& positions, std::string& clipped) const {
		unsigned int peak = 0;
		for (pileup_t::const_iterator pos = pileup.begin(); pos != pileup.end(); ++pos) { const unsigned int cov = pos->second.total(); if (cov > peak) peak = cov; }
		const float low_fraction = 0.10f;
		pileup_t::const_iterator first = pileup.begin(), last = pileup.end();
		for (pileup_t::const_iterator pos = pileup.begin(); pos != pileup.end(); ++pos) {
			const unsigned int cov = pos->second.total();
			if (direction == DOWNSTREAM) { if (cov < peak * low_fraction) first = pos; else break; }
			else if (cov > peak * low_fraction) last = pos;
		}
		if (last != pileup.end()) ++last;
		bool intron_open = false, intron_closed = true;
		const u32 contig = ref.genes[gene].contig;
		std::vector<std::pair<std::string, unsigned int> > column;
		for (pileup_t::const_iterator pos = first; pos != last; ++pos) {
			if (pos != first && std::prev(pos)->first < pos->first - 1 && !intron_open) { sequence += "..."; positions.resize(positions.size() + 3, -1); }
			std::string ref_base = "N";
			if (has_assembly(contig) && (u32) pos->first < ref.seq_len[contig]) ref_base = std::string(1, ref.sequence(contig)[pos->first]);
			pos->second.entries(column);
			auto best = column.end(); unsigned int cov = 0;
			for (auto b = column.begin(); b != column.end(); ++b) {
				const bool is_intron = b->first == "_" || b->first == ">" || b->first == "<";
				if (best == column.end() || b->second > best->second ||
				    (b->second == best->second && ((b->first == ref_base && best->first != "_" && best->first != ">" && best->first != "<") || (b->first == "<" && best->first != "_" && best->first != ">") || (b->first == "_" || b->first == ">")))) best = b;
				if (!is_intron) cov += b->second;
			}
			std::string call = (((best->first == "_" || best->first == ">" || best->first == "<") && best->second >= cov) || best->second >= 0.75 * cov || best->first == ref_base) ? best->first : "?";
			if (call == "_") { if (!intron_open) { sequence += "...___"; positions.resize(positions.size() + 6, -1); intron_open = true; intron_closed = false; } }
			else if (call == ">") { if (!intron_open) { sequence += "___"; positions.resize(positions.size() + 3, -1); intron_open = true; intron_closed = false; } }
			else if (call == "<") { if (!intron_open) { sequence += "...___"; positions.resize(positions.size() + 6, -1); } intron_open = true; intron_closed = true; }
			else {
				if (!intron_closed) { sequence += "..."; positions.resize(positions.size() + 3, -1); }
				intron_open = false; intron_closed = true;
				if (call.size() > 1 || (call != ref_base && ref_base != "N")) for (size_t i = 0; i < call.size(); ++i) call[i] = (char) tolower(call[i]);
				if (call.size() > 1) { // insertion: [inserted]next
					call = "[" + call.substr(0, call.size() - 1) + "]" + call[call.size() - 1];
					positions.resize(positions.size() + call.size() - 1, -1);
					if (toupper(call[call.size() - 1]) == ref_base[0]) call[call.size() - 1] = (char) toupper(call[call.size() - 1]);
				}
				if ((direction == UPSTREAM && pos->first < breakpoint) || (direction == DOWNSTREAM && pos->first > breakpoint)) clipped += call;
				else { sequence += call; positions.push_back(pos->first); }
			}
		}
	}

	static bool lower_acgt(char c) { return c == 'a' || c == 't' || c == 'c' || c == 'g'; }

	// ---- fusion transcript (output_fusions.cpp:242-466)
	// the two consensus sequences of a candidate with the positions of their characters, the bases beyond the breakpoints, and the non-template count:
	// from the device (csrc/consensus_hd.h) or, for the rows it left over, from the pileups below
	struct side_strings { std::string s1, s2, c1, c2; std::vector<i32> p1, p2; unsigned int non_template; };
	bool transcript_unknown(u32 k) const { return (e.bits[k] & CB_PSTRANDS_AMBIGUOUS) || (e.bits2[k] & 1); }
	void transcript_sequence(u32 k, std::string& sequence, std::vector<i32>& positions, const side_strings* from_device = NULL) const {
		if (transcript_unknown(k)) { sequence = "."; positions.push_back(-1); return; }
		if (from_device) { side_strings copy = *from_device; finish_transcript(k, copy, sequence, positions); return; }
		side_strings sides; host_sides(k, sides); finish_transcript(k, sides, sequence, positions);
	}
	void host_sides(u32 k, side_strings& out) const {
		const u32 d1 = e.dir1[k], d2 = e.dir2[k]; const i32 bp1 = e.bp1[k], bp2 = e.bp2[k];
		static thread_local pile_builder build1, build2;
		pile_builder& pile1 = build1; pile_builder& pile2 = build2;
		pile1.reset(bp1); pile2.reset(bp2);
		const u32 a1 = e.list1_off[k], b1 = e.list1_off[k + 1], a2 = e.list2_off[k], b2 = e.list2_off[k + 1], ad = e.listd_off[k], bd = e.listd_off[k + 1];
		pileup_reads(e.list1, a1, b1, SPLIT_READ, false, d1, bp1, pile1);
		pileup_reads(e.list1, a1, b1, MATE1, false, d1, bp1, pile1);
		pileup_reads(e.list1, a1, b1, SUPPLEMENTARY, d1 == d2, d2, bp2, pile2);
		pileup_reads(e.list2, a2, b2, SPLIT_READ, false, d2, bp2, pile2);
		pileup_reads(e.list2, a2, b2, MATE1, false, d2, bp2, pile2);
		pileup_reads(e.list2, a2, b2, SUPPLEMENTARY, d1 == d2, d1, bp1, pile1);
		pileup_reads(e.listd, ad, bd, MATE1, false, d1, bp1, pile1);
		pileup_reads(e.listd, ad, bd, MATE2, false, d1, bp1, pile1);
		pileup_reads(e.listd, ad, bd, MATE1, false, d2, bp2, pile2);
		pileup_reads(e.listd, ad, bd, MATE2, false, d2, bp2, pile2);
		// non-template bases between the fused segments: most frequent surplus of clipped bases over the read length
		unsigned int non_template = 0; std::map<unsigned int, unsigned int> count;
		for (int which = 0; which < 2; ++which) {
			const column<u32>& list = which == 0 ? e.list1 : e.list2;
			for (u32 x = which == 0 ? a1 : a2; x < (which == 0 ? b1 : b2); ++x) {
				const u32 s = f.idx(list[x], SPLIT_READ), u = f.idx(list[x], SUPPLEMENTARY);
				const unsigned int cs = f.fwd(s) ? f.preclip(s) : f.postclip(s), cu = f.fwd(u) ? f.postclip(u) : f.preclip(u);
				if (cs + cu >= f.seq_len[s]) { const unsigned int unmapped = cs + cu - f.seq_len[s]; if (++count[unmapped] > count[non_template]) non_template = unmapped; }
			}
		}
		pileup_t columns;
		pile1.flatten(columns); consensus(columns, bp1, d1, e.gene1[k], out.s1, out.p1, out.c1);
		pile2.flatten(columns); consensus(columns, bp2, d2, e.gene2[k], out.s2, out.p2, out.c2);
		out.non_template = non_template;
	}
	void finish_transcript(u32 k, side_strings& sides, std::string& sequence, std::vector<i32>& positions) const {
		const u32 d1 = e.dir1[k], d2 = e.dir2[k];
		std::string& s1 = sides.s1; std::string& s2 = sides.s2; std::string& c1 = sides.c1; std::string& c2 = sides.c2; std::vector<i32>& p1 = sides.p1; std::vector<i32>& p2 = sides.p2;
		const unsigned int non_template = sides.non_template;
		if (e.n_list1(k) + e.n_list2(k) == 0) { // breakpoints are not known exactly
			if (d1 == DOWNSTREAM) { s1 += "..."; p1.resize(p1.size() + 3, -1); } else { s1 = "..." + s1; p1.insert(p1.begin(), 3, -1); }
			if (d2 == DOWNSTREAM) { s2 += "..."; p2.resize(p2.size() + 3, -1); } else { s2 = "..." + s2; p2.insert(p2.begin(), 3, -1); }
		}
		if (non_template > 0) {
			auto lower = [](std::string& s) { for (size_t i = 0; i < s.size(); ++i) s[i] = (char) tolower(s[i]); };
			if (c1.size() >= non_template) {
				lower(c1);
				if (d1 == UPSTREAM) { s1 = c1.substr(c1.size() - non_template) + s1; p1.insert(p1.begin(), non_template, -1); } else { s1 += c1.substr(0, non_template); p1.resize(p1.size() + non_template, -1); }
			} else if (c2.size() >= non_template) {
				lower(c2);
				if (d2 == UPSTREAM) { s2 = c2.substr(c2.size() - non_template) + s2; p2.insert(p2.begin(), non_template, -1); } else { s2 += c2.substr(0, non_template); p2.resize(p2.size() + non_template, -1); }
			}
		}
		// mismatching (lower-case) bases right at the junction are set off by a pipe
		auto mark = [&](std::string& s, std::vector<i32>& pos, u32 direction) {
			if (direction == UPSTREAM) {
				int b = 0; while (b < (int) s.size() && lower_acgt(s[b])) ++b;
				if (b > 0 && b < (int) s.size()) { s = s.substr(0, b) + "|" + s.substr(b); std::fill(pos.begin(), pos.begin() + b, -1); pos.insert(pos.begin() + b, -1); return true; }
			} else {
				int b = (int) s.size() - 1; while (b >= 0 && lower_acgt(s[b])) --b;
				if (b + 1 < (int) s.size() && b >= 0) { s = s.substr(0, b + 1) + "|" + s.substr(b + 1); std::fill(pos.begin() + b + 1, pos.end(), -1); pos.insert(pos.begin() + b + 1, -1); return true; }
			}
			return false;
		};
		const bool nt1 = mark(s1, p1, d1), nt2 = mark(s2, p2, d2);
		const bool ps1 = e.bits[k] & CB_PSTRAND1, ps2 = e.bits[k] & CB_PSTRAND2;
		if (e.bits[k] & CB_TSTART_GENE1) {
			sequence = ps1 ? s1 : revcomp(s1); if (!ps1) std::reverse(p1.begin(), p1.end()); positions = p1;
			if (!nt1 || !nt2) { sequence += "|"; positions.push_back(-1); }
			sequence += d2 == UPSTREAM ? s2 : revcomp(s2); if (d2 != UPSTREAM) std::reverse(p2.begin(), p2.end());
			positions.insert(positions.end(), p2.begin(), p2.end());
		} else {
			sequence = ps2 ? s2 : revcomp(s2); if (!ps2) std::reverse(p2.begin(), p2.end()); positions = p2;
			if (!nt2 || !nt1) { sequence += "|"; positions.push_back(-1); }
			sequence += d1 == UPSTREAM ? s1 : revcomp(s1); if (d1 != UPSTREAM) std::reverse(p1.begin(), p1.end());
			positions.insert(positions.end(), p1.begin(), p1.end());
		}
		// "...A..." and the like collapse to "..."
		size_t e1 = 0, e2 = std::string::npos;
		while ((e1 = sequence.find("...", e1)) < sequence.size()) {
			if ((e2 = sequence.find("...", e1 + 3)) < e1 + 10 + 3 && sequence.find('|', e1 + 3) > e2) { sequence.replace(e1 + 3, e2 - e1, ""); positions.erase(positions.begin() + e1 + 3, positions.begin() + e2 + 3); }
			else e1 += 3;
		}
		static const char* simplify[][2] = {{"...___|", "|"}, {"|___...", "|"}, {"___|", "...|"}, {"|___", "|..."}, {"______", "___"}, {"___...___", "___"}, {"...___...", "..."}, {"......", "..."}};
		size_t at = std::string::npos;
		do {
			for (size_t r = 0; r < 8; ++r) {
				const std::string from = simplify[r][0], to = simplify[r][1];
				if ((at = sequence.find(from)) < sequence.size()) { sequence.replace(at, from.size(), to); if (from.size() > to.size()) positions.erase(positions.begin() + at, positions.begin() + at + from.size() - to.size()); break; }
			}
		} while (at != std::string::npos);
		while (sequence.substr(0, 3) == "..." || sequence.substr(0, 3) == "___") { sequence = sequence.substr(3); positions.erase(positions.begin(), positions.begin() + 3); }
		while (sequence.size() >= 3 && (sequence.substr(sequence.size() - 3) == "..." || sequence.substr(sequence.size() - 3) == "___")) { sequence = sequence.substr(0, sequence.size() - 3); positions.erase(positions.begin() + positions.size() - 3, positions.end()); }
		if (sequence == "" || sequence == "|" || sequence == "...|" || sequence == "|..." || sequence == "...|...") { sequence = "."; positions.clear(); positions.push_back(-1); return; }
		for (size_t i = 0; i < sequence.size(); ++i) if (sequence[i] == 'n' || sequence[i] == 'N') sequence[i] = '?';
	}

	// ---- annotated transcripts matching the transcribed bases (output_fusions.cpp:720-818)
	void matching_transcripts(const std::string& seq, const std::vector<i32>& bases, u32 gene, bool strand, bool strand_ambiguous, int which_end, std::vector<i32>& best) const {
		if (strand_ambiguous || strand != ref.genes[gene].forward) return;
		size_t from, to, breakpoint;
		if (which_end == 5) {
			from = 0; to = seq.find('|'); if (to >= seq.size()) return;
			while (to > 0 && bases[to] == -1) --to;
			if (bases[to] == -1) return;
			breakpoint = to;
		} else {
			from = seq.find_last_of('|');
			while (from < seq.size() && bases[from] == -1) ++from;
			if (from >= seq.size()) return;
			breakpoint = from; to = seq.size() - 1;
		}
		if (bases[from] > bases[to]) std::swap(from, to);
		std::map<u32, unsigned int> score, peak, utr; std::map<u32, bool> coding_at_bp;
		const region_index& ix = ref.exon_index;
		const u32 contig = ref.genes[gene].contig, lo = ix.begin[contig], hi = ix.begin[contig + 1];
		size_t position = from;
		const size_t pmin = std::min(from, to), pmax = std::max(from, to);
		for (u32 r = (u32) (std::lower_bound(ix.end.begin() + lo, ix.end.begin() + hi, bases[from]) - ix.end.begin()); r < hi && position >= pmin && position <= pmax; ++r) {
			i32 last_transcribed = bases[to];
			while (position >= pmin && position <= pmax && bases[position] <= ix.end[r]) {
				for (u32 x = ix.off[r]; x < ix.off[r + 1]; ++x) {
					const u32 ex = ix.items[x]; const exon_rec& E = ref.exons[ex];
					if (E.gene != gene || bases[position] < E.start || bases[position] > E.end) continue;
					const transcript_rec& T = ref.transcripts[E.transcript];
					++score[E.transcript]; last_transcribed = bases[position];
					if ((i32) ex == T.first_exon || (i32) ex == T.last_exon) ++utr[E.transcript];
					if (position == breakpoint) {
						if (bases[position] >= E.cds_start && bases[position] <= E.cds_end) coding_at_bp[E.transcript] = true;
						if ((std::abs(bases[position] - E.start) <= 2 && (i32) ex != T.first_exon) || (std::abs(bases[position] - E.end) <= 2 && (i32) ex != T.last_exon)) score[E.transcript] += 10;
					}
				}
				position += (from <= to) ? +1 : -1;
			}
			for (u32 x = ix.off[r]; x < ix.off[r + 1]; ++x) {
				const exon_rec& E = ref.exons[ix.items[x]];
				if (E.gene != gene) continue;
				peak[E.transcript] = std::max(score[E.transcript], peak[E.transcript]);
				const i32 exon_start = r != lo ? ix.end[r - 1] : E.start - 1;
				const unsigned int exon_length = std::min(ix.end[r], bases[to]) - std::max(last_transcribed + 1, exon_start) + 1;
				score[E.transcript] -= std::min(exon_length, score[E.transcript]);
			}
		}
		if (peak.empty()) return;
		// the reference walks an unordered_map keyed by pointer; transcripts are visited in id order here
		best.push_back((i32) peak.begin()->first);
		for (std::map<u32, unsigned int>::iterator t = std::next(peak.begin()); t != peak.end(); ++t) {
			const u32 b0 = (u32) best[0];
			if (t->second == peak[b0] && coding_at_bp[b0] == coding_at_bp[t->first]) best.push_back((i32) t->first);
			else if (t->second > peak[b0] || (!coding_at_bp[b0] && coding_at_bp[t->first] && (t->second == peak[b0] || (utr[t->first] > 0 && utr[b0] > 0 && t->second - utr[t->first] >= peak[b0] - utr[b0])))) { best.clear(); best.push_back((i32) t->first); }
		}
		if (peak[(u32) best[0]] == 0) best.clear();
		std::sort(best.begin(), best.end(), [&](i32 x, i32 y) {
			const transcript_rec& X = ref.transcripts[x]; const transcript_rec& Y = ref.transcripts[y];
			const int lx = ref.exons[X.last_exon].end - ref.exons[X.first_exon].start, ly = ref.exons[Y.last_exon].end - ref.exons[Y.first_exon].start;
			return X.coding_length > Y.coding_length || (X.coding_length == Y.coding_length && lx > ly) || (X.coding_length == Y.coding_length && lx == ly && X.id < Y.id);
		});
		if (best.size() > 1) best.push_back(best[0]);
	}

	// ---- peptide (annotate_protein_domains.cpp:164-400)
	static char translate(const std::string& triplet) {
		// all three letters plain bases: table built once from the general rule below
		struct codon_table { char aa[64]; codon_table() { static const char L[] = "ACGT"; for (int x = 0; x < 64; ++x) { std::string t3; t3 += L[x >> 4]; t3 += L[x >> 2 & 3]; t3 += L[x & 3]; aa[x] = translate_general(t3); } } };
		static const codon_table table; // initialised once, by whichever row-formatting thread comes first (the language guards the initialisation of a local static)
		auto code = [](char c) { switch (c) { case 'A': case 'a': return 0; case 'C': case 'c': return 1; case 'G': case 'g': return 2; case 'T': case 't': return 3; default: return -1; } };
		if (triplet.size() == 3) { const int a = code(triplet[0]), b = code(triplet[1]), c = code(triplet[2]); if (a >= 0 && b >= 0 && c >= 0) return table.aa[a << 4 | b << 2 | c]; }
		return translate_general(triplet);
	}
	static char translate_general(const std::string& triplet) {
		std::string t = triplet; for (size_t i = 0; i < t.size(); ++i) t[i] = (char) toupper(t[i]);
		const std::string d = t.substr(0, 2);
		if (d == "GC") return 'A'; if (t == "TGT" || t == "TGC") return 'C'; if (t == "GAT" || t == "GAC") return 'D'; if (t == "GAA" || t == "GAG") return 'E';
		if (t == "TTT" || t == "TTC") return 'F'; if (d == "GG") return 'G'; if (t == "CAT" || t == "CAC") return 'H'; if (t == "ATT" || t == "ATC" || t == "ATA") return 'I';
		if (t == "AAA" || t == "AAG") return 'K'; if (d == "CT" || t == "TTA" || t == "TTG") return 'L'; if (t == "ATG") return 'M'; if (t == "AAT" || t == "AAC") return 'N';
		if (d == "CC") return 'P'; if (t == "CAA" || t == "CAG") return 'Q'; if (d == "CG" || t == "AGA" || t == "AGG") return 'R'; if (d == "TC" || t == "AGT" || t == "AGC") return 'S';
		if (d == "AC") return 'T'; if (d == "GT") return 'V'; if (t == "TGG") return 'W'; if (t == "TAT" || t == "TAC") return 'Y'; if (t == "TAA" || t == "TAG" || t == "TGA") return '*';
		return '?';
	}
	i32 next_in_transcript(i32 ex, bool forward) const { if (ex < 0) return -1; const i32 n = forward ? ref.exons[ex].next : ref.exons[ex].prev; return n >= 0 ? n : -1; }
	// amino acid at the genomic position of the last base of every codon of a transcript, with the warning the reference prints while translating it
	struct protein_t {
		std::vector<std::pair<i32, char> > by_pos; std::string warning;
		const char* find(i32 pos) const { std::vector<std::pair<i32, char> >::const_iterator it = std::lower_bound(by_pos.begin(), by_pos.end(), std::make_pair(pos, (char) 0)); return it != by_pos.end() && it->first == pos ? &it->second : NULL; }
	};
	const protein_t& cached_protein(i32 start_exon) const { // per thread; the same transcripts recur in consecutive rows
		static thread_local std::unordered_map<i32, protein_t> cache; static thread_local const void* owner = NULL;
		if (owner != this || cache.size() > 512) { cache.clear(); owner = this; }
		std::unordered_map<i32, protein_t>::iterator it = cache.find(start_exon);
		if (it == cache.end()) {
			protein_t pr; std::map<i32, char> m; std::string* const outer = warning_sink; warning_sink = &pr.warning;
			reference_protein(start_exon, m);
			warning_sink = outer;
			pr.by_pos.assign(m.begin(), m.end());
			it = cache.insert(std::make_pair(start_exon, pr)).first;
		}
		if (!it->second.warning.empty()) { if (warning_sink) *warning_sink += it->second.warning; else std::cerr << it->second.warning; } // printed on every use, like the reference
		return it->second;
	}
	void reference_protein(i32 start_exon, std::map<i32, char>& protein) const {
		if (start_exon < 0) return;
		const bool fwd = ref.genes[ref.exons[start_exon].gene].forward;
		const char* seq = ref.sequence(ref.genes[ref.exons[start_exon].gene].contig);
		std::string codon; bool reported = false;
		for (i32 ex = start_exon; ex >= 0; ex = next_in_transcript(ex, fwd)) {
			const exon_rec& E = ref.exons[ex];
			for (i32 pos = fwd ? E.cds_start : E.cds_end; pos != -1 && pos >= E.cds_start && pos <= E.cds_end; pos += fwd ? +1 : -1) {
				codon += fwd ? seq[pos] : comp_char(seq[pos]);
				if (codon.size() == 3) {
					protein[pos] = translate(codon); codon.clear();
					if (!reported && pos < E.cds_end && pos > E.cds_start && protein[pos] == '*') {
						std::ostringstream w; w << "WARNING: encountered early stop codon in transcript " << ref.transcripts[E.transcript].name << " at amino acid " << protein.size() << " (error in GTF file?) => predicted peptide sequence may be wrong\n";
						if (warning_sink) *warning_sink += w.str(); else std::cerr << w.str();
						reported = true;
					}
				}
			}
		}
	}
	int reading_frame(const std::vector<i32>& bases, int from, int to, i32 transcript, u32 gene, i32& start_exon) const {
		const bool fwd = ref.genes[gene].forward;
		start_exon = transcript < 0 ? -1 : (fwd ? ref.transcripts[transcript].first_exon : ref.transcripts[transcript].last_exon);
		while (start_exon >= 0 && ref.exons[start_exon].cds_start == -1) start_exon = next_in_transcript(start_exon, fwd);
		if (start_exon < 0) return -1;
		const u32 contig = ref.genes[gene].contig;
		std::string first_codon;
		{
			const i64 at = fwd ? (i64) ref.exons[start_exon].cds_start : (i64) ref.exons[start_exon].cds_end - 2;
			for (i64 x = at; x < at + 3; ++x) if (x >= 0 && x < (i64) ref.seq_len[contig]) first_codon += ref.sequence(contig)[x];
			if (!fwd) first_codon = revcomp(first_codon);
		}
		if (first_codon != "ATG") return -1;
		int frame = -1; i32 coding_base = -1;
		for (i32 ex = start_exon; ex >= 0 && ref.exons[ex].cds_start != -1 && coding_base == -1; ex = next_in_transcript(ex, fwd)) {
			const exon_rec& E = ref.exons[ex];
			for (int pos = from; pos <= to && coding_base == -1; ++pos) if (E.cds_start <= bases[pos] && E.cds_end >= bases[pos]) coding_base = pos;
			if (coding_base == -1) frame = (frame + E.cds_end - E.cds_start + 1) % 3;
			else { frame += fwd ? bases[coding_base] - E.cds_start : E.cds_end - bases[coding_base]; frame = (frame + 1) % 3; }
		}
		if (coding_base == -1) return -1;
		for (int pos = coding_base - 1; pos >= from; --pos) if (bases[pos] != -1) frame = frame == 0 ? 2 : frame - 1;
		return frame;
	}
	std::string peptide(const std::string& seq, const std::vector<i32>& pos, u32 gene5, u32 gene3, i32 tr5, i32 tr3, bool strand3) const {
		if (seq.empty() || seq == "." || seq.find("...|") < seq.size() || seq.find("|...") < seq.size()) return ".";
		if (!has_assembly(ref.genes[gene5].contig) || !has_assembly(ref.genes[gene3].contig)) return ".";
		size_t end5 = seq.find('|') - 1, start5 = seq.rfind("...", end5);
		if (start5 >= seq.size()) start5 = 0; else while (pos[start5] == -1 && seq[start5] != '|') ++start5;
		size_t nt_len = seq.find('|', end5 + 2);
		if (nt_len >= seq.size()) nt_len = 0; else nt_len -= end5 + 2;
		size_t start3 = end5 + 2; if (nt_len > 0) start3 += nt_len + 1;
		size_t end3 = seq.find("...", start3);
		if (end3 >= seq.size()) end3 = seq.size() - 1; else --end3;
		i32 ex5 = -1, ex3 = -1;
		int frame5 = reading_frame(pos, (int) start5, (int) end5, tr5, gene5, ex5);
		if (frame5 == -1) return "."; else if (frame5 != 0) frame5 = 3 - frame5;
		int frame3 = -1;
		if (ref.genes[gene3].forward == strand3) frame3 = reading_frame(pos, (int) start3, (int) end3, tr3, gene3, ex3);
		const protein_t& prot5 = cached_protein(ex5); const protein_t& prot3 = cached_protein(ex3);
		std::string pep; int c5 = 0, c3 = 0; bool started = false; std::string codon;
		const bool g5fwd = ref.genes[gene5].forward;
		for (size_t i = start5 + frame5; i < end3; ++i) {
			if (!started) {
				if (pos[i] != -1 && ((g5fwd && pos[i] >= ref.exons[ex5].cds_start) || (!g5fwd && pos[i] <= ref.exons[ex5].cds_end))) started = true; else continue;
			}
			const char ch = seq[i];
			if (ch == 'A' || ch == 'T' || ch == 'C' || ch == 'G' || ch == 'a' || ch == 't' || ch == 'c' || ch == 'g' || ch == '?') {
				if (codon.empty()) { c5 = 0; c3 = 0; }
				if (i <= end5) ++c5; else if (i >= start3) ++c3;
				codon += ch;
			}
			if (codon.size() == 3) {
				char aa = translate(codon);
				const protein_t& prot = i <= end5 ? prot5 : prot3;
				const char* hit = prot.find(pos[i]);
				if ((i > end5 && i < start3) || hit == NULL || aa != *hit || (c5 != 3 && i <= end5) || (c3 != 3 && i >= start3) || (i >= start3 && frame3 == -1)) aa = (char) tolower(aa);
				pep += aa; codon.clear();
				if (c3 >= 2 && aa == '*') break;
			}
			if ((i == end5 && codon.size() <= 1) || (c5 == 2 && codon.size() == 0)) if (pep.empty() || pep[pep.size() - 1] != '|') pep += '|';
			if (nt_len > 0 && ((i + 2 == start3 && codon.size() <= 1) || (c3 == 1 && codon.size() == 0))) if (pep.empty() || pep[pep.size() - 1] != '|') pep += '|';
		}
		return pep.empty() ? "." : pep;
	}
	static std::string frame_label(const std::string& pep) { // is_in_frame (annotate_protein_domains.cpp:402-446)
		if (pep == "." || pep.empty() || pep[pep.size() - 1] == '|') return ".";
		const size_t junction = pep.rfind('|'), stop = pep.rfind('*', junction);
		size_t start_after = pep.find('m', stop); if (start_after >= junction) start_after = pep.find('M', stop);
		if (stop < junction && start_after >= junction) return "stop-codon";
		auto upper_in = [&](size_t a, size_t b) { for (size_t i = a; i < b; ++i) if (pep[i] >= 'A' && pep[i] <= 'Z') return true; return false; };
		if (stop < junction && upper_in(0, stop) && !upper_in(stop + 1, junction)) return "stop-codon";
		const bool in5 = upper_in(stop < junction ? stop + 1 : 0, junction), in3 = upper_in(junction + 1, pep.size());
		return in5 && in3 ? "in-frame" : "out-of-frame";
	}

	// ---- small descriptive columns
	std::string gene_name(u32 gene, u32 contig, i32 bp) const { // output_fusions.cpp:498-545
		if (!ref.genes[gene].is_dummy) return ref.genes[gene].name;
		const region_index& ix = ref.gene_index; const u32 lo = ix.begin[contig], hi = ix.begin[contig + 1];
		const u32 hit = (u32) (std::lower_bound(ix.end.begin() + lo, ix.end.begin() + hi, bp) - ix.end.begin());
		auto annotated = [&](u32 r) { return ix.off[r + 1] > ix.off[r] && !ref.genes[ix.items[ix.off[r]]].is_dummy; };
		std::string result;
		i64 up = (i64) hit - 1; while (up >= (i64) lo && !annotated((u32) up)) --up;
		if (up >= (i64) lo) for (u32 x = ix.off[up]; x < ix.off[up + 1]; ++x) { const gene_rec& g = ref.genes[ix.items[x]]; if (g.is_dummy) continue; if (!result.empty()) result += ","; result += g.name + "(" + std::to_string((long long) (bp - g.end)) + ")"; }
		u32 down = hit; while (down < hi && !annotated(down)) ++down;
		if (down < hi) for (u32 x = ix.off[down]; x < ix.off[down + 1]; ++x) { const gene_rec& g = ref.genes[ix.items[x]]; if (g.is_dummy) continue; if (!result.empty()) result += ","; result += g.name + "(" + std::to_string((long long) (g.start - bp)) + ")"; }
		return result.empty() ? "." : result;
	}
	std::string fusion_type(u32 k) const { // output_fusions.cpp:547-633
		const gene_rec& g1 = ref.genes[e.gene1[k]]; const gene_rec& g2 = ref.genes[e.gene2[k]];
		const u32 d1 = e.dir1[k], d2 = e.dir2[k]; const bool dummy = g1.is_dummy || g2.is_dummy;
		if (e.contig1[k] != e.contig2[k]) {
			if (dummy || (d1 == d2 && g1.forward != g2.forward) || (d1 != d2 && g1.forward == g2.forward)) return "translocation";
			if (((d1 == UPSTREAM && g1.forward) || (d1 == DOWNSTREAM && !g1.forward)) && ((d2 == UPSTREAM && g2.forward) || (d2 == DOWNSTREAM && !g2.forward))) return "translocation/3'-3'";
			return "translocation/5'-5'";
		}
		const bool rt = e.is_read_through(k);
		if (d1 == DOWNSTREAM && d2 == UPSTREAM) {
			if (dummy || g1.forward == g2.forward) return rt ? "deletion/read-through" : "deletion";
			if (g1.forward || !g2.forward) return rt ? "deletion/read-through/5'-5'" : "deletion/5'-5'";
			return rt ? "deletion/read-through/3'-3'" : "deletion/3'-3'";
		}
		if (d1 == d2) { if (dummy || g1.forward != g2.forward) return "inversion"; return (d1 == UPSTREAM && !g1.forward) ? "inversion/5'-5'" : "inversion/3'-3'"; }
		if (dummy || g1.forward == g2.forward) {
			if (e.gene1[k] == e.gene2[k] && e.spliced1(k) && e.spliced2(k)) return "duplication/non-canonical_splicing";
			if (e.gene1[k] == e.gene2[k] && ((unsigned int) e.bp2[k] - (unsigned int) e.bp1[k]) < p.opt.params.max_itd_length && d1 == UPSTREAM && d2 == DOWNSTREAM) return "duplication/ITD";
			return "duplication";
		}
		return !g1.forward ? "duplication/5'-5'" : "duplication/3'-3'";
	}
	std::string strand_column(bool strand, u32 gene, bool ambiguous) const { std::string r = ref.genes[gene].is_dummy ? "." : (ref.genes[gene].forward ? "+" : "-"); r += "/"; r += ambiguous ? "." : (strand ? "+" : "-"); return r; }
	std::string site(u32 gene, bool spliced, bool exonic, u32 contig, i32 bp) const { // output_fusions.cpp:635-709
		const gene_rec& g = ref.genes[gene];
		if (g.is_dummy || bp < g.start || bp > g.end) return "intergenic";
		if (!exonic) return "intron";
		const annot_view an = const_cast<refdata&>(ref).host_view();
		bool overlapping = false, utr = true; unsigned int end3 = 0, end5 = 0;
		index_query<4096>(exon_index(an), contig, bp, bp, [&](const u32* exons, u32 n_exons) {
		for (u32 x = 0; x < n_exons; ++x) {
			const exon_rec& E = ref.exons[exons[x]];
			if (E.gene != gene) continue;
			overlapping = true;
			if (E.cds_start <= bp && E.cds_end >= bp) utr = false;
			if (utr && g.is_protein_coding) {
				if (E.cds_start != -1 && E.cds_start > bp) { if (g.forward) ++end5; else ++end3; }
				else if (E.cds_end != -1 && E.cds_end < bp) { if (!g.forward) ++end5; else ++end3; }
				else {
					i32 nx = E.next >= 0 ? E.next : -1; while (nx >= 0 && ref.exons[nx].cds_start == -1) nx = ref.exons[nx].next >= 0 ? ref.exons[nx].next : -1;
					i32 pv = E.prev >= 0 ? E.prev : -1; while (pv >= 0 && ref.exons[pv].cds_start == -1) pv = ref.exons[pv].prev >= 0 ? ref.exons[pv].prev : -1;
					if (pv >= 0 || nx >= 0) { if ((nx < 0) != (!g.forward)) ++end3; else ++end5; }
				}
			}
		}
		}, "too many overlapping annotation records at one locus");
		std::string s;
		if (!overlapping) s = "intron";
		else if (g.is_protein_coding) { if (utr) s = end3 > end5 ? "3'UTR" : end3 < end5 ? "5'UTR" : end3 + end5 == 0 ? "exon" : "UTR"; else s = "CDS"; }
		else s = "exon";
		if (spliced && s != "intron") s += "/splice-site";
		return s;
	}

	bool by_support(u32 x, u32 y) const { // output_fusions.cpp:468-483
		if (e.confidence[x] != e.confidence[y]) return e.confidence[x] > e.confidence[y];
		if (e.supporting_reads(x) != e.supporting_reads(y)) return e.supporting_reads(x) > e.supporting_reads(y);
		if (e.evalue[x] != e.evalue[y]) return e.evalue[x] < e.evalue[y];
		if (e.gene1[x] != e.gene1[y]) return e.gene1[x] < e.gene1[y];
		if (e.gene2[x] != e.gene2[y]) return e.gene2[x] < e.gene2[y];
		if (e.bp1[x] != e.bp1[y]) return e.bp1[x] < e.bp1[y];
		return e.bp2[x] < e.bp2[y];
	}

	// Rows are written in the reference's order (support, or the hash order of its candidate map), candidates and their reads therefore lie all over the
	// tables: the columns of a row a few rows ahead are requested early, then (once the list offsets have arrived) its first read lists and their labels.
	void prefetch_candidate(u32 k) const {
		__builtin_prefetch(&e.gene1[k]); __builtin_prefetch(&e.gene2[k]); __builtin_prefetch(&e.contig1[k]); __builtin_prefetch(&e.contig2[k]); __builtin_prefetch(&e.bp1[k]); __builtin_prefetch(&e.bp2[k]);
		__builtin_prefetch(&e.dir1[k]); __builtin_prefetch(&e.dir2[k]); __builtin_prefetch(&e.bits[k]); __builtin_prefetch(&e.filter[k]); __builtin_prefetch(&e.confidence[k]);
		__builtin_prefetch(&e.split_reads1[k]); __builtin_prefetch(&e.split_reads2[k]); __builtin_prefetch(&e.discordant_mates[k]);
		__builtin_prefetch(&e.list1_off[k]); __builtin_prefetch(&e.list2_off[k]); __builtin_prefetch(&e.listd_off[k]);
	}
	void prefetch_lists(u32 k) const { __builtin_prefetch(&e.list1[e.list1_off[k]]); __builtin_prefetch(&e.list2[e.list2_off[k]]); __builtin_prefetch(&e.listd[e.listd_off[k]]); __builtin_prefetch(&ref.genes[e.gene1[k]]); __builtin_prefetch(&ref.genes[e.gene2[k]]); }
	void prefetch_labels(u32 k) const {
		for (u32 r = e.list1_off[k]; r < e.list1_off[k + 1] && r < e.list1_off[k] + 8; ++r) __builtin_prefetch(&p.labels[e.list1[r]]);
		for (u32 r = e.list2_off[k]; r < e.list2_off[k + 1] && r < e.list2_off[k] + 8; ++r) __builtin_prefetch(&p.labels[e.list2[r]]);
		for (u32 r = e.listd_off[k]; r < e.listd_off[k + 1] && r < e.listd_off[k] + 8; ++r) __builtin_prefetch(&p.labels[e.listd[r]]);
	}

	// closest_genomic_breakpoint column (output_fusions.cpp:1195-1205)
	std::string genomic_breakpoint(u32 contig, i32 bp, i32 genomic) const {
		if (genomic < 0) return ".";
		return ref.original_names[contig] + ":" + std::to_string((long long) (genomic + 1)) + "(" + std::to_string((long long) std::abs(bp - genomic)) + ")";
	}

	// -I: the filled sides of one row (fill_gaps_hd.h), P5 per 5' transcript and S3 per 3' transcript, in a block of the writer's
	struct filled_row {
		struct half { i32 transcript; bool three; u32 off, len; };
		std::vector<half> halves; const std::string* chars; const std::vector<i32>* pos;
		filled_row(): chars(NULL), pos(NULL) {}
		const half* find(i32 t, bool three) const { for (size_t h = 0; h < halves.size(); ++h) if (halves[h].transcript == t && halves[h].three == three) return &halves[h]; return NULL; }
		// the sequence of the pair (t5, t3): P5 + seq[b5 .. b3] + S3 (a side without a transcript, -1, stays as it is)
		void assemble(i32 t5, i32 t3, const std::string& seq, const std::vector<i32>& positions, std::string& s, std::vector<i32>& p) const {
			s = seq; p = positions;
			const size_t b5 = seq.find('|'), b3 = seq.rfind('|');
			if (b5 >= seq.size()) return; // no transcripts: nothing to fill
			const half* h5 = t5 >= 0 ? find(t5, false) : NULL; const half* h3 = t3 >= 0 ? find(t3, true) : NULL;
			s.clear(); p.clear();
			if (h5) { s.append(*chars, h5->off, h5->len); p.insert(p.end(), pos->begin() + h5->off, pos->begin() + h5->off + h5->len); }
			else { s.append(seq, 0, b5); p.insert(p.end(), positions.begin(), positions.begin() + b5); }
			s.append(seq, b5, b3 - b5 + 1); p.insert(p.end(), positions.begin() + b5, positions.begin() + b3 + 1);
			if (h3) { s.append(*chars, h3->off, h3->len); p.insert(p.end(), pos->begin() + h3->off, pos->begin() + h3->off + h3->len); }
			else { s.append(seq, b3 + 1, std::string::npos); p.insert(p.end(), positions.begin() + b3 + 1, positions.end()); }
		}
	};
	// the unfilled transcript sequence of a row and the transcripts that match its two sides (output_fusions.cpp:1133-1141)
	struct row_transcripts { std::string tseq; std::vector<i32> positions, t5, t3; };
	void transcripts_of_row(u32 k, const side_strings* from_device, row_transcripts& r) const {
		u32 g5 = e.gene1[k], g3 = e.gene2[k]; bool st5 = e.bits[k] & CB_PSTRAND1, st3 = e.bits[k] & CB_PSTRAND2;
		if (!(e.bits[k] & CB_TSTART_GENE1)) { std::swap(g5, g3); std::swap(st5, st3); }
		const bool ambiguous = e.bits[k] & CB_PSTRANDS_AMBIGUOUS;
		r.tseq = ".";
		transcript_sequence(k, r.tseq, r.positions, from_device);
		matching_transcripts(r.tseq, r.positions, g5, st5, ambiguous, 5, r.t5);
		matching_transcripts(r.tseq, r.positions, g3, st3, ambiguous, 3, r.t3);
	}
	bool is_itd(u32 k) const { return e.gene1[k] == e.gene2[k] && ((unsigned int) e.bp2[k] - (unsigned int) e.bp1[k]) < p.opt.params.max_itd_length && e.dir1[k] == UPSTREAM && e.dir2[k] == DOWNSTREAM; }

	// a row with the columns of -X (fusion transcript, peptide, reading frame, read names): every row formatted on the host has them (the discarded file
	// without -X is formatted on the device, format_discarded_rows_on_device). With -I, `pre` holds the row's transcripts and `fill` its filled sides.
	void format_row(row_buffer& out, u32 k, const side_strings* from_device = NULL, row_transcripts* pre = NULL, const filled_row* fill = NULL) const {
			static const char* CONF[] = {"low", "medium", "high", "high"};
			std::string site5 = site(e.gene1[k], e.spliced1(k), e.exonic1(k), e.contig1[k], e.bp1[k]), site3 = site(e.gene2[k], e.spliced2(k), e.exonic2(k), e.contig2[k], e.bp2[k]);
			u32 g5 = e.gene1[k], g3 = e.gene2[k], c5 = e.contig1[k], c3 = e.contig2[k], d5 = e.dir1[k], d3 = e.dir2[k], s5 = e.split_reads1[k], s3 = e.split_reads2[k];
			i32 b5 = e.bp1[k], b3 = e.bp2[k]; bool st5 = e.bits[k] & CB_PSTRAND1, st3 = e.bits[k] & CB_PSTRAND2;
			i32 gb5 = e.closest1.empty() ? -1 : e.closest1[k], gb3 = e.closest2.empty() ? -1 : e.closest2[k];
			const bool ambiguous = e.bits[k] & CB_PSTRANDS_AMBIGUOUS;
			if (!(e.bits[k] & CB_TSTART_GENE1)) { std::swap(g5, g3); std::swap(c5, c3); std::swap(d5, d3); std::swap(s5, s3); std::swap(b5, b3); std::swap(st5, st3); std::swap(site5, site3); std::swap(gb5, gb3); }
			const int cov5 = p.coverage.get_coverage(c5, b5, d5 == UPSTREAM ? DOWNSTREAM : UPSTREAM), cov3 = p.coverage.get_coverage(c3, b3, d3 == UPSTREAM ? DOWNSTREAM : UPSTREAM);
			std::string pep = ".", frame = "."; i32 tr5 = -1, tr3 = -1;
			row_transcripts own;
			row_transcripts& rt = pre ? *pre : own;
			if (!pre) transcripts_of_row(k, from_device, rt);
			std::string& tseq = rt.tseq; const std::vector<i32>& positions = rt.positions; const std::vector<i32>& t5 = rt.t5; const std::vector<i32>& t3 = rt.t3;
			std::string filled; std::vector<i32> filled_positions;
			for (size_t i = 0; (t5.empty() || i < t5.size()) && frame != "in-frame"; ++i) { // try transcript pairs until one is in-frame
				if (i < t5.size()) tr5 = t5[i];
				for (size_t j = 0; (t3.empty() || j < t3.size()) && frame != "in-frame"; ++j) {
					if (j < t3.size()) tr3 = t3[j];
					if (fill) { fill->assemble(tr5, tr3, tseq, positions, filled, filled_positions); pep = peptide(filled, filled_positions, g5, g3, tr5, tr3, st3); }
					else pep = peptide(tseq, positions, g5, g3, tr5, tr3, st3);
					frame = frame_label(pep);
					if (j >= t3.size()) break;
				}
				if (i >= t5.size() || t3.empty()) break;
			}
			if (frame == "stop-codon") pep = ".";
			if (fill) tseq.swap(filled); // the sequence of the last pair tried
			out << gene_name(g5, c5, b5) << "\t" << gene_name(g3, c3, b3) << "\t" << strand_column(st5, g5, ambiguous) << "\t" << strand_column(st3, g3, ambiguous) << "\t"
			    << ref.original_names[c5] << ":" << (b5 + 1) << "\t" << ref.original_names[c3] << ":" << (b3 + 1) << "\t" << site5 << "\t" << site3 << "\t"
			    << fusion_type(k) << "\t" << s5 << "\t" << s3 << "\t" << e.discordant_mates[k] << "\t"
			    << (cov5 >= 0 ? std::to_string((long long) cov5) : ".") << "\t" << (cov3 >= 0 ? std::to_string((long long) cov3) : ".") << "\t" << CONF[e.confidence[k] & 3] << "\t" << frame
			    << "\t" << p.tags_of(k) << "\t" << p.domains_of(k) << "\t" << genomic_breakpoint(c5, b5, gb5) << "\t" << genomic_breakpoint(c3, b3, gb3);
			// filters column: the candidate's own filter and, with counts, the filters of its supporting reads, in alphabetical order (output_fusions.cpp:1187-1213)
			unsigned int filter_count[38]; bool filter_present[38];
			for (int f = 0; f < 38; ++f) { filter_count[f] = 0; filter_present[f] = false; }
			if (e.filter[k] != F_none) filter_present[e.filter[k]] = true;
			auto tally = [&](const column<u32>& list, u32 lo, u32 hi) { for (u32 r = lo; r < hi; ++r) { if (r + 32 < hi) __builtin_prefetch(&p.labels[list[r + 32]]); const u8 l = p.labels[list[r]]; if (l != F_none && l < 38) { filter_present[l] = true; ++filter_count[l]; } } };
			tally(e.list1, e.list1_off[k], e.list1_off[k + 1]); tally(e.list2, e.list2_off[k], e.list2_off[k + 1]); tally(e.listd, e.listd_off[k], e.listd_off[k + 1]);
			out << "\t" << (ref.genes[g5].is_dummy ? "." : ref.genes[g5].gene_id) << "\t" << (ref.genes[g3].is_dummy ? "." : ref.genes[g3].gene_id)
			    << "\t" << (tr5 < 0 ? "." : ref.transcripts[tr5].name) << "\t" << (tr3 < 0 ? "." : ref.transcripts[tr3].name)
			    << "\t" << (d5 == UPSTREAM ? "upstream" : "downstream") << "\t" << (d3 == UPSTREAM ? "upstream" : "downstream") << "\t";
			bool any = false;
			for (int x = 0; x < 38; ++x) {
				const int f = filters_by_name[x];
				if (f == F_none || !filter_present[f]) continue;
				if (any) out << ",";
				out << FILTER_NAMES[f]; if (filter_count[f] != 0) out << "(" << filter_count[f] << ")";
				any = true;
			}
			if (!any) out << ".";
			out << "\t" << tseq << "\t" << pep << "\t";
			if (e.n_list1(k) + e.n_list2(k) + e.n_listd(k) > 0) {
				bool first_name = true;
				auto names = [&](const column<u32>& list, u32 lo, u32 hi) {
					for (u32 r = lo; r < hi; ++r) {
						if (r + 8 < hi) __builtin_prefetch(&p.frags.name_off[list[r + 8]]);
						if (r + 4 < hi) __builtin_prefetch(p.frags.names.data() + p.frags.name_off[list[r + 4]]);
						if (!first_name) out << ",";
						first_name = false;
						const char* nm = p.frags.names.data() + p.frags.name_off[list[r]]; u64 len = p.frags.name_off[list[r] + 1] - p.frags.name_off[list[r]];
						u64 cut = len; while (cut > 0 && nm[cut - 1] != ',') --cut;
						out.write(nm, cut > 0 ? cut - 1 : len);
					}
				};
				names(e.list1, e.list1_off[k], e.list1_off[k + 1]); names(e.list2, e.list2_off[k], e.list2_off[k + 1]); names(e.listd, e.listd_off[k], e.listd_off[k + 1]);
			} else out << ".";
			out << "\n";
	}

	// A file is produced in two steps, so that the (lock-bound) copy of one file into the page cache can run beside the (CPU-bound) formatting of the other
	struct formatted { std::string header; std::vector<std::string> slices, warnings; column<char> blob; /* rows formatted on the device: one block instead of slices */ };
	static std::string header_line() { return "#gene1\tgene2\tstrand1(gene/fusion)\tstrand2(gene/fusion)\tbreakpoint1\tbreakpoint2\tsite1\tsite2\ttype\tsplit_reads1\tsplit_reads2\tdiscordant_mates\tcoverage1\tcoverage2\tconfidence\treading_frame\ttags\tretained_protein_domains\tclosest_genomic_breakpoint1\tclosest_genomic_breakpoint2\tgene_id1\tgene_id2\ttranscript_id1\ttranscript_id2\tdirection1\tdirection2\tfilters\tfusion_transcript\tpeptide_sequence\tread_identifiers\n"; }
	// the discarded file without -X: every column follows from resident device state; the rows are formatted there (csrc/rows_hd.h) and come back as one block
	void format_discarded_rows_on_device(formatted& out) const {
		output_laps laps;
		sort_filters_by_name();
		pipeline& pl = p;
		if (!pl.row_texts_on_device) {
			std::vector<char> gn, gi, cn, fn; std::vector<u32> gno(1, 0), gio(1, 0), cno(1, 0), fno(1, 0);
			for (size_t g = 0; g < ref.genes.size(); ++g) { gn.insert(gn.end(), ref.genes[g].name.begin(), ref.genes[g].name.end()); gno.push_back((u32) gn.size()); gi.insert(gi.end(), ref.genes[g].gene_id.begin(), ref.genes[g].gene_id.end()); gio.push_back((u32) gi.size()); }
			for (size_t c = 0; c < ref.contig_ids.size(); ++c) { const std::string& nm = ref.original_names[c]; cn.insert(cn.end(), nm.begin(), nm.end()); cno.push_back((u32) cn.size()); }
			for (int f = 0; f < 38; ++f) { fn.insert(fn.end(), FILTER_NAMES[f], FILTER_NAMES[f] + strlen(FILTER_NAMES[f])); fno.push_back((u32) fn.size()); }
			std::vector<i32> prev(ref.exons.size()), next(ref.exons.size());
			for (size_t x = 0; x < ref.exons.size(); ++x) { prev[x] = ref.exons[x].prev >= 0 ? ref.exons[x].prev : -1; next[x] = ref.exons[x].next >= 0 ? ref.exons[x].next : -1; }
			gn.push_back(0); gi.push_back(0); cn.push_back(0); fn.push_back(0);
			arb_row_texts t; memset(&t, 0, sizeof(t));
			t.n_genes = (u32) ref.genes.size(); t.n_exons = (u32) ref.exons.size(); t.n_contigs = (u32) ref.contig_ids.size();
			t.gene_name = gn.data(); t.gene_name_off = gno.data(); t.gene_id = gi.data(); t.gene_id_off = gio.data(); t.contig_name = cn.data(); t.contig_name_off = cno.data(); t.filter_name = fn.data(); t.filter_name_off = fno.data();
			t.exon_prev = prev.data(); t.exon_next = next.data();
			for (int x = 0; x < 38; ++x) t.filters_by_name[x] = (u8) filters_by_name[x];
			t.max_itd_length = p.opt.params.max_itd_length;
			if (arb_set_row_texts(pl.ctx, &t) != 0) throw std::runtime_error(std::string("arb_set_row_texts: ") + arb_last_error(pl.ctx));
			pl.row_texts_on_device = true;
		}
		pl.ensure_coverage_on_device();
		if (arb_set_fragment_filters(pl.ctx, pl.labels.data()) != 0) throw std::runtime_error(std::string("arb_set_fragment_filters: ") + arb_last_error(pl.ctx));
		pl.push_candidate_state();
		uint64_t n_rows = 0, n_bytes = 0;
		if (arb_format_discarded_rows(pl.ctx, e.confidence.data(), &n_rows, &n_bytes) != 0) throw std::runtime_error(std::string("arb_format_discarded_rows: ") + arb_last_error(pl.ctx));
		out.blob.resize(n_bytes ? n_bytes : 1);
		if (n_bytes && arb_get_row_text(pl.ctx, out.blob.data()) != 0) throw std::runtime_error(std::string("arb_get_row_text: ") + arb_last_error(pl.ctx));
		out.blob.resize(n_bytes);
		out.header = header_line();
		out.slices.clear(); out.warnings.clear();
		laps.lap("discarded", "rows formatted (device)");
	}
	// pileups and consensus sequences of the rows of fusions.tsv on the device, in batches of rows; what the device leaves over (verdict != 0) is done by host_sides
	struct device_consensus {
		enum { BATCH = 65536 };
		struct batch { column<u32> seq_off, pos_off, clip_off, non_template; column<u8> verdict; column<char> seq, clip; column<i32> pos; }; // page-locked blocks, not zeroed
		std::vector<batch> batches; std::vector<u32> slot_of_row; // row x -> index among the rows handed to the device, or ~0
		bool get(size_t x, side_strings& out) const {
			if (x >= slot_of_row.size() || slot_of_row[x] == ~0u) return false;
			const batch& b = batches[slot_of_row[x] / BATCH]; const u32 r = slot_of_row[x] % BATCH, j = 2 * r;
			if (b.verdict[j] != 0 || b.verdict[j + 1] != 0 || b.non_template[r] == 0xFFFFFFFFu) return false;
			out.s1.assign(b.seq.data() + b.seq_off[j], b.seq_off[j + 1] - b.seq_off[j]); out.s2.assign(b.seq.data() + b.seq_off[j + 1], b.seq_off[j + 2] - b.seq_off[j + 1]);
			out.c1.assign(b.clip.data() + b.clip_off[j], b.clip_off[j + 1] - b.clip_off[j]); out.c2.assign(b.clip.data() + b.clip_off[j + 1], b.clip_off[j + 2] - b.clip_off[j + 1]);
			out.p1.assign(b.pos.data() + b.pos_off[j], b.pos.data() + b.pos_off[j + 1]); out.p2.assign(b.pos.data() + b.pos_off[j + 1], b.pos.data() + b.pos_off[j + 2]);
			out.non_template = b.non_template[r];
			return true;
		}
	};
	void consensus_on_device(const std::vector<u32>& rows, device_consensus& out) const {
		pipeline& pl = p;
		std::vector<u32> cands; out.slot_of_row.assign(rows.size(), ~0u);
		for (size_t x = 0; x < rows.size(); ++x) if (!transcript_unknown(rows[x])) { out.slot_of_row[x] = (u32) cands.size(); cands.push_back(rows[x]); }
		if (cands.empty()) return;
		output_laps laps;
		if (arb_set_fragment_filters(pl.ctx, pl.labels.data()) != 0) throw std::runtime_error(std::string("arb_set_fragment_filters: ") + arb_last_error(pl.ctx));
		pl.push_candidate_state();
		laps.lap("fusions", "consensus: labels + state -> device");
		u64 left_to_host = 0, retried = 0, reasons[8] = {0, 0, 0, 0, 0, 0, 0, 0};
		for (size_t lo = 0; lo < cands.size(); lo += device_consensus::BATCH) {
			const u32 n = (u32) std::min<size_t>(device_consensus::BATCH, cands.size() - lo);
			arb_consensus_info info;
			if (arb_build_consensus(pl.ctx, cands.data() + lo, n, &info) != 0) throw std::runtime_error(std::string("arb_build_consensus: ") + arb_last_error(pl.ctx));
			laps.lap("fusions", "consensus: kernels");
			out.batches.emplace_back(); device_consensus::batch& b = out.batches.back();
			b.seq_off.resize(2 * (size_t) n + 1); b.pos_off.resize(2 * (size_t) n + 1); b.clip_off.resize(2 * (size_t) n + 1); b.verdict.resize(2 * (size_t) n); b.non_template.resize(n);
			b.seq.resize(info.seq_bytes + 1); b.pos.resize(info.pos_count + 1); b.clip.resize(info.clip_bytes + 1);
			if (arb_get_consensus(pl.ctx, b.seq_off.data(), b.pos_off.data(), b.clip_off.data(), b.verdict.data(), b.non_template.data(), b.seq.data(), b.pos.data(), b.clip.data()) != 0) throw std::runtime_error(std::string("arb_get_consensus: ") + arb_last_error(pl.ctx));
			laps.lap("fusions", "consensus: strings -> host");
			for (size_t j = 0; j < b.verdict.size(); ++j) if (b.verdict[j]) { ++left_to_host; for (int q = 0; q < 8; ++q) if (b.verdict[j] >> q & 1) ++reasons[q]; }
			retried += info.retried_jobs;
		}
		if (getenv("ARB_TRACE")) fprintf(stderr, "[laps] output fusions    consensus jobs %zu, second launch %llu, left to the host %llu (tiles %llu, side list %llu, introns %llu, empty key %llu, counters %llu, output %llu, odd column %llu)\n", cands.size() * 2, (unsigned long long) retried, (unsigned long long) left_to_host,
			(unsigned long long) reasons[0], (unsigned long long) reasons[2], (unsigned long long) reasons[3], (unsigned long long) reasons[4], (unsigned long long) reasons[5], (unsigned long long) reasons[6], (unsigned long long) reasons[7]);
	}
	void format_rows(bool discarded, bool extra_info, formatted& out) const {
		if (discarded && !extra_info) { format_discarded_rows_on_device(out); return; }
		sort_filters_by_name();
		output_laps laps; const char* const which = discarded ? "discarded" : "fusions";
		std::vector<u32> rows;
		for (size_t q = 0; q < e.order.size(); ++q) { const u32 k = e.order[q]; if (discarded != (e.filter[k] == F_none)) rows.push_back(k); }
		if (!discarded) {
			std::map<std::pair<u32, u32>, u32> best; // best-supported candidate per gene pair
			for (size_t x = 0; x < rows.size(); ++x) {
				std::pair<std::map<std::pair<u32, u32>, u32>::iterator, bool> ins = best.insert(std::make_pair(std::make_pair(e.gene1[rows[x]], e.gene2[rows[x]]), rows[x]));
				if (!ins.second && by_support(rows[x], ins.first->second)) ins.first->second = rows[x];
			}
			// same sort, same comparisons, but a row carries its gene pair's best candidate instead of looking it up in the map twice per comparison
			std::vector<std::pair<u32, u32> > keyed(rows.size());
			for (size_t x = 0; x < rows.size(); ++x) keyed[x] = std::make_pair(rows[x], best.at(std::make_pair(e.gene1[rows[x]], e.gene2[rows[x]])));
			std::sort(keyed.begin(), keyed.end(), [&](const std::pair<u32, u32>& x, const std::pair<u32, u32>& y) { return x.second != y.second ? by_support(x.second, y.second) : by_support(x.first, y.first); });
			for (size_t x = 0; x < rows.size(); ++x) rows[x] = keyed[x].first;
			laps.lap(which, "rows selected and ordered");
		}
		const std::string header = header_line();
		device_consensus from_device;
		if (!discarded && (getenv("ARB_DEVICE_CONSENSUS") == NULL || atoi(getenv("ARB_DEVICE_CONSENSUS")) != 0)) { consensus_on_device(rows, from_device); laps.lap(which, "pileups + consensus (device)"); }
		if (p.opt.fill_sequence_gaps) { out.header = header; format_filled_rows(rows, from_device, out, which); return; }
		// Rows are independent and cost very different amounts (the best-supported fusions come first and carry hundreds of reads each): threads draw small
		// chunks of rows from a shared counter; every chunk is formatted into its own string and later copied to its offset of the file (flush_rows).
		const size_t CHUNK = 32;
		const size_t n_chunks = (rows.size() + CHUNK - 1) / CHUNK;
		const int T = std::max(1, std::min(p.threads, (int) (n_chunks ? n_chunks : 1)));
		out.header = header;
		std::vector<std::string>& slices = out.slices; std::vector<std::string>& warnings = out.warnings;
		slices.assign(n_chunks, std::string()); warnings.assign(n_chunks, std::string()); std::vector<std::string> errors(T);
		{
			std::atomic<size_t> next_chunk(0);
			std::vector<std::thread> pool;
			for (int t = 0; t < T; ++t) pool.emplace_back([&, t]() {
				try {
					for (;;) {
						const size_t c = next_chunk.fetch_add(1);
						if (c >= n_chunks) break;
						warning_sink = &warnings[c]; // warnings of a chunk are printed after it, in row order like the reference's
						row_buffer text; text.s.reserve(CHUNK * 4096);
						for (size_t x = c * CHUNK; x < rows.size() && x < (c + 1) * CHUNK; ++x) {
							if (x + 6 < rows.size()) prefetch_candidate(rows[x + 6]);
							if (x + 4 < rows.size()) prefetch_lists(rows[x + 4]);
							if (x + 2 < rows.size()) prefetch_labels(rows[x + 2]);
							side_strings sides;
							format_row(text, rows[x], from_device.get(x, sides) ? &sides : NULL);
						}
						slices[c].swap(text.s);
					}
				} catch (const std::exception& ex) { errors[t] = ex.what(); }
				warning_sink = NULL;
			});
			for (size_t t = 0; t < pool.size(); ++t) pool[t].join();
		}
		for (int t = 0; t < T; ++t) if (!errors[t].empty()) throw std::runtime_error(errors[t]);
		laps.lap(which, "rows formatted");
	}
	// -I: the rows in blocks of ROW_BLOCK; per block (A) the transcript sequences and matching transcripts of the rows on the host threads, (B) every
	// distinct (row, side, transcript) job filled on the device (fill_gaps_hd.h), in calls of at most FILL_CHARS output characters, (C) the transcript pairs
	// of every row tried in the reference's order on the host threads and the rows formatted. Warnings stay with the chunk of rows that printed them (C).
	enum { ROW_BLOCK = 32 * 1024, FILL_CHARS = 32 << 20 };
	template <class F> void for_chunks(size_t lo, size_t hi, size_t chunk, F fn) const { // chunks [lo, hi) of `chunk` rows drawn by the host threads
		const size_t n_chunks = (hi - lo + chunk - 1) / chunk;
		const int T = std::max(1, std::min(p.threads, (int) (n_chunks ? n_chunks : 1)));
		std::vector<std::string> errors(T); std::atomic<size_t> next_chunk(0); std::vector<std::thread> pool;
		for (int t = 0; t < T; ++t) pool.emplace_back([&, t]() {
			try { for (;;) { const size_t c = next_chunk.fetch_add(1); if (c >= n_chunks) break; fn(lo / chunk + c, lo + c * chunk, std::min(hi, lo + (c + 1) * chunk)); } }
			catch (const std::exception& ex) { errors[t] = ex.what(); }
			warning_sink = NULL;
		});
		for (size_t t = 0; t < pool.size(); ++t) pool[t].join();
		for (int t = 0; t < T; ++t) if (!errors[t].empty()) throw std::runtime_error(errors[t]);
	}
	void upload_fill_transcripts() const {
		pipeline& pl = p;
		if (pl.fill_transcripts_on_device) return;
		const size_t n = ref.transcripts.size(), E = ref.exons.size();
		std::vector<i32> first(n ? n : 1, 0), last(n ? n : 1, 0), next(E ? E : 1, -1), prev(E ? E : 1, -1); std::vector<u32> contig(n ? n : 1, 0);
		for (size_t t = 0; t < n; ++t) {
			const transcript_rec& T = ref.transcripts[t];
			if (T.first_exon < 0 || T.last_exon < 0) continue; // a transcript without exons matches no row (matching_transcripts finds transcripts by their exons)
			first[t] = T.first_exon; last[t] = T.last_exon; contig[t] = ref.genes[ref.exons[T.first_exon].gene].contig;
		}
		for (size_t x = 0; x < E; ++x) { next[x] = ref.exons[x].next >= 0 ? ref.exons[x].next : -1; prev[x] = ref.exons[x].prev >= 0 ? ref.exons[x].prev : -1; }
		if (arb_set_fill_transcripts(pl.ctx, (u32) n, first.data(), last.data(), contig.data(), next.data(), prev.data()) != 0) throw std::runtime_error(std::string("arb_set_fill_transcripts: ") + arb_last_error(pl.ctx));
		pl.fill_transcripts_on_device = true;
	}
	// an upper bound of the characters a job writes: its side of the sequence, and every exon of the transcript with its "___" and the marks
	u64 fill_bound(i32 t, size_t side) const {
		u64 b = side + 8;
		for (i32 ex = ref.transcripts[t].first_exon; ex >= 0; ex = ref.exons[ex].next >= 0 ? ref.exons[ex].next : -1) b += (u64) std::max(0, ref.exons[ex].end - ref.exons[ex].start + 1) + 3;
		return b;
	}
	void format_filled_rows(const std::vector<u32>& rows, const device_consensus& from_device, formatted& out, const char* which) const {
		output_laps laps;
		upload_fill_transcripts();
		pipeline& pl = p;
		const size_t CHUNK = 32, n_chunks = (rows.size() + CHUNK - 1) / CHUNK;
		out.slices.assign(n_chunks, std::string()); out.warnings.assign(n_chunks, std::string());
		std::vector<row_transcripts> pre; std::vector<filled_row> fill;
		std::deque<std::string> block_chars; std::deque<std::vector<i32> > block_pos; // the outputs of the calls of a block (a deque keeps them in place)
		u64 n_jobs = 0, n_chars = 0;
		for (size_t lo = 0; lo < rows.size(); lo += ROW_BLOCK) {
			const size_t hi = std::min(rows.size(), lo + (size_t) ROW_BLOCK);
			pre.assign(hi - lo, row_transcripts()); fill.assign(hi - lo, filled_row());
			// (A)
			for_chunks(lo, hi, CHUNK, [&](size_t, size_t a, size_t b) {
				for (size_t y = a; y < b; ++y) { side_strings sides; transcripts_of_row(rows[y], from_device.get(y, sides) ? &sides : NULL, pre[y - lo]); }
			});
			// (B) the distinct transcripts of each side; calls cut at FILL_CHARS characters of bound
			std::vector<u32> job_row, job_tr; std::vector<u8> job_flags; std::vector<size_t> job_x; // job_x: the row of a job in this block
			block_chars.clear(); block_pos.clear();
			size_t x = 0;
			while (x < hi - lo) {
				std::string text; std::vector<i32> tpos; std::vector<u32> row_off(1, 0), pos_off(1, 0); u64 bound = 0;
				job_row.clear(); job_tr.clear(); job_flags.clear(); job_x.clear();
				for (; x < hi - lo && (bound < (u64) FILL_CHARS || job_row.empty()); ++x) {
					const row_transcripts& r = pre[x];
					if (r.t5.empty() && r.t3.empty()) continue;
					const u32 k = rows[lo + x];
					bool st5 = e.bits[k] & CB_PSTRAND1, st3 = e.bits[k] & CB_PSTRAND2;
					if (!(e.bits[k] & CB_TSTART_GENE1)) std::swap(st5, st3);
					const u8 itd = is_itd(k) ? (u8) ARB_FILL_ITD : (u8) 0;
					const size_t b5 = r.tseq.find('|'), b3 = r.tseq.rfind('|');
					const u32 row = (u32) row_off.size() - 1;
					for (int side = 0; side < 2; ++side) {
						const std::vector<i32>& ts = side == 0 ? r.t5 : r.t3;
						for (size_t i = 0; i < ts.size(); ++i) {
							if (std::find(ts.begin(), ts.begin() + i, ts[i]) != ts.begin() + i) continue; // the best transcript comes twice
							job_row.push_back(row); job_tr.push_back((u32) ts[i]); job_x.push_back(x);
							job_flags.push_back((u8) ((side ? ARB_FILL_THREE : 0) | ((side ? st3 : st5) ? ARB_FILL_FORWARD : 0) | itd));
							bound += fill_bound(ts[i], side ? r.tseq.size() - b3 : b5);
						}
					}
					text += r.tseq; tpos.insert(tpos.end(), r.positions.begin(), r.positions.end()); row_off.push_back((u32) text.size()); pos_off.push_back((u32) tpos.size());
				}
				if (job_row.empty()) continue;
				uint64_t chars = 0;
				if (arb_fill_gaps(pl.ctx, (u32) row_off.size() - 1, text.data(), row_off.data(), tpos.data(), pos_off.data(), (u32) job_row.size(), job_row.data(), job_tr.data(), job_flags.data(), &chars) != 0) {
					std::string what = arb_last_error(pl.ctx);
					const size_t at = what.find("(row "); // name the fusion of the row
					if (at != std::string::npos) { const u32 r = (u32) atol(what.c_str() + at + 5); for (size_t j = 0; j < job_row.size(); ++j) if (job_row[j] == r) { const u32 k = rows[lo + job_x[j]]; what += " (fusion " + ref.original_names[e.contig1[k]] + ":" + std::to_string((long long) e.bp1[k] + 1) + " / " + ref.original_names[e.contig2[k]] + ":" + std::to_string((long long) e.bp2[k] + 1) + ")"; break; } }
					throw std::runtime_error("arb_fill_gaps: " + what);
				}
				block_chars.emplace_back(chars, '\0'); block_pos.emplace_back(chars + 1);
				std::vector<u32> off(job_row.size() + 1);
				if (arb_get_filled(pl.ctx, off.data(), &block_chars.back()[0], block_pos.back().data()) != 0) throw std::runtime_error(std::string("arb_get_filled: ") + arb_last_error(pl.ctx));
				for (size_t j = 0; j < job_row.size(); ++j) {
					filled_row& f = fill[job_x[j]];
					filled_row::half h; h.transcript = (i32) job_tr[j]; h.three = job_flags[j] & ARB_FILL_THREE; h.off = off[j]; h.len = off[j + 1] - off[j];
					f.halves.push_back(h); f.chars = &block_chars.back(); f.pos = &block_pos.back(); // a row's jobs are all in one call
				}
				n_jobs += job_row.size(); n_chars += chars;
			}
			laps.lap(which, "gap filling (host A + device B)");
			// (C)
			for_chunks(lo, hi, CHUNK, [&](size_t c, size_t a, size_t b) {
				warning_sink = &out.warnings[c];
				row_buffer text; text.s.reserve(CHUNK * 4096);
				for (size_t y = a; y < b; ++y) format_row(text, rows[y], NULL, &pre[y - lo], &fill[y - lo]);
				out.slices[c].swap(text.s);
			});
		}
		if (getenv("ARB_TRACE")) fprintf(stderr, "[laps] output %-10s gap filling jobs %llu, filled characters %llu\n", which, (unsigned long long) n_jobs, (unsigned long long) n_chars);
		laps.lap(which, "rows formatted");
	}
	static int open_output(const std::string& path) {
		const int fd = ::open(path.c_str(), O_RDWR | O_CREAT | O_TRUNC, 0666);
		if (fd < 0) throw std::runtime_error("failed to open output file");
		return fd;
	}
	void flush_rows(int fd, const formatted& text, bool discarded) const { // writes and closes; the warnings of the rows go to stderr afterwards
		output_laps laps; const char* const which = discarded ? "discarded" : "fusions";
		const std::string& header = text.header; const std::vector<std::string>& slices = text.slices; const std::vector<std::string>& warnings = text.warnings;
		const size_t n_chunks = slices.size();
		const u64 blob_bytes = text.blob.size(); const char* const blob = text.blob.data(); // rows formatted on the device (then there are no slices)
		// write() in 8 MiB pieces: on an overlay file system one writer fills the page cache faster than a shared mapping of the file filled by all threads
		auto write_all = [&](const char* data, size_t n) { while (n > 0) { const ssize_t w = ::write(fd, data, std::min<size_t>(n, (size_t) 8 << 20)); if (w <= 0) return false; data += w; n -= (size_t) w; } return true; };
		bool ok = write_all(header.data(), header.size());
		for (size_t c = 0; c < n_chunks && ok; ) { // the slices of 32 rows go out a thousand at a time (writev): no copy, few system calls
			struct iovec v[512]; int nv = 0; size_t bytes = 0;
			for (; c < n_chunks && nv < 512; ++c) if (!slices[c].empty()) { v[nv].iov_base = (void*) slices[c].data(); v[nv].iov_len = slices[c].size(); bytes += slices[c].size(); ++nv; }
			for (int first = 0; bytes > 0 && ok; ) {
				const ssize_t w = ::writev(fd, v + first, nv - first);
				if (w <= 0) { ok = false; break; }
				bytes -= (size_t) w;
				size_t done = (size_t) w; while (first < nv && done >= v[first].iov_len) { done -= v[first].iov_len; ++first; }
				if (first < nv) { v[first].iov_base = (char*) v[first].iov_base + done; v[first].iov_len -= done; }
			}
		}
		if (ok && blob_bytes) { // the block of device-formatted rows: a few threads with pwrite() on disjoint ranges (one writer loses its CPU to the formatting threads now and then)
			struct stat st2; const bool regular = ::fstat(fd, &st2) == 0 && S_ISREG(st2.st_mode);
			const off_t base = regular ? ::lseek(fd, 0, SEEK_CUR) : (off_t) -1;
			if (base < 0 || blob_bytes < ((u64) 64 << 20)) ok = write_all(blob, blob_bytes);
			else {
				const int W = 4; std::vector<std::thread> pool; std::vector<int> good(W, 1);
				for (int t = 0; t < W; ++t) pool.emplace_back([&, t]() {
					const u64 lo = (blob_bytes * t / W) & ~(u64) 4095, hi = t + 1 == W ? blob_bytes : (blob_bytes * (t + 1) / W) & ~(u64) 4095;
					for (u64 at = lo; at < hi; ) { const ssize_t w = ::pwrite(fd, blob + at, (size_t) std::min<u64>(hi - at, (u64) 8 << 20), base + (off_t) at); if (w <= 0) { good[t] = 0; return; } at += (u64) w; }
				});
				for (size_t t = 0; t < pool.size(); ++t) pool[t].join();
				for (int t = 0; t < W; ++t) ok = ok && good[t];
			}
		}
		ok = ::close(fd) == 0 && ok;
		laps.lap(which, "file written");
		for (size_t c = 0; c < n_chunks; ++c) if (!warnings[c].empty()) std::cerr << warnings[c] << std::flush;
		if (!ok) throw std::runtime_error("failed to write to file");
	}
};

} // namespace

const char* const FILTER_NAMES[38] = {"", "duplicates", "inconsistently_clipped", "homopolymer", "read_through", "same_gene", "small_insert_size", "long_gap", "hairpin",
	"multimappers", "mismatches", "mismappers", "relative_support", "intronic", "non_coding_neighbors", "intragenic_exonic", "internal_tandem_duplication", "min_support",
	"known_fusions", "spliced", "blacklist", "end_to_end", "in_vitro", "merge_adjacent", "select_best", "marginal_read_through", "short_anchor", "no_coverage", "many_spliced",
	"no_genomic_support", "uninteresting_contigs", "viral_contigs", "top_expressed_viral_contigs", "low_coverage_viral_contigs", "genomic_support", "isoforms", "low_entropy", "homologs"};

void pipeline::write_output() {
	order_ready();
	const double t0 = std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
	writer w(*this);
	const bool fusions = !opt.output_file.empty(), discarded = !opt.discarded_output_file.empty();
	// files are opened and announced in the reference's order (output_fusions.cpp:1043, arriba.cpp:601-612)
	int fd_fusions = -1, fd_discarded = -1;
	if (!opt.tags_file.empty() && (fusions || discarded)) annotate_tags(); // arriba.cpp:591-595: the tags are loaded before any output file is opened
	if (!opt.protein_domains_file.empty() && (fusions || discarded)) load_protein_domains(); // arriba.cpp:597-602: the protein domains after the tags
	if (fusions) fd_fusions = writer::open_output(opt.output_file);
	if (discarded) { try { fd_discarded = writer::open_output(opt.discarded_output_file); } catch (...) { if (fd_fusions >= 0) ::close(fd_fusions); throw; } }
	writer::formatted text_fusions, text_discarded;
	std::thread copier; std::string copier_error;
	// The discarded file (a gigabyte on a large sample) is formatted first and copied into the page cache by a helper WHILE the rows of the fusions file, which
	// cost pileups and consensus sequences, are formatted. Only without -X: with it the discarded rows print warnings too, and stderr keeps the reference's order.
	const bool overlap = fusions && discarded && !opt.print_extra_info_for_discarded_fusions;
	try {
		if (fusions) say("Writing fusions to file '" + opt.output_file + "'");
		if (overlap) {
			w.format_rows(true, false, text_discarded);
			const int fd = fd_discarded; fd_discarded = -1; // closed by the helper
			copier = std::thread([&, fd]() { try { w.flush_rows(fd, text_discarded, true); } catch (const std::exception& x) { copier_error = x.what(); } });
		}
		if (fusions) { w.format_rows(false, true, text_fusions); const int fd = fd_fusions; fd_fusions = -1; w.flush_rows(fd, text_fusions, false); }
		if (discarded) say("Writing discarded fusions to file '" + opt.discarded_output_file + "'");
		if (overlap) { copier.join(); if (!copier_error.empty()) throw std::runtime_error(copier_error); }
		else if (discarded) { w.format_rows(true, opt.print_extra_info_for_discarded_fusions, text_discarded); const int fd = fd_discarded; fd_discarded = -1; w.flush_rows(fd, text_discarded, true); }
	} catch (...) {
		if (copier.joinable()) copier.join();
		if (fd_fusions >= 0) ::close(fd_fusions);
		if (fd_discarded >= 0) ::close(fd_discarded);
		throw;
	}
	t_output = std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count() - t0;
}

}} // namespace
