// blacklist_hd.h -- rules of a blacklist file (-b) matched to the candidates: filter_blacklisted_ranges (filter_blacklisted_ranges.cpp:138-300).
//
// The reference indexes the ELIGIBLE candidates (no filter yet, or closest_genomic_breakpoint1 >= 0 with -d) under the 100 kb bins of four ranges: both
// breakpoints and both genes. Every rule then visits the candidates of the bins of its positional items, each widened by max_mate_gap, and blacklists those
// for which (item1 matches breakpoint 1 and item2 breakpoint 2) or (item1 matches breakpoint 2 and item2 breakpoint 1). Removing a candidate from a bin's set
// only stops it from being tested again, and the test reads nothing the loop writes: the verdict is "eligible and some rule that shares a bin with the
// candidate matches", whatever the order of the file or of the candidates. Here the rules' bins become (contig, bin) keys, sorted into a key table with one
// rule list per key; every eligible candidate looks up its own bins and tests the rules listed there.
// The files of known fusions (-k, recover_known_fusions.cpp:14-100) and of tags (-t, annotate_tags.cpp) have the same format and the same item test. They
// differ in three ways: the rules' bins are not widened by max_mate_gap; the match is directional (item 1 against the 5' side, item 2 against the 3' side,
// known fusions also swapped when the transcript start is ambiguous and the breakpoints are far apart); and a tag needs every matching rule, not just one.
// So the rule columns, the key table, the candidate's bins and the item test are shared by three searches, each with its own set of rules.
#pragma once
#include "model.h"
#include "prims.h"        // append_slot
#include "read_filters.h" // lane_group
#include "../../include/arriba_b200.h" // ARB_RULE_*
#include "events_hd.h"    // cand_state
#include "genomic_hd.h"   // wrap_add / wrap_sub
#include <climits>

namespace arb {

// rules in file order, one column per field of each of the two items (type: ARB_RULE_*, strand: ARB_RULE_STRAND_*)
struct rule_columns {
	u32 n;
	const u8* type[2]; const u8* strand[2]; const u16* contig[2]; const i32* start[2]; const i32* end[2]; const u32* gene[2];
};

ARB_HD bool rule_item_positional(u32 type) { return type == ARB_RULE_RANGE || type == ARB_RULE_POSITION || type == ARB_RULE_GENE; }

// get_genome_bins_from_range (:226-230): bins start / 100000 ... (end + 99999) / 100000 of a 100 kb grid, division truncating toward zero.
// Computed in 64 bits; bins beyond +-21475 hold no int position and no candidate, and are dropped so that every key fits 16 bits of bin.
static const i64 RULE_BIN_SIZE = 100000, RULE_BIN_LIMIT = 21475;
ARB_HD void rule_bins(i64 start, i64 end, i32& lo, i32& hi) {
	i64 a = start / RULE_BIN_SIZE, b = (end + RULE_BIN_SIZE - 1) / RULE_BIN_SIZE;
	if (a < -RULE_BIN_LIMIT) a = -RULE_BIN_LIMIT;
	if (b > RULE_BIN_LIMIT) b = RULE_BIN_LIMIT;
	lo = (i32) a; hi = (i32) b; // lo > hi: no bins
}
// the same for int coordinates (every candidate range), in 32-bit arithmetic: a 64-bit division is a called subroutine on the device
ARB_HD void rule_bins32(i32 start, i32 end, i32& lo, i32& hi) {
	lo = start / (i32) RULE_BIN_SIZE;
	hi = end <= INT_MAX - 99999 ? (end + 99999) / (i32) RULE_BIN_SIZE : end / (i32) RULE_BIN_SIZE + (end % (i32) RULE_BIN_SIZE != 0);
}
ARB_HD u32 rule_bin_key(u32 contig, i32 bin) { return contig << 16 | (u32) (bin + 32768); }

// the bins a positional item of a rule is looked up under: (contig, start - widen, end + widen); widen is max_mate_gap for the blacklist (:272-275) and 0 for
// known fusions and tags (recover_known_fusions.cpp:32-34, annotate_tags.cpp:36-38)
ARB_HD void rule_item_bins(const rule_columns& r, u32 rule, u32 side, i32 widen, i32& lo, i32& hi) {
	rule_bins((i64) r.start[side][rule] - widen, (i64) r.end[side][rule] + widen, lo, hi);
}

// overlapping_fraction (:123-135): the quotient in double, returned as float; the four branches as written (the second has no "+ 1")
ARB_HD float overlapping_fraction(i32 start1, i32 end1, i32 start2, i32 end2) {
	if (start1 >= start2 && end1 <= end2) return 1;
	if (start1 < start2 && end1 > end2) return (float) (1.0 * wrap_sub(end2, start2) / wrap_add(wrap_sub(end1, start1), 1));
	if (start1 >= start2 && start1 <= end2) return (float) (1.0 * wrap_sub(end2, start1) / wrap_add(wrap_sub(end1, start1), 1));
	if (end1 >= start2 && end1 <= end2) return (float) (1.0 * wrap_sub(end1, start2) / wrap_add(wrap_sub(end1, start1), 1));
	return 0;
}

// matches_blacklist_item (:138-223) on the resident candidate columns
struct rule_match {
	rule_columns r; cand_state c; annot_view an;
	i32 max_mate_gap; float evalue_cutoff;

	ARB_HD bool item(u32 rule, u32 side, u32 k, u32 which) const {
		const u32 sr1 = c.split_reads1[k], sr2 = c.split_reads2[k], dm = c.discordant_mates[k]; const u8 bits = c.bits[k];
		const bool spliced1 = bits & CB_SPLICED1, spliced2 = bits & CB_SPLICED2;
		switch (r.type[side][rule]) {
			case ARB_RULE_ANY: return true;
			case ARB_RULE_SPLIT_READ_DONOR: return (which == 1 && dm + sr1 == 0) || (which == 2 && dm + sr2 == 0);
			case ARB_RULE_SPLIT_READ_ACCEPTOR: return (which == 1 && dm + sr2 == 0) || (which == 2 && dm + sr1 == 0);
			case ARB_RULE_SPLIT_READ_ANY: return dm == 0;
			case ARB_RULE_DISCORDANT_MATES: return sr1 + sr2 == 0;
			case ARB_RULE_READ_THROUGH: return c.contig1[k] == c.contig2[k] && c.bp2[k] - c.bp1[k] < 400000 && c.dir1[k] == DOWNSTREAM && c.dir2[k] == UPSTREAM; // is_read_through (common.hpp:265-269)
			case ARB_RULE_LOW_SUPPORT: return c.evalue[k] > evalue_cutoff;
			case ARB_RULE_FILTER_SPLICED: return c.evalue[k] > evalue_cutoff && spliced1 && spliced2;
			case ARB_RULE_NOT_BOTH_SPLICED: return !spliced1 || !spliced2;
			case ARB_RULE_GENE: return (which == 1 ? c.gene1[k] : c.gene2[k]) == r.gene[side][rule];
			case ARB_RULE_POSITION: case ARB_RULE_RANGE: {
				if ((which == 1 ? c.contig1[k] : c.contig2[k]) != r.contig[side][rule]) return false;
				const u8 strand = r.strand[side][rule];
				if (strand != ARB_RULE_STRAND_NONE && !(bits & CB_PSTRANDS_AMBIGUOUS)) { // strands that could not be predicted match any
					const bool forward = bits & (which == 1 ? CB_PSTRAND1 : CB_PSTRAND2);
					if (forward != (strand == ARB_RULE_STRAND_FORWARD)) return false;
				}
				const i32 start = r.start[side][rule];
				if (r.type[side][rule] == ARB_RULE_RANGE) {
					const u32 g = which == 1 ? c.gene1[k] : c.gene2[k];
					return overlapping_fraction(an.gene_start[g], an.gene_end[g], start, r.end[side][rule]) > 0.5f;
				}
				const i32 bp = which == 1 ? c.bp1[k] : c.bp2[k];
				if (bp == start) return true;
				if (sr1 + sr2 == 0) { // only discordant mates: near the position and pointing towards it
					const u8 dir = which == 1 ? c.dir1[k] : c.dir2[k];
					if (dir == DOWNSTREAM && bp <= start && (i64) bp >= (i64) start - max_mate_gap) return true;
					if (dir == UPSTREAM && bp >= start && (i64) bp <= (i64) start + max_mate_gap) return true;
				}
				return false;
			}
		}
		return false;
	}
	ARB_HD bool operator()(u32 rule, u32 k) const { // both orders of the two items (:280-283)
		return (item(rule, 0, k, 1) && item(rule, 1, k, 2)) || (item(rule, 0, k, 2) && item(rule, 1, k, 1));
	}
	// item 1 against the 5' side and item 2 against the 3' side (recover_known_fusions.cpp:65-68, annotate_tags.cpp:62-65); swapped: the other way round
	ARB_HD bool directional(u32 rule, u32 k, bool swapped) const {
		const u32 g5 = (c.bits[k] & CB_TSTART_GENE1) ? 1 : 2, g3 = 3 - g5;
		return swapped ? item(rule, 0, k, g3) && item(rule, 1, k, g5) : item(rule, 0, k, g5) && item(rule, 1, k, g3);
	}
};

// ---- key table of the rules (blacklist.cu: build_rule_keys): counts, scan, fill, sort, then one entry per distinct key
struct rule_key_count_fn { // number of (contig, bin) keys of every rule
	rule_columns r; i32 widen; u32* count; unsigned long long* total;
	ARB_HD void operator()(u32 rule) const {
		u32 n = 0;
		for (u32 side = 0; side < 2; ++side) {
			if (!rule_item_positional(r.type[side][rule])) continue;
			i32 lo, hi; rule_item_bins(r, rule, side, widen, lo, hi);
			if (hi >= lo) n += (u32) (hi - lo + 1);
		}
		count[rule] = n;
#ifdef __CUDA_ARCH__
		atomicAdd(total, (unsigned long long) n);
#else
		*total += n;
#endif
	}
};
struct rule_key_fill_fn { // the keys of rule `rule` at its offset, the rule as their value
	rule_columns r; i32 widen; const u32* offset; u32* key; u32* rule_of;
	ARB_HD void operator()(u32 rule) const {
		u32 at = offset[rule];
		for (u32 side = 0; side < 2; ++side) {
			if (!rule_item_positional(r.type[side][rule])) continue;
			i32 lo, hi; rule_item_bins(r, rule, side, widen, lo, hi);
			for (i32 b = lo; b <= hi; ++b) { key[at] = rule_bin_key(r.contig[side][rule], b); rule_of[at] = rule; ++at; }
		}
	}
};
struct rule_key_head_fn { // 1 where a run of equal sorted keys begins
	const u32* key; u32* head;
	ARB_HD void operator()(u32 i) const { head[i] = i == 0 || key[i] != key[i - 1]; }
};
struct rule_key_table_fn { // distinct keys and where their rule lists begin; the last item closes the table
	const u32* key; const u32* head; const u32* slot; u32* table_key; u32* table_begin; u32 n;
	ARB_HD void operator()(u32 i) const {
		if (head[i]) { table_key[slot[i]] = key[i]; table_begin[slot[i]] = i; }
		if (i + 1 == n) table_begin[slot[i] + head[i]] = n;
	}
};

struct rule_key_table {
	u32 n_keys;
	const u32* key;      // distinct (contig, bin) keys, ascending
	const u32* begin;    // n_keys + 1: the rules of key q are rules[begin[q] .. begin[q + 1])
	const u32* rules;
	ARB_HD bool find(u32 k, u32& lo, u32& hi) const {
		u32 a = 0, b = n_keys;
		while (a < b) { const u32 m = a + (b - a) / 2; if (key[m] < k) a = m + 1; else b = m; }
		if (a == n_keys || key[a] != k) return false;
		lo = begin[a]; hi = begin[a + 1];
		return true;
	}
};

// ---- the rule lists a candidate meets: the bins of its four ranges, each distinct bin once
struct cand_bins {
	cand_state c; annot_view an; rule_key_table t;
	// the four ranges a candidate is indexed under (:244-247, recover_known_fusions.cpp:53-57, annotate_tags.cpp:48-52): both breakpoints, then both genes
	ARB_HD void range(u32 k, u32 x, u32& contig, i32& lo, i32& hi) const {
		contig = (x & 1) ? c.contig2[k] : c.contig1[k];
		if (x < 2) { const i32 bp = x ? c.bp2[k] : c.bp1[k]; rule_bins32(bp, bp, lo, hi); }
		else { const u32 g = x == 2 ? c.gene1[k] : c.gene2[k]; rule_bins32(an.gene_start[g], an.gene_end[g], lo, hi); }
	}
	// a bin already listed by an earlier range of the same candidate is looked up once (every search's verdict is the same either way)
	ARB_HD bool listed_before(u32 k, u32 x, u32 contig, i32 bin) const {
		for (u32 y = 0; y < x; ++y) { u32 cy; i32 lo, hi; range(k, y, cy, lo, hi); if (cy == contig && bin >= lo && bin <= hi) return true; }
		return false;
	}
	// v(a, e) for the rule list rules[a .. e) of every distinct bin of candidate k, until v returns true; returns whether it did
	template <class V> ARB_HD bool visit(u32 k, V& v) const {
		for (u32 x = 0; x < 4; ++x) {
			u32 contig; i32 lo, hi; range(k, x, contig, lo, hi);
			for (i32 b = lo; b <= hi; ++b) {
				u32 a, e;
				if (listed_before(k, x, contig, b) || !t.find(rule_bin_key(contig, b), a, e)) continue;
				if (v(a, e)) return true;
			}
		}
		return false;
	}
};

// ---- "does some listed rule pass Test": one thread per candidate id; a candidate with a long rule list goes to a group of lanes
// Test: ARB_HD bool operator()(u32 rule, u32 k)
template <class Test> struct rule_search {
	cand_bins b; Test test;
	const u32* ids; u8* verdict;        // candidates, one verdict byte each
	u32 short_list;                     // lists up to this length are walked by the candidate's own thread
	u32* heavy; u32* n_heavy;           // positions in `ids` of the candidates queued for a group of lanes

	struct lanes_fn { // lane `lane` of `lanes` tests rules a + lane, a + lane + lanes, ... of a list
		const rule_search* s; u32 k, lane, lanes;
		ARB_HD bool operator()(u32 a, u32 e) const { for (u32 q = a + lane; q < e; q += lanes) if (s->test(s->b.t.rules[q], k)) return true; return false; }
	};
	struct thread_fn { // the whole list, or 2 when it is too long for one thread
		const rule_search* s; u32 k; u32 result;
		ARB_HD bool operator()(u32 a, u32 e) {
			if (e - a > s->short_list) { result = 2; return true; }
			for (u32 q = a; q < e; ++q) if (s->test(s->b.t.rules[q], k)) { result = 1; return true; }
			return false;
		}
	};
	// a single thread is lane 0 of 1
	ARB_HD bool lane_walk(u32 k, u32 lane, u32 lanes) const { lanes_fn v = {this, k, lane, lanes}; return b.visit(k, v); }
	ARB_HD void operator()(u32 i) const {
		thread_fn v = {this, ids[i], 0};
		b.visit(ids[i], v);
		if (v.result == 2) heavy[append_slot(n_heavy)] = i;
		else verdict[i] = (u8) v.result;
	}
};

typedef rule_search<rule_match> blacklist_search;

// ---- known fusions (recover_known_fusions.cpp:41-92): a rule rescues an eligible candidate if it matches it directionally (or swapped, when the transcript
// start is ambiguous and the breakpoints are not within 1 Mb on one contig), and either both of its items are positions or the candidate is well supported:
// >= 2 reads, or both breakpoints spliced with coverage < 200 at them, on different contigs or more than 1 Mb apart. The rules are read in order, but the
// outcome is a plain "some rule rescues it".
ARB_HD i64 abs_i64(i64 a) { return a < 0 ? -a : a; }
ARB_HD bool cand_close(const cand_state& c, u32 k) { return c.contig1[k] == c.contig2[k] && abs_i64((i64) c.bp2[k] - c.bp1[k]) < 1000000; }
// the per-candidate half of the rescue condition (:81-85), computed once per eligible candidate before the search: indexed by candidate id
struct known_support_fn {
	cand_state c; annot_view an; coverage_view cov; const u32* ids; u8* supported;
	ARB_HD void operator()(u32 i) const {
		const u32 k = ids[i];
		bool ok = cand_support(c, k) >= 2;
		if (!ok && cand_both_spliced(c, an, k)) {
			const int cov1 = cov.get(c.contig1[k], c.bp1[k], c.dir1[k] == UPSTREAM ? DOWNSTREAM : UPSTREAM), cov2 = cov.get(c.contig2[k], c.bp2[k], c.dir2[k] == UPSTREAM ? DOWNSTREAM : UPSTREAM);
			ok = cov1 + cov2 < 200 && (c.contig1[k] != c.contig2[k] || abs_i64((i64) c.bp2[k] - c.bp1[k]) > 1000000);
		}
		supported[k] = ok ? 1 : 0;
	}
};
struct known_fusion_test {
	rule_match m; const u8* supported;
	ARB_HD bool operator()(u32 rule, u32 k) const {
		if (!supported[k] && !(m.r.type[0][rule] == ARB_RULE_POSITION && m.r.type[1][rule] == ARB_RULE_POSITION)) return false; // a match would not rescue
		const u32 orders = m.c.bits2[k] && !cand_close(m.c, k) ? 2 : 1; // the swapped order only for an ambiguous transcript start, breakpoints not within 1 Mb
		for (u32 o = 0; o < orders; ++o) if (m.directional(rule, k, o != 0)) return true;
		return false;
	}
};
typedef rule_search<known_fusion_test> known_fusion_search;

// ---- tags (annotate_tags.cpp:45-83): the ranks of the tags of every rule that matches a row directionally. Pass 1 counts them per row, pass 2 (offset set)
// writes (rank, candidate) pairs at the row's offset. Duplicates (a rule listed under two bins of the row, two rules with one tag) are removed afterwards.
struct tag_search {
	cand_bins b; rule_match m; const u32* rank; // rank of every rule's tag among the distinct tags in bytewise order
	const u32* ids; u32 short_list;
	u8* heavy_mark; u32* heavy; u32* n_heavy;   // pass 1 queues the rows with a long list; pass 2 leaves them to the lane groups as well
	u32* count; const u32* offset;              // pass 1 writes count, pass 2 reads offset
	unsigned long long* total;                  // pass 1: the sum of all counts, in 64 bits (the 32-bit offsets are used only once it is known to fit)
	u32* out_rank; u32* out_cand;

	struct lanes_fn { // lane `lane` of `lanes`: rules a + lane, a + lane + lanes, ...; pass 2 writes at `at`, which advances
		const tag_search* s; u32 k, lane, lanes, n; u32 at;
		ARB_HD bool operator()(u32 a, u32 e) {
			for (u32 q = a + lane; q < e; q += lanes) {
				const u32 rule = s->b.t.rules[q];
				if (!s->m.directional(rule, k, false)) continue;
				if (s->offset) { s->out_rank[at] = s->rank[rule]; s->out_cand[at] = k; ++at; }
				++n;
			}
			return false;
		}
	};
	struct long_fn { const tag_search* s; ARB_HD bool operator()(u32 a, u32 e) const { return e - a > s->short_list; } };
	// a single thread is lane 0 of 1; returns the number of matches of this lane
	ARB_HD u32 lane_walk(u32 k, u32 lane, u32 lanes, u32 at) const { lanes_fn v = {this, k, lane, lanes, 0, at}; b.visit(k, v); return v.n; }
	ARB_HD void operator()(u32 i) const {
		const u32 k = ids[i];
		if (offset) { if (!heavy_mark[i]) lane_walk(k, 0, 1, offset[i]); return; }
		long_fn l = {this};
		if (b.visit(k, l)) { heavy_mark[i] = 1; count[i] = 0; heavy[append_slot(n_heavy)] = i; return; }
		heavy_mark[i] = 0; count[i] = lane_walk(k, 0, 1, 0);
		add_total(count[i]);
	}
	ARB_HD void add_total(u32 n) const {
		if (!n) return;
#ifdef __CUDA_ARCH__
		atomicAdd(total, (unsigned long long) n);
#else
		*total += n;
#endif
	}
};

// the distinct (candidate, rank) pairs after the sort by (candidate, rank): a pair is kept if it differs from the one before it
struct tag_head_fn {
	const u32* cand; const u32* rank; u32* head;
	ARB_HD void operator()(u32 j) const { head[j] = j == 0 || cand[j] != cand[j - 1] || rank[j] != rank[j - 1]; }
};
struct tag_compact_fn { // pair j -> slot[j] of the CSR, and one more tag for its candidate
	const u32* cand; const u32* rank; const u32* head; const u32* slot; u32* csr_rank; u32* per_cand;
	ARB_HD void operator()(u32 j) const { if (head[j]) { csr_rank[slot[j]] = rank[j]; atomic_add_u32(&per_cand[cand[j]], 1); } }
};

#ifdef ARB_DEVICE_BUILD
// a group of lanes per queued candidate: every lane tests its share of every list, __any_sync combines them
template <class Test> __device__ inline void rule_search_group(const lane_group& g, const rule_search<Test>& s, u32 i) {
	const bool found = s.lane_walk(s.ids[i], g.lane, g.lanes);
	const bool any = __any_sync(g.mask, found);
	if (g.lane == 0) s.verdict[i] = any ? 1 : 0;
}
// a group of lanes per queued row: every lane tests its share of a list, the ballot counts the matches and gives every lane its write position
struct tag_group_fn {
	const tag_search* s; const lane_group* g; u32 k, n, at;
	__device__ bool operator()(u32 a, u32 e) {
		for (u32 base = a; base < e; base += g->lanes) {
			const u32 q = base + g->lane;
			const u32 rule = q < e ? s->b.t.rules[q] : 0;
			const bool hit = q < e && s->m.directional(rule, k, false);
			const u32 mask = __ballot_sync(g->mask, hit);
			if (hit && s->offset) { const u32 j = at + n + __popc(mask & ((1u << g->lane) - 1u)); s->out_rank[j] = s->rank[rule]; s->out_cand[j] = k; }
			n += __popc(mask);
		}
		return false;
	}
};
__device__ inline void tag_group(const lane_group& g, const tag_search& s, u32 i) {
	tag_group_fn v = {&s, &g, s.ids[i], 0, s.offset ? s.offset[i] : 0};
	s.b.visit(v.k, v);
	if (!s.offset && g.lane == 0) { s.count[i] = v.n; s.add_total(v.n); }
}
#endif

} // namespace arb
