// blacklist_hd.h -- rules of a blacklist file (-b) matched to the candidates: filter_blacklisted_ranges (filter_blacklisted_ranges.cpp:138-300).
//
// The reference indexes the ELIGIBLE candidates (no filter yet, or closest_genomic_breakpoint1 >= 0 with -d) under the 100 kb bins of four ranges: both
// breakpoints and both genes. Every rule then visits the candidates of the bins of its positional items, each widened by max_mate_gap, and blacklists those
// for which (item1 matches breakpoint 1 and item2 breakpoint 2) or (item1 matches breakpoint 2 and item2 breakpoint 1). Removing a candidate from a bin's set
// only stops it from being tested again, and the test reads nothing the loop writes: the verdict is "eligible and some rule that shares a bin with the
// candidate matches", whatever the order of the file or of the candidates. Here the rules' bins become (contig, bin) keys, sorted into a key table with one
// rule list per key; every eligible candidate looks up its own bins and tests the rules listed there.
// The rule columns and rule_match do not depend on the blacklist: a file of known fusions (-k) has the same format and the same item test.
#pragma once
#include "model.h"
#include "prims.h"        // append_slot
#include "read_filters.h" // lane_group
#include "../../include/arriba_b200.h" // ARB_RULE_*
#include "events_hd.h"    // cand_state
#include "genomic_hd.h"   // wrap_add / wrap_sub

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
ARB_HD u32 rule_bin_key(u32 contig, i32 bin) { return contig << 16 | (u32) (bin + 32768); }

// the bins a positional item of a rule is looked up under: (contig, start - max_mate_gap, end + max_mate_gap) (:272-275)
ARB_HD void rule_item_bins(const rule_columns& r, u32 rule, u32 side, i32 max_mate_gap, i32& lo, i32& hi) {
	rule_bins((i64) r.start[side][rule] - max_mate_gap, (i64) r.end[side][rule] + max_mate_gap, lo, hi);
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
};

// ---- key table of the rules (engine: filter_blacklist): counts, scan, fill, sort, then one entry per distinct key
struct rule_key_count_fn { // number of (contig, bin) keys of every rule
	rule_columns r; i32 max_mate_gap; u32* count; unsigned long long* total;
	ARB_HD void operator()(u32 rule) const {
		u32 n = 0;
		for (u32 side = 0; side < 2; ++side) {
			if (!rule_item_positional(r.type[side][rule])) continue;
			i32 lo, hi; rule_item_bins(r, rule, side, max_mate_gap, lo, hi);
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
	rule_columns r; i32 max_mate_gap; const u32* offset; u32* key; u32* rule_of;
	ARB_HD void operator()(u32 rule) const {
		u32 at = offset[rule];
		for (u32 side = 0; side < 2; ++side) {
			if (!rule_item_positional(r.type[side][rule])) continue;
			i32 lo, hi; rule_item_bins(r, rule, side, max_mate_gap, lo, hi);
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

// ---- the search: one thread per eligible candidate; a candidate with a long rule list goes to a group of lanes
struct blacklist_search {
	rule_match m; rule_key_table t;
	const u32* ids; u8* verdict;        // eligible candidates, one verdict byte each
	u32 short_list;                     // lists up to this length are walked by the candidate's own thread
	u32* heavy; u32* n_heavy;           // positions in `ids` of the candidates queued for a group of lanes

	// the four ranges a candidate is indexed under (:244-247): both breakpoints, then both genes
	ARB_HD void range(u32 k, u32 x, u32& contig, i32& lo, i32& hi) const {
		const cand_state& c = m.c;
		contig = (x & 1) ? c.contig2[k] : c.contig1[k];
		if (x < 2) { const i32 bp = x ? c.bp2[k] : c.bp1[k]; rule_bins(bp, bp, lo, hi); }
		else { const u32 g = x == 2 ? c.gene1[k] : c.gene2[k]; rule_bins(m.an.gene_start[g], m.an.gene_end[g], lo, hi); }
	}
	// a bin already listed by an earlier range of the same candidate is looked up once
	ARB_HD bool listed_before(u32 k, u32 x, u32 contig, i32 bin) const {
		for (u32 y = 0; y < x; ++y) { u32 cy; i32 lo, hi; range(k, y, cy, lo, hi); if (cy == contig && bin >= lo && bin <= hi) return true; }
		return false;
	}
	// lane `lane` of `lanes` tests rules lo + lane, lo + lane + lanes, ... of every list of candidate k; a single thread is lane 0 of 1
	ARB_HD bool lane_walk(u32 k, u32 lane, u32 lanes) const {
		for (u32 x = 0; x < 4; ++x) {
			u32 contig; i32 lo, hi; range(k, x, contig, lo, hi);
			for (i32 b = lo; b <= hi; ++b) {
				u32 a, e;
				if (listed_before(k, x, contig, b) || !t.find(rule_bin_key(contig, b), a, e)) continue;
				for (u32 q = a + lane; q < e; q += lanes) if (m(t.rules[q], k)) return true;
			}
		}
		return false;
	}
	ARB_HD void operator()(u32 i) const {
		const u32 k = ids[i];
		for (u32 x = 0; x < 4; ++x) {
			u32 contig; i32 lo, hi; range(k, x, contig, lo, hi);
			for (i32 b = lo; b <= hi; ++b) {
				u32 a, e;
				if (listed_before(k, x, contig, b) || !t.find(rule_bin_key(contig, b), a, e)) continue;
				if (e - a > short_list) { heavy[append_slot(n_heavy)] = i; return; }
				for (u32 q = a; q < e; ++q) if (m(t.rules[q], k)) { verdict[i] = 1; return; }
			}
		}
		verdict[i] = 0;
	}
};

#ifdef ARB_DEVICE_BUILD
// a group of lanes per queued candidate: every lane tests its share of every list, __any_sync combines them
__device__ inline void blacklist_group(const lane_group& g, const blacklist_search& s, u32 i) {
	const bool found = s.lane_walk(s.ids[i], g.lane, g.lanes);
	const bool any = __any_sync(g.mask, found);
	if (g.lane == 0) s.verdict[i] = any ? 1 : 0;
}
#endif

} // namespace arb
