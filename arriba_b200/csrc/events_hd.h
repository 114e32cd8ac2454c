// events_hd.h -- candidate-level ("event-level") device stages: merging of adjacent breakpoints and the e-value model.
//
// Reference behaviour: merge_adjacent_fusions (merge_adjacent_fusions.cpp:19-108), estimate_expected_fusions
// (filter_relative_support.cpp:17-207), filter_relative_support (:209-223).
//
// merge_adjacent is sequential in coordinate order and updates the very counters it compares, but two candidates can only
// interact when their first breakpoints lie within max_distance on the same contig. After a radix sort by
// (contig1, breakpoint1, contig2, breakpoint2) the table therefore splits into independent clusters (gap > max_distance
// or contig change); one thread replays one cluster sequentially, clusters run in parallel.
#pragma once
#include "model.h"
#include "annot_hd.h"
#include "prims.h"

namespace arb {

struct cand_state { // mutable event-level columns, device copies
	u32 n;
	const u32* gene1; const u32* gene2; const u16* contig1; const u16* contig2; const i32* bp1; const i32* bp2; const u8* dir1; const u8* dir2; const u8* bits; const u8* bits2; // bits2: 1 = transcript start ambiguous
	u32* split_reads1; u32* split_reads2; u32* discordant_mates; u8* filter; float* evalue;
	u32* n_list1; u32* n_list2; // current sizes of the split-read lists (grow when ITD lists are merged)
};

ARB_HD bool cand_is_itd(const cand_state& c, u32 k, u32 max_itd_length) { // common.hpp:270-274
	return c.gene1[k] == c.gene2[k] && ((u32) c.bp2[k] - (u32) c.bp1[k]) < max_itd_length && c.dir1[k] == UPSTREAM && c.dir2[k] == DOWNSTREAM;
}
ARB_HD u32 cand_support(const cand_state& c, u32 k) { return c.split_reads1[k] + c.split_reads2[k] + c.discordant_mates[k]; }
ARB_HD bool cand_both_spliced(const cand_state& c, const annot_view& an, u32 k) { // both_breakpoints_spliced (common.hpp:280-284)
	const u8 bits = c.bits[k];
	const bool f1 = an.gene_strand[c.gene1[k]], f2 = an.gene_strand[c.gene2[k]];
	return (bits & CB_SPLICED1) && (bits & CB_SPLICED2) && ((f1 == f2 && c.dir1[k] != c.dir2[k]) || (f1 != f2 && c.dir1[k] == c.dir2[k]));
}

struct merge_eligible_fn { // candidates that take part: unfiltered, or ITD-shaped (merge_adjacent_fusions.cpp:23-26)
	cand_state c; u32 max_itd_length; u32* flag;
	ARB_HD void operator()(u32 k) const { flag[k] = (c.filter[k] == F_none || cand_is_itd(c, k, max_itd_length)) ? 1 : 0; }
};
struct merge_gather_fn { const u32* flag_scan; u32* ids; ARB_HD void operator()(u32 k) const { if (flag_scan[k + 1] != flag_scan[k]) ids[flag_scan[k]] = k; } };
// sort keys, least significant first: bp2, contig2, bp1, contig1 (stable LSD passes on the same permutation)
struct merge_key_fn {
	cand_state c; const u32* ids; u32* key; int which;
	ARB_HD void operator()(u32 j) const {
		const u32 k = ids[j];
		key[j] = which == 0 ? (u32) c.bp2[k] : which == 1 ? (u32) c.contig2[k] : which == 2 ? (u32) c.bp1[k] : (u32) c.contig1[k];
	}
};
struct merge_cluster_head_fn { // position j starts a cluster if it cannot interact with position j-1
	cand_state c; const u32* ids; u32* head; i32 max_distance;
	ARB_HD void operator()(u32 j) const {
		if (j == 0) { head[j] = 1; return; }
		const u32 a = ids[j - 1], b = ids[j];
		head[j] = (c.contig1[a] != c.contig1[b] || c.bp1[b] - c.bp1[a] > max_distance) ? 1 : 0;
	}
};
struct merge_cluster_start_fn { const u32* head_scan; u32* start; u32 n; u32 n_clusters; ARB_HD void operator()(u32 j) const { if (head_scan[j + 1] != head_scan[j]) start[head_scan[j]] = j; if (j == n - 1) start[n_clusters] = n; } };

struct merge_cluster_fn {
	cand_state c; const u32* ids; const u32* cluster_start; i32 max_distance; u32 max_itd_length;
	u32* itd_log; u32* itd_log_count; u32 itd_log_capacity; // (winner, loser, sorted position of winner) triples
	ARB_HD bool partner(u32 f, u32 o, bool itd, bool o_is_before) const {
		if (!(c.gene1[o] == c.gene1[f] && c.gene2[o] == c.gene2[f] && c.dir1[o] == c.dir1[f] && c.dir2[o] == c.dir2[f] && c.contig2[o] == c.contig2[f])) return false;
		const i32 sign = (c.dir1[f] == c.dir2[f]) ? +1 : -1;
		const i32 shift = o_is_before ? (c.bp1[f] - c.bp1[o]) * sign : (c.bp1[o] - c.bp1[f]) * -sign; // breakpoints must be shifted in the same sense
		if (!(c.bp2[o] == c.bp2[f] + shift || (itd && hd_abs(c.bp2[f] - c.bp2[o]) <= max_distance))) return false;
		return c.split_reads1[o] + c.split_reads2[o] > 0 || (itd && c.n_list1[o] + c.n_list2[o] > 0);
	}
	ARB_HD void operator()(u32 cl) const {
		const u32 lo = cluster_start[cl], hi = cluster_start[cl + 1];
		for (u32 j = lo; j < hi; ++j) {
			const u32 f = ids[j];
			const bool itd = cand_is_itd(c, f, max_itd_length);
			if ((!itd && c.split_reads1[f] + c.split_reads2[f] == 0) || (itd && c.n_list1[f] + c.n_list2[f] == 0)) continue;
			// neighbours: upstream (descending), then downstream (ascending), as the reference collects them; decide + sum in that order
			u32 sum1 = 0, sum2 = 0; bool most = true;
			for (int pass = 0; pass < 2 && most; ++pass) {
				if (pass == 0) {
					for (u32 q = j; q-- > lo;) {
						const u32 o = ids[q];
						if (c.bp1[o] < c.bp1[f] - max_distance) break;
						if (!partner(f, o, itd, true)) continue;
						if (cand_support(c, f) < cand_support(c, o) || (cand_support(c, f) == cand_support(c, o) && c.n_list1[f] + c.n_list2[f] < c.n_list1[o] + c.n_list2[o])) { most = false; break; }
						sum1 += c.split_reads1[o]; sum2 += c.split_reads2[o];
					}
				} else {
					for (u32 q = j + 1; q < hi; ++q) {
						const u32 o = ids[q];
						if (c.bp1[o] > c.bp1[f] + max_distance) break;
						if (!partner(f, o, itd, false)) continue;
						if (cand_support(c, f) < cand_support(c, o) || (cand_support(c, f) == cand_support(c, o) && c.n_list1[f] + c.n_list2[f] < c.n_list1[o] + c.n_list2[o])) { most = false; break; }
						sum1 += c.split_reads1[o]; sum2 += c.split_reads2[o];
					}
				}
			}
			if (!most) continue;
			c.split_reads1[f] += sum1; c.split_reads2[f] += sum2;
			for (int pass = 0; pass < 2; ++pass) {
				if (pass == 0) {
					for (u32 q = j; q-- > lo;) { const u32 o = ids[q]; if (c.bp1[o] < c.bp1[f] - max_distance) break; if (partner(f, o, itd, true)) absorb(f, o, itd, j); }
				} else {
					for (u32 q = j + 1; q < hi; ++q) { const u32 o = ids[q]; if (c.bp1[o] > c.bp1[f] + max_distance) break; if (partner(f, o, itd, false)) absorb(f, o, itd, j); }
				}
			}
		}
	}
	ARB_HD void absorb(u32 f, u32 o, bool itd, u32 pos) const {
		c.filter[o] = F_merge_adjacent;
		if (itd) { // discarded reads matter for ITDs: the loser's lists are appended to the winner's (done by the caller from this log)
			const u32 at = atomic_add_u32(itd_log_count, 1);
			if (at < itd_log_capacity) { itd_log[3 * at] = f; itd_log[3 * at + 1] = o; itd_log[3 * at + 2] = pos; }
			c.n_list1[f] += c.n_list1[o]; c.n_list2[f] += c.n_list2[o];
		}
	}
};

// ------------------------------------------------------------------------------------------- e-value
struct evalue_inputs { // host-computed, order-dependent global statistics (filter_relative_support.cpp:19-127) and pow() tables
	const i32* partner_count;      // per gene: fusion_partner_count (0 if absent)
	u32 spliced_breakpoints, exonic_breakpoints, intronic_breakpoints, exonic_intronic_breakpoints;
	u32 intragenic_duplications, intragenic_inversions, spliced_same_gene, spliced_different_genes;
	float read_through_fraction;
	u64 mapped_reads;
	const double* pow_reads;       // pow(0.02, n - 2) as the reference evaluates it, n = supporting reads (index clamped to table size)
	const double* pow_intragenic;  // pow(n - 0.42, -2.11) * pow(10, -1.11)
	const double* pow_intergenic;  // pow(n - 0.73, -2.28) * pow(10, -1.75)
	u32 n_read_table;
	const double* pow_spliced1000; // pow(max(400, d) / 1000.0, -2), d < 1000
	const double* pow_spliced400;  // pow(max(1, d) / 400.0, -4.58), d < 400
	const double* pow_read_through;// pow(max(1, d) / 400000.0, -0.63), d < 400000
	const double* pow_proximal;    // pow(max(1, d) / 400000.0, -1.53), d < 400000
	double read_through_penalty;   // 1 + pow((fraction - 0.25) * 20, 2)
	float cutoff; u32 apply_filter;
};

struct evalue_fn {
	cand_state c; annot_view an; evalue_inputs in;
	ARB_HD void operator()(u32 k) const {
		const u32 g1 = c.gene1[k], g2 = c.gene2[k];
		const i32 bp1 = c.bp1[k], bp2 = c.bp2[k];
		const u32 d1 = c.dir1[k], d2 = c.dir2[k];
		const u32 reads = cand_support(c, k);
		const double a = 10000.0 / an.gene_exonic_length[g1] * hd_max(in.partner_count[g1] - 1, 1);
		const double b = 10000.0 / an.gene_exonic_length[g2] * hd_max(in.partner_count[g2] - 1, 1);
		const float max_partners = (float) (a > b ? a : b);
		const u32 ri = reads < in.n_read_table ? reads : in.n_read_table - 1;
		const double scale = (double) in.mapped_reads / 20000000.0 * in.pow_reads[ri];
		float e = (float) ((double) max_partners * (1.0 > scale ? 1.0 : scale));
		const i32 g1s = an.gene_start[g1], g1e = an.gene_end[g1], g2s = an.gene_start[g2], g2e = an.gene_end[g2];
		const bool intragenic = g1 == g2 || (bp1 >= g2s - 10000 && bp1 <= g2e + 10000 && bp2 >= g1s - 10000 && bp2 <= g1e + 10000);
		const bool read_through = c.contig1[k] == c.contig2[k] && bp2 - bp1 < 400000 && d1 == DOWNSTREAM && d2 == UPSTREAM;
		if (intragenic) {
			e = (float) ((double) e * (2.0 / (in.intragenic_duplications + in.intragenic_inversions)));
			if (d1 == UPSTREAM && d2 == DOWNSTREAM) e = (float) ((float) e * (float) in.intragenic_duplications); // float *= unsigned: float arithmetic
			else if (d1 == d2) e = (float) ((float) e * (float) in.intragenic_inversions);
			if (reads >= 1) {
				e = (float) ((double) e * in.pow_intragenic[ri]);
				const i32 sd = spliced_distance(an, c.contig1[k], bp1, bp2, g1);
				if (sd < 1000) {
					e = (float) ((double) e * in.pow_spliced1000[sd < 0 ? 0 : sd]);
					if (sd < 400) e = (float) ((double) e * in.pow_spliced400[sd < 0 ? 0 : sd]);
				}
			}
			const double penalty = (double) in.spliced_same_gene / 0.25 / (double) in.spliced_different_genes;
			e = (float) ((double) e * (1.0 > penalty ? 1.0 : penalty));
		} else if (reads >= 1) {
			e = (float) ((double) e * in.pow_intergenic[ri]);
			const i32 dist = bp2 - bp1;
			if (read_through) e = (float) ((double) e * in.pow_read_through[dist < 1 ? 0 : dist]);
			else if (c.contig1[k] == c.contig2[k] && dist < 400000) e = (float) ((double) e * in.pow_proximal[dist < 1 ? 0 : dist]);
		}
		e = (float) ((double) e * (4.0 / (in.spliced_breakpoints + in.exonic_breakpoints + in.intronic_breakpoints + in.exonic_intronic_breakpoints)));
		const u8 bits = c.bits[k];
		u32 factor;
		if (bits & (CB_SPLICED1 | CB_SPLICED2)) factor = in.spliced_breakpoints;
		else if ((bits & CB_EXONIC1) && (bits & CB_EXONIC2)) factor = hd_max(in.spliced_breakpoints, in.exonic_breakpoints);
		else if (!(bits & CB_EXONIC1) && !(bits & CB_EXONIC2)) factor = hd_max(in.spliced_breakpoints, in.intronic_breakpoints);
		else factor = hd_max(in.spliced_breakpoints, in.exonic_intronic_breakpoints);
		e = e * (float) factor;
		if (in.read_through_fraction > 0.25 && read_through) e = (float) ((double) e * in.read_through_penalty);
		c.evalue[k] = e;
	}
};

struct relative_support_fn { // filter_relative_support.cpp:209-223
	cand_state c; annot_view an; float cutoff;
	ARB_HD void operator()(u32 k) const {
		if (c.filter[k] != F_none) return;
		const u32 g1 = c.gene1[k], g2 = c.gene2[k];
		const i32 bp1 = c.bp1[k], bp2 = c.bp2[k];
		const bool intragenic = g1 == g2 || (bp1 >= an.gene_start[g2] - 10000 && bp1 <= an.gene_end[g2] + 10000 && bp2 >= an.gene_start[g1] - 10000 && bp2 <= an.gene_end[g1] + 10000);
		if (!(c.evalue[k] < cutoff && !(intragenic && c.split_reads1[k] + c.split_reads2[k] == 0))) c.filter[k] = F_relative_support;
	}
};

// ---- global tallies of the e-value model (filter_relative_support.cpp:62-127): breakpoint locations, intragenic duplications / inversions, spliced pairs, genes
// with fusions / with read-through fusions, and the largest number of supporting reads (size of the pow tables the caller builds)
enum { ET_SPLICED = 0, ET_EXONIC, ET_INTRONIC, ET_MIXED, ET_DUPLICATIONS, ET_INVERSIONS, ET_SPLICED_SAME, ET_SPLICED_DIFFERENT, ET_GENES_WITH_FUSIONS, ET_GENES_WITH_READ_THROUGH, ET_MAX_READS, ET_COUNT };
struct evalue_tally_fn {
	cand_state c; annot_view an; u32* tally; u8* with_fusion; u8* with_read_through;
	ARB_HD void operator()(u32 k) const {
		const u32 g1 = c.gene1[k], g2 = c.gene2[k];
		const bool dummy = (an.gene_flags[g1] & GF_DUMMY) || (an.gene_flags[g2] & GF_DUMMY);
		const u32 split = c.split_reads1[k] + c.split_reads2[k], support = split + c.discordant_mates[k];
		const u8 b = c.bits[k]; const bool unfiltered = c.filter[k] == F_none;
		if (unfiltered && (c.contig1[k] != c.contig2[k] || c.bp2[k] - c.bp1[k] > 500000) && support >= 2 && split > 0 && !dummy)
			atomic_add_u32(&tally[(b & (CB_SPLICED1 | CB_SPLICED2)) ? ET_SPLICED : ((b & CB_EXONIC1) && (b & CB_EXONIC2)) ? ET_EXONIC : (!(b & CB_EXONIC1) && !(b & CB_EXONIC2)) ? ET_INTRONIC : ET_MIXED], 1);
		if (unfiltered && g1 == g2 && split >= 2) { if (c.dir1[k] == UPSTREAM && c.dir2[k] == DOWNSTREAM) atomic_add_u32(&tally[ET_DUPLICATIONS], 1); else if (c.dir1[k] == c.dir2[k]) atomic_add_u32(&tally[ET_INVERSIONS], 1); }
		if ((b & CB_SPLICED1) && (b & CB_SPLICED2)) atomic_add_u32(&tally[g1 == g2 ? ET_SPLICED_SAME : ET_SPLICED_DIFFERENT], 1);
		if (!dummy && split > 0) {
			with_fusion[g1] = 1; with_fusion[g2] = 1;
			if (c.contig1[k] == c.contig2[k] && c.bp2[k] - c.bp1[k] < 400000 && c.dir1[k] == DOWNSTREAM && c.dir2[k] == UPSTREAM) { with_read_through[g1] = 1; with_read_through[g2] = 1; }
		}
#ifdef __CUDA_ARCH__
		if (support > tally[ET_MAX_READS]) atomicMax(&tally[ET_MAX_READS], support);
#else
		if (support > tally[ET_MAX_READS]) tally[ET_MAX_READS] = support;
#endif
	}
};
struct evalue_gene_tally_fn { const u8* with_fusion; const u8* with_read_through; u32* tally;
	ARB_HD void operator()(u32 g) const { if (with_fusion[g]) atomic_add_u32(&tally[ET_GENES_WITH_FUSIONS], 1); if (with_read_through[g]) atomic_add_u32(&tally[ET_GENES_WITH_READ_THROUGH], 1); } };

// ---- select_best (select_best.cpp): the candidates of one (gene1, gene2, direction1, direction2) compete in the order the reference visits them -- the comparison is
// not a total order, so the order matters: stable sorts by (key, iteration rank), then every group is one sequential scan
struct select_eligible_fn { cand_state c; u32* flag; ARB_HD void operator()(u32 k) const { flag[k] = c.filter[k] == F_none ? 1u : 0u; } };
struct select_key_fn { // which: 0 = iteration rank, 1 = low word of the key (gene2 << 4 | directions), 2 = high word (gene1)
	cand_state c; const u32* rank; const u32* ids; u32* key; int which;
	ARB_HD void operator()(u32 j) const {
		const u32 k = ids[j];
		key[j] = which == 0 ? rank[k] : which == 1 ? (c.gene2[k] << 2 | (c.dir1[k] != 0 ? 2u : 0u) | (c.dir2[k] != 0 ? 1u : 0u)) : c.gene1[k];
	}
};
struct select_head_fn { cand_state c; const u32* ids; u32* head;
	ARB_HD void operator()(u32 j) const {
		if (j == 0) { head[j] = 1; return; }
		const u32 a = ids[j - 1], b = ids[j];
		head[j] = (c.gene1[a] != c.gene1[b] || c.gene2[a] != c.gene2[b] || (c.dir1[a] != 0) != (c.dir1[b] != 0) || (c.dir2[a] != 0) != (c.dir2[b] != 0)) ? 1u : 0u;
	}
};
struct select_group_fn {
	cand_state c; const u32* ids; const u32* group_start;
	ARB_HD u32 rank(u32 k) const { const bool s1 = c.split_reads1[k] != 0, s2 = c.split_reads2[k] != 0, d = c.discordant_mates[k] != 0; return (s1 && s2) ? 3u : ((s1 || s2) && d) ? 2u : (s1 || s2) ? 1u : 0u; }
	ARB_HD bool challenger_wins(u32 k, u32 b) const { // select_best.cpp:22-60
		if (rank(k) > rank(b)) return true;
		if (rank(k) != rank(b)) return false;
		if (cand_support(c, k) > cand_support(c, b)) return true;
		if (cand_support(c, k) != cand_support(c, b)) return false;
		const bool k1 = c.bits[k] & CB_EXONIC1, k2 = c.bits[k] & CB_EXONIC2, b1 = c.bits[b] & CB_EXONIC1, b2 = c.bits[b] & CB_EXONIC2;
		if ((k1 && !b1) || (k2 && !b2)) return true;
		if ((!b1 || k1 == b1) && (!b2 || k2 == b2)) {
			if ((c.dir1[k] == DOWNSTREAM && c.bp1[k] > c.bp1[b]) || (c.dir1[k] == UPSTREAM && c.bp1[k] < c.bp1[b])) return true;
			if (c.bp1[k] == c.bp1[b]) return (c.dir2[k] == DOWNSTREAM && c.bp2[k] > c.bp2[b]) || (c.dir2[k] == UPSTREAM && c.bp2[k] < c.bp2[b]);
		}
		return false;
	}
	ARB_HD void operator()(u32 g) const {
		const u32 lo = group_start[g], hi = group_start[g + 1];
		u32 best = ids[lo];
		for (u32 x = lo + 1; x < hi; ++x) if (challenger_wins(ids[x], best)) best = ids[x];
		for (u32 x = lo; x < hi; ++x) if (ids[x] != best) c.filter[ids[x]] = F_select_best;
	}
};

// ---- per-candidate predicates of the event chain that only look at the candidate itself: filter_non_coding_neighbors.cpp, filter_intragenic_both_exonic.cpp,
// filter_min_support.cpp; `remaining` counts the candidates that are still unfiltered afterwards (the stage's "(remaining=N)" line)
enum { SIMPLE_NON_CODING_NEIGHBORS = 0, SIMPLE_INTRAGENIC_EXONIC = 1, SIMPLE_MIN_SUPPORT = 2 };
struct simple_filter_fn {
	cand_state c; annot_view an; int stage; float exonic_fraction; int min_support; u32* remaining;
	ARB_HD bool read_through(u32 k) const { return c.contig1[k] == c.contig2[k] && c.bp2[k] - c.bp1[k] < 400000 && c.dir1[k] == DOWNSTREAM && c.dir2[k] == UPSTREAM; } // common.hpp:265-269
	ARB_HD bool overlaps_both(u32 k) const { // common.hpp:260-264
		const u32 g1 = c.gene1[k], g2 = c.gene2[k];
		return (c.bp1[k] >= an.gene_start[g2] && c.bp1[k] <= an.gene_end[g2]) || (c.bp2[k] >= an.gene_start[g1] && c.bp2[k] <= an.gene_end[g1]);
	}
	ARB_HD void operator()(u32 k) const {
		if (c.filter[k] != F_none) return;
		const u32 g1 = c.gene1[k], g2 = c.gene2[k];
		u8 verdict = F_none;
		if (stage == SIMPLE_NON_CODING_NEIGHBORS) {
			if (!(an.gene_flags[g1] & GF_CODING) && !(an.gene_flags[g2] & GF_CODING) && read_through(k)) verdict = F_non_coding_neighbors;
		} else if (stage == SIMPLE_INTRAGENIC_EXONIC) {
			const u8 b = c.bits[k];
			if ((overlaps_both(k) || g1 == g2) && (b & CB_EXONIC1) && (b & CB_EXONIC2) && !((b & CB_SPLICED1) && (b & CB_SPLICED2))) {
				const int sd = spliced_distance(an, c.contig1[k], c.bp1[k], c.bp2[k], g1);
				const int distance = c.bp2[k] - c.bp1[k];
				if (sd == distance || 1.0 * sd / distance < exonic_fraction) verdict = F_intragenic_exonic;
			}
		} else {
			const int split = (int) (c.split_reads1[k] + c.split_reads2[k]);
			if (split + (int) c.discordant_mates[k] < min_support || (overlaps_both(k) && split < min_support)) verdict = F_min_support;
		}
		if (verdict != F_none) c.filter[k] = verdict; else atomic_add_u32(remaining, 1);
	}
};

// ---- expression per gene (filter_in_vitro.cpp:48-83): supporting fragments per gene of MATE1 and of the last alignment
struct reads_by_gene_fn {
	frag_view f; u32* reads;
	ARB_HD void operator()(u32 i) const {
		const u32 a = f.idx(i, 0), b = f.idx(i, f.n_aln[i] == 2 ? 1 : 2);
		for (u32 g = 0; g < f.genes_cnt[a]; ++g) atomic_add_u32(&reads[f.genes[f.genes_off[a] + g]], 1);
		for (u32 g = 0; g < f.genes_cnt[b]; ++g) atomic_add_u32(&reads[f.genes[f.genes_off[b] + g]], 1);
	}
};

// coverage windows on the device (read_stats.cpp:268-306): 20 bp windows per contig, one flat array
struct coverage_view {
	const u16* windows; const u64* contig_off; const u32* contig_windows; u32 n_contigs;
	ARB_HD int get(u32 contig, i32 position, u32 direction) const {
		if (contig >= n_contigs || contig_windows[contig] == 0) return -1;
		const u16* c = windows + contig_off[contig];
		if (direction == UPSTREAM) return position < 20 ? 0 : (int) c[position / 20 - 1];
		return (int) c[position / 20 + 1];
	}
};

// ---- filter_in_vitro (filter_in_vitro.cpp:85-228), one thread per candidate: the verdict of a candidate does not depend on the other verdicts
struct in_vitro_inputs { const u32* reads_by_gene; u32 threshold; const u64* exonic_pairs; u64 n_pairs; };
struct in_vitro_fn {
	cand_state c; frag_view f; annot_view an; coverage_view cov; in_vitro_inputs in;
	const u32* listd_off; const u32* listd;
	ARB_HD u32 higher_expressed(u16 contig, i32 bp, u32 gene) const { // the most expressed gene at the breakpoint, the candidate's own gene unless another one has more reads
		u32 highest = in.reads_by_gene[gene];
		if (contig >= an.n_contigs) return gene;
		const u32 lo = an.gene_region_begin[contig], hi = an.gene_region_begin[contig + 1];
		const u32 r = region_lower_bound(an.gene_region_end, lo, hi, bp);
		if (r < hi) for (u32 x = an.gene_region_off[r]; x < an.gene_region_off[r + 1]; ++x) { const u32 g = an.gene_region_items[x]; if (in.reads_by_gene[g] > highest) { highest = in.reads_by_gene[g]; gene = g; } }
		return gene;
	}
	ARB_HD u32 pair_count(u32 a, u32 b) const { // width of the equal range of (a, b) in the sorted pair list
		const u64 key = (u64) a << 32 | b;
		u64 lo = 0, hi = in.n_pairs;
		while (lo < hi) { const u64 mid = lo + ((hi - lo) >> 1); if (in.exonic_pairs[mid] < key) lo = mid + 1; else hi = mid; }
		u64 lo2 = lo, hi2 = in.n_pairs;
		while (lo2 < hi2) { const u64 mid = lo2 + ((hi2 - lo2) >> 1); if (in.exonic_pairs[mid] <= key) lo2 = mid + 1; else hi2 = mid; }
		return (u32) (lo2 - lo);
	}
	ARB_HD void operator()(u32 k) const {
		const u8 fl = c.filter[k]; const u8 bits = c.bits[k];
		const bool spliced1 = bits & CB_SPLICED1, spliced2 = bits & CB_SPLICED2, exonic1 = bits & CB_EXONIC1, exonic2 = bits & CB_EXONIC2;
		if (fl != F_none && !((spliced1 || spliced2) && (fl == F_relative_support || fl == F_min_support || fl == F_homopolymer))) return;
		float rt = 0;
		if (!exonic1) rt += 0.5f; else if (!spliced1) rt += 1;
		if (!exonic2) rt += 0.5f; else if (!spliced2) rt += 1;
		const u32 own_split = c.split_reads1[k] + c.split_reads2[k], dm = c.discordant_mates[k];
		if (own_split > 2 && own_split * 2 > dm) return; // total_split >= own_split: "total_split * 2 <= discordant_mates || total_split <= 2" cannot hold
		const u16 contig1 = c.contig1[k], contig2 = c.contig2[k]; const i32 bp1 = c.bp1[k], bp2 = c.bp2[k];
		const u32 g1 = higher_expressed(contig1, bp1, c.gene1[k]), g2 = higher_expressed(contig2, bp2, c.gene2[k]);
		const u32 x1 = in.reads_by_gene[g1], x2 = in.reads_by_gene[g2];
		if (!(x1 + x2 > in.threshold)) return; // only breakpoints in highly expressed genes are suspected
		u32 clipped1 = 0, clipped2 = 0;
		for (u32 p = listd_off[k]; p < listd_off[k + 1]; ++p) {
			const u32 i = listd[p];
			if (f.filter[i] != F_none) continue;
			for (u32 s = 0; s < f.n_aln[i]; ++s) {
				const u32 a = f.idx(i, s);
				if (f.fwd(a) && f.postclip(a) >= 3) { if (f.contig[a] == contig1 && f.end[a] == bp1) ++clipped1; else if (f.contig[a] == contig2 && f.end[a] == bp2) ++clipped2; }
				else if (!f.fwd(a) && f.preclip(a) >= 3) { if (f.contig[a] == contig1 && f.start[a] == bp1) ++clipped1; else if (f.contig[a] == contig2 && f.start[a] == bp2) ++clipped2; }
			}
		}
		const u32 total_split = hd_min(clipped1, clipped2) + own_split;
		if (!(total_split * 2 <= dm || total_split <= 2)) return;
		if (!((double) total_split <= 2 + 0.0001 * (double) (x1 + x2))) return;
		const u32 sup = own_split + dm;
		if (sup >= 10 && (spliced1 || spliced2) && ((spliced1 || !exonic1) && (spliced2 || !exonic2))) {
			const int cov1 = cov.get(contig1, bp1, c.dir1[k] == UPSTREAM ? DOWNSTREAM : UPSTREAM), cov2 = cov.get(contig2, bp2, c.dir2[k] == UPSTREAM ? DOWNSTREAM : UPSTREAM);
			if (((int) sup * 4) >= hd_max(cov1, cov2) && cov1 > (int) sup && cov2 > (int) sup) return; // well covered on both sides: kept
		}
		const u32 threshold = in.threshold;
		if (rt > 1 || (rt > 0 && (x1 > threshold || x2 > threshold)) || x1 > 2 * threshold || x2 > 2 * threshold || (x1 > threshold && x2 > threshold) || sup <= 1 ||
		    hd_max(pair_count(g1, g2), pair_count(c.gene1[k], c.gene2[k])) > 8)
			c.filter[k] = F_in_vitro;
	}
};

// ---- recover_both_spliced: spliced support of a candidate (recover_both_spliced.cpp:15-62), a pure function of the candidate
struct spliced_support_fn {
	cand_state c; frag_view f; annot_view an; coverage_view cov; const u32* reads_by_gene; u32 threshold;
	const u32* l1o; const u32* l1; const u32* l2o; const u32* l2; const u32* ldo; const u32* ld; u32* support; // 0xFFFFFFFF: not eligible
	ARB_HD bool both_spliced(u32 k) const { return cand_both_spliced(c, an, k); }
	ARB_HD bool long_exon_at(u16 contig, i32 bp) const { // any exon over the breakpoint longer than 1000 bases (a point query returns the region's items)
		if (contig >= an.n_contigs) return false;
		const u32 lo = an.exon_region_begin[contig], hi = an.exon_region_begin[contig + 1];
		const u32 r = region_lower_bound(an.exon_region_end, lo, hi, bp);
		if (r < hi) for (u32 x = an.exon_region_off[r]; x < an.exon_region_off[r + 1]; ++x) { const u32 e = an.exon_region_items[x]; if (an.exon_end[e] + 1 - an.exon_start[e] > 1000) return true; }
		return false;
	}
	ARB_HD void scan(const u32* off, const u32* list, u32 k, u32& multi, u32& unique) const {
		for (u32 p = off[k]; p < off[k + 1]; ++p) { const u32 i = list[p]; if (f.fflags[i] & FF_MULTIMAPPER) ++multi; else if (f.filter[i] == F_none) ++unique; }
	}
	ARB_HD u32 spliced_support(u32 k) const {
		const u32 max_coverage = 1000; // arriba.cpp:492
		const bool bs = both_spliced(k);
		if (reads_by_gene[c.gene1[k]] > threshold || reads_by_gene[c.gene2[k]] > threshold) return (bs && c.discordant_mates[k] <= c.split_reads1[k] + c.split_reads2[k]) ? 1u : 0u;
		if (!bs) {
			const u32 cov1 = (u32) cov.get(c.contig1[k], c.bp1[k], c.dir1[k] == UPSTREAM ? DOWNSTREAM : UPSTREAM), cov2 = (u32) cov.get(c.contig2[k], c.bp2[k], c.dir2[k] == UPSTREAM ? DOWNSTREAM : UPSTREAM);
			if (cov1 + cov2 > cand_support(c, k) * max_coverage) return 0;
			if (long_exon_at(c.contig1[k], c.bp1[k]) || long_exon_at(c.contig2[k], c.bp2[k])) return 0;
		}
		u32 multi = 0, unique = 0;
		scan(l1o, l1, k, multi, unique); scan(l2o, l2, k, multi, unique); scan(ldo, ld, k, multi, unique);
		const u32 listed = (l1o[k + 1] - l1o[k]) + (l2o[k + 1] - l2o[k]) + (ldo[k + 1] - ldo[k]);
		if ((double) multi >= 0.5 * (double) listed) return 0;
		return unique == 0 ? 1u : unique;
	}
	ARB_HD void operator()(u32 k) const {
		support[k] = 0xFFFFFFFFu;
		const u8 fl = c.filter[k];
		if (fl == F_merge_adjacent) return;
		if (fl == F_none || fl == F_in_vitro || fl == F_intronic || fl == F_relative_support || fl == F_min_support || (fl == F_inconsistently_clipped && both_spliced(k))) {
			const u32 s = spliced_support(k);
			if (s > 0) support[k] = s;
		}
	}
};

// ---- filter_multimappers (filter_multimappers.cpp:14-168)
// alignment score of a fragment (:14-77): matches +1, insertions / deletions / introns off splice sites -1
ARB_HD bool any_gene_spliced(const frag_view& f, const annot_view& an, u32 a, i32 pos, u32 direction) {
	for (u32 k = 0; k < f.genes_cnt[a]; ++k) if (is_breakpoint_spliced(an, f.genes[f.genes_off[a] + k], direction, pos)) return true;
	return false;
}
ARB_HD int segment_score(const frag_view& f, const annot_view& an, u32 a, const u8* seq, u32 seq_len, bool revcomp) {
	const u32 contig = f.contig[a];
	if (an.contig_len[contig] == 0) return 0;
	int score = 0; i32 ref = f.start[a]; u32 rp = 0;
	const u32* c = f.cig(a);
	const u64 base = an.contig_seq_off[contig];
	for (u32 k = 0; k < f.cigar_cnt[a]; ++k) {
		const u32 op = cig_op(c[k]), len = cig_len(c[k]);
		switch (op) {
			case C_S: case C_H: rp += len; break;
			case C_D: --score; ref += (i32) len; break;
			case C_N: if (!any_gene_spliced(f, an, a, ref, DOWNSTREAM) || !any_gene_spliced(f, an, a, ref + (i32) len, UPSTREAM)) --score; ref += (i32) len; break;
			case C_I: --score; rp += len; break;
			case C_EQ: score += (int) len; ref += (i32) len; rp += len; break;
			case C_X: ref += (i32) len; rp += len; break;
			case C_M:
				for (u32 j = 0; j < len; ++j, ++ref, ++rp) {
					if (rp >= seq_len) continue;
					const u32 code = revcomp ? nt16_complement(nt16_at(seq, seq_len - 1 - rp)) : nt16_at(seq, rp);
					if ((u32) ref < an.contig_len[contig] && nt16_char(code) == an.assembly[base + (u32) ref]) ++score;
				}
				break;
			default: break;
		}
	}
	return score;
}
ARB_HD int alignment_score(const frag_view& f, const annot_view& an, u32 i) {
	const u32 a0 = f.idx(i, 0), a1 = f.idx(i, 1), a2 = f.idx(i, 2);
	int score = segment_score(f, an, a0, f.sq(a0), f.seq_len[a0], false) + segment_score(f, an, a1, f.sq(a1), f.seq_len[a1], false);
	if (f.n_aln[i] == 3) {
		score += segment_score(f, an, a2, f.sq(a1), f.seq_len[a1], f.fwd(a2) != f.fwd(a1));
		if (!any_gene_spliced(f, an, a2, f.fwd(a2) ? f.end[a2] : f.start[a2], f.fwd(a2) ? DOWNSTREAM : UPSTREAM) || !any_gene_spliced(f, an, a1, f.fwd(a1) ? f.start[a1] : f.end[a1], f.fwd(a1) ? UPSTREAM : DOWNSTREAM)) --score;
	}
	return score;
}
// total order "has more support" (filter_multimappers.cpp:79-113): is candidate x better than y?
ARB_HD bool cand_better(const cand_state& c, const annot_view& an, u32 x, u32 y) {
	const u32 sx = cand_support(c, x), sy = cand_support(c, y);
	if (sy != sx) return sy < sx;
	const bool c1x = an.gene_flags[c.gene1[x]] & GF_CODING, c1y = an.gene_flags[c.gene1[y]] & GF_CODING;
	if (c1x != c1y) return c1x;
	const bool c2x = an.gene_flags[c.gene2[x]] & GF_CODING, c2y = an.gene_flags[c.gene2[y]] & GF_CODING;
	if (c2x != c2y) return c2x;
	if (c.contig1[x] != c.contig1[y]) return c.contig1[x] < c.contig1[y];
	if (c.contig2[x] != c.contig2[y]) return c.contig2[x] < c.contig2[y];
	if (c.bp1[x] != c.bp1[y]) return c.bp1[x] < c.bp1[y];
	if (c.bp2[x] != c.bp2[y]) return c.bp2[x] < c.bp2[y];
	if (c.dir1[x] != c.dir1[y]) return c.dir1[x] < c.dir1[y];
	if (c.dir2[x] != c.dir2[y]) return c.dir2[x] < c.dir2[y];
	if (c.gene1[x] != c.gene1[y]) return c.gene1[x] < c.gene1[y];
	return c.gene2[x] < c.gene2[y];
}
// most supported candidate per multi-mapping fragment: the order is total, so the result does not depend on who comes first (compare-and-swap per fragment)
struct multimapper_best_fn {
	cand_state c; annot_view an; frag_view f; const u32* l1o; const u32* l1; const u32* l2o; const u32* l2; const u32* ldo; const u32* ld; u32* best;
	ARB_HD void consider(u32 cand, u32 frag) const {
		if (!(f.fflags[frag] & FF_MULTIMAPPER)) return;
		u32 seen = *(volatile u32*) &best[frag];
		for (;;) {
			if (!(seen == 0xFFFFFFFFu || cand_better(c, an, cand, seen))) return;
			const u32 was = atomic_cas_u32(&best[frag], seen, cand);
			if (was == seen) return;
			seen = was;
		}
	}
	ARB_HD void operator()(u32 k) const {
		for (u32 p = l1o[k]; p < l1o[k + 1]; ++p) consider(k, l1[p]);
		for (u32 p = l2o[k]; p < l2o[k + 1]; ++p) consider(k, l2[p]);
		for (u32 p = ldo[k]; p < ldo[k + 1]; ++p) consider(k, ld[p]);
	}
};
// clusters = maximal runs of fragments that share the read name (FF_SAME_NAME_AS_PREVIOUS marks the members after the first); one thread per cluster:
// the member with the best alignment score survives, ties go to the one whose best candidate has more support (:128-151)
struct multimapper_cluster_fn {
	cand_state c; annot_view an; frag_view f; const u32* best;
	ARB_HD bool more_support(u32 fa, u32 fb) const {
		const u32 x = best[fa], y = best[fb];
		if (x == 0xFFFFFFFFu) return false;
		if (y == 0xFFFFFFFFu) return true;
		return cand_better(c, an, x, y);
	}
	ARB_HD void operator()(u32 i) const {
		const u8 fl = f.fflags[i];
		if (!(fl & FF_MULTIMAPPER) || (fl & FF_SAME_NAME_AS_PREVIOUS)) return;
		u32 j = i + 1;
		while (j < f.n && (f.fflags[j] & FF_SAME_NAME_AS_PREVIOUS)) ++j;
		if (j - i <= 1) return;
		u32 best_frag = 0xFFFFFFFFu; int best_score = (int) 0x80000000;
		for (u32 x = i; x < j; ++x) {
			const int s = alignment_score(f, an, x);
			if (best_score < s) { best_frag = x; best_score = s; }
			else if (best_score == s && more_support(x, best_frag)) best_frag = x;
		}
		for (u32 x = i; x < j; ++x) if (x != best_frag && f.filter[x] == F_none) f.filter[x] = F_multimappers;
	}
};
struct multimapper_recount_fn { // :153-166
	cand_state c; frag_view f; const u32* l1o; const u32* l1; const u32* l2o; const u32* l2; const u32* ldo; const u32* ld;
	ARB_HD void operator()(u32 k) const {
		if (c.filter[k] != F_none || cand_support(c, k) == 0) return;
		u32 s1 = c.split_reads1[k], s2 = c.split_reads2[k], dm = c.discordant_mates[k];
		for (u32 p = l1o[k]; p < l1o[k + 1]; ++p) if (f.filter[l1[p]] == F_multimappers && s1 > 0) --s1;
		for (u32 p = l2o[k]; p < l2o[k + 1]; ++p) if (f.filter[l2[p]] == F_multimappers && s2 > 0) --s2;
		for (u32 p = ldo[k]; p < ldo[k + 1]; ++p) if (f.filter[ld[p]] == F_multimappers && dm > 0) --dm;
		c.split_reads1[k] = s1; c.split_reads2[k] = s2; c.discordant_mates[k] = dm;
		if (s1 + s2 + dm == 0) c.filter[k] = F_multimappers;
	}
};

// ---- iteration order of the reference's candidate map (fusions_t = std::unordered_map, common.hpp:286-314), which several event stages and the discarded
// file depend on. libstdc++ keeps all nodes in one list; a new node goes to the FRONT of its bucket's run, or -- first node of its bucket -- to the front
// of the whole list; growing re-inserts the nodes, in list order, into the new bucket array by the same rule (bits/hashtable.h: _M_insert_bucket_begin,
// _M_rehash_aux). So for an insertion sequence S into an empty table of B buckets the list reads: buckets by DESCENDING time of their first node, inside a
// bucket nodes by DESCENDING time -- a sort, not a simulation. The whole history is a chain of such sorts: at every growth the current list, followed by the
// candidates inserted until the next growth, is the sequence of the next sort. The caller supplies the growth schedule (the library's own policy object).
struct order_code_fn { // value-identical to the reference's recursive tuple hash: h(e0) ^ (H(rest) << 4), H() = 0; std::hash of an integer is the integer
	cand_state c; u64* code;
	ARB_HD void operator()(u32 k) const {
		u64 h = 0;
		h = (u64) (c.dir2[k] != 0) ^ (h << 4); h = (u64) (c.dir1[k] != 0) ^ (h << 4);
		h = (u64) (i64) c.bp2[k] ^ (h << 4); h = (u64) (i64) c.bp1[k] ^ (h << 4);
		h = (u64) c.contig2[k] ^ (h << 4); h = (u64) c.contig1[k] ^ (h << 4);
		h = (u64) c.gene2[k] ^ (h << 4); h = (u64) c.gene1[k] ^ (h << 4);
		code[k] = h;
	}
};
struct order_bucket_fn { const u32* seq; const u64* code; u64 n_buckets; u32* bucket; u32* first; ARB_HD void operator()(u32 i) const { const u32 b = (u32) (code[seq[i]] % n_buckets); bucket[i] = b; atomic_min_u32(&first[b], i); } };
struct order_key_fn { // position i' of the reversed sequence: key ascending = first node of the bucket descending
	const u32* seq; const u32* bucket; const u32* first; u32 m; u32* key; u32* val;
	ARB_HD void operator()(u32 r) const { const u32 i = m - 1 - r; key[r] = m - 1 - first[bucket[i]]; val[r] = seq[i]; }
};
struct order_append_fn { u32* seq; u32 from; ARB_HD void operator()(u32 k) const { seq[from + k] = from + k; } };
struct order_rank_fn { const u32* order; u32* rank; ARB_HD void operator()(u32 q) const { rank[order[q]] = q; } };

// ---- fusion partners per gene for the e-value model (filter_relative_support.cpp:19-60). Of the candidates that share (gene, breakpoint1, breakpoint2) --
// the same breakpoints annotated with overlapping partner genes -- only the one the reference visits FIRST contributes its partner (`overlap_duplicates`):
// first = smallest rank in the iteration order. Sort the (gene, breakpoints, rank) occurrences, keep group heads, make the (gene, partner) pairs unique.
struct partner_eligible_fn { cand_state c; u32* flag; ARB_HD void operator()(u32 k) const { flag[k] = (c.filter[k] == F_none && c.gene1[k] != c.gene2[k]) ? 1u : 0u; } };
struct partner_emit_fn { // occurrence 2e: (gene2 sees partner gene1), 2e + 1: (gene1 sees partner gene2)
	cand_state c; const u32* flag_scan; u32* occ_cand;
	ARB_HD void operator()(u32 k) const { if (flag_scan[k + 1] != flag_scan[k]) { const u32 e = flag_scan[k]; occ_cand[2 * e] = k << 1; occ_cand[2 * e + 1] = k << 1 | 1u; } }
};
ARB_HD u32 occ_gene(const cand_state& c, u32 o) { return (o & 1u) ? c.gene1[o >> 1] : c.gene2[o >> 1]; }
ARB_HD u32 occ_partner(const cand_state& c, u32 o) { return (o & 1u) ? c.gene2[o >> 1] : c.gene1[o >> 1]; }
struct partner_key_fn { // which: 0 rank, 1 breakpoint2, 2 breakpoint1, 3 gene (least significant first)
	cand_state c; const u32* rank; const u32* occ; u32* key; int which;
	ARB_HD void operator()(u32 i) const { const u32 o = occ[i], k = o >> 1; key[i] = which == 0 ? rank[k] : which == 1 ? (u32) c.bp2[k] : which == 2 ? (u32) c.bp1[k] : occ_gene(c, o); }
};
struct partner_head_fn { // first occurrence of its (gene, breakpoint1, breakpoint2) group
	cand_state c; const u32* occ; u32* head;
	ARB_HD void operator()(u32 i) const {
		if (i == 0) { head[i] = 1; return; }
		const u32 a = occ[i - 1], b = occ[i];
		head[i] = (occ_gene(c, a) != occ_gene(c, b) || c.bp1[a >> 1] != c.bp1[b >> 1] || c.bp2[a >> 1] != c.bp2[b >> 1]) ? 1u : 0u;
	}
};
struct partner_pair_fn { cand_state c; const u32* occ; const u32* head_scan; u32* gene; u32* partner; ARB_HD void operator()(u32 i) const { if (head_scan[i + 1] != head_scan[i]) { gene[head_scan[i]] = occ_gene(c, occ[i]); partner[head_scan[i]] = occ_partner(c, occ[i]); } } };
struct partner_unique_fn { const u32* gene; const u32* partner; u32* flag; u32* n_partners; ARB_HD void operator()(u32 i) const { const u32 u = (i == 0 || gene[i] != gene[i - 1] || partner[i] != partner[i - 1]) ? 1u : 0u; flag[i] = u; if (u) atomic_add_u32(&n_partners[gene[i]], 1); } };
struct partner_count_fn { const u32* gene; const u32* partner; const u32* flag; const u32* n_partners; u32* count; ARB_HD void operator()(u32 i) const { if (flag[i] && n_partners[gene[i]] >= n_partners[partner[i]]) atomic_add_u32(&count[gene[i]], 1); } };

} // namespace arb
