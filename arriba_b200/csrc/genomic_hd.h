// genomic_hd.h -- genomic breakpoints from whole-genome sequencing (-d) matched to the candidates: mark_genomic_support (filter_genomic_support.cpp:169-212).
//
// The reference keeps the breakpoints in map[(contig1, contig2, direction1, direction2)][position1] -> position2 list (file order) and walks it per candidate:
//   * UPSTREAM direction1: from the last position1 below breakpoint1 + 5 DOWNWARDS while is_genomic_breakpoint_close_enough (:62-78) holds, i.e. over the
//     position1 keys in [most distal position, breakpoint1 + 5) in descending order;
//   * DOWNSTREAM direction1: the key at lower_bound(breakpoint1 - 5) and then one step DOWN, which is always below breakpoint1 - 5 and so never close enough:
//     at most ONE position1 key is visited (a quirk of the reference, reproduced);
//   * within a key the position2 values in file order; an entry that passes the closeness test on side 2 and the deletion / duplication / ITD / inversion
//     checks (:190-194) replaces the current choice if that is unset (a coordinate < 0) or has a strictly larger distance sum (:197-201).
// Here the records are sorted by (key, position1, file order), a small key table gives every key its range, and a candidate's visits are a CONTIGUOUS range
// of records. Without negative coordinates the sequential rule picks the first entry of smallest distance sum in visiting order, i.e. the smallest
// (distance sum, -position1, record index): lanes can split a long range and combine their picks in any order. An entry with a negative coordinate makes the
// next one win unconditionally, which no such combination reproduces: a range that holds one is walked by one lane.
#pragma once
#include "model.h"
#include "read_filters.h" // lane_group
#include "events_hd.h"  // cand_state

namespace arb {

struct genomic_index { // sorted records and the key table (engine: set_genomic_breakpoints)
	u32 n_keys;
	const u64* key;        // (contig1 << 32 | contig2 << 16 | direction1 << 8 | direction2), ascending
	const u32* key_begin;  // n_keys + 1: records of key q are [key_begin[q], key_begin[q + 1])
	const i32* pos1; const i32* pos2; // per record, sorted by (key, pos1, file order)
};

ARB_HD u64 genomic_key(u32 contig1, u32 contig2, u32 dir1, u32 dir2) { return (u64) contig1 << 32 | (u64) contig2 << 16 | (u64) dir1 << 8 | (u64) dir2; }

// int arithmetic of the reference, wrapping like the machine does
ARB_HD i32 wrap_add(i32 a, i32 b) { return (i32) ((u32) a + (u32) b); }
ARB_HD i32 wrap_sub(i32 a, i32 b) { return (i32) ((u32) a - (u32) b); }
ARB_HD i32 wrap_abs(i32 a) { return a < 0 ? (i32) (0u - (u32) a) : a; }

ARB_HD u32 lower_bound_i32(const i32* v, u32 lo, u32 hi, i32 x) { while (lo < hi) { const u32 m = lo + (hi - lo) / 2; if (v[m] < x) lo = m + 1; else hi = m; } return lo; }
ARB_HD u32 upper_bound_i32(const i32* v, u32 lo, u32 hi, i32 x) { while (lo < hi) { const u32 m = lo + (hi - lo) / 2; if (v[m] <= x) lo = m + 1; else hi = m; } return lo; }

struct genomic_search {
	genomic_index ix; cand_state c; annot_view an;
	i32 max_distance, max_itd_length;
	i32* closest1; i32* closest2;
	u32 short_range;                 // ranges up to this length are walked by the candidate's own thread
	u32* heavy; u32* n_heavy;        // the others are queued for a group of lanes
	u32* range_lo; u32* range_hi;    // per candidate

	// most distal genomic position that still counts (is_genomic_breakpoint_close_enough)
	ARB_HD i32 most_distal(u32 dir, i32 bp, u32 gene) const {
		const bool dummy = an.gene_flags[gene] & GF_DUMMY;
		if (dir == UPSTREAM) return wrap_sub(dummy ? bp : an.gene_start[gene], max_distance);
		return wrap_add(dummy ? bp : an.gene_end[gene], max_distance);
	}
	ARB_HD bool close_enough(u32 dir, i32 genomic, i32 bp, u32 gene) const {
		const i32 distal = most_distal(dir, bp, gene);
		if (dir == UPSTREAM) return genomic >= distal && genomic <= wrap_add(bp, 5);
		return genomic <= distal && genomic >= wrap_sub(bp, 5);
	}
	// side 2 and the extra checks of deletions, duplications / ITDs and inversions (filter_genomic_support.cpp:189-194)
	ARB_HD bool passes(u32 k, i32 p1, i32 p2) const {
		const u32 d1 = c.dir1[k], d2 = c.dir2[k]; const i32 b1 = c.bp1[k], b2 = c.bp2[k];
		if (!close_enough(d2, p2, b2, c.gene2[k])) return false;
		if (c.contig1[k] != c.contig2[k]) return true;
		if (d1 == UPSTREAM && d2 == DOWNSTREAM) {
			const bool itd = c.gene1[k] == c.gene2[k] && (u32) b2 - (u32) b1 < (u32) max_itd_length; // is_internal_tandem_duplication (common.hpp:270-274)
			return !itd || (wrap_sub(b1, p1) < max_itd_length && wrap_sub(p2, b2) < max_itd_length);
		}
		if (d1 == DOWNSTREAM && d2 == UPSTREAM) return p1 < b2 && p2 > b1;
		if (d1 == UPSTREAM && d2 == UPSTREAM) return p2 > b1;
		return p1 < b2;
	}
	ARB_HD i32 distance(u32 k, i32 p1, i32 p2) const { return wrap_add(wrap_abs(wrap_sub(p1, c.bp1[k])), wrap_abs(wrap_sub(c.bp2[k], p2))); }

	// the reference's update rule, entry by entry in visiting order
	ARB_HD void visit(u32 k, u32 r, i32& g1, i32& g2) const {
		const i32 p1 = ix.pos1[r], p2 = ix.pos2[r];
		if (!passes(k, p1, p2)) return;
		if (g1 < 0 || g2 < 0 || distance(k, g1, g2) > distance(k, p1, p2)) { g1 = p1; g2 = p2; }
	}
	// records [lo, hi) in visiting order: position1 runs from the highest down, file order inside a run
	ARB_HD void walk(u32 k, u32 lo, u32 hi, i32& g1, i32& g2) const {
		u32 end = hi;
		while (end > lo) {
			u32 begin = end - 1;
			while (begin > lo && ix.pos1[begin - 1] == ix.pos1[end - 1]) --begin;
			for (u32 r = begin; r < end; ++r) visit(k, r, g1, g2);
			end = begin;
		}
	}

	// the range of records candidate k visits; lo == hi: none
	ARB_HD void range(u32 k, u32& lo, u32& hi) const {
		lo = hi = 0;
		const u64 key = genomic_key(c.contig1[k], c.contig2[k], c.dir1[k], c.dir2[k]);
		u32 a = 0, b = ix.n_keys;
		while (a < b) { const u32 m = a + (b - a) / 2; if (ix.key[m] < key) a = m + 1; else b = m; }
		if (a == ix.n_keys || ix.key[a] != key) return;
		const u32 first = ix.key_begin[a], last = ix.key_begin[a + 1];
		const i32 b1 = c.bp1[k]; const u32 g1 = c.gene1[k];
		if (c.dir1[k] == UPSTREAM) {
			hi = lower_bound_i32(ix.pos1, first, last, wrap_add(b1, 5));
			lo = lower_bound_i32(ix.pos1, first, hi, most_distal(UPSTREAM, b1, g1));
		} else {
			lo = lower_bound_i32(ix.pos1, first, last, wrap_sub(b1, 5));
			if (lo == last || !close_enough(DOWNSTREAM, ix.pos1[lo], b1, g1)) { lo = hi = 0; return; }
			hi = upper_bound_i32(ix.pos1, lo, last, ix.pos1[lo]);
		}
	}

	// one thread per candidate; long ranges go to the queue
	ARB_HD void operator()(u32 k) const {
		u32 lo, hi; range(k, lo, hi);
		i32 g1 = -1, g2 = -1;
		if (hi - lo > short_range) {
			range_lo[k] = lo; range_hi[k] = hi;
#ifdef __CUDA_ARCH__
			heavy[atomicAdd(n_heavy, 1u)] = k;
#else
			heavy[(*n_heavy)++] = k;
#endif
			return;
		}
		walk(k, lo, hi, g1, g2);
		closest1[k] = g1; closest2[k] = g2;
	}
};

// what one lane found in its share of a long range
struct genomic_pick {
	i32 dist, pos1; u32 rec; u32 flags; // flags: 1 found, 2 an entry with a negative coordinate passed
	ARB_HD bool better_than(const genomic_pick& o) const { // first entry of smallest distance in visiting order: (distance, -position1, record)
		if (!(flags & 1)) return false;
		if (!(o.flags & 1)) return true;
		if (dist != o.dist) return dist < o.dist;
		if (pos1 != o.pos1) return pos1 > o.pos1;
		return rec < o.rec;
	}
	ARB_HD void merge(const genomic_pick& o) { const u32 neg = (flags | o.flags) & 2u; if (o.better_than(*this)) *this = o; flags |= neg; }
};

// lane `lane` of `lanes` looks at records lo + lane, lo + lane + lanes, ...
ARB_HD genomic_pick genomic_lane_pick(const genomic_search& s, u32 k, u32 lo, u32 hi, u32 lane, u32 lanes) {
	genomic_pick best; best.dist = 0; best.pos1 = 0; best.rec = 0; best.flags = 0;
	for (u32 r = lo + lane; r < hi; r += lanes) {
		const i32 p1 = s.ix.pos1[r], p2 = s.ix.pos2[r];
		if (!s.passes(k, p1, p2)) continue;
		genomic_pick x; x.dist = s.distance(k, p1, p2); x.pos1 = p1; x.rec = r; x.flags = 1u | (p1 < 0 || p2 < 0 ? 2u : 0u);
		best.merge(x);
	}
	return best;
}

// the combined pick of all lanes decides; a range where an entry with a negative coordinate passed is walked with the reference's rule
ARB_HD void genomic_finish(const genomic_search& s, u32 k, const genomic_pick& p) {
	i32 g1 = -1, g2 = -1;
	if (p.flags & 2u) s.walk(k, s.range_lo[k], s.range_hi[k], g1, g2);
	else if (p.flags & 1u) { g1 = s.ix.pos1[p.rec]; g2 = s.ix.pos2[p.rec]; }
	s.closest1[k] = g1; s.closest2[k] = g2;
}

#ifdef ARB_DEVICE_BUILD
// a group of lanes per queued candidate: every lane picks from its share, the picks are combined by shuffles
__device__ inline void genomic_group(const lane_group& g, const genomic_search& s, u32 k) {
	genomic_pick p = genomic_lane_pick(s, k, s.range_lo[k], s.range_hi[k], g.lane, g.lanes);
	for (u32 d = g.lanes >> 1; d; d >>= 1) {
		genomic_pick o;
		o.dist = __shfl_xor_sync(g.mask, p.dist, d); o.pos1 = __shfl_xor_sync(g.mask, p.pos1, d); o.rec = __shfl_xor_sync(g.mask, p.rec, d); o.flags = __shfl_xor_sync(g.mask, p.flags, d);
		p.merge(o);
	}
	if (g.lane == 0) genomic_finish(s, k, p);
}
#endif

} // namespace arb
