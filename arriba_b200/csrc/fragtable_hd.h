// fragtable_hd.h -- the fragment table from the fragment pools the record replay writes (records.cu; fragtable.cu drives it; the CPU stand-in runs the same functors).
//   ft_normalise : brings a fragment's alignments into the canonical slots or rejects it (read_chimeric_alignments.cpp:340-373 disjoin_split_read_segments,
//                  :377-506 remove_malformed_alignments), without writing anything: the rewritten CIGAR operations are kept as overrides of the pool's,
//   ft_keep_fn   : one thread per fragment of the pools: kept or not, its CIGAR operations, sequence units and name length,
//   ft_key_fn    : the name key of one round of the name sort, ft_fill_fn : every column of one fragment in name order, ft_multimap_fn : the neighbour flags.
#pragma once
#include "model.h"
#include "../../include/arriba_b200.h"

namespace arb {

// the pools of all workers back to back; base[k * (n_workers + 1) + w] = first item of worker w in pool k (FT_FRAGS ... FT_SEQS)
enum { FT_FRAGS = 0, FT_ALNS = 1, FT_NAMES = 2, FT_CIGARS = 3, FT_SEQS = 4, FT_POOLS = 5 };
struct ft_pools {
	const arb_pool_fragment* frags; const arb_pool_alignment* alns; const char* names; const u32* cigars; const u8* seqs;
	const u64* base; u32 n_workers;
	ARB_HD u64 at(u32 pool, u32 w) const { return base[pool * (n_workers + 1) + w]; }
	ARB_HD u32 worker_of(u32 g) const { // the last worker whose first fragment is <= g (workers without fragments share their first index with the next)
		u32 lo = 0, hi = n_workers;
		while (hi - lo > 1) { const u32 mid = (lo + hi) / 2; if (at(FT_FRAGS, mid) <= g) lo = mid; else hi = mid; }
		return lo;
	}
	ARB_HD const char* name(u32 g, u32& len) const { const u32 w = worker_of(g); const arb_pool_fragment& f = frags[g]; len = f.name_len; return names + at(FT_NAMES, w) + f.name_off; }
};

// one alignment during normalisation: its fields, and its CIGAR as the source's operations with at most four of them rewritten
// (normalisation only touches the first two and the last two operations). OPS: where the operations come from -- the pool (const u32*), or a record of
// the record store (records_hd.h), whose CIGAR need not be 4-byte aligned.
template <class OPS> struct ft_slot_t {
	u16 contig; u8 supplementary, first_in_pair, forward; i32 start, end; u32 seq_len, cnt; u64 seq_off; OPS ops;
	u32 n_set, set_at[4], set_to[4];
	// fixed trip counts: the arrays stay in registers
	ARB_HD u32 op(u32 k) const {
#pragma unroll
		for (u32 j = 0; j < 4; ++j) if (j < n_set && set_at[j] == k) return set_to[j];
		return ops[k];
	}
	ARB_HD void set(u32 k, u32 v) {
#pragma unroll
		for (u32 j = 0; j < 4; ++j) if (j < n_set && set_at[j] == k) { set_to[j] = v; return; }
#pragma unroll
		for (u32 j = 0; j < 4; ++j) if (j == n_set) { set_at[j] = k; set_to[j] = v; }
		++n_set;
	}
	ARB_HD u32 front() const { return op(0); }
	ARB_HD u32 back() const { return op(cnt - 1); }
	ARB_HD u32 clip(bool at_front) const { const u32 c = at_front ? front() : back(), o = c & 15; return (o == C_S || o == C_H) ? c >> 4 : 0; }
};
typedef ft_slot_t<const u32*> ft_slot;
template <class S> ARB_HD void ft_swap(S& a, S& b) { const S t = a; a = b; b = t; }

template <class S> ARB_HD bool ft_disjoin(S& split, S& supp) {
	const u32 clipped_split = split.forward ? split.clip(true) : split.clip(false);
	const u32 clipped_supp = supp.forward ? supp.clip(false) : supp.clip(true);
	const int overlap = (int) split.seq_len - (int) clipped_split - (int) clipped_supp;
	if (overlap <= 0) return true;
	const u32 clipped_op = supp.forward ? supp.cnt - 1 : 0;
	const u32 matching_op = supp.forward ? clipped_op - 1 : 1;
	if (supp.cnt < 2 || (supp.op(matching_op) & 15) != C_M || (int) (supp.op(matching_op) >> 4) < overlap + 10) return false;
	const u32 c = supp.op(clipped_op), m = supp.op(matching_op);
	supp.set(clipped_op, ((c >> 4) + overlap) << 4 | (c & 15));
	supp.set(matching_op, ((m >> 4) - overlap) << 4 | (m & 15));
	if (supp.forward) supp.end -= overlap; else supp.start += overlap;
	return true;
}

// the fragment sizes remove_malformed_alignments accepts at all
ARB_HD bool ft_count_ok(bool single_end, u32 count) { return single_end ? count == 2 : (count == 2 || count == 3); }

// The rule itself, on the fragment's alignments m[0, count) in the order the loop added them: brings them into the slots MATE1, MATE2 / SPLIT_READ,
// SUPPLEMENTARY and returns how many it keeps, 0 = rejected. The fragment table applies it to the pools (ft_normalise); the record replay applies it to the
// alignments that a separate chimeric file gave a read (records_hd.h), to learn whether the first pass over the map keeps them.
template <class S> ARB_HD u32 ft_decide(bool single_end, u32 count, S (&m)[3]) {
	if (!ft_count_ok(single_end, count)) return 0;
	if (single_end) {
		if (m[0].supplementary == m[1].supplementary) return 0;
		// the longer anchor becomes the split read; it is duplicated into the MATE1 slot to imitate paired-end data
		if (m[0].end - m[0].start > m[1].end - m[1].start) { m[2] = m[1]; m[1] = m[0]; }
		else { m[2] = m[0]; m[0] = m[1]; }
		// sequence: MATE1 and SPLIT_READ carry it, SUPPLEMENTARY does not
		if (!m[0].supplementary) { m[1].seq_off = m[0].seq_off; m[1].seq_len = m[0].seq_len; }
		else if (!m[1].supplementary) { m[0].seq_off = m[1].seq_off; m[0].seq_len = m[1].seq_len; }
		else { m[0].seq_off = m[1].seq_off = m[2].seq_off; m[0].seq_len = m[1].seq_len = m[2].seq_len; }
		m[2].seq_len = 0;
		for (int s = 0; s < 2; ++s) {
			if ((m[s].front() & 15) == C_H) m[s].set(0, (m[s].front() >> 4) << 4 | C_S);
			if ((m[s].back() & 15) == C_H) {
				// the reference takes the length for SPLIT_READ's last op from MATE1's CIGAR at the same index (read_chimeric_alignments.cpp:415)
				const u32 len = s == 0 ? m[0].back() >> 4 : (m[1].cnt - 1 < m[0].cnt ? m[0].op(m[1].cnt - 1) >> 4 : 0);
				m[s].set(m[s].cnt - 1, len << 4 | C_S);
			}
		}
		m[2].supplementary = 1; m[0].supplementary = 0; m[1].supplementary = 0;
		const bool same = m[1].forward == m[2].forward;
		const u32 len = m[1].seq_len;
		const u32 lhs = len - m[1].clip(true) - (same ? m[2].clip(false) : m[2].clip(true));
		const u32 rhs = len - m[1].clip(false) - (same ? m[2].clip(true) : m[2].clip(false));
		const bool flip = lhs < rhs ? (m[1].forward != 0) : (m[1].forward == 0);
		if (flip) m[0].forward = !m[0].forward; else { m[1].forward = !m[1].forward; m[2].forward = !m[2].forward; }
		m[0].first_in_pair = !flip; m[1].first_in_pair = flip; m[2].first_in_pair = flip;
		if (!ft_disjoin(m[1], m[2])) return 0;
	} else if (count == 3) {
		if (m[0].supplementary) ft_swap(m[0], m[2]); else if (m[1].supplementary) ft_swap(m[1], m[2]);
		if (m[1].first_in_pair != m[2].first_in_pair) ft_swap(m[0], m[1]);
		if (m[0].supplementary || m[1].supplementary || !m[2].supplementary) return 0;
		if (m[0].contig != m[1].contig || m[0].forward == m[1].forward) return 0;
		if (!ft_disjoin(m[1], m[2])) return 0;
	} else {
		if (m[0].supplementary || m[1].supplementary) return 0;
	}
	for (int s = 0; s < 2; ++s) if ((m[s].front() & 15) == C_H || (m[s].back() & 15) == C_H) return 0; // anchors need their full sequence
	return single_end ? 3 : count;
}

// the slots of fragment g of the pools (0 = rejected), in the order MATE1, MATE2 / SPLIT_READ, SUPPLEMENTARY
ARB_HD u32 ft_normalise(const ft_pools& p, u32 g, ft_slot (&m)[3]) {
	const arb_pool_fragment& f = p.frags[g];
	const bool single_end = f.single_end != 0;
	if (!ft_count_ok(single_end, f.count)) return 0;
	const u32 w = p.worker_of(g);
	const u64 aln0 = p.at(FT_ALNS, w), cig0 = p.at(FT_CIGARS, w), seq0 = p.at(FT_SEQS, w);
	i32 a = f.head;
#pragma unroll
	for (u32 s = 0; s < 3; ++s) {
		if (s >= f.count) break;
		const arb_pool_alignment& x = p.alns[aln0 + (u32) a];
		m[s].contig = x.contig; m[s].supplementary = x.supplementary; m[s].first_in_pair = x.first_in_pair; m[s].forward = x.forward;
		m[s].start = x.start; m[s].end = x.end; m[s].seq_len = x.seq_len; m[s].seq_off = seq0 + x.seq_off; m[s].cnt = x.cigar_cnt; m[s].ops = p.cigars + cig0 + x.cigar_off;
		m[s].n_set = 0;
		a = x.next;
	}
	return ft_decide(single_end, f.count, m);
}

ARB_HD u32 ft_seq_units(u32 seq_len) { return ((seq_len + 1) / 2 + 15) / 16; }

// per fragment of the pools: keep[g] (0/1), its CIGAR operations, sequence units and name length (0 for a rejected one); the longest kept name.
// Fragments of a separate chimeric file (Chimeric.out.sam) went through remove_malformed_alignments twice in the reference: once after their own file
// (the replay's counting pass counts that pass's verdicts) and once more with the main file's. The second pass keeps what the first kept, except single-end
// fragments: the first pass made three alignments of their two and left them single-end, which the second pass rejects.
struct ft_keep_fn {
	ft_pools p; u32 *keep, *n_ops, *n_units, *name_len, *max_name_len;
	ARB_HD void operator()(u32 g) const {
		ft_slot m[3];
		u32 n = ft_normalise(p, g, m);
		const arb_pool_fragment& f = p.frags[g];
		if (f.chimeric_file && f.single_end) n = 0;
		u32 ops = 0, units = 0;
#pragma unroll
		for (u32 s = 0; s < 3; ++s) if (s < n) { ops += m[s].cnt; if (s < 2) units += ft_seq_units(m[s].seq_len); }
		const u32 len = n ? p.frags[g].name_len : 0;
		keep[g] = n ? 1 : 0; n_ops[g] = ops; n_units[g] = units; name_len[g] = len;
#ifdef __CUDA_ARCH__
		if (len) atomicMax(max_name_len, len);
#else
		if (len > *max_name_len) *max_name_len = len;
#endif
	}
};
struct ft_compact_fn { const u32* at; u32* ids; ARB_HD void operator()(u32 g) const { if (at[g + 1] != at[g]) ids[at[g]] = g; } };

// word `word` of a name, big-endian, zero bytes past its end: names hold no zero byte, so zero padding orders a name before every longer name it begins
struct ft_key_fn {
	ft_pools p; const u32* ids; u32* keys; u32 word;
	ARB_HD void operator()(u32 i) const {
		u32 len; const char* s = p.name(ids[i], len);
		u32 k = 0;
		for (u32 b = 0; b < 4; ++b) { const u32 at = 4 * word + b; k = k << 8 | (at < len ? (u32) (u8) s[at] : 0u); }
		keys[i] = k;
	}
};
struct ft_gather_fn { const u32* ids; const u32 *a, *b, *c; u32 *a_out, *b_out, *c_out; ARB_HD void operator()(u32 i) const { const u32 g = ids[i]; a_out[i] = a[g]; b_out[i] = b[g]; c_out[i] = c[g]; } };

struct ft_fill_fn { // fragment i of the name order: every column of arb_soa_chunk but the gene sets (zero), and its name
	ft_pools p; const u32* ids; const u32 *cig_at, *seq_at, *name_at; frag_view f; char* names; u64* name_off;
	ARB_HD void operator()(u32 i) const {
		const u32 g = ids[i];
		ft_slot m[3];
		const u32 n = ft_normalise(p, g, m);
		const arb_pool_fragment& fb = p.frags[g];
		f.n_aln[i] = (u8) n; f.fflags[i] = (fb.single_end ? FF_SINGLE_END : 0) | (fb.duplicate ? FF_DUPLICATE : 0); f.filter[i] = 0;
		u32 len; const char* s = p.name(g, len);
		for (u32 k = 0; k < len; ++k) names[name_at[i] + k] = s[k];
		name_off[i] = name_at[i];
		u32 c = cig_at[i], sq = seq_at[i];
#pragma unroll
		for (u32 slot = 0; slot < 3; ++slot) {
			const u32 x = f.idx(i, slot);
			f.genes_off[x] = 0; f.genes_cnt[x] = 0;
			if (slot >= n) { // unused slot
				f.contig[x] = 0; f.start[x] = 0; f.end[x] = 0; f.aflags[x] = 0; f.cigar_off[x] = 0; f.cigar_cnt[x] = 0;
				if (slot < 2) { f.seq_off[x] = 0; f.seq_len[x] = 0; }
				continue;
			}
			const ft_slot& a = m[slot];
			f.contig[x] = a.contig; f.start[x] = a.start; f.end[x] = a.end;
			f.aflags[x] = (a.supplementary ? AF_SUPPLEMENTARY : 0) | (a.first_in_pair ? AF_FIRST_IN_PAIR : 0) | (a.forward ? AF_FORWARD : 0) | AF_PRED_AMBIGUOUS;
			f.cigar_off[x] = c; f.cigar_cnt[x] = (u16) a.cnt;
			for (u32 k = 0; k < a.cnt; ++k) f.cigar[c + k] = a.op(k);
			c += a.cnt;
			if (slot < 2) {
				f.seq_off[x] = sq; f.seq_len[x] = (u16) a.seq_len;
				// whole 16-byte units, the bytes past the sequence zero (the pool's sequences are 16-byte aligned; what follows one is not read into the table)
				const u32 bytes = (a.seq_len + 1) / 2, units = ft_seq_units(a.seq_len);
				const u32* src = (const u32*) (p.seqs + a.seq_off); u32* dst = (u32*) (f.seq + (u64) sq * 16);
				for (u32 k = 0; k < units * 4; ++k) {
					const u32 have = bytes > 4 * k ? bytes - 4 * k : 0;
					dst[k] = have >= 4 ? src[k] : have == 0 ? 0u : src[k] & ((1u << (8 * have)) - 1u);
				}
				sq += units;
			}
		}
	}
};
struct ft_tail_fn { // behind the last fragment: the CIGAR terminator, 16 zero bytes behind the sequences, the end of the last name
	frag_view f; u32 n_ops, n_units, n_name_bytes; u64* name_off; u32 n;
	ARB_HD void operator()(u32) const { f.cigar[n_ops] = 0; for (u32 k = 0; k < 16; ++k) f.seq[(u64) n_units * 16 + k] = 0; name_off[n] = n_name_bytes; }
};

// multimappers: neighbours in name order that share the name up to the last comma (read_chimeric_alignments.cpp:792-802)
struct ft_multimap_fn {
	const char* names; const u64* name_off; u8* fflags; u32 n; u32* pairs; // pairs: neighbours with the same stem (mark_multimappers' count)
	ARB_HD u64 stem(u32 i) const { const char* s = names + name_off[i]; const u64 l = name_off[i + 1] - name_off[i]; u64 k = l; while (k > 0 && s[k - 1] != ',') --k; return k > 0 ? k - 1 : l; }
	ARB_HD bool same(u32 i) const { // fragments i and i + 1
		const u64 la = stem(i), lb = stem(i + 1);
		if (la != lb) return false;
		for (u64 k = 0; k < la; ++k) if (names[name_off[i] + k] != names[name_off[i + 1] + k]) return false;
		return true;
	}
	ARB_HD void operator()(u32 i) const {
		const bool before = i > 0 && same(i - 1), after = i + 1 < n && same(i);
		if (before || after) fflags[i] |= FF_MULTIMAPPER;
		if (before) fflags[i] |= FF_SAME_NAME_AS_PREVIOUS;
#ifdef __CUDA_ARCH__
		const unsigned active = __activemask(), votes = __ballot_sync(active, after);
		if (votes && (threadIdx.x & 31u) == (unsigned) __ffs((int) active) - 1u) atomicAdd(pairs, (u32) __popc(votes));
#else
		if (after) ++*pairs;
#endif
	}
};

} // namespace arb
