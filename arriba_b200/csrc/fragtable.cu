// fragtable.cu -- the resident fragment table, built on the device from the fragment pools of the record replay (records.cu; functors: fragtable_hd.h).
// The device
//   1. normalises the slots of every fragment and rejects the malformed ones (one thread per fragment, the alignment chain walked in the pool),
//   2. orders the kept fragments by name: stable LSD radix sort of (name word, fragment), 4-byte words from the last one any name has to the first,
//   3. lays out the columns: exclusive scans of CIGAR operations, sequence units and name bytes in name order, then one thread per fragment writes them,
//   4. sets the multimapper flags from the neighbours' names.
// The table is the resident one afterwards (what arb_push_chunk_begin leaves); the host gets its copy with one download per column.
#include "engine.h"
#include "fragtable_hd.h"

namespace arb {

void engine::fragment_table_build(u64 sizes[6]) {
	if (pool_workers == 0) throw arb_error("arb_fragment_table_build without arb_records_finish");
	const u32 W = pool_workers;
	std::vector<u64> base(pool_base.size()); pool_base.download(ex, base.data(), base.size());
	const u32 N = (u32) base[FT_FRAGS * (W + 1) + W];
	const ft_pools p = {pool_frags.ptr(), pool_alns.ptr(), pool_names.ptr(), pool_cigars.ptr(), pool_seqs.ptr(), pool_base.ptr(), W};
	// 1. normalisation: what every fragment keeps
	dbuf<u32> keep((size_t) N + 1), n_ops(N), n_units(N), name_len(N), max_len(1);
	max_len.zero(ex, 1);
	ft_keep_fn kf = {p, keep.ptr(), n_ops.ptr(), n_units.ptr(), name_len.ptr(), max_len.ptr()};
	for_each(ex, N, kf);
	exclusive_scan_u32(ex, keep.ptr(), keep.ptr(), N);
	u32 head[2] = {0, 0};
	keep.download(ex, head, 1, N); max_len.download(ex, head + 1, 1);
	const u32 n = head[0], longest = head[1];
	dbuf<u32> ids((size_t) n + 1), keys((size_t) n + 1), tk((size_t) n + 1), tv((size_t) n + 1);
	ft_compact_fn cf = {keep.ptr(), ids.ptr()};
	for_each(ex, N, cf);
	// 2. name order (std::string::compare): least significant word first, every pass stable
	for (u32 word = (longest + 3) / 4; word-- > 0;) {
		ft_key_fn key = {p, ids.ptr(), keys.ptr(), word};
		for_each(ex, n, key);
		radix_sort_pairs_u32(ex, keys.ptr(), ids.ptr(), tk.ptr(), tv.ptr(), n, 32);
	}
	// 3. offsets in name order
	dbuf<u32> cig_at((size_t) n + 1), seq_at((size_t) n + 1), name_at((size_t) n + 1);
	ft_gather_fn gf = {ids.ptr(), n_ops.ptr(), n_units.ptr(), name_len.ptr(), cig_at.ptr(), seq_at.ptr(), name_at.ptr()};
	for_each(ex, n, gf);
	exclusive_scan_u32(ex, cig_at.ptr(), cig_at.ptr(), n); exclusive_scan_u32(ex, seq_at.ptr(), seq_at.ptr(), n); exclusive_scan_u32(ex, name_at.ptr(), name_at.ptr(), n);
	// the scans are 32-bit: the pools bound what they can reach (a fragment's slots hold at most its own operations, the single-end copy of one anchor included,
	// and at most two sequences of the pool, each at most one unit longer than it is)
	const u64 pool_ops = base[FT_CIGARS * (W + 1) + W], pool_seq = base[FT_SEQS * (W + 1) + W], pool_names_bytes = base[FT_NAMES * (W + 1) + W];
	if (2 * pool_ops >= 0xFFFFFFFFull || 2 * (pool_seq / 16 + N) >= 0xFFFFFFFFull || pool_names_bytes >= 0xFFFFFFFFull)
		throw arb_error("chunk too large: more than 2^32 CIGAR operations or 64 GiB of sequence");
	u32 tot[3] = {0, 0, 0};
	cig_at.download(ex, tot, 1, n); seq_at.download(ex, tot + 1, 1, n); name_at.download(ex, tot + 2, 1, n);
	// 4. the columns
	frags.n = n;
	frags.n_aln.ensure(n); frags.fflags.ensure(n); frags.filter.ensure(n); frags.early.ensure(n); frags.swapped.ensure(n); frags.swapped.zero(ex, n);
	frags.contig.ensure(3 * (size_t) n); frags.start.ensure(3 * (size_t) n); frags.end.ensure(3 * (size_t) n); frags.aflags.ensure(3 * (size_t) n);
	frags.cigar_off.ensure(3 * (size_t) n); frags.cigar_cnt.ensure(3 * (size_t) n); frags.seq_off.ensure(2 * (size_t) n); frags.seq_len.ensure(2 * (size_t) n);
	frags.genes_off.ensure(3 * (size_t) n); frags.genes_cnt.ensure(3 * (size_t) n);
	frags.cigar.ensure((size_t) tot[0] + 1); frags.seq.ensure((size_t) tot[1] * 16 + 16);
	frag_names.ensure((size_t) tot[2] + 1); frag_name_off.ensure((size_t) n + 1);
	const frag_view v = frags.view();
	ft_fill_fn ff = {p, ids.ptr(), cig_at.ptr(), seq_at.ptr(), name_at.ptr(), v, frag_names.ptr(), frag_name_off.ptr()};
	for_each(ex, n, ff);
	ft_tail_fn tf = {v, tot[0], tot[1], tot[2], frag_name_off.ptr(), n};
	for_each(ex, 1, tf);
	dbuf<u32> pairs(1); pairs.zero(ex, 1);
	ft_multimap_fn mf = {frag_names.ptr(), frag_name_off.ptr(), frags.fflags.ptr(), n, pairs.ptr()};
	for_each(ex, n, mf);
	u32 same_name_pairs = 0; pairs.download(ex, &same_name_pairs, 1);
	frag_name_bytes = tot[2];
	adopt_table(ex, (u64) tot[0] + 1, (u64) tot[1] * 16 + 16);
	sizes[0] = n; sizes[1] = N - n; sizes[2] = tot[0]; sizes[3] = (u64) tot[1] * 16 + 16; sizes[4] = tot[2]; sizes[5] = same_name_pairs;
}

void engine::fragment_table_download(const arb_soa_chunk& c, char* names, u64* name_off) {
	const u32 n = frags.n;
	if (c.n_fragments != n) throw arb_error("arb_fragment_table_download: the columns are sized for another table");
	frags.n_aln.download(ex, (u8*) c.n_aln, n); frags.fflags.download(ex, (u8*) c.fflags, n); frags.filter.download(ex, (u8*) c.filter, n);
	frags.contig.download(ex, (u16*) c.contig, 3 * (size_t) n); frags.start.download(ex, (i32*) c.start, 3 * (size_t) n); frags.end.download(ex, (i32*) c.end, 3 * (size_t) n);
	frags.aflags.download(ex, (u8*) c.aflags, 3 * (size_t) n); frags.cigar_off.download(ex, (u32*) c.cigar_off, 3 * (size_t) n); frags.cigar_cnt.download(ex, (u16*) c.cigar_cnt, 3 * (size_t) n);
	frags.seq_off.download(ex, (u32*) c.seq_off, 2 * (size_t) n); frags.seq_len.download(ex, (u16*) c.seq_len, 2 * (size_t) n);
	frags.genes_off.download(ex, (u32*) c.genes_off, 3 * (size_t) n); frags.genes_cnt.download(ex, (u16*) c.genes_cnt, 3 * (size_t) n);
	frags.cigar.download(ex, (u32*) c.cigar, c.n_cigar); frags.seq.download(ex, (u8*) c.seq, c.n_seq_bytes);
	frag_names.download(ex, names, frag_name_bytes); frag_name_off.download(ex, name_off, (size_t) n + 1);
}

} // namespace arb
