// fusions.cu -- driver of candidate generation (see fusions_hd.h for the stage design and reference citations).
#include <cstdlib>
#include "engine.h"
#include "fusions_hd.h"

namespace arb {

static u32 bits_for(u32 n) { u32 b = 1; while (b < 32 && ((u64) 1 << b) < n) ++b; return b; }

#ifdef ARB_DEVICE_BUILD
// Pass B on the device: one WARP per unfiltered candidate that has a bucket. The bucket's discordant mates lie in name order in bucket-ordered columns
// (breakpoints, fragment, label), so a warp reads them coalesced, 32 at a time; the two geometric tests (fusions.cpp:383-398) are independent per mate and
// are taken with a ballot. The order-dependent part -- the subsampling counters `listed` / `counted` (fusions.cpp:400-406) -- only matters once a counter
// can reach the threshold inside the chunk: until then every mate that passes is listed (rank = prefix popcount of the ballot); chunks where the threshold
// is in reach are replayed serially from the ballot (same statements as walk_b_fn, which stays the host-build path and the statement of the rule).
struct bucket_columns { const i32* bp1; const i32* bp2; const u32* frag; const u8* label; };
struct gather_bucket_fn { record_view r; const u32* drec; const u32* bperm; i32* bp1; i32* bp2; u32* frag; u8* label;
	ARB_HD void operator()(u32 p) const { const u32 k = drec[bperm[p]]; bp1[p] = r.bp1[k]; bp2[p] = r.bp2[k]; frag[p] = r.frag[k]; label[p] = (u8) (r.meta[k] >> 8); } };
struct probe_bucket_fn { // bucket of every candidate pass B looks at (0xFFFFFFFF: none), and the flag of the compaction
	record_view r; cand_out c; hash_index_view bucket_table; const u32* drec; const u32* bucket_head_scan; u32* bucket; u32* active;
	ARB_HD void operator()(u32 cand) const {
		u32 b = 0xFFFFFFFFu;
		if (c.filter[cand] == F_none) {
			const u32 d1 = c.dir1[cand], d2 = c.dir2[cand];
			bucket_probe probe = {r, drec, c.gene1[cand], c.gene2[cand], (d1 ? 1u : 0u) | (d2 ? 2u : 0u)};
			const u32 slot = bucket_table.find(probe);
			if (slot != hash_index_view::EMPTY) b = bucket_head_scan[bucket_table.mn[slot]];
		}
		bucket[cand] = b; active[cand] = b != 0xFFFFFFFFu; c.n_listd[cand] = 0;
	}
};
// lists of the one-pass variant: from the candidates' stretches of the scratch buffer to their places in the CSR list, one warp per candidate
__global__ void __launch_bounds__(256) k_walk_b_pack(const u32* active_cands, u32 n_active, const u32* scratch, const u32* stretch_off, const u32* listd_off, u32* listd) {
	const u32 warp = (blockIdx.x * 256u + threadIdx.x) >> 5, lane = threadIdx.x & 31u;
	if (warp >= n_active) return;
	const u32 cand = active_cands[warp], lo = listd_off[cand], n = listd_off[cand + 1] - lo;
	for (u32 x = lane; x < n; x += 32) listd[lo + x] = scratch[stretch_off[warp] + x];
}
struct stretch_size_fn { const u32* active_cands; const u32* bucket_of_cand; const u32* bseg_off; u64 cap; u32* size;
	ARB_HD void operator()(u32 w) const { const u32 b = bucket_of_cand[active_cands[w]]; const u64 n = bseg_off[b + 1] - bseg_off[b]; size[w] = (u32) (n < cap ? n : cap); } };
static bool sf_fits(u32 n_active, const dbuf<u32>&, u32 threshold) { return (u64) n_active * 2 * (u64) threshold < (1ull << 32); } // the scan adds in 32 bits: only when even the largest possible total fits
static const u32 WALK_B_THREADS = 256;
__global__ void __launch_bounds__(WALK_B_THREADS) k_walk_b(const u32* active_cands, u32 n_active, const u32* bucket_of_cand, bucket_columns bc, const u32* bseg_off,
                                                            frag_view f, annot_view an, cand_out c, const u32* listd_off, u32* listd, u32* need_swap, i32 max_mate_gap, u32 threshold, u32 fill) {
	// fill: 0 = count, 1 = fill the CSR list (listd_off per candidate), 2 = count and fill in ONE walk: listd_off then holds the start of each WARP's stretch of a scratch buffer
	const u32 warp = (blockIdx.x * WALK_B_THREADS + threadIdx.x) >> 5, lane = threadIdx.x & 31u;
	if (warp >= n_active) return;
	const u32 FULL = 0xFFFFFFFFu;
	const u32 cand = active_cands[warp], b = bucket_of_cand[cand];
	const u32 g1 = c.gene1[cand], g2 = c.gene2[cand], d1 = c.dir1[cand], d2 = c.dir2[cand];
	const i32 bp1 = c.bp1[cand], bp2 = c.bp2[cand];
	const i32 overlap = (c.n_list1[cand] + c.n_list2[cand] > 0) ? 2 : max_mate_gap;
	const i32 lim1 = d1 == DOWNSTREAM ? bp1 + overlap : bp1 - overlap, lim2 = d2 == DOWNSTREAM ? bp2 + overlap : bp2 - overlap;
	const i32 g1s = an.gene_start[g1], g1e = an.gene_end[g1], g2s = an.gene_start[g2], g2e = an.gene_end[g2];
	const bool intragenic = g1 == g2 || (bp1 >= g2s - 10000 && bp1 <= g2e + 10000 && bp2 >= g1s - 10000 && bp2 <= g1e + 10000);
	u32 listed = 0, counted = 0;
	i32 an1 = c.anchor1[cand], an2 = c.anchor2[cand];
	u32 w = fill == 2 ? listd_off[warp] : fill ? listd_off[cand] : 0;
	const u32 seg_end = bseg_off[b + 1];
	bool done = false;
	for (u32 base = bseg_off[b]; base < seg_end && !done; base += 32) {
		const u32 p = base + lane;
		bool pass = false; u32 frag = 0; u8 fl = 0;
		if (p < seg_end) {
			const i32 m1 = bc.bp1[p], m2 = bc.bp2[p];
			pass = ((d1 == DOWNSTREAM && m1 <= lim1) || (d1 == UPSTREAM && m1 >= lim1)) && ((d2 == DOWNSTREAM && m2 <= lim2) || (d2 == UPSTREAM && m2 >= lim2)) &&
			       ((!intragenic && !(m1 >= g2s && m1 <= g2e) && !(m2 >= g1s && m2 <= g1e)) || (hd_abs(bp1 - m1) <= max_mate_gap && hd_abs(bp2 - m2) <= max_mate_gap));
			if (pass) { frag = bc.frag[p]; fl = bc.label[p]; }
		}
		u32 mask = __ballot_sync(FULL, pass);
		if (mask == 0) continue;
		const u32 none_mask = __ballot_sync(FULL, pass && fl == F_none);
		if (listed >= threshold) { // labelled mates are no longer listed (fusions.cpp:400): only the unlabelled ones count from here on
			mask = none_mask; pass = pass && fl == F_none;
			if (mask == 0) continue;
		}
		// the values the anchors and the canonical mate order need, per listed mate
		i32 v1 = 0, v2 = 0; bool out_of_order = false;
		if (pass) {
			u32 x = f.idx(frag, MATE1), y = f.idx(frag, MATE2);
			const i32 xs = f.start[x], xe = f.end[x], ys = f.start[y], ye = f.end[y];
			const u16 xc = f.contig[x], yc = f.contig[y];
			const i32 xb = f.fwd(x) ? xe : xs, yb = f.fwd(y) ? ye : ys;
			out_of_order = xc > yc || (xc == yc && xb > yb);
			const i32 s1 = out_of_order ? ys : xs, e1 = out_of_order ? ye : xe, s2 = out_of_order ? xs : ys, e2 = out_of_order ? xe : ye;
			v1 = d1 == DOWNSTREAM ? s1 : e1; v2 = d2 == DOWNSTREAM ? s2 : e2;
		}
		const u32 n_pass = __popc(mask), n_none = __popc(mask & none_mask);
		const bool zero_value = __any_sync(FULL, pass && (v1 <= 0 || v2 <= 0)); // 0 means "unset" to expand_anchor: such a chunk is replayed statement by statement
		const bool in_reach = listed >= threshold ? counted + n_none > threshold : listed + n_pass > threshold;
		if (!in_reach && !zero_value) {
			if (fill && pass) { listd[w + __popc(mask & ((1u << lane) - 1u))] = frag; if (out_of_order) need_swap[frag] = 1; }
			w += n_pass; listed += n_pass; counted += n_none;
			// anchors: minimum (downstream) / maximum (upstream) of the listed mates' values and the anchor so far
			i32 r1 = pass ? v1 : (d1 == DOWNSTREAM ? 0x7FFFFFFF : (i32) 0x80000000), r2 = pass ? v2 : (d2 == DOWNSTREAM ? 0x7FFFFFFF : (i32) 0x80000000);
			for (int o = 16; o > 0; o >>= 1) {
				const i32 t1 = __shfl_xor_sync(FULL, r1, o), t2 = __shfl_xor_sync(FULL, r2, o);
				r1 = d1 == DOWNSTREAM ? (t1 < r1 ? t1 : r1) : (t1 > r1 ? t1 : r1); r2 = d2 == DOWNSTREAM ? (t2 < r2 ? t2 : r2) : (t2 > r2 ? t2 : r2);
			}
			expand_anchor(an1, d1, r1, r1); expand_anchor(an2, d2, r2, r2);
		} else {
			for (u32 m = mask; m; m &= m - 1) {
				const int src = __ffs((int) m) - 1;
				const u32 fl_s = __shfl_sync(FULL, (u32) fl, src), frag_s = __shfl_sync(FULL, frag, src);
				const i32 v1_s = __shfl_sync(FULL, v1, src), v2_s = __shfl_sync(FULL, v2, src);
				const bool ooo_s = __shfl_sync(FULL, (u32) out_of_order, src) != 0;
				if (fl_s != F_none && listed >= threshold) continue;
				if (counted >= threshold) { done = true; break; }
				++listed; if (fl_s == F_none) ++counted;
				expand_anchor(an1, d1, v1_s, v1_s); expand_anchor(an2, d2, v2_s, v2_s);
				if (fill && lane == 0) { listd[w] = frag_s; if (ooo_s) need_swap[frag_s] = 1; }
				++w;
			}
		}
	}
	if (lane == 0) {
		if (fill != 1) c.n_listd[cand] = listed;
		if (fill) { c.discordant_mates[cand] = counted; c.anchor1[cand] = an1; c.anchor2[cand] = an2; }
	}
}
#endif

struct fill_u32_fn { u32* p; u32 v; ARB_HD void operator()(u32 i) const { p[i] = v; } };

void engine::find_fusions(i32 max_mate_gap) {
	if (!has_annotation) throw arb_error("arb_find_fusions: annotation must be set first");
	const u32 n = frags.n;
	const u32 T = params.subsampling_threshold;
	frag_view f = frags.view();
	annot_view an = annot.view();
	stage_timer t_all(ex);

	// 1. records
	dbuf<u32> rec_off((size_t) n + 1);
	emit_count_fn ec = {f, rec_off.ptr(), work_parts > 1 ? work_owned.ptr() : NULL};
	for_each(ex, n, ec);
	exclusive_scan_u32(ex, rec_off.ptr(), rec_off.ptr(), n);
	u32 R = 0; rec_off.download(ex, &R, 1, n);
	dbuf<u32> r_gene1(R), r_gene2(R), r_contigs(R), r_meta(R), r_frag(R); dbuf<i32> r_bp1(R), r_bp2(R), r_an1(R), r_an2(R);
	record_view r = {r_gene1.ptr(), r_gene2.ptr(), r_contigs.ptr(), r_bp1.ptr(), r_bp2.ptr(), r_meta.ptr(), r_frag.ptr(), r_an1.ptr(), r_an2.ptr()};
	emit_fill_fn ef = {f, rec_off.ptr(), r};
	for_each(ex, n, ef);

	// 2. group records by candidate key; candidate id = rank of the group's first record
	dbuf<u32> first(R), slot(R), head((size_t) R + 1), cand_of(R), perm(R), tmp_k(R), tmp_v(R);
	record_key_ops kops = {r};
	group_min_index(ex, table, R, kops, (const u8*) NULL, slot.ptr(), first.ptr());
	head_flag_fn hf = {first.ptr(), head.ptr()};
	for_each(ex, R, hf);
	exclusive_scan_u32(ex, head.ptr(), head.ptr(), R);
	u32 C = 0; head.download(ex, &C, 1, R);
	group_id_fn gi = {first.ptr(), head.ptr(), cand_of.ptr(), perm.ptr()};
	for_each(ex, R, gi);

	// 3. contiguous, name-ordered segment per candidate
	radix_sort_pairs_u32(ex, cand_of.ptr(), perm.ptr(), tmp_k.ptr(), tmp_v.ptr(), R, bits_for(C));
	dbuf<u32> seg_off((size_t) C + 1);
	segment_offsets_fn so = {cand_of.ptr(), seg_off.ptr(), R, C};
	for_each(ex, R, so);

	cands.first_frag.ensure(C);
	first_fragment_fn ff = {r.frag, perm.ptr(), seg_off.ptr(), cands.first_frag.ptr()};
	for_each(ex, C, ff);

	// 4. pass A
	cands.n = C; cands.genomic_marked = false; has_tag_csr = false;
	cands.gene1.ensure(C); cands.gene2.ensure(C); cands.contig1.ensure(C); cands.contig2.ensure(C); cands.bp1.ensure(C); cands.bp2.ensure(C);
	cands.dir1.ensure(C); cands.dir2.ensure(C); cands.split_reads1.ensure(C); cands.split_reads2.ensure(C); cands.discordant_mates.ensure(C);
	cands.filter.ensure(C); cands.bits.ensure(C); cands.bits2.ensure(C); cands.anchor1.ensure(C); cands.anchor2.ensure(C); cands.evalue.ensure(C);
	cands.list1_off.ensure((size_t) C + 1); cands.list2_off.ensure((size_t) C + 1); cands.listd_off.ensure((size_t) C + 1);
	cand_out co = {cands.gene1.ptr(), cands.gene2.ptr(), cands.contig1.ptr(), cands.contig2.ptr(), cands.bp1.ptr(), cands.bp2.ptr(), cands.dir1.ptr(), cands.dir2.ptr(),
	               cands.split_reads1.ptr(), cands.split_reads2.ptr(), cands.discordant_mates.ptr(), cands.filter.ptr(), cands.bits.ptr(), cands.bits2.ptr(),
	               cands.anchor1.ptr(), cands.anchor2.ptr(), cands.evalue.ptr(), cands.list1_off.ptr(), cands.list2_off.ptr(), cands.listd_off.ptr()};
	dbuf<u8> kept(R);
	walk_a_fn wa = {r, perm.ptr(), seg_off.ptr(), co, kept.ptr(), T};
	for_each(ex, C, wa);
	// list sizes were written into the *_off arrays; keep copies of the counts, then scan in place
	dbuf<u32> n_list1((size_t) C + 1), n_list2((size_t) C + 1), n_listd((size_t) C + 1);
#ifdef ARB_DEVICE_BUILD
	ARB_CUDA_CHECK(cudaMemcpyAsync(n_list1.ptr(), cands.list1_off.ptr(), (size_t) C * 4, cudaMemcpyDeviceToDevice, ex.stream));
	ARB_CUDA_CHECK(cudaMemcpyAsync(n_list2.ptr(), cands.list2_off.ptr(), (size_t) C * 4, cudaMemcpyDeviceToDevice, ex.stream));
#else
	memcpy(n_list1.ptr(), cands.list1_off.ptr(), (size_t) C * 4); memcpy(n_list2.ptr(), cands.list2_off.ptr(), (size_t) C * 4);
#endif
	exclusive_scan_u32(ex, cands.list1_off.ptr(), cands.list1_off.ptr(), C);
	exclusive_scan_u32(ex, cands.list2_off.ptr(), cands.list2_off.ptr(), C);
	u32 L1 = 0, L2 = 0; cands.list1_off.download(ex, &L1, 1, C); cands.list2_off.download(ex, &L2, 1, C);
	cands.n_list1 = L1; cands.n_list2 = L2;
	cands.list1.ensure(L1); cands.list2.ensure(L2);
	fill_split_lists_fn fl = {r, perm.ptr(), seg_off.ptr(), kept.ptr(), cands.list1_off.ptr(), cands.list2_off.ptr(), cands.list1.ptr(), cands.list2.ptr()};
	for_each(ex, C, fl);

	// 5. discordant mates bucketed by (gene1, gene2, direction1, direction2), buckets in name order
	dbuf<u32> dflag((size_t) R + 1);
	flag_discordant_fn fd = {r, dflag.ptr()};
	for_each(ex, R, fd);
	exclusive_scan_u32(ex, dflag.ptr(), dflag.ptr(), R);
	u32 D = 0; dflag.download(ex, &D, 1, R);
	dbuf<u32> drec(D), bfirst(D), bslot(D), bhead((size_t) D + 1), bucket_of(D), bperm(D), btmp_k(D), btmp_v(D);
	compact_fn cf = {dflag.ptr(), NULL, drec.ptr(), R};
	for_each(ex, R, cf);
	hash_index bucket_table;
	bucket_key_ops bops = {r, drec.ptr()};
	group_min_index(ex, bucket_table, D, bops, (const u8*) NULL, bslot.ptr(), bfirst.ptr());
	head_flag_fn bhf = {bfirst.ptr(), bhead.ptr()};
	for_each(ex, D, bhf);
	exclusive_scan_u32(ex, bhead.ptr(), bhead.ptr(), D);
	u32 B = 0; bhead.download(ex, &B, 1, D);
	group_id_fn bgi = {bfirst.ptr(), bhead.ptr(), bucket_of.ptr(), bperm.ptr()};
	for_each(ex, D, bgi);
	radix_sort_pairs_u32(ex, bucket_of.ptr(), bperm.ptr(), btmp_k.ptr(), btmp_v.ptr(), D, bits_for(B));
	dbuf<u32> bseg_off((size_t) B + 1);
	segment_offsets_fn bso = {bucket_of.ptr(), bseg_off.ptr(), D, B};
	for_each(ex, D, bso);

	// 6. pass B (count, scan, fill) + canonical mate order
	cand_out cob = co; cob.n_list1 = n_list1.ptr(); cob.n_list2 = n_list2.ptr(); cob.n_listd = n_listd.ptr();
	dbuf<u32> need_swap(n); need_swap.zero(ex, n);
#ifdef ARB_DEVICE_BUILD
	{
		dbuf<i32> o_bp1(D), o_bp2(D); dbuf<u32> o_frag(D); dbuf<u8> o_label(D);
		gather_bucket_fn gb = {r, drec.ptr(), bperm.ptr(), o_bp1.ptr(), o_bp2.ptr(), o_frag.ptr(), o_label.ptr()};
		for_each(ex, D, gb);
		dbuf<u32> bucket_of_cand(C), act((size_t) C + 1), active_cands(C);
		probe_bucket_fn pb = {r, cob, bucket_table.view(), drec.ptr(), bhead.ptr(), bucket_of_cand.ptr(), act.ptr()};
		for_each(ex, C, pb);
		exclusive_scan_u32(ex, act.ptr(), act.ptr(), C);
		u32 A = 0; act.download(ex, &A, 1, C);
		compact_fn ca = {act.ptr(), NULL, active_cands.ptr(), C};
		for_each(ex, C, ca);
		bucket_columns bcols = {o_bp1.ptr(), o_bp2.ptr(), o_frag.ptr(), o_label.ptr()};
		const u32 blocks = (u32) (((u64) A * 32 + WALK_B_THREADS - 1) / WALK_B_THREADS);
		// A list holds at most 2 x threshold mates (fusions.cpp:400-406: labelled mates are listed while fewer than `threshold` are, unlabelled ones until `threshold`
		// of them are) and never more than its bucket has: with a stretch of that size per candidate ONE walk writes the lists, a copy packs them. When the stretches
		// would not fit (huge -U, or millions of candidates on big buckets) the count / fill walks remain.
		dbuf<u32> stretch_off((size_t) A + 1), stretches; u32 S = 0;
		if (A) { stretch_size_fn sf = {active_cands.ptr(), bucket_of_cand.ptr(), bseg_off.ptr(), 2 * (u64) T, stretch_off.ptr()}; for_each(ex, A, sf); exclusive_scan_u32(ex, stretch_off.ptr(), stretch_off.ptr(), A); stretch_off.download(ex, &S, 1, A); }
		const bool one_pass = A != 0 && S < (1u << 31) && sf_fits(A, bseg_off, T) && getenv("ARB_WALK_B_TWO_PASS") == NULL;
		if (one_pass) stretches.alloc((size_t) S + 1);
		if (A) { k_walk_b<<<blocks, WALK_B_THREADS, 0, ex.stream>>>(active_cands.ptr(), A, bucket_of_cand.ptr(), bcols, bseg_off.ptr(), f, an, cob, one_pass ? stretch_off.ptr() : NULL, one_pass ? stretches.ptr() : NULL, need_swap.ptr(), max_mate_gap, T, one_pass ? 2 : 0); ARB_CUDA_CHECK(cudaGetLastError()); ++stats().kernels; }
		exclusive_scan_u32(ex, n_listd.ptr(), cands.listd_off.ptr(), C);
		u32 LD = 0; cands.listd_off.download(ex, &LD, 1, C);
		cands.n_listd = LD; cands.listd.ensure(LD);
		if (one_pass) { k_walk_b_pack<<<blocks, 256, 0, ex.stream>>>(active_cands.ptr(), A, stretches.ptr(), stretch_off.ptr(), cands.listd_off.ptr(), cands.listd.ptr()); ARB_CUDA_CHECK(cudaGetLastError()); ++stats().kernels; }
		else if (A) { k_walk_b<<<blocks, WALK_B_THREADS, 0, ex.stream>>>(active_cands.ptr(), A, bucket_of_cand.ptr(), bcols, bseg_off.ptr(), f, an, cob, cands.listd_off.ptr(), cands.listd.ptr(), need_swap.ptr(), max_mate_gap, T, 1); ARB_CUDA_CHECK(cudaGetLastError()); ++stats().kernels; }
	}
#else
	walk_b_fn wb = {r, f, an, cob, bucket_table.view(), drec.ptr(), bhead.ptr(), bperm.ptr(), bseg_off.ptr(), NULL, NULL, need_swap.ptr(), max_mate_gap, T, 0};
	for_each(ex, C, wb);
	exclusive_scan_u32(ex, n_listd.ptr(), cands.listd_off.ptr(), C);
	u32 LD = 0; cands.listd_off.download(ex, &LD, 1, C);
	cands.n_listd = LD; cands.listd.ensure(LD);
	wb.listd_off = cands.listd_off.ptr(); wb.listd = cands.listd.ptr(); wb.fill = 1;
	for_each(ex, C, wb);
#endif
	swap_mates_fn sm = {f, need_swap.ptr(), frags.swapped.ptr()};
	for_each(ex, n, sm);

	// 7. pass C
	walk_c_fn wc = {f, an, cob, cands.list1_off.ptr(), cands.list2_off.ptr(), cands.listd_off.ptr(), cands.list1.ptr(), cands.list2.ptr(), cands.listd.ptr()};
	for_each(ex, C, wc);
	timings.find_fusions_ms = t_all.stop();
	ex.sync();
}

void engine::get_candidates(arb_candidates& o) {
	const u32 C = cands.n;
	cands.gene1.download(ex, o.gene1, C); cands.gene2.download(ex, o.gene2, C); cands.contig1.download(ex, o.contig1, C); cands.contig2.download(ex, o.contig2, C);
	cands.bp1.download(ex, o.breakpoint1, C); cands.bp2.download(ex, o.breakpoint2, C); cands.dir1.download(ex, o.direction1, C); cands.dir2.download(ex, o.direction2, C);
	cands.split_reads1.download(ex, o.split_reads1, C); cands.split_reads2.download(ex, o.split_reads2, C); cands.discordant_mates.download(ex, o.discordant_mates, C);
	cands.filter.download(ex, o.filter, C); cands.bits.download(ex, o.bits, C); cands.bits2.download(ex, o.bits2, C);
	cands.anchor1.download(ex, o.anchor_start1, C); cands.anchor2.download(ex, o.anchor_start2, C); cands.evalue.download(ex, o.evalue, C);
	cands.list1_off.download(ex, o.list1_off, (size_t) C + 1); cands.list2_off.download(ex, o.list2_off, (size_t) C + 1); cands.listd_off.download(ex, o.listd_off, (size_t) C + 1);
	cands.list1.download(ex, o.list1, cands.n_list1); cands.list2.download(ex, o.list2, cands.n_list2); cands.listd.download(ex, o.listd, cands.n_listd);
	o.n = C;
}

void engine::get_slot_swaps(u8* out) { frags.swapped.download(ex, out, frags.n); }

} // namespace arb
