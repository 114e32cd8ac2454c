// blacklist.cu -- driver of the blacklist filter (see blacklist_hd.h).
#include <cstdlib>
#include "engine.h"
#include "blacklist_hd.h"

namespace arb {

static const u32 BLACKLIST_LANES = 32, BLACKLIST_THREADS = 256;

#ifdef ARB_DEVICE_BUILD
__global__ void __launch_bounds__(BLACKLIST_THREADS) k_blacklist_groups(blacklist_search s, const u32* heavy, u32 n_heavy) {
	const u32 q = blockIdx.x * (BLACKLIST_THREADS / BLACKLIST_LANES) + threadIdx.x / BLACKLIST_LANES;
	if (q >= n_heavy) return;
	lane_group g; g.lane = threadIdx.x % BLACKLIST_LANES; g.lanes = BLACKLIST_LANES; g.mask = 0xFFFFFFFFu;
	blacklist_group(g, s, heavy[q]);
}
#endif

static u32 bits_for(u32 n) { u32 b = 1; while (b < 32 && ((u64) 1 << b) < n) ++b; return b; }

// the rules in file order, as parsed by the caller
void engine::set_blacklist(u32 n, const u8* type1, const u8* type2, const u8* strand1, const u8* strand2, const u16* contig1, const u16* contig2,
                           const i32* start1, const i32* end1, const i32* start2, const i32* end2, const u32* gene1, const u32* gene2) {
	for (u32 k = 0; k < n; ++k)
		if (type1[k] > ARB_RULE_NOT_BOTH_SPLICED || type2[k] > ARB_RULE_NOT_BOTH_SPLICED) throw arb_error("arb_set_blacklist: unknown item type in rule " + std::to_string(k));
	blacklist_n = n;
	bl_type1.upload(ex, type1, n); bl_type2.upload(ex, type2, n); bl_strand1.upload(ex, strand1, n); bl_strand2.upload(ex, strand2, n);
	bl_contig1.upload(ex, contig1, n); bl_contig2.upload(ex, contig2, n); bl_start1.upload(ex, start1, n); bl_end1.upload(ex, end1, n);
	bl_start2.upload(ex, start2, n); bl_end2.upload(ex, end2, n); bl_gene1.upload(ex, gene1, n); bl_gene2.upload(ex, gene2, n);
	ex.sync();
	has_blacklist = true;
}

u32 engine::filter_blacklist(u32 n_ids, const u32* ids, float evalue_cutoff, i32 max_mate_gap, u8* verdicts) {
	if (!has_blacklist) throw arb_error("arb_filter_blacklist: arb_set_blacklist must be called first");
	if (!has_annotation) throw arb_error("arb_filter_blacklist: no annotation");
	if (max_mate_gap < 0) throw arb_error("arb_filter_blacklist: max_mate_gap must not be negative");
	const u32 C = cands.n;
	for (u32 i = 0; i < n_ids; ++i) if (ids[i] >= C) throw arb_error("arb_filter_blacklist: candidate id out of range");
	blacklist_heavy = 0;
	if (n_ids == 0) { timings.blacklist_ms = 0; return 0; }
	stage_timer t(ex);
	const u32 R = blacklist_n;
	rule_columns r;
	r.n = R;
	r.type[0] = bl_type1.ptr(); r.type[1] = bl_type2.ptr(); r.strand[0] = bl_strand1.ptr(); r.strand[1] = bl_strand2.ptr();
	r.contig[0] = bl_contig1.ptr(); r.contig[1] = bl_contig2.ptr(); r.start[0] = bl_start1.ptr(); r.start[1] = bl_start2.ptr();
	r.end[0] = bl_end1.ptr(); r.end[1] = bl_end2.ptr(); r.gene[0] = bl_gene1.ptr(); r.gene[1] = bl_gene2.ptr();

	// key table: the (contig, bin) keys of every rule, sorted, one entry per distinct key
	dbuf<u32> offset((size_t) R + 1); dbuf<unsigned long long> total(1);
	total.zero(ex, 1);
	u64 K = 0;
	if (R) {
		rule_key_count_fn cnt = {r, max_mate_gap, offset.ptr(), total.ptr()};
		for_each(ex, R, cnt);
		unsigned long long k = 0; total.download(ex, &k, 1); K = k;
	}
	if (K >= ((u64) 1 << 31)) throw arb_error("arb_filter_blacklist: the rules span " + std::to_string((unsigned long long) K) + " (contig, 100 kb bin) keys, more than 2^31");
	dbuf<u32> key((size_t) K), rule_of((size_t) K), key_tmp((size_t) K + 1), rule_tmp((size_t) K), head((size_t) K), table_key((size_t) K), table_begin((size_t) K + 1);
	u32 n_keys = 0;
	if (K) {
		exclusive_scan_u32(ex, offset.ptr(), offset.ptr(), R);
		rule_key_fill_fn fill = {r, max_mate_gap, offset.ptr(), key.ptr(), rule_of.ptr()};
		for_each(ex, R, fill);
		radix_sort_pairs_u32(ex, key.ptr(), rule_of.ptr(), key_tmp.ptr(), rule_tmp.ptr(), (u32) K, 16 + bits_for(annot.n_contigs + 1));
		rule_key_head_fn hf = {key.ptr(), head.ptr()};
		for_each(ex, (u32) K, hf);
		exclusive_scan_u32(ex, head.ptr(), key_tmp.ptr(), (u32) K); // slot of every head; the number of distinct keys lands at [K]
		rule_key_table_fn tf = {key.ptr(), head.ptr(), key_tmp.ptr(), table_key.ptr(), table_begin.ptr(), (u32) K};
		for_each(ex, (u32) K, tf);
		key_tmp.download(ex, &n_keys, 1, (size_t) K);
	}

	// the search over the eligible candidates
	dbuf<u32> d_ids(n_ids), heavy(n_ids), n_heavy(1); dbuf<u8> verdict(n_ids);
	d_ids.upload(ex, ids, n_ids);
	n_heavy.zero(ex, 1);
	blacklist_search s;
	s.m.r = r; s.m.c = make_state_for_rows(); s.m.an = annot.view(); s.m.max_mate_gap = max_mate_gap; s.m.evalue_cutoff = evalue_cutoff;
	s.t.n_keys = n_keys; s.t.key = table_key.ptr(); s.t.begin = table_begin.ptr(); s.t.rules = rule_of.ptr();
	s.ids = d_ids.ptr(); s.verdict = verdict.ptr();
	s.short_list = 64;
	if (const char* e = getenv("ARB_BLACKLIST_SHORT_LIST")) s.short_list = (u32) atol(e); // test hook: send short lists to the lane groups too
	s.heavy = heavy.ptr(); s.n_heavy = n_heavy.ptr();
	if (n_keys) {
		for_each(ex, n_ids, s);
		u32 H = 0; n_heavy.download(ex, &H, 1);
		blacklist_heavy = H;
#ifdef ARB_DEVICE_BUILD
		if (H) {
			const u32 per_block = BLACKLIST_THREADS / BLACKLIST_LANES;
			k_blacklist_groups<<<(H + per_block - 1) / per_block, BLACKLIST_THREADS, 0, ex.stream>>>(s, heavy.ptr(), H);
			ARB_CUDA_CHECK(cudaGetLastError());
			++stats().kernels;
		}
#else
		// the stand-in plays the lanes of a group one after the other and ORs their findings like __any_sync does
		std::vector<u32> queue = heavy.to_host(ex, H);
		hostsim_visit(H, [&](u32 q) {
			const u32 i = queue[q];
			bool any = false;
			for (u32 lane = 0; lane < BLACKLIST_LANES; ++lane) any = s.lane_walk(ids[i], lane, BLACKLIST_LANES) || any;
			verdict.ptr()[i] = any ? 1 : 0;
		});
		if (H) ++stats().kernels;
#endif
	} else verdict.zero(ex, n_ids); // no rule has a positional item that could share a bin
	verdict.download(ex, verdicts, n_ids);
	timings.blacklist_ms = t.stop();
	u32 blacklisted = 0;
	for (u32 i = 0; i < n_ids; ++i) blacklisted += verdicts[i] != 0;
	return blacklisted;
}

} // namespace arb
