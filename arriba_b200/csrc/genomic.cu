// genomic.cu -- driver of the genomic-support search (see genomic_hd.h).
#include <algorithm>
#include <cstdlib>
#include <numeric>
#include "engine.h"
#include "genomic_hd.h"

namespace arb {

static const u32 GENOMIC_LANES = 32, GENOMIC_THREADS = 256;

#ifdef ARB_DEVICE_BUILD
__global__ void __launch_bounds__(GENOMIC_THREADS) k_genomic_groups(genomic_search s, const u32* heavy, u32 n_heavy) {
	const u32 q = blockIdx.x * (GENOMIC_THREADS / GENOMIC_LANES) + threadIdx.x / GENOMIC_LANES;
	if (q >= n_heavy) return;
	lane_group g; g.lane = threadIdx.x % GENOMIC_LANES; g.lanes = GENOMIC_LANES; g.mask = 0xFFFFFFFFu;
	genomic_group(g, s, heavy[q]);
}
#endif

// the records in file order, as parsed by the caller: sorted here by (key, position1), stable, and the key table built
void engine::set_genomic_breakpoints(u32 n, const u16* c1, const u16* c2, const u8* d1, const u8* d2, const i32* p1, const i32* p2) {
	std::vector<u32> perm(n);
	std::iota(perm.begin(), perm.end(), 0u);
	auto key = [&](u32 r) { return genomic_key(c1[r], c2[r], d1[r] ? UPSTREAM : DOWNSTREAM, d2[r] ? UPSTREAM : DOWNSTREAM); };
	std::stable_sort(perm.begin(), perm.end(), [&](u32 a, u32 b) { const u64 ka = key(a), kb = key(b); return ka != kb ? ka < kb : p1[a] < p1[b]; });
	std::vector<i32> s1(n), s2(n); std::vector<u64> keys; std::vector<u32> begin;
	for (u32 x = 0; x < n; ++x) {
		const u32 r = perm[x];
		s1[x] = p1[r]; s2[x] = p2[r];
		if (keys.empty() || keys.back() != key(r)) { keys.push_back(key(r)); begin.push_back(x); }
	}
	begin.push_back(n);
	genomic_n = n; genomic_keys = (u32) keys.size();
	genomic_pos1.upload(ex, s1.data(), n); genomic_pos2.upload(ex, s2.data(), n);
	genomic_key_table.upload(ex, keys.data(), keys.size()); genomic_key_begin.upload(ex, begin.data(), begin.size());
	ex.sync();
	has_genomic_breakpoints = true;
}

u32 engine::mark_genomic_support(i32 max_distance, i32 max_itd_length) {
	if (!has_genomic_breakpoints) throw arb_error("arb_mark_genomic_support: arb_set_genomic_breakpoints must be called first");
	if (!has_annotation) throw arb_error("arb_mark_genomic_support: no annotation");
	const u32 C = cands.n;
	cands.closest1.ensure(C); cands.closest2.ensure(C);
	cands.genomic_marked = true;
	if (C == 0) { timings.genomic_support_ms = 0; return 0; }
	stage_timer t(ex);
	dbuf<u32> heavy(C), n_heavy(1), range_lo(C), range_hi(C);
	n_heavy.zero(ex, 1);
	genomic_search s;
	s.ix.n_keys = genomic_keys; s.ix.key = genomic_key_table.ptr(); s.ix.key_begin = genomic_key_begin.ptr(); s.ix.pos1 = genomic_pos1.ptr(); s.ix.pos2 = genomic_pos2.ptr();
	s.c = make_state_for_rows(); s.an = annot.view();
	s.max_distance = max_distance; s.max_itd_length = max_itd_length;
	s.closest1 = cands.closest1.ptr(); s.closest2 = cands.closest2.ptr();
	s.short_range = 64;
	if (const char* e = getenv("ARB_GENOMIC_SHORT_RANGE")) s.short_range = (u32) atol(e); // test hook: send short ranges to the lane groups too
	s.heavy = heavy.ptr(); s.n_heavy = n_heavy.ptr(); s.range_lo = range_lo.ptr(); s.range_hi = range_hi.ptr();
	for_each(ex, C, s);
	u32 H = 0; n_heavy.download(ex, &H, 1);
	genomic_heavy = H;
#ifdef ARB_DEVICE_BUILD
	if (H) {
		const u32 per_block = GENOMIC_THREADS / GENOMIC_LANES;
		k_genomic_groups<<<(H + per_block - 1) / per_block, GENOMIC_THREADS, 0, ex.stream>>>(s, heavy.ptr(), H);
		ARB_CUDA_CHECK(cudaGetLastError());
		++stats().kernels;
	}
#else
	// the stand-in plays the lanes of a group one after the other and combines their picks like the shuffles do
	std::vector<u32> queue = heavy.to_host(ex, H);
	hostsim_visit(H, [&](u32 q) {
		const u32 k = queue[q];
		genomic_pick p = genomic_lane_pick(s, k, range_lo.ptr()[k], range_hi.ptr()[k], 0, GENOMIC_LANES);
		for (u32 lane = 1; lane < GENOMIC_LANES; ++lane) p.merge(genomic_lane_pick(s, k, range_lo.ptr()[k], range_hi.ptr()[k], lane, GENOMIC_LANES));
		genomic_finish(s, k, p);
	});
	if (H) ++stats().kernels;
#endif
	std::vector<i32> c1 = cands.closest1.to_host(ex, C);
	timings.genomic_support_ms = t.stop();
	u32 marked = 0;
	for (u32 k = 0; k < C; ++k) if (c1[k] >= 0) ++marked;
	return marked;
}

void engine::get_genomic_support(i32* closest1, i32* closest2) {
	if (!cands.genomic_marked) throw arb_error("arb_get_genomic_support: arb_mark_genomic_support must be called first");
	cands.closest1.download(ex, closest1, cands.n); cands.closest2.download(ex, closest2, cands.n);
}

} // namespace arb
