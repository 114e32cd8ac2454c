// prims.cu -- hand-written sm_90a implementations of the primitives declared in prims.h
// (exclusive scan, stable LSD radix sort). HBM-bound integer kernels: coalesced 128-bit loads, shared-memory
// staging, warp shuffles / match; no tensor-core work and no library calls.
#include "prims.h"

namespace arb {

#ifdef ARB_DEVICE_BUILD
// =========================================================================================== scan
static const u32 SCAN_THREADS = 256, SCAN_ITEMS = 8, SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

__device__ __forceinline__ u32 warp_inclusive_scan(u32 v, u32 lane) {
	#pragma unroll
	for (u32 d = 1; d < 32; d <<= 1) { u32 t = __shfl_up_sync(0xFFFFFFFFu, v, d); if (lane >= d) v += t; }
	return v;
}

// loads the thread's 8 consecutive items (zero beyond n)
__device__ __forceinline__ void load8(const u32* in, u32 base, u32 n, u32 (&x)[SCAN_ITEMS]) {
	if (base + SCAN_ITEMS <= n) {
		const uint4 a = *reinterpret_cast<const uint4*>(in + base), b = *reinterpret_cast<const uint4*>(in + base + 4);
		x[0] = a.x; x[1] = a.y; x[2] = a.z; x[3] = a.w; x[4] = b.x; x[5] = b.y; x[6] = b.z; x[7] = b.w;
	} else {
		#pragma unroll
		for (u32 k = 0; k < SCAN_ITEMS; ++k) x[k] = base + k < n ? in[base + k] : 0;
	}
}

__global__ void __launch_bounds__(SCAN_THREADS) k_scan_block_sums(const u32* __restrict__ in, u32* __restrict__ block_sums, u32 n) {
	__shared__ u32 warp_sums[SCAN_THREADS / 32];
	const u32 base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
	u32 x[SCAN_ITEMS]; load8(in, base, n, x);
	u32 s = 0;
	#pragma unroll
	for (u32 k = 0; k < SCAN_ITEMS; ++k) s += x[k];
	#pragma unroll
	for (u32 d = 16; d > 0; d >>= 1) s += __shfl_xor_sync(0xFFFFFFFFu, s, d);
	if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = s;
	__syncthreads();
	if (threadIdx.x == 0) { u32 t = 0; for (u32 w = 0; w < SCAN_THREADS / 32; ++w) t += warp_sums[w]; block_sums[blockIdx.x] = t; }
}

// out[i] = block_offsets[block] + exclusive prefix within the tile; in may alias out
__global__ void __launch_bounds__(SCAN_THREADS) k_scan_apply(const u32* in, u32* out, const u32* __restrict__ block_offsets, u32 n) {
	__shared__ u32 warp_sums[SCAN_THREADS / 32];
	const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const u32 base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
	u32 x[SCAN_ITEMS]; load8(in, base, n, x);
	u32 s = 0;
	#pragma unroll
	for (u32 k = 0; k < SCAN_ITEMS; ++k) s += x[k];
	const u32 incl = warp_inclusive_scan(s, lane);
	if (lane == 31) warp_sums[warp] = incl;
	__syncthreads();
	if (warp == 0) {
		u32 w = lane < SCAN_THREADS / 32 ? warp_sums[lane] : 0;
		u32 wi = warp_inclusive_scan(w, lane);
		if (lane < SCAN_THREADS / 32) warp_sums[lane] = wi - w; // exclusive
	}
	__syncthreads();
	u32 run = block_offsets[blockIdx.x] + warp_sums[warp] + (incl - s);
	#pragma unroll
	for (u32 k = 0; k < SCAN_ITEMS; ++k) { if (base + k < n) out[base + k] = run; run += x[k]; }
}

// arrays of at most a few tiles: one block walks the tiles with a running carry
__global__ void __launch_bounds__(SCAN_THREADS) k_scan_small(const u32* in, u32* out, u32 n, u32* total_out) {
	__shared__ u32 warp_sums[SCAN_THREADS / 32];
	__shared__ u32 tile_total;
	const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	u32 carry = 0;
	for (u32 tile = 0; tile < n; tile += SCAN_TILE) {
		const u32 base = tile + threadIdx.x * SCAN_ITEMS;
		u32 x[SCAN_ITEMS]; load8(in, base, n, x);
		u32 s = 0;
		#pragma unroll
		for (u32 k = 0; k < SCAN_ITEMS; ++k) s += x[k];
		const u32 incl = warp_inclusive_scan(s, lane);
		if (lane == 31) warp_sums[warp] = incl;
		__syncthreads();
		if (warp == 0) {
			u32 w = lane < SCAN_THREADS / 32 ? warp_sums[lane] : 0;
			u32 wi = warp_inclusive_scan(w, lane);
			if (lane < SCAN_THREADS / 32) warp_sums[lane] = wi - w;
			if (lane == SCAN_THREADS / 32 - 1) tile_total = wi;
		}
		__syncthreads();
		u32 run = carry + warp_sums[warp] + (incl - s);
		#pragma unroll
		for (u32 k = 0; k < SCAN_ITEMS; ++k) { if (base + k < n) out[base + k] = run; run += x[k]; }
		carry += tile_total;
		__syncthreads();
	}
	if (threadIdx.x == 0 && total_out) *total_out = carry;
}

// scans `n` items; level buffers are carved from `scratch` (needs >= n/SCAN_TILE*1.01 + 64 words)
static void scan_level(const exec_ctx& ex, const u32* in, u32* out, u32 n, u32* scratch, u32* total_out) {
	if (n <= 4 * SCAN_TILE) {
		k_scan_small<<<1, SCAN_THREADS, 0, ex.stream>>>(in, out, n, total_out);
		ARB_CUDA_CHECK(cudaGetLastError()); ++stats().kernels;
		return;
	}
	const u32 blocks = (n + SCAN_TILE - 1) / SCAN_TILE;
	u32* sums = scratch;
	k_scan_block_sums<<<blocks, SCAN_THREADS, 0, ex.stream>>>(in, sums, n);
	ARB_CUDA_CHECK(cudaGetLastError()); ++stats().kernels;
	scan_level(ex, sums, sums, blocks, scratch + ((blocks + 63) & ~63u), total_out);
	k_scan_apply<<<blocks, SCAN_THREADS, 0, ex.stream>>>(in, out, sums, n);
	ARB_CUDA_CHECK(cudaGetLastError()); ++stats().kernels;
}

void exclusive_scan_u32(const exec_ctx& ex, const u32* in, u32* out, u32 n) {
	if (!ex.scratch) throw arb_error("exclusive_scan_u32: the execution context has no scratch set");
	dbuf<u32>& scratch = ex.scratch->scan;
	scratch.ensure((size_t) n / SCAN_TILE * 2 + 8192);
	scan_level(ex, in, out, n, scratch.ptr(), out + n);
}

// =========================================================================================== radix sort
static const u32 RS_THREADS = 256, RS_ITEMS = 8, RS_TILE = RS_THREADS * RS_ITEMS, RS_WARPS = RS_THREADS / 32;

__global__ void __launch_bounds__(RS_THREADS) k_radix_hist(const u32* __restrict__ keys, u32* __restrict__ hist, u32 n, u32 shift, u32 nblocks) {
	__shared__ u32 h[256];
	h[threadIdx.x] = 0;
	__syncthreads();
	const u32 tile = blockIdx.x * RS_TILE;
	#pragma unroll
	for (u32 r = 0; r < RS_ITEMS; ++r) {
		const u32 i = tile + r * RS_THREADS + threadIdx.x;
		if (i < n) atomicAdd(&h[(keys[i] >> shift) & 255u], 1u);
	}
	__syncthreads();
	hist[threadIdx.x * nblocks + blockIdx.x] = h[threadIdx.x]; // digit-major: a scan of this array yields stable global offsets
}

__global__ void __launch_bounds__(RS_THREADS) k_radix_scatter(const u32* __restrict__ keys, const u32* __restrict__ vals, u32* __restrict__ keys_out, u32* __restrict__ vals_out,
                                                              const u32* __restrict__ offsets, u32 n, u32 shift, u32 nblocks) {
	__shared__ u32 warp_hist[RS_WARPS][256];
	__shared__ u32 gbase[256];
	const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	for (u32 k = threadIdx.x; k < RS_WARPS * 256; k += RS_THREADS) (&warp_hist[0][0])[k] = 0;
	gbase[threadIdx.x] = offsets[threadIdx.x * nblocks + blockIdx.x];
	__syncthreads();
	// warp w owns the contiguous sub-tile [w*256, (w+1)*256) of the tile, visited in 8 rounds of 32 consecutive items (stable order)
	const u32 warp_base = blockIdx.x * RS_TILE + warp * (32 * RS_ITEMS);
	u32 key[RS_ITEMS], val[RS_ITEMS], rank[RS_ITEMS];
	#pragma unroll
	for (u32 r = 0; r < RS_ITEMS; ++r) {
		const u32 i = warp_base + r * 32 + lane;
		const bool valid = i < n;
		key[r] = valid ? keys[i] : 0; val[r] = valid ? vals[i] : 0;
		const u32 d = valid ? (key[r] >> shift) & 255u : 256u + lane; // invalid lanes form singleton groups
		const u32 peers = __match_any_sync(0xFFFFFFFFu, d);
		const u32 before = __popc(peers & ((1u << lane) - 1u));
		u32 old = 0;
		if (valid) old = warp_hist[warp][d];
		__syncwarp();
		if (valid && before == 0) warp_hist[warp][d] = old + __popc(peers);
		__syncwarp();
		rank[r] = old + before;
	}
	__syncthreads();
	{ // per digit: exclusive prefix over the warps of this block
		const u32 d = threadIdx.x;
		u32 run = 0;
		#pragma unroll
		for (u32 w = 0; w < RS_WARPS; ++w) { u32 c = warp_hist[w][d]; warp_hist[w][d] = run; run += c; }
	}
	__syncthreads();
	#pragma unroll
	for (u32 r = 0; r < RS_ITEMS; ++r) {
		const u32 i = warp_base + r * 32 + lane;
		if (i < n) {
			const u32 d = (key[r] >> shift) & 255u;
			const u32 dst = gbase[d] + warp_hist[warp][d] + rank[r];
			keys_out[dst] = key[r]; vals_out[dst] = val[r];
		}
	}
}

void radix_sort_pairs_u32(const exec_ctx& ex, u32* keys, u32* vals, u32* keys_tmp, u32* vals_tmp, u32 n, u32 bits) {
	if (n <= 1 || bits == 0) return;
	const u32 nblocks = (n + RS_TILE - 1) / RS_TILE;
	if (!ex.scratch) throw arb_error("radix_sort_pairs_u32: the execution context has no scratch set");
	dbuf<u32>& hist = ex.scratch->radix;
	hist.ensure((size_t) 256 * nblocks + 1);
	u32 *ki = keys, *vi = vals, *ko = keys_tmp, *vo = vals_tmp;
	for (u32 shift = 0; shift < bits; shift += 8) {
		k_radix_hist<<<nblocks, RS_THREADS, 0, ex.stream>>>(ki, hist.ptr(), n, shift, nblocks);
		ARB_CUDA_CHECK(cudaGetLastError()); ++stats().kernels;
		exclusive_scan_u32(ex, hist.ptr(), hist.ptr(), 256 * nblocks);
		k_radix_scatter<<<nblocks, RS_THREADS, 0, ex.stream>>>(ki, vi, ko, vo, hist.ptr(), n, shift, nblocks);
		ARB_CUDA_CHECK(cudaGetLastError()); ++stats().kernels;
		u32* t = ki; ki = ko; ko = t; t = vi; vi = vo; vo = t;
	}
	if (ki != keys) {
		ARB_CUDA_CHECK(cudaMemcpyAsync(keys, ki, (size_t) n * sizeof(u32), cudaMemcpyDeviceToDevice, ex.stream));
		ARB_CUDA_CHECK(cudaMemcpyAsync(vals, vi, (size_t) n * sizeof(u32), cudaMemcpyDeviceToDevice, ex.stream));
	}
}

#else // ======================================================================================= hostsim stand-ins

void exclusive_scan_u32(const exec_ctx&, const u32* in, u32* out, u32 n) {
	u32 run = 0;
	for (u32 i = 0; i < n; ++i) { u32 t = in[i]; out[i] = run; run += t; }
	out[n] = run;
}

void radix_sort_pairs_u32(const exec_ctx&, u32* keys, u32* vals, u32* keys_tmp, u32* vals_tmp, u32 n, u32 bits) {
	(void) keys_tmp; (void) vals_tmp;
	if (n <= 1 || bits == 0) return;
	const u32 passes = (bits + 7) / 8;
	const u32 mask = passes >= 4 ? 0xFFFFFFFFu : ((1u << (passes * 8)) - 1u);
	std::vector<std::pair<u32, u32> > v(n);
	for (u32 i = 0; i < n; ++i) v[i] = std::make_pair(keys[i], vals[i]);
	std::stable_sort(v.begin(), v.end(), [mask](const std::pair<u32, u32>& a, const std::pair<u32, u32>& b) { return (a.first & mask) < (b.first & mask); });
	for (u32 i = 0; i < n; ++i) { keys[i] = v[i].first; vals[i] = v[i].second; }
}

#endif

} // namespace arb
