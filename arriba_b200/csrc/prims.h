// prims.h -- data-parallel primitives used by every stage: device buffers, for_each, exclusive scan,
// stable LSD radix sort of (key,value) pairs, and an exact "group by key, smallest index wins" hash index.
//
// Two builds of the SAME interface:
//   * product (nvcc, sm_90a): hand-written CUDA kernels below (#ifdef ARB_DEVICE_BUILD). No CUB/Thrust.
//   * tests/hostsim (g++ -DARB_HOSTSIM): sequential stand-ins, used only by the CPU test-suite to check the
//     per-element rules against the oracle. The product library is never built this way.
#pragma once
#include "hd.h"
#include <stdlib.h>
#include <string.h>
#include <stdexcept>
#include <string>
#include <vector>
#include <mutex>
#include <atomic>
#include <algorithm>

#ifdef ARB_DEVICE_BUILD
#include <cuda_runtime.h>
#endif

namespace arb {

struct arb_error: public std::runtime_error { explicit arb_error(const std::string& m): std::runtime_error(m) {} };

#ifdef ARB_DEVICE_BUILD
#define ARB_CUDA_CHECK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) throw arb::arb_error(std::string("CUDA error: ") + cudaGetErrorString(e_) + " at " + __FILE__ + ":" + std::to_string(__LINE__)); } while (0)
#endif

// launch statistics (bench.py reports gpu_launches from here)
struct launch_stats { std::atomic<u64> kernels; launch_stats(): kernels(0) {} }; // contexts on several threads count into the same total
inline launch_stats& stats() { static launch_stats s; return s; }

struct scratch_set; // per-context scratch of the scan and the radix sort (defined after dbuf)
struct exec_ctx {
	scratch_set* scratch; // owned by the context (engine): a context is bound to one device and one stream, so is its scratch
#ifdef ARB_DEVICE_BUILD
	cudaStream_t stream;
	exec_ctx(): scratch(0), stream(0) {}
	void sync() const { ARB_CUDA_CHECK(cudaStreamSynchronize(stream)); }
#else
	exec_ctx(): scratch(0) {}
	void sync() const {}
#endif
};

// ------------------------------------------------------------------------------------------- device memory pool
// Stage-local scratch buffers come and go many times per run; cudaMalloc/cudaFree would serialise the stream each time (cudaFree synchronises the
// device, cudaMalloc costs up to a millisecond). Blocks are carved out of large slabs, one list of free blocks per size class (steps of at most 25 %),
// per device; slabs go back to the driver only through pool_trim() (arb_release_device_memory) or when an allocation fails.
// size classes of the pool: steps of at most 25 %, every class a multiple of 512 bytes because blocks are carved back to back out of a slab
inline size_t pool_size_class(size_t bytes) { size_t c = 512; while (c < bytes) { c += c < (1u << 20) ? c : c / 4 >= (1u << 20) ? c / 4 : (1u << 20); c = (c + 511) & ~(size_t) 511; } return c; }
#ifdef ARB_DEVICE_BUILD
struct device_pool {
	struct slab { char* base; size_t size, used; };
	struct per_device { std::vector<std::pair<size_t, void*> > free_blocks; std::vector<slab> slabs; size_t outstanding; per_device(): outstanding(0) {} };
	std::vector<per_device> dev; std::mutex lock;
	static size_t size_class(size_t bytes) { return pool_size_class(bytes); }
	per_device& current() { int d = 0; ARB_CUDA_CHECK(cudaGetDevice(&d)); if ((size_t) d >= dev.size()) dev.resize((size_t) d + 1); return dev[(size_t) d]; }
	void* get(size_t bytes, size_t& granted) {
		std::lock_guard<std::mutex> g(lock);
		per_device& d = current();
		granted = size_class(bytes);
		++d.outstanding;
		for (size_t k = d.free_blocks.size(); k-- > 0; ) if (d.free_blocks[k].first == granted) {
			void* p = d.free_blocks[k].second; d.free_blocks[k] = d.free_blocks.back(); d.free_blocks.pop_back(); return p;
		}
		for (size_t k = d.slabs.size(); k-- > 0; ) if (d.slabs[k].size - d.slabs[k].used >= granted) { void* p = d.slabs[k].base + d.slabs[k].used; d.slabs[k].used += granted; return p; }
		slab s; s.size = std::max<size_t>(granted, (size_t) 512 << 20); s.used = granted; s.base = NULL;
		cudaError_t e = cudaMalloc((void**) &s.base, s.size);
		if (e != cudaSuccess) { cudaGetLastError(); s.size = granted; e = cudaMalloc((void**) &s.base, s.size); }
		if (e != cudaSuccess) { --d.outstanding; cudaGetLastError(); throw arb_error(std::string("out of device memory (") + cudaGetErrorString(e) + ")"); }
		d.slabs.push_back(s);
		return s.base;
	}
	void put(void* p, size_t granted) { std::lock_guard<std::mutex> g(lock); per_device& d = current(); d.free_blocks.push_back(std::make_pair(granted, p)); --d.outstanding; }
	void trim() { // only when nothing is handed out on the current device (blocks point into the slabs)
		std::lock_guard<std::mutex> g(lock);
		per_device& d = current();
		if (d.outstanding != 0) return;
		for (size_t k = 0; k < d.slabs.size(); ++k) cudaFree(d.slabs[k].base);
		d.slabs.clear(); d.free_blocks.clear();
	}
};
inline device_pool& pool() { static device_pool p; return p; }
inline void pool_trim() { pool().trim(); }
#else
inline void pool_trim() {}
#endif

// ------------------------------------------------------------------------------------------- device buffer
template <class T> class dbuf {
	T* p_; size_t n_; size_t granted_;
	dbuf(const dbuf&); dbuf& operator=(const dbuf&);
public:
	dbuf(): p_(NULL), n_(0), granted_(0) {}
	explicit dbuf(size_t n): p_(NULL), n_(0), granted_(0) { alloc(n); }
	~dbuf() { release(); }
	void release() {
		if (!p_) return;
#ifdef ARB_DEVICE_BUILD
		pool().put(p_, granted_);
#else
		free(p_);
#endif
		p_ = NULL; n_ = 0; granted_ = 0;
	}
	void alloc(size_t n) {
		release();
		n_ = n;
		size_t bytes = (n ? n : 1) * sizeof(T) + 64; // slack for vectorised tail reads
#ifdef ARB_DEVICE_BUILD
		p_ = (T*) pool().get(bytes, granted_);
#else
		p_ = (T*) malloc(bytes);
		if (!p_) throw arb_error("out of memory");
		// the device pool hands out recycled blocks with whatever the last user left in them, malloc hands out fresh (zero) pages for anything large: with
		// ARB_HOSTSIM_POISON set the stand-in fills new buffers with a pattern, so that a functor that counts on zeroed scratch shows in the CPU tests
		static const bool poison = getenv("ARB_HOSTSIM_POISON") != NULL;
		if (poison) memset((void*) p_, 0xA5, bytes);
#endif
	}
	void ensure(size_t n) { if (n > n_) alloc(n + n / 4); }
	void swap(dbuf& o) { std::swap(p_, o.p_); std::swap(n_, o.n_); std::swap(granted_, o.granted_); }
	T* ptr() const { return p_; }
	size_t size() const { return n_; }
	void zero(const exec_ctx& ex, size_t n) { fill_bytes(ex, 0, n); }
	void fill_bytes(const exec_ctx& ex, int byte, size_t n) {
		(void) ex;
#ifdef ARB_DEVICE_BUILD
		ARB_CUDA_CHECK(cudaMemsetAsync(p_, byte, n * sizeof(T), ex.stream));
#else
		memset(p_, byte, n * sizeof(T));
#endif
	}
	void upload(const exec_ctx& ex, const T* host, size_t n) {
		(void) ex;
		ensure(n);
		if (!n) return;
#ifdef ARB_DEVICE_BUILD
		ARB_CUDA_CHECK(cudaMemcpyAsync(p_, host, n * sizeof(T), cudaMemcpyHostToDevice, ex.stream));
#else
		memcpy(p_, host, n * sizeof(T));
#endif
	}
	void upload_at(const exec_ctx& ex, const T* host, size_t n, size_t offset) { // into [offset, offset + n) of a buffer already large enough
		(void) ex;
		if (!n) return;
		if (offset + n > n_) throw arb_error("dbuf::upload_at past the end of the buffer");
#ifdef ARB_DEVICE_BUILD
		ARB_CUDA_CHECK(cudaMemcpyAsync(p_ + offset, host, n * sizeof(T), cudaMemcpyHostToDevice, ex.stream));
#else
		memcpy(p_ + offset, host, n * sizeof(T));
#endif
	}
	void download(const exec_ctx& ex, T* host, size_t n, size_t offset = 0) const {
		(void) ex;
		if (!n) return;
#ifdef ARB_DEVICE_BUILD
		ARB_CUDA_CHECK(cudaMemcpyAsync(host, p_ + offset, n * sizeof(T), cudaMemcpyDeviceToHost, ex.stream));
		ARB_CUDA_CHECK(cudaStreamSynchronize(ex.stream));
#else
		memcpy(host, p_ + offset, n * sizeof(T));
#endif
	}
	std::vector<T> to_host(const exec_ctx& ex, size_t n) const { std::vector<T> v(n); download(ex, v.data(), n); return v; }
};

struct scratch_set { dbuf<u32> scan, radix; };

// ------------------------------------------------------------------------------------------- for_each
#ifdef ARB_DEVICE_BUILD
template <class F> __global__ void __launch_bounds__(256) k_for_each(u32 n, F f) {
	u32 i = blockIdx.x * 256u + threadIdx.x;
	if (i < n) f(i);
}
template <class F> void for_each(const exec_ctx& ex, u32 n, const F& f) {
	if (n == 0) return;
	k_for_each<F><<<(n + 255) / 256, 256, 0, ex.stream>>>(n, f);
	ARB_CUDA_CHECK(cudaGetLastError());
	++stats().kernels;
}
// same, with a register cap: at least MIN_BLOCKS resident 256-thread blocks per SM (the cooperative re-alignment kernels, whose many threads per item want occupancy)
template <int MIN_BLOCKS, class F> __global__ void __launch_bounds__(256, MIN_BLOCKS) k_for_each_occ(u32 n, F f) {
	u32 i = blockIdx.x * 256u + threadIdx.x;
	if (i < n) f(i);
}
template <int MIN_BLOCKS, class F> void for_each_occ(const exec_ctx& ex, u32 n, const F& f) {
	if (n == 0) return;
	k_for_each_occ<MIN_BLOCKS, F><<<(n + 255) / 256, 256, 0, ex.stream>>>(n, f);
	ARB_CUDA_CHECK(cudaGetLastError());
	++stats().kernels;
}
// functor with a private scratch array of WORDS 32-bit words per thread, kept in shared memory and interleaved by thread
// (word k of thread t at [k * BLOCK + t]: dynamically indexed, yet free of bank conflicts); f(i, scratch, stride)
template <u32 WORDS, u32 BLOCK, class F> __global__ void __launch_bounds__(BLOCK) k_for_each_scratch(u32 n, F f) {
	__shared__ u32 scratch[WORDS * BLOCK];
	u32 i = blockIdx.x * BLOCK + threadIdx.x;
	if (i < n) f(i, scratch + threadIdx.x, BLOCK);
}
template <u32 WORDS, class F> void for_each_scratch(const exec_ctx& ex, u32 n, const F& f) {
	if (n == 0) return;
	const u32 BLOCK = 128;
	k_for_each_scratch<WORDS, BLOCK, F><<<(n + BLOCK - 1) / BLOCK, BLOCK, 0, ex.stream>>>(n, f);
	ARB_CUDA_CHECK(cudaGetLastError());
	++stats().kernels;
}
#else
// The stand-in visits the items of a launch one after the other. A GPU visits them in no particular order, so a functor must not depend on it: with
// ARB_HOSTSIM_ORDER=1 the stand-in walks backwards, with 2 in a scattered order (a stride coprime to n), and the CPU tests must give the same results.
inline int hostsim_order() { static const int mode = getenv("ARB_HOSTSIM_ORDER") ? atoi(getenv("ARB_HOSTSIM_ORDER")) : 0; return mode; }
template <class G> inline void hostsim_visit(u32 n, const G& g) {
	const int mode = hostsim_order();
	if (mode == 0 || n < 2) { for (u32 i = 0; i < n; ++i) g(i); return; }
	if (mode == 1) { for (u32 i = n; i-- > 0;) g(i); return; }
	u64 stride = (u64) n * 5 / 13 + 1; // some stride near 0.38 n, made coprime to n
	auto gcd = [](u64 a, u64 b) { while (b) { const u64 t = a % b; a = b; b = t; } return a; };
	while (gcd(stride, n) != 1) ++stride;
	u64 at = n / 3;
	for (u32 k = 0; k < n; ++k) { g((u32) at); at = (at + stride) % n; }
}
template <class F> void for_each(const exec_ctx&, u32 n, const F& f) { hostsim_visit(n, [&](u32 i) { f(i); }); ++stats().kernels; }
template <int MIN_BLOCKS, class F> void for_each_occ(const exec_ctx& ex, u32 n, const F& f) { for_each(ex, n, f); }
template <u32 WORDS, class F> void for_each_scratch(const exec_ctx&, u32 n, const F& f) { u32 scratch[WORDS]; hostsim_visit(n, [&](u32 i) { f(i, scratch, 1); }); ++stats().kernels; }
#endif

// ------------------------------------------------------------------------------------------- atomics usable from HD functors
ARB_HD u32 atomic_cas_u32(u32* p, u32 expected, u32 desired) {
#ifdef __CUDA_ARCH__
	return atomicCAS(p, expected, desired);
#else
	u32 old = *p; if (old == expected) *p = desired; return old;
#endif
}
ARB_HD u32 atomic_min_u32(u32* p, u32 v) {
#ifdef __CUDA_ARCH__
	return atomicMin(p, v);
#else
	u32 old = *p; if (v < old) *p = v; return old;
#endif
}
ARB_HD u32 atomic_add_u32(u32* p, u32 v) {
#ifdef __CUDA_ARCH__
	return atomicAdd(p, v);
#else
	u32 old = *p; *p = old + v; return old;
#endif
}
// next free slot of an append-only list; on the device one atomic per warp (the active lanes take consecutive slots)
ARB_HD u32 append_slot(u32* counter) {
#ifdef __CUDA_ARCH__
	const unsigned active = __activemask();
	const unsigned lane = threadIdx.x & 31u, leader = (unsigned) __ffs((int) active) - 1u;
	u32 base = 0;
	if (lane == leader) base = atomicAdd(counter, (u32) __popc(active));
	base = __shfl_sync(active, base, (int) leader);
	return base + (u32) __popc(active & ((1u << lane) - 1u));
#else
	return (*counter)++;
#endif
}
ARB_HD u64 atomic_cas_u64(u64* p, u64 expected, u64 desired) {
#ifdef __CUDA_ARCH__
	return (u64) atomicCAS((unsigned long long*) p, (unsigned long long) expected, (unsigned long long) desired);
#else
	const u64 old = *p; if (old == expected) *p = desired; return old;
#endif
}
ARB_HD i32 atomic_min_i32(i32* p, i32 v) {
#ifdef __CUDA_ARCH__
	return atomicMin(p, v);
#else
	const i32 old = *p; if (v < old) *p = v; return old;
#endif
}
ARB_HD u32 atomic_or_u32(u32* p, u32 v) {
#ifdef __CUDA_ARCH__
	return atomicOr(p, v);
#else
	u32 old = *p; *p = old | v; return old;
#endif
}

// ------------------------------------------------------------------------------------------- exclusive scan (u32)
// out[i] = sum(in[0..i)), returns nothing; total is written to out[n] (out must hold n+1 elements). in may alias out.
void exclusive_scan_u32(const exec_ctx& ex, const u32* in, u32* out, u32 n);

// ------------------------------------------------------------------------------------------- stable radix sort of pairs
// Sorts (keys, vals) ascending by the low `bits` bits of the 32-bit key; stable. Uses (keys_tmp, vals_tmp) as ping-pong
// space; on return the sorted data is in keys/vals.
void radix_sort_pairs_u32(const exec_ctx& ex, u32* keys, u32* vals, u32* keys_tmp, u32* vals_tmp, u32 n, u32 bits);

// ------------------------------------------------------------------------------------------- exact group-by with smallest-index representative
// hash_index: open-addressing table over item indices. Each slot holds a representative item (`rep`, claimed by CAS)
// and the smallest item index with an equal key (`mn`). Keys are compared in full through KeyOps, so grouping is exact.
//   KeyOps requirements:  u64 hash(u32 item) const;  bool equal(u32 item_a, u32 item_b) const;
struct hash_index_view {
	u32* rep; u32* mn; u32 mask;
	static const u32 EMPTY = 0xFFFFFFFFu;
	template <class K> ARB_HD u32 insert(const K& k, u32 item) const { // returns slot
		u32 h = (u32) k.hash(item) & mask;
		for (;;) {
			u32 r = atomic_cas_u32(&rep[h], EMPTY, item);
			if (r == EMPTY || r == item || k.equal(r, item)) { atomic_min_u32(&mn[h], item); return h; }
			h = (h + 1) & mask;
		}
	}
	// lookup by an external probe object: P must provide  u64 hash() const;  bool equal_item(u32 item) const;
	template <class P> ARB_HD u32 find(const P& probe) const { // returns slot or EMPTY
		u32 h = (u32) probe.hash() & mask;
		for (;;) {
			u32 r = rep[h];
			if (r == EMPTY) return EMPTY;
			if (probe.equal_item(r)) return h;
			h = (h + 1) & mask;
		}
	}
};

struct hash_index {
	dbuf<u32> rep, mn; u32 cap;
	hash_index(): cap(0) {}
	hash_index_view view() const { hash_index_view v = {rep.ptr(), mn.ptr(), cap - 1}; return v; }
	void reset(const exec_ctx& ex, u32 n_items) {
		u32 c = 1024; while (c < 2 * (u64) n_items + 16) c <<= 1;
		cap = c;
		rep.ensure(c); mn.ensure(c);
		rep.fill_bytes(ex, 0xFF, c); mn.fill_bytes(ex, 0xFF, c);
	}
};

template <class K> struct group_insert_fn {
	hash_index_view t; K k; u32* slot_of; const u8* participate;
	ARB_HD void operator()(u32 i) const { slot_of[i] = (participate == NULL || participate[i]) ? t.insert(k, i) : hash_index_view::EMPTY; }
};
struct group_first_fn {
	hash_index_view t; const u32* slot_of; u32* first;
	ARB_HD void operator()(u32 i) const { first[i] = slot_of[i] == hash_index_view::EMPTY ? i : t.mn[slot_of[i]]; }
};
// first[i] = smallest j with key(j) == key(i) among participating items (first[i] = i for non-participants)
template <class K> void group_min_index(const exec_ctx& ex, hash_index& table, u32 n, const K& k, const u8* participate, u32* slot_scratch, u32* first) {
	table.reset(ex, n);
	group_insert_fn<K> ins = {table.view(), k, slot_scratch, participate};
	for_each(ex, n, ins);
	group_first_fn fin = {table.view(), slot_scratch, first};
	for_each(ex, n, fin);
}

} // namespace arb
