// mismap.cu -- drivers of the k-mer index, gene homology and re-alignment stages (see mismap_hd.h).
#include <algorithm>
#include <cstdlib>
#include "engine.h"
#include "mismap_hd.h"

namespace arb {

#ifdef ARB_DEVICE_BUILD
// pass 1 of the re-alignment: MISMAP_GROUP_LANES lanes per (candidate, read) item, worklist of continuations in shared memory (mismap_hd.h, evaluate_group)
static const u32 MISMAP_THREADS = 256, MISMAP_WORKLIST = 64, MISMAP_GROUP_LANES = 16;
template <u32 LANES> __global__ void __launch_bounds__(MISMAP_THREADS, 3) k_mismap_items(mismap_items it, u32 n_items, int budget, u32* heavy, u32* n_heavy) {
	const u32 GROUPS = MISMAP_THREADS / LANES;
	__shared__ realign_work tasks[GROUPS][MISMAP_WORKLIST];
	__shared__ u32 tops[GROUPS];
	const u32 group = threadIdx.x / LANES;
	lane_group g; g.lane = threadIdx.x % LANES; g.lanes = LANES; g.mask = (LANES >= 32 ? 0xFFFFFFFFu : ((1u << (LANES & 31u)) - 1u)) << ((threadIdx.x & 31u) / LANES * LANES);
	const u32 j = blockIdx.x * GROUPS + group;
	if (j >= n_items || it.skip(j)) return;
	const u32 i = it.item_frag[j];
	if (((const volatile u8*) it.mismapper)[i]) return; // another candidate's evaluation of this fragment already decided (the label is an OR)
	realign_worklist wl = {tasks[group], &tops[group], MISMAP_WORKLIST};
	realign_tally tally = {0, 0, 0};
	const u32 verdict = evaluate_group(g, it, j, wl, budget, tally);
	if (it.tallies) { // sequences and bases are the same on every lane, the hits are per lane
		const u32 hits = g.sum(tally.hits);
		if (g.lane == 0) { unsigned long long* t = it.tallies + 3 * (j % mismap_items::TALLY_SLOTS); atomicAdd(t, (unsigned long long) tally.sequences); atomicAdd(t + 1, (unsigned long long) tally.bases); atomicAdd(t + 2, (unsigned long long) hits); }
	}
	if (g.lane == 0) {
		if (verdict == REALIGN_FOUND) it.mismapper[i] = 1;
		else if (verdict == REALIGN_EXHAUSTED) heavy[atomicAdd(n_heavy, 1u)] = j;
	}
}
#endif

void engine::set_splice_sites(const u32* off, const i32* sites) {
	splice_off.upload(ex, off, (size_t) annot.n_genes + 1);
	splice_sites.upload(ex, sites, off[annot.n_genes]); n_splice_sites = off[annot.n_genes];
	ex.sync();
	has_splice_sites = true;
}

u64 engine::build_kmer_index(const u32* contig, const i32* start, const i32* end, u32 n, u32 n_index_contigs) {
	// an empty index has no blocks (no lookup reaches the block table: every bucket is empty)
	kmer_index_contigs = n_index_contigs; kmer_indexed = 0; kmer_block_shift = 0; kmer_blocks = 0;
	kmer_block_base.ensure((size_t) n_index_contigs + 1); kmer_block_base.zero(ex, (size_t) n_index_contigs + 1);
	stage_timer t_all(ex);
	const size_t n_buckets = (size_t) n_index_contigs * 65536;
	kmer_bucket_off.ensure(n_buckets + 2);
	kmer_bucket_off.zero(ex, n_buckets + 2);
	std::vector<u32> first((size_t) n + 1, 0);
	for (u32 k = 0; k < n; ++k) { if (end[k] < start[k]) throw arb_error("arb_build_kmer_index: malformed interval"); const u64 t = (u64) first[k] + (u64) (end[k] - start[k]); if (t > 0xFFFFFFF0ull) throw arb_error("arb_build_kmer_index: more than 2^32 positions"); first[k + 1] = (u32) t; }
	const u32 P = first[n];
	if (P == 0) { ex.sync(); return 0; }
	dbuf<u32> d_contig, d_first; dbuf<i32> d_start, d_end;
	d_contig.upload(ex, contig, n); d_start.upload(ex, start, n); d_end.upload(ex, end, n); d_first.upload(ex, first.data(), (size_t) n + 1);
	interval_view iv = {d_contig.ptr(), d_start.ptr(), d_end.ptr(), d_first.ptr(), n};
	dbuf<u32> flag((size_t) P + 1);
	kmer_flag_fn ff = {iv, annot.view(), flag.ptr()};
	for_each(ex, P, ff);
	exclusive_scan_u32(ex, flag.ptr(), flag.ptr(), P);
	u32 K = 0; flag.download(ex, &K, 1, P);
	kmer_indexed = K;
	if (K == 0) return 0;
	dbuf<u32> key(K), pos(K), tk(K), tv(K);
	kmer_emit_fn ef = {iv, annot.view(), flag.ptr(), key.ptr(), pos.ptr()};
	for_each(ex, P, ef);
	u32 bits = 16; while (bits < 32 && ((u64) 1 << bits) < (u64) n_index_contigs * 65536) ++bits;
	radix_sort_pairs_u32(ex, key.ptr(), pos.ptr(), tk.ptr(), tv.ptr(), K, bits); // stable: positions stay ascending inside a bucket
	bucket_count_fn bc = {key.ptr(), kmer_bucket_off.ptr()};
	for_each(ex, K, bc);
	exclusive_scan_u32(ex, kmer_bucket_off.ptr(), kmer_bucket_off.ptr(), (u32) n_buckets);
	kmer_pos.ensure(K);
#ifdef ARB_DEVICE_BUILD
	ARB_CUDA_CHECK(cudaMemcpyAsync(kmer_pos.ptr(), pos.ptr(), (size_t) K * 4, cudaMemcpyDeviceToDevice, ex.stream));
#else
	memcpy(kmer_pos.ptr(), pos.ptr(), (size_t) K * 4);
#endif
	{ // block table (mismap_hd.h, kmer_index_view): blocks of 128 kb, larger where the table would exceed 2 GiB
		u32 shift = 17;
		std::vector<u32> base(n_index_contigs + 1, 0);
		for (;; ++shift) {
			u64 total = 0;
			for (u32 c = 0; c < n_index_contigs; ++c) { base[c] = (u32) total; total += ((u64) (c < annot.h_contig_len.size() ? annot.h_contig_len[c] : 0) >> shift) + 1; }
			base[n_index_contigs] = (u32) total;
			if (total * 65536 * 4 <= ((u64) 2 << 30) || shift >= 24) break;
		}
		kmer_block_shift = shift; kmer_blocks = base[n_index_contigs];
		kmer_block_base.upload(ex, base.data(), (size_t) n_index_contigs + 1);
		const u64 cells = (u64) kmer_blocks << 16;
		kmer_block_first.ensure(cells); kmer_block_first.fill_bytes(ex, 0xFF, cells);
		block_first_min_fn mn = {key.ptr(), kmer_pos.ptr(), kmer_block_base.ptr(), kmer_block_shift, kmer_block_first.ptr()};
		for_each(ex, K, mn);
		block_first_sweep_fn sf = {kmer_bucket_off.ptr(), kmer_block_base.ptr(), kmer_block_first.ptr()};
		for_each(ex, n_index_contigs << 16, sf);
	}
	timings.kmer_index_ms = t_all.stop(); timings.kmer_positions = K;
	ex.sync();
	return K;
}

kmer_index_view engine::index_view() {
	kmer_index_view ix = {kmer_pos.ptr(), kmer_bucket_off.ptr(), kmer_index_contigs, kmer_block_first.ptr(), kmer_block_base.ptr(), kmer_block_shift};
	return ix;
}

void engine::probe_kmer_lookup(const u32* contig, const u32* kmer, const i32* from, u32 n, u32* out) {
	if (n == 0) return;
	for (u32 j = 0; j < n; ++j) {
		if (contig[j] >= kmer_index_contigs || kmer[j] > 0xFFFFu) throw arb_error("arb_selftest_kmer_lookup: contig not indexed or 8-mer out of range");
		if (from[j] > 0 && (u64) from[j] >= (u64) (contig[j] < annot.h_contig_len.size() ? annot.h_contig_len[contig[j]] : 0)) throw arb_error("arb_selftest_kmer_lookup: bound past the contig's end");
	}
	dbuf<u32> c, k, o((size_t) n * 6); dbuf<i32> f;
	c.upload(ex, contig, n); k.upload(ex, kmer, n); f.upload(ex, from, n);
	kmer_lookup_fn fn = {index_view(), c.ptr(), k.ptr(), f.ptr(), o.ptr()};
	for_each(ex, n, fn);
	o.download(ex, out, (size_t) n * 6);
}

void engine::homolog_pairs(const u32* ga, const u32* gb, u32 n, u8* out) {
	if (n == 0) return;
	dbuf<u32> a, b; dbuf<u8> o(n);
	a.upload(ex, ga, n); b.upload(ex, gb, n);
	kmer_index_view ix = index_view();
	stage_timer t_all(ex);
	if (homolog_lanes > 1 && (u64) n * homolog_lanes < 0x80000000ull) { // a few pairs of long, similar genes dominate: lanes per pair (mismap_hd.h, homolog_count_fn)
		dbuf<u32> count(n); count.zero(ex, n);
		homolog_count_fn cf = {annot.view(), ix, a.ptr(), b.ptr(), count.ptr(), homolog_lanes, params.max_homolog_identity};
		for_each(ex, n * homolog_lanes, cf);
		homolog_decide_fn df = {annot.view(), ix, a.ptr(), b.ptr(), count.ptr(), o.ptr(), params.max_homolog_identity};
		for_each(ex, n, df);
	} else {
		homolog_pairs_fn fn = {annot.view(), ix, a.ptr(), b.ptr(), o.ptr(), params.max_homolog_identity};
		for_each(ex, n, fn);
	}
	timings.homologs_ms += t_all.stop();
	o.download(ex, out, n);
}

// work items j = part, part + parts, ... of the item list (items of one candidate are consecutive: a stride spreads the expensive candidates over the parts)
struct item_stride_fn {
	const u32* cand; const u32* frag; const u8* kind; u32 part, parts; u32* o_cand; u32* o_frag; u8* o_kind;
	ARB_HD void operator()(u32 k) const { const u32 j = k * parts + part; o_cand[k] = cand[j]; o_frag[k] = frag[j]; o_kind[k] = kind[j]; }
};
struct verdict_or_fn { const u8* v; u8* mism; ARB_HD void operator()(u32 i) const { if (v[i]) mism[i] = 1; } };

u64 engine::filter_mismappers(i32 max_mate_gap) {
	void* v; u64 b;
	filter_mismappers_part(max_mate_gap, 0, 1, &v, &b);
	return filter_mismappers_finish();
}

// re-aligns this part's share of the work items; the verdicts (one byte per fragment, 1 = some evaluation says mis-mapped) stay on the device for the caller to
// combine across parts (MAX) before filter_mismappers_finish
void engine::filter_mismappers_part(i32 max_mate_gap, int part, int parts, void** verdicts, u64* bytes) {
	if (!has_splice_sites) throw arb_error("arb_filter_mismappers: arb_set_splice_sites must be called first");
	if (parts < 1 || part < 0 || part >= parts) throw arb_error("arb_filter_mismappers_part: invalid part");
	const u32 C = cands.n, N = frags.n;
	mismap_verdicts.ensure(N); mismap_verdicts.zero(ex, N);
	*verdicts = mismap_verdicts.ptr(); *bytes = N;
	mismap_items_total = 0; mismap_ms_part = 0;
	if (C == 0) { ex.sync(); return; }
	stage_timer t_all(ex);
	dbuf<u32> item_off((size_t) C + 1);
	item_count_fn ic = {cands.filter.ptr(), cands.list1_off.ptr(), cands.list2_off.ptr(), cands.listd_off.ptr(), item_off.ptr()};
	for_each(ex, C, ic);
	exclusive_scan_u32(ex, item_off.ptr(), item_off.ptr(), C);
	u32 I = 0; item_off.download(ex, &I, 1, C);
	mismap_items_total = I;
	dbuf<u32> item_cand(I), item_frag(I); dbuf<u8> item_kind(I); dbuf<u8>& mism = mismap_verdicts;
	item_fill_fn ifn = {cands.filter.ptr(), cands.list1_off.ptr(), cands.list1.ptr(), cands.list2_off.ptr(), cands.list2.ptr(), cands.listd_off.ptr(), cands.listd.ptr(), item_off.ptr(), item_cand.ptr(), item_frag.ptr(), item_kind.ptr()};
	for_each(ex, C, ifn);
	if (parts > 1) { // this part's share
		const u32 mine = I > (u32) part ? (I - (u32) part + (u32) parts - 1) / (u32) parts : 0;
		dbuf<u32> c2(mine), f2(mine); dbuf<u8> k2(mine);
		item_stride_fn st = {item_cand.ptr(), item_frag.ptr(), item_kind.ptr(), (u32) part, (u32) parts, c2.ptr(), f2.ptr(), k2.ptr()};
		for_each(ex, mine, st);
		ex.sync();
		item_cand.swap(c2); item_frag.swap(f2); item_kind.swap(k2);
		I = mine;
	}
	kmer_index_view ix = index_view();
	gene_splice_view sp = {splice_off.ptr(), splice_sites.ptr()};
	mismap_params mp = {max_mate_gap, params.max_mismapper_fraction};
	dbuf<unsigned long long> tallies(3 * (size_t) mismap_items::TALLY_SLOTS); tallies.zero(ex, 3 * (size_t) mismap_items::TALLY_SLOTS);
	mismap_items items = {frags.view(), annot.view(), ix, sp, mp, item_cand.ptr(), item_frag.ptr(), item_kind.ptr(), cands.contig1.ptr(), cands.contig2.ptr(), cands.filter.ptr(), mism.ptr(), tallies.ptr()};
	// pass 1: a group of lanes per item, bounded; pass 2: the few items it gives up on (stuck in repeats), `lanes` threads each (mismap_hd.h, realign_ctl)
	dbuf<u32> heavy(I), n_heavy(1);
	n_heavy.zero(ex, 1);
	stage_timer t1(ex);
#ifdef ARB_DEVICE_BUILD
	if (I) {
		const u32 GROUPS = MISMAP_THREADS / MISMAP_GROUP_LANES;
		k_mismap_items<MISMAP_GROUP_LANES><<<(I + GROUPS - 1) / GROUPS, MISMAP_THREADS, 0, ex.stream>>>(items, I, mismap_budget, heavy.ptr(), n_heavy.ptr());
		ARB_CUDA_CHECK(cudaGetLastError()); ++stats().kernels;
	}
#else
	mismap_item_group_fn mi = {items, mismap_budget, heavy.ptr(), n_heavy.ptr()};
	for_each(ex, I, mi);
#endif
	timings.mismappers_pass1_ms = t1.stop();
	{ // SURVEY.md section 8(d): per re-aligned sequence of length l: 3l/8 (read) + 8(l - 8) (bucket offsets) + 4 * hits + l/2 (extension windows)
		std::vector<unsigned long long> t(3 * (size_t) mismap_items::TALLY_SLOTS);
		tallies.download(ex, t.data(), t.size());
		u64 sequences = 0, bases = 0, hits = 0;
		for (size_t k = 0; k < t.size(); k += 3) { sequences += t[k]; bases += t[k + 1]; hits += t[k + 2]; }
		timings.mismapper_sequences = sequences; timings.mismapper_hits = hits;
		timings.mismapper_algorithmic_bytes = bases * 3 / 8 + 8 * (bases - 8 * sequences) + 4 * hits + bases / 2;
		items.tallies = NULL; // the cooperative passes are not part of the budget
	}
	u32 H = 0; n_heavy.download(ex, &H, 1);
	stage_timer t2(ex);
	// pass 2 and the task rounds: continuations are registered (mismap_hd.h, realign_ctl) and run as tasks, one per distinct continuation
	// one table for all cooperative items (a read in a long repeat registers thousands of continuations, most reads a handful): 4,096 slots of 16 bytes per
	// item, at least 2^20 and at most 2^26 slots; the pass 2 kernels keep 4 resident 256-thread blocks per SM (prims.h, for_each_occ)
	u32 K = 1u << 20; while (K < (1u << 26) && (u64) K < (u64) H * 4096) K <<= 1;
	if (const char* s = getenv("ARB_MISMAP_TABLE_TOTAL")) { K = 1; while (K < (u32) std::max(1, atoi(s))) K <<= 1; } // test hook: a first table that overflows
	if (H >= (1u << 24)) throw arb_error("too many reads need the cooperative re-alignment");
	timings.mismapper_heavy_items = H; timings.mismapper_table_slots = K;
	u64 spawned = 0; u32 rounds = 0, overflows = 0;
	dbuf<u32> n_tasks(1), overflow(1), n_redo(1);
	for (u32 n = H; n; ) { // attempts: the items of this one are heavy[0, n)
		dbuf<continuation_slot> tables((size_t) K + 1); dbuf<realign_task> tasks((size_t) K + 1); dbuf<u8> incomplete(n);
		overflow.zero(ex, 1); incomplete.zero(ex, n);
		continuation_init_fn ci = {tables.ptr()}; for_each(ex, K, ci);
		const continuation_registry reg = {tables.ptr(), K, overflow.ptr(), incomplete.ptr()};
		for (u32 done = 0; done < n; ) { // launches of at most 2^31 threads
			const u32 batch = std::min<u32>(n - done, 0x80000000u / mismap_lanes);
			mismap_heavy_fn mh = {items, heavy.ptr(), mismap_lanes, done, reg};
			for_each_occ<4>(ex, batch * mismap_lanes, mh);
			done += batch;
		}
		for (;;) {
			n_tasks.zero(ex, 1);
			continuation_collect_fn cc = {tables.ptr(), K, heavy.ptr(), item_frag.ptr(), mism.ptr(), tasks.ptr(), n_tasks.ptr()};
			for_each(ex, K, cc);
			u32 Q = 0; n_tasks.download(ex, &Q, 1);
			if (Q == 0) break;
			spawned += Q; ++rounds;
			for (u32 done = 0; done < Q; ) {
				const u32 batch = std::min<u32>(Q - done, 0x80000000u / mismap_task_lanes);
				mismap_task_fn mt = {items, tasks.ptr() + done, mismap_task_lanes, reg};
				for_each_occ<4>(ex, batch * mismap_task_lanes, mt);
				done += batch;
			}
		}
		u32 o = 0; overflow.download(ex, &o, 1); overflows += o;
		if (o == 0) break;
		// a registration did not fit: its continuation was dropped, so the undecided items it belonged to are re-aligned again with a larger table
		dbuf<u32> redo(n); n_redo.zero(ex, 1);
		incomplete_collect_fn ic = {incomplete.ptr(), heavy.ptr(), item_frag.ptr(), mism.ptr(), redo.ptr(), n_redo.ptr()};
		for_each(ex, n, ic);
		n_redo.download(ex, &n, 1);
		heavy.swap(redo);
		u64 next = K; while (next < std::max<u64>(4 * (u64) K, (u64) n * 4096)) next <<= 1;
		if (n && next > (1u << 31)) throw arb_error("the continuation registry of the re-alignment would exceed 2^31 slots");
		K = (u32) next;
	}
	timings.mismapper_tasks = spawned; timings.mismapper_rounds = rounds; timings.mismapper_overflow = overflows;
	timings.mismappers_pass2_ms = t2.stop();
	mismap_ms_part = t_all.stop();
	ex.sync();
}

// labels the mis-mapped fragments and discards the candidates most of whose reads are (filter_mismappers.cpp:232-244, :336-356)
u64 engine::filter_mismappers_finish() {
	const u32 C = cands.n, N = frags.n;
	if (C == 0) return 0;
	stage_timer t_all(ex);
	dbuf<u8>& mism = mismap_verdicts;
	mismap_apply_fn ma = {mism.ptr(), frags.filter.ptr()};
	for_each(ex, N, ma);
	mismap_count_fn mc = {frags.filter.ptr(), cands.list1_off.ptr(), cands.list1.ptr(), cands.list2_off.ptr(), cands.list2.ptr(), cands.listd_off.ptr(), cands.listd.ptr(),
	                      cands.split_reads1.ptr(), cands.split_reads2.ptr(), cands.discordant_mates.ptr(), cands.filter.ptr(), params.max_mismapper_fraction};
	for_each(ex, C, mc);
	timings.mismappers_ms = mismap_ms_part + t_all.stop(); timings.mismapper_items = mismap_items_total;
	ex.sync();
	return mismap_items_total;
}

} // namespace arb
