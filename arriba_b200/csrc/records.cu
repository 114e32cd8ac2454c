// records.cu -- the reference's record loop on the device (functors: records_hd.h).
//   records_begin  : the BAM header's contig map, the contig flags, the coverage windows' layout,
//   records_source : a separate chimeric file (-c) ahead of the main file: which file the following chunks belong to, and its header's contig map,
//   records_bgzf_stage : stream input: the raw BGZF blocks of a chunk go up as they were read, and the inflated chunk is assembled on the device
//                    (stage_hd.h) where records_upload would have put it,
//   records_chunk  : per chunk of inflated payload: copy it up behind the unfinished record of the previous chunk, find the records (bamscan.cu), classify
//                    them and append the kept ones to the record store, which lives across chunks (mates and supplementaries of one key may sit anywhere
//                    in the file),
//   records_finish : sort the store by key hash (two stable 32-bit passes: file order inside a hash), replay every run of equal hashes (count and log
//                    the searches' outcomes, scan, write from the log) into the fragment pools that fragment_table_build reads, saturate the coverage
//                    counts into packed 16-bit windows, and bring the windows and the counters back.
#include <cstdlib>
#include <cstdio>
#include <type_traits>
#include "engine.h"
#include "records_hd.h"
#include "fragtable_hd.h"
#include "stage_hd.h"

namespace arb {

// b grows to hold `want` items; its first `used` items are kept
template <class T> static void grow_keep(const exec_ctx& ex, dbuf<T>& b, size_t used, size_t want) {
	if (want <= b.size()) return;
	dbuf<T> bigger(want);
	if (used) {
#ifdef ARB_DEVICE_BUILD
		ARB_CUDA_CHECK(cudaMemcpyAsync(bigger.ptr(), b.ptr(), used * sizeof(T), cudaMemcpyDeviceToDevice, ex.stream));
#else
		(void) ex; memcpy(bigger.ptr(), b.ptr(), used * sizeof(T));
#endif
	}
	b.swap(bigger);
}

// n items from the device to the host, queued on the stream (the caller synchronises)
template <class T> static void copy_to_host(const exec_ctx& ex, T* host, const T* dev, size_t n) {
#ifdef ARB_DEVICE_BUILD
	ARB_CUDA_CHECK(cudaMemcpyAsync(host, dev, n * sizeof(T), cudaMemcpyDeviceToHost, ex.stream));
#else
	(void) ex; memcpy(host, dev, n * sizeof(T));
#endif
}

void engine::records_begin(const u16* tid_to_contig, u32 n_tid, const u8* interesting, const u8* viral, const u64* n_windows, u32 n_contigs,
                           u32 max_itd_length, bool external_duplicate_marking, u64 expected_bytes) {
	ex.sync(); // kernels of the previous sample may still read the buffers that are about to be overwritten
	if (n_contigs != annot.n_contigs) throw arb_error("arb_records_begin: the contig table on the device has " + std::to_string(annot.n_contigs) + " contigs, the BAM header " + std::to_string(n_contigs));
	rec_n_tid = n_tid; rec_n_contigs = n_contigs; rec_max_itd = max_itd_length; rec_external_dup = external_duplicate_marking; rec_expected_bytes = expected_bytes;
	rec_tid.upload(ex, tid_to_contig, n_tid ? n_tid : 0); rec_tid.ensure(1);
	rec_interesting.upload(ex, interesting, n_contigs); rec_viral.upload(ex, viral, n_contigs); rec_interesting.ensure(1); rec_viral.ensure(1);
	std::vector<u64> off((size_t) n_contigs + 1, 0); std::vector<u32> n(n_contigs);
	for (u32 c = 0; c < n_contigs; ++c) { if (n_windows[c] > 0xFFFFFFFFull) throw arb_error("arb_records_begin: contig too long"); n[c] = (u32) n_windows[c]; off[c + 1] = off[c] + n[c]; }
	rec_cov_windows = off[n_contigs];
	rec_cov_off.upload(ex, off.data(), off.size()); rec_cov_n.upload(ex, n.data(), n_contigs); rec_cov_n.ensure(1);
	rec_cov_words.ensure(rec_cov_windows / 2 + 1); rec_cov_words.zero(ex, rec_cov_windows / 2 + 1);
	rec_cov_starts.ensure(rec_cov_windows + 1); rec_cov_starts.zero(ex, rec_cov_windows + 1);
	rec_cov_ends.ensure(rec_cov_windows + 1); rec_cov_ends.zero(ex, rec_cov_windows + 1);
	rec_counters.ensure((size_t) REC_CTR_VIRAL + n_contigs); rec_counters.zero(ex, (size_t) REC_CTR_VIRAL + n_contigs);
	const u64 none = ~(u64) 0; rec_error.upload(ex, &none, 1);
	rec_n = 0; rec_arena_used = 0; rec_carry = 0; rec_carry_at = 0; rec_error_record.clear();
	rec_src_chimeric = rec_has_chimeric = false; rec_pos_base = rec_pos_end = rec_chimeric_end = 0;
	// test hook: keys share their hash far more often than 64-bit hashes ever do, so that runs of one hash hold many keys
	const char* bits = getenv("ARB_KEY_HASH_BITS");
	rec_hash_mask = bits && atoi(bits) > 0 && atoi(bits) < 64 ? ((u64) 1 << atoi(bits)) - 1 : ~(u64) 0;
	timings.bam_scan_ms = 0; timings.h2d_ms = 0; timings.h2d_bytes = 0;
	timings.rec_chunk_copy_ms = timings.rec_chunk_kernels_ms = timings.rec_sort_ms = timings.rec_count_ms = timings.rec_scan_ms = timings.rec_write_ms = timings.rec_download_ms = timings.rec_text_parse_ms = 0;
	timings.rec_unwrap_ms = 0; timings.rec_store_grows = 0; timings.rec_store_bytes = 0; timings.rec_h2d_bytes = 0;
	rec_stage_pending = false; rec_staged = 0;
	rec_open = true;
}

// The records of the chunks that follow belong to the -c file (chimeric_file) or to the main file, whose header maps its references by tid_to_contig.
// Every file's positions start behind those of the files before it (first_position): the store then orders a key's records by file, then by position,
// and the earliest record error is the one the reference meets first.
void engine::records_source(bool chimeric_file, const u16* tid_to_contig, u32 n_tid, u64* first_position) {
	if (!rec_open) throw arb_error("arb_records_source without arb_records_begin");
	if (rec_carry) throw arb_error("arb_records_source: the previous file ended inside a record");
	if (rec_has_chimeric && !rec_src_chimeric && chimeric_file) throw arb_error("arb_records_source: the -c file must come before the main file");
	if (!chimeric_file && rec_src_chimeric) rec_chimeric_end = rec_pos_end;
	rec_has_chimeric = rec_has_chimeric || chimeric_file; rec_src_chimeric = chimeric_file;
	rec_pos_base = rec_pos_end; *first_position = rec_pos_base;
	rec_n_tid = n_tid; rec_tid.upload(ex, tid_to_contig, n_tid); rec_tid.ensure(1);
	rec_text_staged = 0; rec_carry_at = 0; rec_stage_pending = false;
}

// the chunk goes to the device behind the unfinished record (or line) at the end of the previous one; returns the bytes of bam_buf now in use. chunk ==
// NULL: the chunk records_bgzf_stage put there (without one, NULL with 0 bytes stays an empty chunk).
u64 engine::records_upload(const u8* chunk, u64 bytes) {
	if (!chunk && (rec_stage_pending || bytes != 0)) {
		if (!rec_stage_pending || bytes != rec_staged) throw arb_error("a NULL chunk takes the chunk of arb_records_bgzf_stage, and as many bytes as it staged");
		rec_stage_pending = false;
		return rec_carry + bytes;
	}
	if (rec_stage_pending) throw arb_error("the chunk of arb_records_bgzf_stage has not been read (pass chunk = NULL)");
	const u64 total = rec_carry + bytes;
	if (total >= 0xFFFFFFF0ull) throw arb_error("failed to load alignments (chunk too large)");
	bam_buf_next.ensure(total + 64);
	if (rec_carry) {
#ifdef ARB_DEVICE_BUILD
		ARB_CUDA_CHECK(cudaMemcpyAsync(bam_buf_next.ptr(), bam_buf.ptr() + rec_carry_at, rec_carry, cudaMemcpyDeviceToDevice, ex.stream));
#else
		memcpy(bam_buf_next.ptr(), bam_buf.ptr() + rec_carry_at, rec_carry);
#endif
	}
	bam_buf_next.upload_at(ex, chunk, bytes, rec_carry);
	timings.rec_h2d_bytes += bytes;
	bam_buf.swap(bam_buf_next);
	return total;
}

void engine::records_bgzf_stage(const u8* raw, u64 raw_bytes, const arb_bgzf_block* blocks, u32 n_blocks) {
	if (!rec_open) throw arb_error("arb_records_bgzf_stage without arb_records_begin");
	if (rec_stage_pending) throw arb_error("arb_records_bgzf_stage: the chunk staged before has not been read");
	if (raw_bytes && !raw) throw arb_error("arb_records_bgzf_stage: no raw bytes");
	u64 out = 0;
	for (u32 k = 0; k < n_blocks; ++k) {
		if (blocks[k].dst != out || blocks[k].src > raw_bytes || blocks[k].bytes > raw_bytes - blocks[k].src) throw arb_error("arb_records_bgzf_stage: block " + std::to_string(k) + " is out of place or outside the raw bytes");
		out += blocks[k].bytes;
	}
	const u64 total = rec_carry + out;
	if (total >= 0xFFFFFFF0ull) throw arb_error("failed to load alignments (chunk too large)");
	stage_timer t_all(ex), t_copy(ex);
	rec_raw.ensure(raw_bytes); rec_raw.upload_at(ex, raw, raw_bytes, 0);
	rec_stage_blocks.upload(ex, blocks, n_blocks); rec_stage_blocks.ensure(1);
	timings.rec_h2d_bytes += raw_bytes + (u64) n_blocks * sizeof(arb_bgzf_block);
	timings.rec_chunk_copy_ms += t_copy.stop();
	stage_timer t_unwrap(ex);
	bam_buf_next.ensure(total + 64);
	const stage_gather_fn g = {bam_buf.ptr() + rec_carry_at, rec_carry, rec_raw.ptr(), rec_stage_blocks.ptr(), n_blocks, total, bam_buf_next.ptr()};
	for_each(ex, (u32) ((total + 15) / 16), g);
	bam_buf.swap(bam_buf_next);
	rec_carry_at = 0; rec_staged = out; rec_stage_pending = true;
	const float ms = t_unwrap.stop();
	timings.rec_unwrap_ms += ms; timings.rec_chunk_kernels_ms += ms;
	timings.bam_scan_ms += t_all.stop();
}

void engine::records_chunk(const u8* chunk, u64 bytes, u64 first, u64 chunk_pos, u64* n_records, u64* carry, u32* malformed, u64* error) {
	if (!rec_open) throw arb_error("arb_records_chunk without arb_records_begin");
	stage_timer t_all(ex), t_copy(ex);
	const u64 first_record = rec_carry ? 0 : first;
	const u64 total = records_upload(chunk, bytes);
	timings.rec_chunk_copy_ms += t_copy.stop();
	stage_timer t_kernels(ex);
	const u64 buf_pos = rec_pos_base + chunk_pos - (total - bytes);
	u64 consumed = 0; u32 R = 0;
	dbuf<u32> rec_off;
	bam_scan(bam_buf.ptr(), total, first_record, (i32) rec_n_tid, rec_off, &consumed, &R, malformed);
	*n_records = R;
	rec_carry_at = consumed; rec_carry = total - consumed; *carry = rec_carry;
	if (*malformed || R == 0) { rec_error.download(ex, error, 1); timings.rec_chunk_kernels_ms += t_kernels.stop(); timings.bam_scan_ms += t_all.stop(); return; }
	records_store(bam_buf, buf_pos, total, rec_off.ptr(), R, chunk_pos + bytes, error);
	timings.rec_chunk_kernels_ms += t_kernels.stop();
	timings.bam_scan_ms += t_all.stop();
}

// the R records of B (block_size at B[rec_off[i]]; B[0] is at position buf_pos of the record stream, `total` bytes of B in use): classified, and the kept
// ones appended to the store. seen = the bytes of the input read so far (with expected_bytes it sizes the store after the first chunk).
void engine::records_store(const dbuf<u8>& B, u64 buf_pos, u64 total, const u32* rec_off, u32 R, u64 seen, u64* error) {
	// classify, then append the kept records to the store
	dbuf<u32> bytes_of((size_t) R + 1), kept((size_t) R + 1); dbuf<u64> hash(R); dbuf<i64> hit(R); dbuf<u8> sa(R);
	const rec_chunk_view cv = {B.ptr(), rec_off, buf_pos, rec_tid.ptr(), (i32) rec_n_tid, annot.contig_len.ptr(), rec_interesting.ptr()};
	rec_pos_end = std::max(rec_pos_end, buf_pos + total);
	if (rec_src_chimeric) {
		rec_extract_t<true> xf = {cv, rec_hash_mask, bytes_of.ptr(), kept.ptr(), hash.ptr(), hit.ptr(), sa.ptr(), rec_counters.ptr(), rec_error.ptr()};
		for_each(ex, R, xf);
	} else {
		rec_extract_fn xf = {cv, rec_hash_mask, bytes_of.ptr(), kept.ptr(), hash.ptr(), hit.ptr(), sa.ptr(), rec_counters.ptr(), rec_error.ptr()};
		for_each(ex, R, xf);
	}
	exclusive_scan_u32(ex, bytes_of.ptr(), bytes_of.ptr(), R); exclusive_scan_u32(ex, kept.ptr(), kept.ptr(), R);
	u32 add_bytes = 0, add_items = 0;
	bytes_of.download(ex, &add_bytes, 1, R); kept.download(ex, &add_items, 1, R);
	const u64 need_bytes = rec_arena_used + add_bytes, need_items = rec_n + add_items;
	if (need_bytes > rec_arena.size() || need_items > rec_at.size()) {
		// sized once from the share of the file seen so far (the first chunk), grown by a quarter where that falls short
		double factor = 1.25;
		if (rec_n == 0 && seen < rec_expected_bytes) factor = 1.03 * (double) rec_expected_bytes / (double) seen;
		const u64 want_bytes = (u64) ((double) need_bytes * factor) + 4096, want_items = (u64) ((double) need_items * factor) + 1024;
		if (want_items >= 0xFFFFFFF0ull) throw arb_error("more than 2^32 BAM records");
		try {
			grow_keep(ex, rec_arena, rec_arena_used, want_bytes); grow_keep(ex, rec_at, rec_n, want_items); grow_keep(ex, rec_pos, rec_n, want_items);
			grow_keep(ex, rec_hash_lo, rec_n, want_items); grow_keep(ex, rec_hash_hi, rec_n, want_items); grow_keep(ex, rec_hit, rec_n, want_items); grow_keep(ex, rec_sa, rec_n, want_items);
			++timings.rec_store_grows;
			timings.rec_store_bytes = std::max<u64>(timings.rec_store_bytes, (u64) rec_arena.size() + (u64) rec_at.size() * (8 + 8 + 4 + 4 + 8 + 1));
		} catch (const arb_error& e) {
			char m[256];
			snprintf(m, sizeof(m), "the BAM record store does not fit in device memory: %llu records in %.2f GB (%s)", (unsigned long long) want_items,
			         ((double) want_bytes + (double) want_items * (8 + 8 + 4 + 4 + 8 + 1)) / 1e9, e.what());
			throw arb_error(m);
		}
	}
	rec_store_fn sf = {cv, bytes_of.ptr(), kept.ptr(), hash.ptr(), hit.ptr(), sa.ptr(), rec_n, rec_arena_used, rec_arena.ptr(),
	                   rec_at.ptr(), rec_pos.ptr(), rec_hash_lo.ptr(), rec_hash_hi.ptr(), rec_hit.ptr(), rec_sa.ptr()};
	for_each(ex, R, sf);
	rec_n = need_items; rec_arena_used = need_bytes;
	rec_error.download(ex, error, 1);
	// the text of a record error names the record: keep a copy while the chunk is still on the device
	if (*error != ~(u64) 0 && rec_error_record.empty()) {
		const u64 at = *error >> 3;
		if (at >= buf_pos && at + 4 <= buf_pos + total) {
			u8 bs[4]; B.download(ex, bs, 4, at - buf_pos);
			const u64 n = std::min<u64>(rec_rd32(bs), buf_pos + total - (at + 4));
			rec_error_record.resize(n); B.download(ex, rec_error_record.data(), n, at - buf_pos + 4);
		}
	}
}

struct rec_seg_flag_fn { const u32* order; const u32* lo; const u32* hi; u32* flag; ARB_HD void operator()(u32 k) const { flag[k] = k == 0 || lo[order[k]] != lo[order[k - 1]] || hi[order[k]] != hi[order[k - 1]]; } };
// at: exclusive scan of the flags (n + 1 entries); item k starts segment at[k] when its flag is set
struct rec_seg_begin_fn { const u32* at; u32 n; u32* begin; ARB_HD void operator()(u32 k) const { if (k == n) begin[at[n]] = n; else if (at[k + 1] != at[k]) begin[at[k]] = k; } };
struct rec_big_list_fn { const u8* big; u32* list; u32* n; ARB_HD void operator()(u32 s) const { if (big[s]) list[append_slot(n)] = s; } };
struct rec_gather_fn { const u32* order; const u32* hi; u32* key; ARB_HD void operator()(u32 k) const { key[k] = hi[order[k]]; } };
// item q * S + s: did row q's exclusive scan step down (wrap past 2^32) between segments s and s + 1?
struct rec_wrap_fn { const u32* scan; u32 stride, S; u32* wraps; ARB_HD void operator()(u32 i) const { const u32 q = i / S, s = i % S; if (scan[q * stride + s + 1] < scan[q * stride + s]) atomic_add_u32(&wraps[q], 1); } };
struct rec_iota_fn { u32* v; ARB_HD void operator()(u32 k) const { v[k] = k; } };

void engine::records_finish(u16* const* coverage, u8* const* starts, u8* const* ends, u64* counters, u64* error) {
	if (!rec_open) throw arb_error("arb_records_finish without arb_records_begin");
	rec_open = false;
	stage_timer t_all(ex), t_sort(ex);
	const u32 n = (u32) rec_n;
	// 1. key order: low word, then high word, both stable (file order inside a key hash)
	dbuf<u32> order((size_t) n + 1), key((size_t) n + 1), tk((size_t) n + 1), tv((size_t) n + 1);
	rec_iota_fn io = {order.ptr()}; for_each(ex, n, io);
	rec_gather_fn g0 = {order.ptr(), rec_hash_lo.ptr(), key.ptr()}; for_each(ex, n, g0);
	radix_sort_pairs_u32(ex, key.ptr(), order.ptr(), tk.ptr(), tv.ptr(), n, 32);
	rec_gather_fn g1 = {order.ptr(), rec_hash_hi.ptr(), key.ptr()}; for_each(ex, n, g1);
	radix_sort_pairs_u32(ex, key.ptr(), order.ptr(), tk.ptr(), tv.ptr(), n, 32);
	// 2. segments: runs of one hash
	dbuf<u32> seg_at((size_t) n + 1);
	rec_seg_flag_fn ff = {order.ptr(), rec_hash_lo.ptr(), rec_hash_hi.ptr(), seg_at.ptr()}; for_each(ex, n, ff);
	exclusive_scan_u32(ex, seg_at.ptr(), seg_at.ptr(), n);
	u32 S = 0; seg_at.download(ex, &S, 1, n);
	dbuf<u32> seg_begin((size_t) S + 1);
	rec_seg_begin_fn bf = {seg_at.ptr(), n, seg_begin.ptr()}; for_each(ex, n + 1, bf);
	timings.rec_sort_ms = t_sort.stop();
	// 3. replay, with the -c file's steps compiled in only when there is one
	dbuf<u64> cov_counts(rec_cov_windows + 2);
	dbuf<u32> chimeric_counts(2); chimeric_counts.zero(ex, 2); // the -c fragments the first malformed pass rejects / keeps (counting pass)
	auto replay = [&](auto chimeric_file) -> bool { // false: the counting pass found a fatal error
		constexpr bool C = decltype(chimeric_file)::value;
		stage_timer t_count(ex);
		// count (sets of up to 32 gene ids, the few segments that need more: 1024), scan, write
		dbuf<u8> big((size_t) S + 1); big.zero(ex, (size_t) S + 1);
		const u32 stride = (S + 4) & ~3u; // S + 1 entries per row, rows 16-byte aligned (the scan loads four items at a time)
		dbuf<u32> tally((size_t) RS_N * stride), big_list((size_t) S + 1), n_big(1);
		dbuf<u64> search_log((size_t) n + 1); // what the counting pass's searches decided, per store position (written before it is read: no zeroing)
		if (rec_src_chimeric) rec_chimeric_end = rec_pos_end; // the -c file was the last one (no main file followed)
		const rec_store_view sv = {rec_arena.ptr(), rec_at.ptr(), rec_pos.ptr(), rec_hit.ptr(), rec_sa.ptr(), order.ptr(), rec_chimeric_end};
		rec_cov_view cov = {NULL, rec_cov_starts.ptr(), rec_cov_ends.ptr(), rec_cov_off.ptr(), rec_cov_n.ptr(), rec_n_contigs}; // counts: writing pass only
		const rec_params prm = {rec_max_itd, (u8) (rec_external_dup ? 1 : 0), rec_viral.ptr()};
		const annot_view an = annot.view();
		rec_replay_fn<32, C> small = {sv, seg_begin.ptr(), NULL, big.ptr(), an, prm, cov, tally.ptr(), tally.ptr(), stride, NULL, NULL, NULL, NULL, NULL, search_log.ptr(), rec_counters.ptr(), rec_error.ptr(), false, chimeric_counts.ptr()};
		for_each(ex, S, small);
		n_big.zero(ex, 1);
		rec_big_list_fn lf = {big.ptr(), big_list.ptr(), n_big.ptr()}; for_each(ex, S, lf);
		u32 B = 0; n_big.download(ex, &B, 1);
		rec_replay_fn<1024, C> large = {sv, seg_begin.ptr(), big_list.ptr(), big.ptr(), an, prm, cov, tally.ptr(), tally.ptr(), stride, NULL, NULL, NULL, NULL, NULL, search_log.ptr(), rec_counters.ptr(), rec_error.ptr(), false, chimeric_counts.ptr()};
		for_each(ex, B, large);
		rec_error.download(ex, error, 1);
		timings.rec_count_ms = t_count.stop();
		if (C) { u32 c[2]; chimeric_counts.download(ex, c, 2); ft_chimeric[0] = c[0]; ft_chimeric[1] = c[1]; }
		else ft_chimeric[0] = ft_chimeric[1] = 0;
		if (*error != ~(u64) 0) return false;
		stage_timer t_scan(ex);
		// The scans are 32-bit. A prefix sum that passes 2^32 wraps, and every wrap shows as a step down between neighbours (each tally is < 2^32): counted,
		// the true totals follow, and a sample whose pools the table cannot address stops here, before anything is written.
		for (u32 q = 0; q < RS_N; ++q) exclusive_scan_u32(ex, tally.ptr() + (size_t) q * stride, tally.ptr() + (size_t) q * stride, S);
		dbuf<u32> wraps(RS_N); wraps.zero(ex, RS_N);
		rec_wrap_fn wf = {tally.ptr(), stride, S, wraps.ptr()}; for_each(ex, RS_N * S, wf);
		u32 tot[RS_N], n_wraps[RS_N];
		for (u32 q = 0; q < RS_N; ++q) tally.download(ex, tot + q, 1, (size_t) q * stride + S);
		wraps.download(ex, n_wraps, RS_N);
		timings.rec_scan_ms = t_scan.stop();
		{
			u64 total[RS_N], limit[RS_N] = {(u64) 1 << 30 /* fragment ids */, (u64) 1 << 31 /* i32 alignment links */, (u64) 1 << 32, (u64) 1 << 32, (u64) 1 << 32};
			const char* hook = getenv("ARB_REPLAY_POOL_LIMIT"); // test hook: the limits lowered, so that a small sample reaches them
			bool over = false;
			for (u32 q = 0; q < RS_N; ++q) {
				total[q] = (u64) n_wraps[q] << 32 | tot[q];
				if (hook && atoll(hook) > 0) limit[q] = std::min<u64>(limit[q], (u64) atoll(hook));
				over = over || total[q] >= limit[q];
			}
			if (over) {
				char m[400];
				snprintf(m, sizeof(m), "the sample is too large for one fragment table: %llu fragments (limit %llu), %llu alignments (limit %llu), %llu name bytes (limit %llu), "
				         "%llu CIGAR operations (limit %llu), %llu sequence bytes (limit %llu)",
				         (unsigned long long) total[RS_FRAGS], (unsigned long long) limit[RS_FRAGS], (unsigned long long) total[RS_ALNS], (unsigned long long) limit[RS_ALNS],
				         (unsigned long long) total[RS_NAMES], (unsigned long long) limit[RS_NAMES], (unsigned long long) total[RS_CIGARS], (unsigned long long) limit[RS_CIGARS],
				         (unsigned long long) total[RS_UNITS] * 16, (unsigned long long) limit[RS_UNITS] * 16);
				throw arb_error(m);
			}
		}
		stage_timer t_write(ex);
		pool_frags.ensure(tot[RS_FRAGS]); pool_alns.ensure(tot[RS_ALNS]); pool_names.ensure(tot[RS_NAMES]); pool_cigars.ensure(tot[RS_CIGARS]); pool_seqs.ensure((size_t) tot[RS_UNITS] * 16);
		cov_counts.zero(ex, rec_cov_windows + 2);
		small.write = large.write = true;
		small.cov.counts = large.cov.counts = cov_counts.ptr();
		small.frags = large.frags = pool_frags.ptr(); small.alns = large.alns = pool_alns.ptr(); small.names = large.names = pool_names.ptr();
		small.cigars = large.cigars = pool_cigars.ptr(); small.seqs = large.seqs = pool_seqs.ptr();
		for_each(ex, S, small);
		for_each(ex, B, large);
		const u64 base[2 * FT_POOLS] = {0, tot[RS_FRAGS], 0, tot[RS_ALNS], 0, tot[RS_NAMES], 0, tot[RS_CIGARS], 0, (u64) tot[RS_UNITS] * 16};
		pool_base.upload(ex, base, 2 * FT_POOLS);
		pool_workers = 1;
		timings.rec_write_ms = t_write.stop();
		return true;
	};
	if (!(rec_has_chimeric ? replay(std::true_type()) : replay(std::false_type()))) {
		// the counters so far: with a -c file, REC_CTR_CHIMERIC tells whether it had chimeric reads (its error comes before the main file's)
		rec_counters.download(ex, counters, (size_t) REC_CTR_VIRAL + rec_n_contigs);
		timings.bam_scan_ms += t_all.stop(); return;
	}
	stage_timer t_download(ex);
	// 4. the by-products: the counts saturated into packed 16-bit windows, then every contig's windows straight into the caller's arrays (the
	// 16-bit counters lie in their 32-bit words in little-endian order, i.e. as a plain u16 array)
	rec_cov_pack_fn pk = {cov_counts.ptr(), rec_cov_words.ptr()}; for_each(ex, (u32) (rec_cov_windows / 2 + 1), pk);
	std::vector<u64> off((size_t) rec_n_contigs + 1); rec_cov_off.download(ex, off.data(), off.size());
	const u16* windows = (const u16*) rec_cov_words.ptr();
	for (u32 c = 0; c < rec_n_contigs; ++c) {
		const u64 w = off[c + 1] - off[c];
		if (!w) continue;
		copy_to_host(ex, coverage[c], windows + off[c], w); copy_to_host(ex, starts[c], rec_cov_starts.ptr() + off[c], w); copy_to_host(ex, ends[c], rec_cov_ends.ptr() + off[c], w);
	}
	rec_counters.download(ex, counters, (size_t) REC_CTR_VIRAL + rec_n_contigs); // synchronises: the copies above are done
	rec_error.download(ex, error, 1);
	timings.rec_download_ms = t_download.stop();
	// the store is not needed any more: its memory goes to the fragment table
	rec_arena.release(); rec_at.release(); rec_pos.release(); rec_hash_lo.release(); rec_hash_hi.release(); rec_hit.release(); rec_sa.release(); bam_buf_next.release();
	timings.bam_scan_ms += t_all.stop();
}

} // namespace arb
