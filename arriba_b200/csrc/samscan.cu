// samscan.cu -- SAM text input: every chunk of text is cut into lines and each line becomes a BAM record body in a staging buffer (functors: sam_hd.h);
// records_store (records.cu) then classifies and stores the staged records exactly as it does the records of a BAM chunk.
//   records_text_names : the @SQ names of the header (RNAME -> tid), sorted here on the host, kept on the device for the sample,
//   records_text_chunk : per chunk: the copy behind the unfinished line of the previous chunk, the line ends, the sizes of the staged records, their scan,
//                        the staged records, then records_store. Staged offsets accumulate over the chunks, so a record's staged position keeps file order:
//                        the record store orders the records of one key by it, and record errors are ordered by it.
#include <algorithm>
#include <cstring>
#include "engine.h"
#include "sam_hd.h"

namespace arb {

void engine::records_text_names(const char* names, const u64* name_off, u32 n) {
	if (!rec_open) throw arb_error("arb_records_text_names without arb_records_begin");
	if (n != rec_n_tid) throw arb_error("arb_records_text_names: " + std::to_string(n) + " names for " + std::to_string(rec_n_tid) + " references");
	std::vector<u32> order(n);
	for (u32 k = 0; k < n; ++k) order[k] = k;
	auto name = [&](u32 k) { return std::string(names + name_off[k], names + name_off[k + 1]); };
	std::stable_sort(order.begin(), order.end(), [&](u32 a, u32 b) { return name(a) < name(b); }); // a repeated name: the first reference that has it
	std::string blob; std::vector<u64> off(1, 0); std::vector<u32> tid;
	for (u32 k = 0; k < n; ++k) {
		if (k > 0 && name(order[k]) == name(order[k - 1])) continue;
		blob += name(order[k]); off.push_back(blob.size()); tid.push_back(order[k]);
	}
	sam_n_names = (u32) tid.size();
	sam_blob.upload(ex, (const u8*) blob.data(), blob.size()); sam_blob.ensure(1);
	sam_name_off.upload(ex, off.data(), off.size()); sam_name_tid.upload(ex, tid.data(), tid.size()); sam_name_tid.ensure(1);
	rec_text_staged = 0;
}

void engine::records_text_chunk(const u8* chunk, u64 bytes, u64 first, u64 chunk_pos, bool last, u64* n_records, u64* carry, u64* error) {
	if (!rec_open) throw arb_error("arb_records_text_chunk without arb_records_begin");
	stage_timer t_all(ex), t_copy(ex);
	const u64 start = rec_carry ? 0 : first;
	const u64 total = records_upload(chunk, bytes);
	// a staged record takes at most four times the bytes of its line, so offsets of a chunk below 1 GiB fit the 32-bit scans
	if (total >= (1ull << 30)) throw arb_error("failed to load alignments (SAM chunk too large)");
	timings.rec_chunk_copy_ms += t_copy.stop();
	stage_timer t_kernels(ex), t_parse(ex);
	// 1. line ends
	const u64 w0 = start / 16, n_words = (total + 15) / 16 - w0;
	const sam_text tx = {bam_buf.ptr(), start, total, w0};
	dbuf<u32> lf_base(n_words + 1);
	sam_lf_count_fn cf = {tx, lf_base.ptr()}; for_each(ex, (u32) n_words, cf);
	exclusive_scan_u32(ex, lf_base.ptr(), lf_base.ptr(), (u32) n_words);
	u32 n_lf = 0; lf_base.download(ex, &n_lf, 1, n_words);
	dbuf<u32> line_end((size_t) n_lf + 2);
	sam_lf_write_fn wf = {tx, lf_base.ptr(), line_end.ptr()}; for_each(ex, (u32) n_words, wf);
	u64 consumed = start;
	if (n_lf) { u32 e = 0; line_end.download(ex, &e, 1, n_lf - 1); consumed = (u64) e + 1; }
	u32 L = n_lf;
	if (last && consumed < total) { const u32 e = (u32) total; line_end.upload_at(ex, &e, 1, n_lf); ++L; consumed = total; } // the last line may end without an LF
	rec_carry_at = consumed; rec_carry = total - consumed; *carry = rec_carry;
	*n_records = L;
	if (L == 0) { rec_error.download(ex, error, 1); timings.rec_text_parse_ms += t_parse.stop(); timings.rec_chunk_kernels_ms += t_kernels.stop(); timings.bam_scan_ms += t_all.stop(); return; }
	// 2. the staged records: sizes, offsets, bodies
	const sam_lines lines = {bam_buf.ptr(), start, line_end.ptr(), n_lf};
	const sam_names nm = {sam_blob.ptr(), sam_name_off.ptr(), sam_name_tid.ptr(), sam_n_names};
	dbuf<u32> at((size_t) L + 1);
	sam_size_fn sf = {lines, nm, at.ptr()}; for_each(ex, L, sf);
	exclusive_scan_u32(ex, at.ptr(), at.ptr(), L);
	u32 staged = 0; at.download(ex, &staged, 1, L);
	sam_stage.ensure((size_t) staged + 64);
	sam_write_fn sw = {lines, nm, at.ptr(), sam_stage.ptr()}; for_each(ex, L, sw);
	timings.rec_text_parse_ms += t_parse.stop();
	// 3. the record loop's classification and store, as for a BAM chunk
	const u64 stage_pos = rec_pos_base + rec_text_staged;
	rec_text_staged += staged;
	records_store(sam_stage, stage_pos, staged, at.ptr(), L, chunk_pos + bytes, error);
	timings.rec_chunk_kernels_ms += t_kernels.stop();
	timings.bam_scan_ms += t_all.stop();
}

} // namespace arb
