// fill_gaps.cu -- driver of the gap filling of fusion transcript sequences (-I, see fill_gaps_hd.h).
#include <cstdlib>
#include "engine.h"
#include "fill_gaps_hd.h"

static_assert((int) arb::FJ_THREE == (int) ARB_FILL_THREE && (int) arb::FJ_FORWARD == (int) ARB_FILL_FORWARD && (int) arb::FJ_ITD == (int) ARB_FILL_ITD, "job flags of the C ABI");

namespace arb {

#ifdef ARB_DEVICE_BUILD
// one block per job; a block that runs out of jobs takes the next one of its stride
template <u32 THREADS> __global__ void __launch_bounds__(THREADS) k_fill_emit(fill_emit_fn f, u32 n_jobs) {
	for (u32 j = blockIdx.x; j < n_jobs; j += gridDim.x) f.run(j, threadIdx.x, THREADS);
}
#endif

static void run_emit(const exec_ctx& ex, int device, const fill_emit_fn& f, u32 n_jobs) {
	if (n_jobs == 0) return;
#ifdef ARB_DEVICE_BUILD
	enum { THREADS = 128 };
	int per_sm = 0, n_sm = 0;
	ARB_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_fill_emit<THREADS>, (int) THREADS, 0));
	ARB_CUDA_CHECK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, device));
	const u32 grid = std::min<u32>(n_jobs, (u32) std::max(1, per_sm) * (u32) n_sm * 4);
	k_fill_emit<THREADS><<<grid, THREADS, 0, ex.stream>>>(f, n_jobs);
	ARB_CUDA_CHECK(cudaGetLastError());
	++stats().kernels;
#else
	(void) device;
	hostsim_visit(n_jobs, [&](u32 j) { f.run(j, 0, 1); });
	++stats().kernels;
#endif
}

// the transcripts of the resident annotation: first and last exon, contig, and the exon chains (next / previous exon of the same transcript, -1: none)
void engine::set_fill_transcripts(u32 n, const i32* first_exon, const i32* last_exon, const u32* contig, const i32* exon_next, const i32* exon_prev) {
	has_fill_transcripts = false;
	if (!has_annotation) throw arb_error("arb_set_fill_transcripts: no annotation");
	const i32 E = (i32) annot.n_exons;
	for (u32 t = 0; t < n; ++t) {
		if (first_exon[t] < 0 || first_exon[t] >= E || last_exon[t] < 0 || last_exon[t] >= E) throw arb_error("arb_set_fill_transcripts: exon out of range in transcript " + std::to_string(t));
		if (contig[t] >= annot.n_contigs) throw arb_error("arb_set_fill_transcripts: contig out of range in transcript " + std::to_string(t));
	}
	for (i32 x = 0; x < E; ++x)
		if (exon_next[x] < -1 || exon_next[x] >= E || exon_prev[x] < -1 || exon_prev[x] >= E) throw arb_error("arb_set_fill_transcripts: exon chain out of range at exon " + std::to_string(x));
	// the kernels walk the chains to their ends: a chain must end (no cycle), in both directions
	for (int dir = 0; dir < 2; ++dir) {
		const i32* link = dir == 0 ? exon_next : exon_prev;
		std::vector<u8> state(E ? E : 1, 0); // 0 unseen, 1 on the current walk, 2 known to end
		for (i32 x = 0; x < E; ++x) {
			i32 y = x;
			while (y >= 0 && state[y] == 0) { state[y] = 1; y = link[y]; }
			if (y >= 0 && state[y] == 1) throw arb_error(std::string("arb_set_fill_transcripts: the chain of ") + (dir == 0 ? "next" : "previous") + " exons starting at exon " + std::to_string(x) + " has a cycle");
			for (y = x; y >= 0 && state[y] == 1; y = link[y]) state[y] = 2;
		}
	}
	stage_timer t(ex);
	fill_first.upload(ex, first_exon, n ? n : 1); fill_last.upload(ex, last_exon, n ? n : 1); fill_contig.upload(ex, contig, n ? n : 1);
	fill_next.upload(ex, exon_next, E ? E : 1); fill_prev.upload(ex, exon_prev, E ? E : 1);
	timings.fill_gaps_ms += t.stop();
	ex.sync();
	fill_transcript_count = n; has_fill_transcripts = true;
}

// n_jobs jobs on the n_rows sequences text[row_off[r] .. row_off[r + 1]) with their positions pos[pos_off[r] .. pos_off[r + 1]); returns the number of characters of all outputs, which stay here
// until arb_get_filled
u64 engine::fill_gaps(u32 n_rows, const char* text, const u32* row_off, const i32* pos, const u32* pos_off, u32 n_jobs, const u32* row, const u32* transcript, const u8* flags) {
	fill_off.assign((size_t) n_jobs + 1, 0); fill_chars_total = 0;
	if (!has_fill_transcripts) throw arb_error("arb_fill_gaps: arb_set_fill_transcripts must be called first");
	if (n_jobs == 0) return 0;
	if (row_off[0] != 0 || pos_off[0] != 0) throw arb_error("arb_fill_gaps: the first row must start at 0");
	for (u32 r = 0; r < n_rows; ++r) {
		if (row_off[r + 1] < row_off[r] || pos_off[r + 1] < pos_off[r]) throw arb_error("arb_fill_gaps: row offsets must not decrease");
		// fewer positions than characters: the reference would read positions beyond the end of the vector
		if (pos_off[r + 1] - pos_off[r] < row_off[r + 1] - row_off[r]) throw arb_error("arb_fill_gaps: row " + std::to_string(r) + " has fewer positions than characters");
	}
	if (row_off[n_rows] >= (1u << 30) || pos_off[n_rows] >= (1u << 30)) throw arb_error("arb_fill_gaps: too many characters in one call");
	for (u32 j = 0; j < n_jobs; ++j) {
		if (row[j] >= n_rows) throw arb_error("arb_fill_gaps: row out of range in job " + std::to_string(j));
		if (transcript[j] >= fill_transcript_count) throw arb_error("arb_fill_gaps: transcript out of range in job " + std::to_string(j));
		const u32 a = row_off[row[j]], b = row_off[row[j] + 1]; bool bar = false;
		for (u32 i = a; i < b && !bar; ++i) bar = text[i] == '|';
		if (!bar) throw arb_error("arb_fill_gaps: the sequence of job " + std::to_string(j) + " has no '|'");
	}
	stage_timer t(ex);
	const u32 chars_in = row_off[n_rows], pos_in = pos_off[n_rows];
	dbuf<char> d_text; dbuf<i32> d_pos; dbuf<u32> d_row_off, d_pos_off, d_row, d_tr; dbuf<u8> d_flags;
	d_text.upload(ex, text, chars_in ? chars_in : 1); d_pos.upload(ex, pos, pos_in ? pos_in : 1); d_row_off.upload(ex, row_off, (size_t) n_rows + 1); d_pos_off.upload(ex, pos_off, (size_t) n_rows + 1);
	d_row.upload(ex, row, n_jobs); d_tr.upload(ex, transcript, n_jobs); d_flags.upload(ex, flags, n_jobs);
	fill_transcripts tr = {fill_first.ptr(), fill_last.ptr(), fill_contig.ptr(), fill_transcript_count, fill_next.ptr(), fill_prev.ptr()};
	fill_jobs jobs = {d_text.ptr(), d_row_off.ptr(), d_pos.ptr(), d_pos_off.ptr(), d_row.ptr(), d_tr.ptr(), d_flags.ptr(), n_jobs};
	dbuf<fill_plan> plan(n_jobs); dbuf<u32> len((size_t) n_jobs + 1), bad(1);
	const u32 none = ~0u; bad.upload(ex, &none, 1);
	{ fill_plan_fn pf = {annot.view(), tr, jobs, plan.ptr(), len.ptr(), bad.ptr()}; for_each(ex, n_jobs, pf); }
	u32 first_bad = 0; bad.download(ex, &first_bad, 1);
	if (first_bad != ~0u) {
		ex.sync();
		throw arb_error("arb_fill_gaps: job " + std::to_string(first_bad) + " (row " + std::to_string(row[first_bad]) + "): an exon of transcript " + std::to_string(transcript[first_bad]) +
		                " lies outside its contig's sequence; the reference would read beyond the end of the contig");
	}
	exclusive_scan_u32(ex, len.ptr(), len.ptr(), n_jobs);
	std::vector<u32> off32((size_t) n_jobs + 1); len.download(ex, off32.data(), (size_t) n_jobs + 1);
	if (off32[n_jobs] >= (1u << 31)) throw arb_error("arb_fill_gaps: too many characters in one call");
	fill_chars.ensure((size_t) off32[n_jobs] + 1); fill_pos.ensure((size_t) off32[n_jobs] + 1);
	{ fill_emit_fn ef = {annot.view(), tr, jobs, plan.ptr(), len.ptr(), fill_chars.ptr(), fill_pos.ptr()}; run_emit(ex, device, ef, n_jobs); }
	timings.fill_gaps_ms += t.stop();
	ex.sync();
	for (u32 j = 0; j <= n_jobs; ++j) fill_off[j] = off32[j];
	fill_chars_total = off32[n_jobs];
	timings.fill_gaps_jobs += n_jobs; timings.fill_gaps_chars += fill_chars_total;
	return fill_chars_total;
}

void engine::get_filled(u32* off, char* chars, i32* pos) {
	for (size_t j = 0; j < fill_off.size(); ++j) off[j] = fill_off[j];
	if (fill_chars_total) { fill_chars.download(ex, chars, fill_chars_total); fill_pos.download(ex, pos, fill_chars_total); }
}

} // namespace arb
