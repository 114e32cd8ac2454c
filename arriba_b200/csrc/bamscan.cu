// bamscan.cu -- BAM record boundaries of a chunk of inflated BGZF payload, on the device.
//
// A BAM record can only be found from the one before it (SAMv1 4.2: block_size, then the record). The reference reads record after record
// (read_chimeric_alignments.cpp:611, sam_read1). Here, on the chunk in device memory (records.cu copies it up),
//   1. every 64 KB piece GUESSES its first record: the first offset from which three records in a row look sane (necessary conditions only);
//   2. every piece hops from its guess to the next piece's guess, counting records;
//   3. one thread VERIFIES: the chain of piece s must arrive exactly at the guess of piece s + 1; where it does not, that stretch is walked serially
//      (errors are therefore raised exactly where a one-thread walk would raise them);
//   4. every piece hops again from its verified start and writes the record offsets, in file order.
// What a record means is records_hd.h / records.cu.
#include <cstdlib>
#include "engine.h"

namespace arb {

struct bam_chunk { const u8* B; u64 end; i32 n_ref; };
ARB_HD u32 bam_rd32(const u8* p) { return (u32) p[0] | (u32) p[1] << 8 | (u32) p[2] << 16 | (u32) p[3] << 24; }
ARB_HD u32 bam_rd16(const u8* p) { return (u32) p[0] | (u32) p[1] << 8; }
ARB_HD bool bam_plausible(const bam_chunk& c, u64 q) { // a BAM record could start at q; a necessary condition only
	if (q + 36 > c.end) return false;
	const u8* B = c.B;
	const u32 bs = bam_rd32(B + q);
	if (bs < 33 || bs > (1u << 26) || q + 4 + bs > c.end) return false;
	const i32 tid = (i32) bam_rd32(B + q + 4), pos = (i32) bam_rd32(B + q + 8), mtid = (i32) bam_rd32(B + q + 24), mpos = (i32) bam_rd32(B + q + 28);
	const u32 lq = B[q + 12], nc = bam_rd16(B + q + 16); const i32 ls = (i32) bam_rd32(B + q + 20);
	if (tid < -1 || tid >= c.n_ref || mtid < -1 || mtid >= c.n_ref || pos < -1 || mpos < -1 || lq == 0 || ls < 0) return false;
	if (32ull + lq + 4ull * nc + ((u64) ls + 1) / 2 + (u64) ls > bs) return false;
	return B[q + 36 + lq - 1] == 0;
}
static const u64 BAM_NONE = ~(u64) 0;

struct bam_guess_fn {
	bam_chunk c; u64 first, piece_bytes; u32 pieces; u64* guess; // guess[pieces] = end
	ARB_HD void operator()(u32 s) const {
		if (s == pieces) { guess[s] = c.end; return; }
		if (s == 0) { guess[0] = first; return; }
		u64 q = first + piece_bytes * s; const u64 give_up = q + (4u << 20) < c.end ? q + (4u << 20) : c.end;
		for (; q < give_up; ++q) {
			if (!bam_plausible(c, q)) continue;
			const u64 q2 = q + 4 + bam_rd32(c.B + q); if (q2 < c.end && !bam_plausible(c, q2)) continue;
			const u64 q3 = q2 < c.end ? q2 + 4 + bam_rd32(c.B + q2) : c.end; if (q3 < c.end && q3 + 36 <= c.end && !bam_plausible(c, q3)) continue;
			break;
		}
		guess[s] = q < give_up ? q : c.end;
	}
};
// records that start in [q, limit); returns where the chain stands afterwards; bad: a block_size < 33 was met (the chain stops there)
ARB_HD u64 bam_hop(const bam_chunk& c, u64 q, u64 limit, u32& count, bool& bad) {
	while (q < limit && q + 4 <= c.end) {
		const u32 bs = bam_rd32(c.B + q);
		if (q + 4 + bs > c.end) break;
		if (bs < 33) { bad = true; break; }
		++count; q += 4 + (u64) bs;
	}
	return q;
}
struct bam_hop_fn {
	bam_chunk c; const u64* guess; u64* stop_at; u32* count; u8* bad;
	ARB_HD void operator()(u32 s) const { u32 n = 0; bool b = false; stop_at[s] = guess[s] < c.end ? bam_hop(c, guess[s], guess[s + 1], n, b) : c.end; count[s] = n; bad[s] = b ? 1 : 0; }
};
struct bam_stitch_fn { // one thread: follows the true chain over the pieces
	bam_chunk c; u64 first; u32 pieces; const u64* guess; const u64* stop_at; u32* count; const u8* bad; u64* start /* pieces + 1 */; u32* base /* pieces + 1 */; u64* result /* consumed, records, malformed */;
	ARB_HD void operator()(u32) const {
		u64 cur = first; u32 total = 0; bool malformed = false;
		for (u32 s = 0; s < pieces && !malformed; ++s) {
			start[s] = cur; base[s] = total;
			if (cur == guess[s] && guess[s] < c.end) { if (bad[s]) malformed = true; total += count[s]; cur = stop_at[s]; }
			else { u32 n = 0; bool b = false; cur = bam_hop(c, cur, guess[s + 1], n, b); count[s] = n; total += n; if (b) malformed = true; } // wrong or missing guess: this stretch is walked here
		}
		start[pieces] = cur; base[pieces] = total;
		result[0] = cur; result[1] = total; result[2] = malformed ? 1 : 0;
	}
};
struct bam_write_fn { // piece s: its records' offsets, file order
	bam_chunk c; const u64* start; const u32* base; const u32* count; u32* rec_off;
	ARB_HD void operator()(u32 s) const {
		u64 q = start[s]; u32 at = base[s];
		for (u32 k = 0; k < count[s]; ++k, ++at) { rec_off[at] = (u32) q; q += 4 + (u64) bam_rd32(c.B + q); }
	}
};

// the records of bytes [first, bytes) of `B` (device memory): rec_off gets their offsets in file order
void engine::bam_scan(const u8* B, u64 bytes, u64 first, i32 n_ref, dbuf<u32>& rec_off, u64* consumed, u32* n_records, u32* malformed) {
	if (bytes >= 0xFFFFFFF0ull) throw arb_error("failed to load alignments (chunk too large)");
	*consumed = first; *n_records = 0; *malformed = 0;
	if (first >= bytes) return;
	const u64 PIECE = getenv("ARB_BAM_SCAN_PIECE") ? (u64) std::max(1L, atol(getenv("ARB_BAM_SCAN_PIECE"))) : (u64) 64 << 10; // env: test hook (pieces smaller than a record)
	const u64 span = bytes - first;
	const u32 pieces = (u32) std::max<u64>(1, std::min<u64>(span / PIECE, 1u << 16));
	const u64 piece_bytes = span / pieces;
	bam_chunk c = {B, bytes, n_ref};
	dbuf<u64> guess((size_t) pieces + 1), stop_at(pieces), start((size_t) pieces + 1), result(3);
	dbuf<u32> count(pieces), base((size_t) pieces + 1); dbuf<u8> bad(pieces);
	bam_guess_fn gf = {c, first, piece_bytes, pieces, guess.ptr()};
	for_each(ex, pieces + 1, gf);
	bam_hop_fn hf = {c, guess.ptr(), stop_at.ptr(), count.ptr(), bad.ptr()};
	for_each(ex, pieces, hf);
	bam_stitch_fn sf = {c, first, pieces, guess.ptr(), stop_at.ptr(), count.ptr(), bad.ptr(), start.ptr(), base.ptr(), result.ptr()};
	for_each(ex, 1, sf);
	u64 res[3]; result.download(ex, res, 3);
	*consumed = res[0]; *malformed = (u32) res[2];
	const u32 R = (u32) res[1];
	*n_records = R;
	if (res[2] || R == 0) return;
	rec_off.ensure(R);
	bam_write_fn wf = {c, start.ptr(), base.ptr(), count.ptr(), rec_off.ptr()};
	for_each(ex, pieces, wf);
}

} // namespace arb
