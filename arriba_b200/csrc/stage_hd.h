// stage_hd.h -- the inflated chunk of a BGZF stream, assembled on the device from the chunk as it was read (records.cu, records_bgzf_stage; the CPU
// stand-in runs the same functor). The output is the unfinished record carried from the previous chunk, then the payload of every block at its dst.
//   stage_gather_fn : one thread per 16-byte word of the output. A word whose 16 bytes come from one stretch of input (the carry, or one block's payload:
//                     nearly all of them) loads the five aligned 32-bit words that cover it and funnel-shifts them into place; a word that straddles a
//                     block boundary (or the end of the chunk) is put together byte by byte. Every word is written with one 16-byte store.
#pragma once
#include "prims.h"
#include "../../include/arriba_b200.h"

namespace arb {

ARB_HD u32 stage_funnel_r(u32 lo, u32 hi, u32 shift) { // the 32 bits of (hi:lo) from bit `shift` on, shift < 32
#ifdef __CUDA_ARCH__
	return __funnelshift_r(lo, hi, shift);
#else
	return shift ? (lo >> shift) | (hi << (32 - shift)) : lo;
#endif
}
ARB_HD u32 stage_load32(const u8* p) { // p 4-byte aligned
#ifdef __CUDA_ARCH__
	return __ldg((const unsigned int*) p);
#else
	u32 v; memcpy(&v, p, 4); return v;
#endif
}

struct stage_gather_fn {
	const u8* carry; u64 n_carry;                                   // the unfinished record of the previous chunk
	const u8* raw; const arb_bgzf_block* blocks; u32 n_blocks;     // blocks[0].dst = 0, each block's dst = the end of the one before
	u64 total;                                                      // n_carry + the payload bytes
	u8* out;                                                        // 16-byte aligned, room for whole words
	// where output byte p (< total) comes from, and how many bytes of that stretch are left from there on
	ARB_HD const u8* locate(u64 p, u64& left) const {
		if (p < n_carry) { left = n_carry - p; return carry + p; }
		const u64 q = p - n_carry;
		u32 lo = 0, hi = n_blocks; // the last block that starts at or before q: the one of equal starts that is not empty
		while (hi - lo > 1) { const u32 mid = (lo + hi) / 2; if (blocks[mid].dst <= q) lo = mid; else hi = mid; }
		left = blocks[lo].dst + blocks[lo].bytes - q;
		return raw + blocks[lo].src + (q - blocks[lo].dst);
	}
	ARB_HD void operator()(u32 k) const {
		const u64 p0 = (u64) k * 16, n = total - p0 < 16 ? total - p0 : 16;
		u64 left = 0;
		const u8* s = locate(p0, left);
		u32 w[4];
		if (n == 16 && left >= 16) {
			const u8* a = (const u8*) ((uintptr_t) s & ~(uintptr_t) 3); // the buffers are aligned and have slack behind their end: the fifth word may be read
			const u32 shift = (u32) ((uintptr_t) s & 3) * 8;
			const u32 v0 = stage_load32(a), v1 = stage_load32(a + 4), v2 = stage_load32(a + 8), v3 = stage_load32(a + 12), v4 = stage_load32(a + 16);
			w[0] = stage_funnel_r(v0, v1, shift); w[1] = stage_funnel_r(v1, v2, shift); w[2] = stage_funnel_r(v2, v3, shift); w[3] = stage_funnel_r(v3, v4, shift);
		} else {
			w[0] = w[1] = w[2] = w[3] = 0;
			for (u32 i = 0; i < (u32) n; ++i) {
				if (left == 0) s = locate(p0 + i, left);
				w[i >> 2] |= (u32) *s++ << (8 * (i & 3));
				--left;
			}
		}
#ifdef __CUDA_ARCH__
		*(uint4*) (out + p0) = make_uint4(w[0], w[1], w[2], w[3]);
#else
		memcpy(out + p0, w, 16);
#endif
	}
};

} // namespace arb
