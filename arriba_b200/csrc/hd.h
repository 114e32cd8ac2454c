// hd.h -- host/device portability layer for arriba-b200.
//
// Every per-fragment / per-candidate rule of the hot path is written once as an ARB_HD functor.
// The product compiles them with nvcc for sm_90a and launches them as CUDA kernels (prims.cuh).
// The SAME functors can be compiled by g++ with -DARB_HOSTSIM into a separate, test-only library
// (tests/hostsim) so that rule logic can be checked against the oracle on machines without a GPU;
// the product library never contains or falls back to that build.
#pragma once
#include <stdint.h>
#include <stddef.h>

#if defined(__CUDACC__) && !defined(ARB_HOSTSIM)
#define ARB_HD __host__ __device__ __forceinline__
#define ARB_DEVICE_BUILD 1
#else
#define ARB_HD inline
#endif

namespace arb {

typedef uint8_t u8;
typedef uint16_t u16;
typedef uint32_t u32;
typedef uint64_t u64;
typedef int16_t i16;
typedef int32_t i32;
typedef int64_t i64;

// filter identifiers: numbering of the reference's registry (common.hpp:30-67), order is part of the file format
enum filter_id {
	F_none = 0, F_duplicates = 1, F_inconsistently_clipped = 2, F_homopolymer = 3, F_read_through = 4, F_same_gene = 5,
	F_small_insert_size = 6, F_long_gap = 7, F_hairpin = 8, F_multimappers = 9, F_mismatches = 10, F_mismappers = 11,
	F_relative_support = 12, F_intronic = 13, F_non_coding_neighbors = 14, F_intragenic_exonic = 15,
	F_internal_tandem_duplication = 16, F_min_support = 17, F_known_fusions = 18, F_spliced = 19, F_blacklist = 20,
	F_end_to_end = 21, F_in_vitro = 22, F_merge_adjacent = 23, F_select_best = 24, F_marginal_read_through = 25,
	F_short_anchor = 26, F_no_coverage = 27, F_many_spliced = 28, F_no_genomic_support = 29, F_uninteresting_contigs = 30,
	F_viral_contigs = 31, F_top_expressed_viral_contigs = 32, F_low_coverage_viral_contigs = 33, F_genomic_support = 34,
	F_isoforms = 35, F_low_entropy = 36, F_homologs = 37, F_COUNT = 38
};

// BAM CIGAR encoding (SAMv1 4.2): low 4 bits op, high 28 bits length
enum { C_M = 0, C_I = 1, C_D = 2, C_N = 3, C_S = 4, C_H = 5, C_P = 6, C_EQ = 7, C_X = 8 };
ARB_HD u32 cig_op(u32 c) { return c & 0xf; }
ARB_HD u32 cig_len(u32 c) { return c >> 4; }
ARB_HD bool cig_is_clip(u32 c) { u32 o = c & 0xf; return o == C_S || o == C_H; }
ARB_HD bool cig_is_match(u32 c) { u32 o = c & 0xf; return o == C_M || o == C_EQ || o == C_X; }

// nt16 4-bit base codes as stored in BAM ("=ACMGRSVTWYHKDBN")
enum { NT_A = 1, NT_C = 2, NT_G = 4, NT_T = 8, NT_N = 15 };
ARB_HD char nt16_char(u32 code) {
	// switch instead of a memory table: compiles to a constant-bank lookup on the device
	switch (code & 15) {
		case 0: return '='; case 1: return 'A'; case 2: return 'C'; case 3: return 'M'; case 4: return 'G'; case 5: return 'R';
		case 6: return 'S'; case 7: return 'V'; case 8: return 'T'; case 9: return 'W'; case 10: return 'Y'; case 11: return 'H';
		case 12: return 'K'; case 13: return 'D'; case 14: return 'B'; default: return 'N';
	}
}
// complement on nt16 codes restricted to what assembly.hpp:9-22 complements (A<->T, C<->G; everything else unchanged)
ARB_HD u32 nt16_complement(u32 code) {
	switch (code) { case NT_A: return NT_T; case NT_T: return NT_A; case NT_C: return NT_G; case NT_G: return NT_C; default: return code; }
}
ARB_HD u32 nt16_at(const u8* seq, u32 i) { return (seq[i >> 1] >> ((~i & 1) << 2)) & 0xf; }
// nt16 code of a reference character; 16 = not in the alphabet (such a base never equals a read base)
ARB_HD u32 nt16_of_char(char c) {
	switch (c) {
		case '=': return 0; case 'A': return 1; case 'C': return 2; case 'M': return 3; case 'G': return 4; case 'R': return 5; case 'S': return 6; case 'V': return 7;
		case 'T': return 8; case 'W': return 9; case 'Y': return 10; case 'H': return 11; case 'K': return 12; case 'D': return 13; case 'B': return 14; case 'N': return 15;
		default: return 16;
	}
}

// ---- bit tricks on words of eight 4-bit bases, first base in the most significant nibble
ARB_HD u32 bswap32(u32 x) {
#ifdef __CUDA_ARCH__
	return __byte_perm(x, 0, 0x0123);
#else
	return __builtin_bswap32(x);
#endif
}
ARB_HD u32 brev32(u32 x) {
#ifdef __CUDA_ARCH__
	return __brev(x);
#else
	x = (x >> 1 & 0x55555555u) | (x & 0x55555555u) << 1; x = (x >> 2 & 0x33333333u) | (x & 0x33333333u) << 2; x = (x >> 4 & 0x0f0f0f0fu) | (x & 0x0f0f0f0fu) << 4;
	return __builtin_bswap32(x);
#endif
}
ARB_HD u32 popc32(u32 x) {
#ifdef __CUDA_ARCH__
	return (u32) __popc(x);
#else
	return (u32) __builtin_popcount(x);
#endif
}
// words of a BAM-order nt16 sequence (two bases per byte, first base in the high nibble); the sequence is padded to whole words
ARB_HD u32 nt16_word(const u8* seq, u32 k, u32 n_words) { return k < n_words ? bswap32(((const u32*) seq)[k]) : 0u; }
// eight bases starting at base `start` (>= -7; bases before the sequence read as 0)
ARB_HD u32 nt16_window(const u8* seq, u32 n_words, i32 start) {
	if (start < 0) return nt16_word(seq, 0, n_words) >> (4 * (u32) -start);
	const u32 k = (u32) start >> 3, sh = ((u32) start & 7) * 4;
	const u32 hi = nt16_word(seq, k, n_words);
	return sh ? hi << sh | nt16_word(seq, k + 1, n_words) >> (32 - sh) : hi;
}
// same for the packed reference (native words, first base in the most significant nibble)
ARB_HD u32 packed_window(const u32* words, u64 start) {
	const u64 k = start >> 3; const u32 sh = ((u32) start & 7) * 4;
	const u32 hi = words[k];
	return sh ? hi << sh | words[k + 1] >> (32 - sh) : hi;
}

template <class T> ARB_HD T hd_min(T a, T b) { return a < b ? a : b; }
template <class T> ARB_HD T hd_max(T a, T b) { return a > b ? a : b; }
ARB_HD i32 hd_abs(i32 a) { return a < 0 ? -a : a; }

} // namespace arb
