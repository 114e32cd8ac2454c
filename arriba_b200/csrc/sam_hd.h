// sam_hd.h -- SAM text lines turned into BAM record bodies on the device (samscan.cu drives it; the CPU stand-in runs the same functors).
//   sam_lf_count_fn / sam_lf_write_fn : one thread per 16-byte word of the chunk: its LFs counted, then (after an exclusive scan) the offsets of the
//                                       line ends written in file order,
//   sam_size_fn  : one thread per line: the line parsed (the rules of DESIGN.md section 5, which follow htslib's sam_parse1), the size of the BAM record
//                  it becomes, or 4 bytes (a block_size of 0) for an unreadable line,
//   sam_write_fn : one thread per line: the same parse, then block_size and the body written at the line's staged offset (an exclusive scan of the
//                  sizes): the 32-byte core, the name, the CIGAR, the nt16 sequence, 0xFF qualities and an aux part that holds only the first HI
//                  (as type i) and, if the line has an SA tag, an empty SA:Z.
// The staged bodies are what records_hd.h classifies and stores for BAM input, so the record loop downstream is the same for both formats.
#pragma once
#include "model.h"
#include "prims.h"
#include "records_hd.h"

namespace arb {

// the @SQ names of the header, sorted bytewise: name k is blob[off[k], off[k + 1]) and belongs to reference tid[k]
struct sam_names { const u8* blob; const u64* off; const u32* tid; u32 n; };

// tid of an RNAME, -1 if no @SQ line names it (names are compared exactly)
ARB_HD i32 sam_find_name(const sam_names& nm, const u8* s, u32 len) {
	u32 lo = 0, hi = nm.n;
	while (lo < hi) {
		const u32 mid = (lo + hi) / 2;
		const u8* t = nm.blob + nm.off[mid]; const u32 tl = (u32) (nm.off[mid + 1] - nm.off[mid]);
		int c = 0;
		for (u32 x = 0; x < len && x < tl && c == 0; ++x) c = (int) s[x] - (int) t[x];
		if (c == 0) c = len < tl ? -1 : len > tl ? 1 : 0;
		if (c == 0) return (i32) nm.tid[mid];
		if (c < 0) hi = mid; else lo = mid + 1;
	}
	return -1;
}

// an unsigned decimal of 1-19 digits; false on anything else or past `max`
ARB_HD bool sam_decimal(const u8* s, u32 len, u64 max, u64& v) {
	if (len == 0 || len > 19) return false;
	v = 0;
	for (u32 x = 0; x < len; ++x) { const u32 d = (u32) s[x] - '0'; if (d > 9) return false; v = v * 10 + d; }
	return v <= max;
}
ARB_HD bool sam_is_alpha(u8 c) { return (c >= 'A' && c <= 'Z') || (c >= 'a' && c <= 'z'); }
ARB_HD bool sam_is_alnum(u8 c) { return sam_is_alpha(c) || (c >= '0' && c <= '9'); }
ARB_HD u32 sam_cigar_op(u8 c) { // BAM operation code, 16 = not an operation
	switch (c) { case 'M': return C_M; case 'I': return C_I; case 'D': return C_D; case 'N': return C_N; case 'S': return C_S; case 'H': return C_H; case 'P': return C_P; case '=': return C_EQ; case 'X': return C_X; default: return 16; }
}
ARB_HD u32 sam_base_code(u8 c) { // nt16 code of a SEQ byte, either case; anything else is N
	if (c >= 'a' && c <= 'z') c = (u8) (c - 32);
	const u32 v = nt16_of_char((char) c);
	return v == 16 ? 15u : v;
}

// what a line says, as offsets into the line
struct sam_line {
	u32 flag, name_at, name_len, cigar_at, cigar_len, n_cigar, seq_at, l_seq; i32 tid, pos, hit; u8 has_hi, has_sa;
	ARB_HD u32 body_bytes() const { return 32u + name_len + 1u + 4u * n_cigar + (l_seq + 1u) / 2u + l_seq + (has_hi ? 7u : 0u) + (has_sa ? 4u : 0u); }
};

// s[0, n): one line without its LF (and without the CR before it); false: unreadable
ARB_HD bool sam_parse(const u8* s, u32 n, const sam_names& nm, sam_line& L) {
	u32 at[11], len[11], p = 0;
	for (u32 k = 0; k < 11; ++k) {
		at[k] = p;
		while (p < n && s[p] != '\t') ++p;
		len[k] = p - at[k];
		if (k < 10) { if (p >= n) return false; ++p; }
	}
	// QNAME, FLAG
	if (len[0] < 1 || len[0] > 254) return false;
	L.name_at = at[0]; L.name_len = len[0];
	u64 v;
	if (!sam_decimal(s + at[1], len[1], 65535, v)) return false;
	L.flag = (u32) v;
	// RNAME: a name without @SQ line makes the record unmapped
	if (len[2] == 1 && s[at[2]] == '*') L.tid = -1;
	else { L.tid = sam_find_name(nm, s + at[2], len[2]); if (L.tid < 0) L.flag |= BF_UNMAP; }
	// POS (1-based in the text)
	if (!sam_decimal(s + at[3], len[3], 0x7FFFFFFFull, v)) return false;
	L.pos = (i32) v - 1;
	if (v == 0 && !(L.flag & BF_UNMAP)) L.flag |= BF_UNMAP;
	// CIGAR
	L.cigar_at = at[5]; L.cigar_len = len[5]; L.n_cigar = 0;
	if (len[5] == 1 && s[at[5]] == '*') { L.cigar_len = 0; if (!(L.flag & BF_UNMAP)) L.flag |= BF_UNMAP; }
	else {
		u32 digits = 0; u64 run = 0;
		for (u32 x = 0; x < len[5]; ++x) {
			const u8 c = s[at[5] + x]; const u32 d = (u32) c - '0';
			if (d <= 9) { if (++digits > 9) return false; run = run * 10 + d; continue; }
			if (digits == 0 || run == 0 || run >= (1u << 28) || sam_cigar_op(c) == 16) return false;
			++L.n_cigar; digits = 0; run = 0;
		}
		if (digits != 0 || L.n_cigar == 0 || L.n_cigar > 65535) return false;
	}
	// SEQ, QUAL
	L.seq_at = at[9]; L.l_seq = len[9] == 1 && s[at[9]] == '*' ? 0 : len[9];
	if (!(len[10] == 1 && s[at[10]] == '*') && len[10] != L.l_seq) return false;
	// tags: XX:T:value; the first HI decides the hit index, SA only counts as present
	L.has_hi = 0; L.has_sa = 0; L.hit = 0;
	while (p < n) {
		++p; // the tab before the field
		const u32 t = p;
		while (p < n && s[p] != '\t') ++p;
		const u32 tl = p - t;
		if (tl < 5 || !sam_is_alpha(s[t]) || !sam_is_alnum(s[t + 1]) || s[t + 2] != ':' || s[t + 4] != ':') return false;
		const u8 type = s[t + 3];
		if (type != 'A' && type != 'i' && type != 'f' && type != 'Z' && type != 'H' && type != 'B') return false;
		if (s[t] == 'H' && s[t + 1] == 'I' && !L.has_hi) {
			L.has_hi = 1;
			if (type == 'i') {
				const bool neg = s[t + 5] == '-' && tl > 5;
				const u32 d0 = t + 5 + (neg || s[t + 5] == '+' ? 1 : 0);
				if (!sam_decimal(s + d0, t + tl - d0, neg ? 0x80000000ull : 0x7FFFFFFFull, v)) return false;
				L.hit = neg ? (i32) (0 - (u32) v) : (i32) v;
			}
		}
		if (s[t] == 'S' && s[t + 1] == 'A') L.has_sa = 1;
	}
	return true;
}

// ------------------------------------------------------------------------------------------- line ends
// the chunk's words [w0, w0 + n_words) of 16 bytes; only bytes in [lo, hi) count
struct sam_text { const u8* B; u64 lo, hi, w0; };
// the LFs of word w, in order: emit(k, offset) for the k-th; returns their number
template <class E> ARB_HD u32 sam_word_lfs(const sam_text& t, u32 w, E emit) {
	const u64 base = (t.w0 + w) * 16;
	u32 n = 0;
#ifdef __CUDA_ARCH__
	const uint4 q = *(const uint4*) (t.B + base); // the buffer is 16-byte aligned and has slack behind its end
	const u32 word[4] = {q.x, q.y, q.z, q.w};
#else
	u32 word[4] = {0, 0, 0, 0};
	for (u32 x = 0; x < 16; ++x) if (base + x < t.hi) word[x >> 2] |= (u32) t.B[base + x] << (8 * (x & 3));
#endif
#pragma unroll
	for (u32 x = 0; x < 16; ++x) {
		const u64 o = base + x;
		if (o >= t.lo && o < t.hi && ((word[x >> 2] >> (8 * (x & 3))) & 0xFF) == '\n') emit(n++, (u32) o);
	}
	return n;
}
struct sam_lf_count_fn { sam_text t; u32* count; ARB_HD void operator()(u32 w) const { count[w] = sam_word_lfs(t, w, [](u32, u32) {}); } };
struct sam_lf_write_fn {
	sam_text t; const u32* base; u32* line_end;
	ARB_HD void operator()(u32 w) const { u32* out = line_end + base[w]; sam_word_lfs(t, w, [&](u32 k, u32 o) { out[k] = o; }); }
};

// ------------------------------------------------------------------------------------------- lines -> staged BAM records
struct sam_lines {
	const u8* B; u64 start /* the first line's offset */; const u32* line_end; u32 n_lf /* lines that end at an LF; a last line without one ends at line_end[n_lf] */;
	ARB_HD void span(u32 k, u32& a, u32& n) const {
		a = k == 0 ? (u32) start : line_end[k - 1] + 1;
		u32 e = line_end[k];
		if (k < n_lf && e > a && B[e - 1] == '\r') --e; // one CR before the LF
		n = e - a;
	}
};
struct sam_size_fn {
	sam_lines l; sam_names nm; u32* bytes;
	ARB_HD void operator()(u32 k) const {
		u32 a, n; l.span(k, a, n);
		sam_line L;
		bytes[k] = sam_parse(l.B + a, n, nm, L) ? 4u + L.body_bytes() : 4u;
	}
};
struct sam_write_fn {
	sam_lines l; sam_names nm; const u32* at; u8* stage;
	ARB_HD static void put32(u8* d, u32 v) { d[0] = (u8) v; d[1] = (u8) (v >> 8); d[2] = (u8) (v >> 16); d[3] = (u8) (v >> 24); }
	ARB_HD void operator()(u32 k) const {
		u32 a, n; l.span(k, a, n);
		const u8* s = l.B + a;
		u8* d = stage + at[k];
		sam_line L;
		if (!sam_parse(s, n, nm, L)) { put32(d, 0); return; } // block_size 0: the record loop reports an unreadable record here
		put32(d, L.body_bytes()); d += 4;
		put32(d, (u32) L.tid); put32(d + 4, (u32) L.pos);
		d[8] = (u8) (L.name_len + 1); d[9] = 255; d[10] = 0; d[11] = 0; // l_read_name, mapq, bin
		d[12] = (u8) L.n_cigar; d[13] = (u8) (L.n_cigar >> 8); d[14] = (u8) L.flag; d[15] = (u8) (L.flag >> 8);
		put32(d + 16, L.l_seq); put32(d + 20, 0xFFFFFFFFu); put32(d + 24, 0xFFFFFFFFu); put32(d + 28, 0); // l_seq, next refID, next pos, tlen
		d += 32;
		for (u32 x = 0; x < L.name_len; ++x) d[x] = s[L.name_at + x];
		d[L.name_len] = 0; d += L.name_len + 1;
		u32 run = 0;
		for (u32 x = 0; x < L.cigar_len; ++x) {
			const u8 c = s[L.cigar_at + x];
			if (c >= '0' && c <= '9') { run = run * 10 + (c - '0'); continue; }
			put32(d, run << 4 | sam_cigar_op(c)); d += 4; run = 0;
		}
		for (u32 x = 0; x < L.l_seq; x += 2) {
			const u32 hi = sam_base_code(s[L.seq_at + x]), lo = x + 1 < L.l_seq ? sam_base_code(s[L.seq_at + x + 1]) : 0;
			*d++ = (u8) (hi << 4 | lo);
		}
		for (u32 x = 0; x < L.l_seq; ++x) *d++ = 0xFF;
		if (L.has_hi) { d[0] = 'H'; d[1] = 'I'; d[2] = 'i'; put32(d + 3, (u32) L.hit); d += 7; }
		if (L.has_sa) { d[0] = 'S'; d[1] = 'A'; d[2] = 'Z'; d[3] = 0; }
	}
};

} // namespace arb
