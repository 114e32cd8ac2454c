// records_hd.h -- what the reference's record loop does with every BAM record (read_chimeric_alignments.cpp:611-749), as host/device code
// (records.cu drives it; the CPU stand-in runs the same functors). The main file (-x) and, ahead of it, a separate chimeric file (-c, STAR's
// Chimeric.out.sam) go into one record store; the replay runs both files' loops for every key.
//   rec_extract_fn : one thread per record of a chunk: the records the loop skips, HI and SA, the two validity checks, the key hash and the size of the
//                    compact copy that the record store keeps across chunks (fixed fields with the contig id, name, CIGAR, nt16 sequence);
//                    rec_extract_t<true> is the -c file's variant,
//   rec_store_fn   : the copy itself,
//   rec_replay_fn  : one thread per run of equal key hashes (the store sorted stably by hash: file order inside a run): every key of the run replays the
//                    loop's steps in file order -- supplementaries, discordant mates, proper pairs (each record alternates between waiting and pairing),
//                    tandem duplications in soft clips, split reads, read-through fragments, pristine viral reads, coverage -- once to count what it
//                    emits, once to write the fragment pools (the layout fragtable.cu reads, one pool). The searches (the genome scan for tandem
//                    duplications, the gene-index queries of the read-through test) run in the counting pass only: it logs what they decided per record,
//                    and the writing pass replays from that log,
//   rec_cov_pack_fn: the coverage counts of the writing pass, saturated to 16 bits and packed two to a 32-bit word.
#pragma once
#include "model.h"
#include "prims.h"
#include "annot_hd.h"
#include "fragtable_hd.h"
#include "../../include/arriba_b200.h"

namespace arb {

enum { BF_PAIRED = 1, BF_PROPER = 2, BF_UNMAP = 4, BF_MUNMAP = 8, BF_REVERSE = 16, BF_READ1 = 64, BF_SECONDARY = 256, BF_DUP = 1024, BF_SUPPLEMENTARY = 2048 };
// fatal record errors, by file position (the smallest position wins: the reference reads serially); the host raises them with their texts (ingest.cpp)
enum { REC_ERR_LOAD = 1, REC_ERR_CIGAR = 2, REC_ERR_BEYOND = 3, REC_ERR_ANNOTATION = 4, REC_ERR_UNMAPPED = 5 /* a -c record without a reference */ };
// device counters of the loop's by-products: [REC_CTR_VIRAL + contig] = pristine reads per viral contig. REC_CTR_CHIMERIC: the loop added an alignment
// (with a -c file only the -c file's loop adds them outside read-through and tandem-duplication fragments; the -x file's loop then never sets it)
enum { REC_CTR_MAPPED = 0, REC_CTR_MALFORMED = 1, REC_CTR_MISSING_HI = 2, REC_CTR_CHIMERIC = 3, REC_CTR_VIRAL = 4 };

ARB_HD u32 rec_rd32(const u8* p) { return (u32) p[0] | (u32) p[1] << 8 | (u32) p[2] << 16 | (u32) p[3] << 24; }
ARB_HD u32 rec_rd16(const u8* p) { return (u32) p[0] | (u32) p[1] << 8; }
ARB_HD u64 rec_atomic_min_u64(u64* p, u64 v) {
#ifdef __CUDA_ARCH__
	return (u64) atomicMin((unsigned long long*) p, (unsigned long long) v);
#else
	const u64 old = *p; if (v < old) *p = v; return old;
#endif
}
ARB_HD void rec_atomic_add_u64(u64* p, u64 v) {
#ifdef __CUDA_ARCH__
	atomicAdd((unsigned long long*) p, (unsigned long long) v);
#else
	*p += v;
#endif
}
// aligned 8- and 16-byte stores: a thread that copies a record byte by byte issues one store per byte, to lines no other lane of its warp touches
ARB_HD void rec_put_u64(u8* d /* 8-byte aligned */, u64 v) {
#ifdef __CUDA_ARCH__
	*(u64*) d = v;
#else
	memcpy(d, &v, 8);
#endif
}
ARB_HD void rec_put_u128(u8* d /* 16-byte aligned */, u64 lo, u64 hi) {
#ifdef __CUDA_ARCH__
	*(ulonglong2*) d = make_ulonglong2(lo, hi);
#else
	memcpy(d, &lo, 8); memcpy(d + 8, &hi, 8);
#endif
}
// bytes [at, at + 8) of src as a little-endian word, zero from byte n on
ARB_HD u64 rec_get_u64(const u8* src, u32 at, u32 n) {
	u64 v = 0;
	for (u32 x = 0; x < 8; ++x) if (at + x < n) v |= (u64) src[at + x] << (8 * x);
	return v;
}
// +1 on a counter that every thread of a launch may bump: on the device one atomic per warp (the active lanes' increments summed)
ARB_HD void rec_count_one(u64* p) {
#ifdef __CUDA_ARCH__
	const unsigned active = __activemask();
	if ((threadIdx.x & 31u) == (unsigned) __ffs((int) active) - 1u) atomicAdd((unsigned long long*) p, (unsigned long long) __popc(active));
#else
	*p += 1;
#endif
}

// ------------------------------------------------------------------------------------------- one record (a BAM record body, or its compact copy: no qualities, no tags)
struct rec_t {
	const u8* base; u32 size;
	i32 tid, pos; u32 flag, n_cigar, l_qname; i32 l_seq;
	const u8* cigar_raw; const u8* seq; const u8* aux; const u8* aux_end;
	ARB_HD bool reverse() const { return flag & BF_REVERSE; }
	ARB_HD const char* qname() const { return (const char*) base + 32; }
	ARB_HD u32 name_len() const { u32 n = 0; while (n < l_qname && base[32 + n]) ++n; return n; } // strnlen
	ARB_HD u32 cig(u32 k) const { return rec_rd32(cigar_raw + 4 * k); }
	ARB_HD i32 ref_len(u32 n_ops) const { i64 l = 0; for (u32 k = 0; k < n_ops; ++k) { u32 c = cig(k), o = c & 15; if (o == C_M || o == C_D || o == C_N || o == C_EQ || o == C_X) l += c >> 4; } return (i32) l; }
	ARB_HD i32 query_len(u32 n_ops) const { i64 l = 0; for (u32 k = 0; k < n_ops; ++k) { u32 c = cig(k), o = c & 15; if (o == C_M || o == C_I || o == C_S || o == C_EQ || o == C_X) l += c >> 4; } return (i32) l; }
	ARB_HD i32 endpos() const { i32 r = (flag & BF_UNMAP) ? 0 : ref_len(n_cigar); if (r == 0) r = 1; return pos + r; }
	ARB_HD u32 base_code(u32 i) const { return nt16_at(seq, i); }
	ARB_HD u32 compact_bytes() const { return (32u + l_qname + 4u * n_cigar + ((u32) l_seq + 1) / 2 + 7) & ~7u; } // 8-byte steps in the store
};

// p: the record body (after block_size); with_tail: the qualities and tags follow the sequence (a BAM record), otherwise it is a compact copy
ARB_HD bool rec_parse(const u8* p, u32 size, rec_t& r, bool with_tail = true) {
	if (size < 32) return false;
	r.base = p; r.size = size;
	r.tid = (i32) rec_rd32(p); r.pos = (i32) rec_rd32(p + 4); r.l_qname = p[8]; r.n_cigar = rec_rd16(p + 12); r.flag = rec_rd16(p + 14); r.l_seq = (i32) rec_rd32(p + 16);
	const u64 need = 32ull + r.l_qname + 4ull * r.n_cigar + ((u64) (u32) r.l_seq + 1) / 2 + (with_tail ? (u64) (u32) r.l_seq : 0);
	if (need > size || r.l_qname == 0) return false;
	r.cigar_raw = p + 32 + r.l_qname; r.seq = r.cigar_raw + 4 * r.n_cigar;
	r.aux = r.seq + ((u32) r.l_seq + 1) / 2 + (with_tail ? (u32) r.l_seq : 0); r.aux_end = p + size;
	return true;
}

ARB_HD const u8* rec_find_aux(const rec_t& r, char a, char b) { // returns pointer to the type byte
	const u8* s = r.aux;
	while (s + 3 <= r.aux_end) {
		const bool hit = s[0] == (u8) a && s[1] == (u8) b;
		const u8* v = s + 2; const u8 t = v[0]; const u8* next;
		switch (t) {
			case 'A': case 'c': case 'C': next = v + 2; break;
			case 's': case 'S': next = v + 3; break;
			case 'i': case 'I': case 'f': next = v + 5; break;
			case 'd': next = v + 9; break;
			case 'Z': case 'H': next = v + 1; while (next < r.aux_end && *next) ++next; ++next; break;
			case 'B': {
				if (v + 6 > r.aux_end) return 0;
				const u8 st = v[1]; const u32 n = rec_rd32(v + 2);
				const u32 sz = (st == 'c' || st == 'C') ? 1 : (st == 's' || st == 'S') ? 2 : 4;
				if ((u64) sz * n > (u64) (r.aux_end - (v + 6))) return 0;
				next = v + 6 + (u64) sz * n; break;
			}
			default: return 0;
		}
		if (next > r.aux_end) return 0; // truncated field: its payload lies past the record (htslib reports corrupted aux data and returns no tag)
		if (hit) return v;
		s = next;
	}
	return 0;
}
ARB_HD i64 rec_aux_int(const u8* v) {
	switch (v[0]) {
		case 'c': return (int8_t) v[1]; case 'C': return v[1]; case 's': return (int16_t) rec_rd16(v + 1); case 'S': return rec_rd16(v + 1);
		case 'i': return (i32) rec_rd32(v + 1); case 'I': return rec_rd32(v + 1); default: return 0;
	}
}
// decimal digits of a hit index, most significant first; returns their number
ARB_HD u32 rec_hit_digits(i64 hit_index, char* out /* 21 */) {
	char d[21]; u32 n = 0; u32 w = 0;
	u64 v = hit_index < 0 ? 0 - (u64) hit_index : (u64) hit_index;
	do { d[n++] = (char) ('0' + v % 10); v /= 10; } while (v);
	if (hit_index < 0) out[w++] = '-';
	while (n > 0) out[w++] = d[--n];
	return w;
}
// FNV-1a over "<qname>,<HI>", folded
ARB_HD u64 rec_key_hash(const char* name, u32 n_name, i64 hit_index) {
	u64 h = 1469598103934665603ULL;
	for (u32 i = 0; i < n_name; ++i) { h ^= (u8) name[i]; h *= 1099511628211ULL; }
	h ^= (u8) ','; h *= 1099511628211ULL;
	char digits[21]; const u32 n = rec_hit_digits(hit_index, digits);
	for (u32 i = 0; i < n; ++i) { h ^= (u8) digits[i]; h *= 1099511628211ULL; }
	h ^= h >> 29;
	return h;
}

// what the loop does not keep (unmapped records, records with unmapped mates, secondaries without HI) and the two validity checks
ARB_HD bool rec_skipped(const rec_t& r) { return (r.flag & BF_UNMAP) || ((r.flag & BF_PAIRED) && (r.flag & BF_MUNMAP)); }
// An alignment that starts before or runs past the end of its contig is not a valid record (SAMv1 1.4), and what the reference does with one is undefined:
// it indexes its coverage vectors and the contig's sequence beyond their ends. Here the same indices would leave the coverage windows and the genome on the
// device: the run stops with an error instead. Likewise a mapped record without CIGAR operations, or whose CIGAR consumes more bases than the record holds:
// the reference dies on those (segmentation fault, or std::out_of_range from substr); everything downstream indexes the sequence by the CIGAR.
// contig: the record's contig id (after tid_to_contig); contig_len: 0 for a contig without sequence.
ARB_HD u32 rec_validate(const rec_t& r, u32 contig_len, i64& query_span) {
	i64 ref_span = 0; query_span = 0;
	for (u32 k = 0; k < r.n_cigar; ++k) { const u32 c = r.cig(k), o = c & 15; if (o == C_M || o == C_EQ || o == C_X) { ref_span += c >> 4; query_span += c >> 4; } else if (o == C_D || o == C_N) ref_span += c >> 4; else if (o == C_I || o == C_S) query_span += c >> 4; }
	if (r.n_cigar == 0 || query_span > (i64) r.l_seq) return REC_ERR_CIGAR;
	if (contig_len > 0 && (r.pos < 0 || (i64) r.pos + (ref_span ? ref_span : 1) > (i64) contig_len)) return REC_ERR_BEYOND;
	return 0;
}

// ------------------------------------------------------------------------------------------- per chunk: classify and copy
struct rec_chunk_view {
	const u8* B; const u32* rec_off; u64 buf_pos /* file position (inflated stream) of B[0] */;
	const u16* tid_to_contig; i32 n_tid; const u32* contig_len; const u8* interesting;
};
// CHIMERIC_FILE: the records of a -c file (read_chimeric_alignments.cpp:611-623 with separate_chimeric_bam_file set, is_rna_bam_file not): none is skipped
// (a record without a reference is an error that names it: the reference indexes tid_to_contig[-1]), HI is not read (every key is "<qname>,1"), nothing is
// counted (the call's interesting_tids stays all false), and the SA tag plays no part.
template <bool CHIMERIC_FILE> struct rec_extract_t {
	rec_chunk_view c; u64 hash_mask;
	u32* bytes /* compact size, 0 = not kept */; u32* kept; u64* hash; i64* hit; u8* has_sa; u64* counters; u64* error;
	ARB_HD void fail(u32 i, u32 kind) const { rec_atomic_min_u64(error, (c.buf_pos + c.rec_off[i]) << 3 | kind); }
	ARB_HD void operator()(u32 i) const {
		bytes[i] = 0; kept[i] = 0;
		const u8* p = c.B + c.rec_off[i];
		rec_t r;
		if (!rec_parse(p + 4, rec_rd32(p), r)) { fail(i, REC_ERR_LOAD); return; }
		i64 hit_index = 1;
		if (CHIMERIC_FILE) {
			if (r.tid < 0) { fail(i, REC_ERR_UNMAPPED); return; }
		} else {
			if (rec_skipped(r)) return;
			const u8* hi = rec_find_aux(r, 'H', 'I');
			if (hi) hit_index = rec_aux_int(hi);
			else if (r.flag & BF_SECONDARY) { rec_count_one(&counters[REC_CTR_MISSING_HI]); return; }
		}
		if (r.tid < 0 || r.tid >= c.n_tid) { fail(i, REC_ERR_LOAD); return; }
		const u32 contig = c.tid_to_contig[r.tid];
		i64 query_span;
		const u32 bad = rec_validate(r, c.contig_len[contig], query_span);
		if (bad) { fail(i, bad); return; }
		if (!CHIMERIC_FILE && !(r.flag & BF_SUPPLEMENTARY) && c.interesting[contig]) rec_count_one(&counters[REC_CTR_MAPPED]);
		bytes[i] = r.compact_bytes(); kept[i] = 1;
		hash[i] = rec_key_hash(r.qname(), r.name_len(), hit_index) & hash_mask; hit[i] = hit_index;
		has_sa[i] = !CHIMERIC_FILE && rec_find_aux(r, 'S', 'A') != 0;
	}
};
typedef rec_extract_t<false> rec_extract_fn;
struct rec_store_fn { // record i of the chunk -> store item n_stored + kept[i] at byte arena_used + at[i] (at, kept: exclusive scans of the sizes / the kept flags)
	rec_chunk_view c; const u32* at; const u32* kept; const u64* hash; const i64* hit; const u8* has_sa;
	u64 n_stored, arena_used; u8* arena; u64* s_at; u64* s_pos; u32* s_hash_lo; u32* s_hash_hi; i64* s_hit; u8* s_sa;
	ARB_HD void operator()(u32 i) const {
		if (kept[i + 1] == kept[i]) return;
		const u8* p = c.B + c.rec_off[i] + 4;
		const u64 k = n_stored + kept[i], dst = arena_used + at[i], size = at[i + 1] - at[i];
		rec_t r; rec_parse(p, rec_rd32(p - 4), r);
		const u32 head = 32u + r.l_qname + 4u * r.n_cigar, n_seq = ((u32) r.l_seq + 1) / 2; // the sequence follows the CIGAR: p[0, head + n_seq)
		u8* d = arena + dst; // 8-byte aligned, `size` a multiple of 8
		const u32 contig = c.tid_to_contig[r.tid];
		rec_put_u64(d, (rec_get_u64(p, 0, head + n_seq) & ~(u64) 0xFFFFFFFFu) | contig); // the contig id in place of the BAM's reference id
		for (u32 b = 8; b < size; b += 8) rec_put_u64(d + b, rec_get_u64(p, b, head + n_seq));
		s_at[k] = dst; s_pos[k] = c.buf_pos + c.rec_off[i]; s_hash_lo[k] = (u32) hash[i]; s_hash_hi[k] = (u32) (hash[i] >> 32); s_hit[k] = hit[i]; s_sa[k] = has_sa[i];
	}
};

// ------------------------------------------------------------------------------------------- after the last chunk: replay
struct rec_store_view {
	const u8* arena; const u64* at; const u64* pos; const i64* hit; const u8* sa; const u32* order /* sorted by key hash, file order inside a hash */;
	u64 chimeric_end; // records at positions below it come from a -c file (which precedes the main file: a key's -c records come first)
	ARB_HD bool from_chimeric_file(u32 k) const { return pos[k] < chimeric_end; }
	ARB_HD void get(u32 k, rec_t& r) const { const u8* p = arena + at[k]; rec_parse(p, 0xFFFFFFFFu, r, false); r.aux = r.aux_end = 0; }
	ARB_HD bool same_key(u32 a, u32 b) const {
		if (hit[a] != hit[b]) return false;
		const u8* pa = arena + at[a]; const u8* pb = arena + at[b];
		rec_t ra, rb; get(a, ra); get(b, rb);
		const u32 na = ra.name_len(), nb = rb.name_len();
		if (na != nb) return false;
		for (u32 x = 0; x < na; ++x) if (pa[32 + x] != pb[32 + x]) return false;
		return true;
	}
};
struct rec_cov_view { u64* counts /* per window; packed by rec_cov_pack_fn */; u8* starts; u8* ends; const u64* off; const u32* n; u32 n_contigs; };
struct rec_params { u32 max_itd_length; u8 external_duplicate_marking; const u8* viral; };
// per segment: fragments, alignments, name bytes, CIGAR operations, 16-byte sequence units; exclusive scans of them turn into the segments' write bases
enum { RS_FRAGS = 0, RS_ALNS = 1, RS_NAMES = 2, RS_CIGARS = 3, RS_UNITS = 4, RS_N = 5 };

// paired-end reads must be clipped at the outer end of the fragment (read_chimeric_alignments.cpp:511-522)
ARB_HD bool clipped_at_correct_end(const rec_t& r) {
	if (!(r.flag & BF_PAIRED)) return true;
	const bool fwd = !r.reverse();
	const u32 k = (r.flag & BF_SUPPLEMENTARY) ? (fwd ? r.n_cigar - 1 : 0) : (fwd ? 0 : r.n_cigar - 1);
	const u32 op = r.cig(k) & 15;
	return op == C_S || op == C_H;
}
ARB_HD bool clipped_sequence_is_adapter(const rec_t& a, const rec_t* bp) { // read_chimeric_alignments.cpp:197-214
	if (!bp) return false;
	const rec_t& b = *bp;
	if (a.pos != b.pos) return false;
	const u32 a0 = a.cig(0), al = a.cig(a.n_cigar - 1), b0 = b.cig(0), bl = b.cig(b.n_cigar - 1);
	if (a.reverse() && (a0 & 15) == C_S && !b.reverse() && (bl & 15) == C_S && (a0 >> 4) == (bl >> 4)) return true;
	if (b.reverse() && (b0 & 15) == C_S && !a.reverse() && (al & 15) == C_S && (b0 >> 4) == (al >> 4)) return true;
	return false;
}
ARB_HD bool spanning_intron(const rec_t& r, i32 gene1_end, i32 gene2_start, u32& op, i32& read_pos) { // read_chimeric_alignments.cpp:19-41
	if (r.n_cigar < 3) return false;
	i32 before = r.pos;
	for (u32 k = 0; k < r.n_cigar; ++k) {
		const u32 c = r.cig(k), o = c & 15;
		const i32 len = (o == C_M || o == C_D || o == C_N || o == C_EQ || o == C_X) ? (i32) (c >> 4) : 0;
		const i32 after = before + len;
		if (o == C_N && ((before <= gene1_end && after > gene1_end) || (before < gene2_start && after >= gene2_start))) { op = k; read_pos = r.query_len(k); return true; }
		before = after;
	}
	return false;
}
ARB_HD bool pristine(const rec_t& r) { // read_chimeric_alignments.cpp:526-558
	for (u32 k = 0; k < r.n_cigar; ++k) { const u32 o = r.cig(k) & 15; if (o != C_N && o != C_M && o != C_X) return false; }
	const u32 n = (u32) r.l_seq;
	for (u32 i = 2, repeat = 0, count = 1; i + 2 < n; i += 2) {
		if (r.base_code(i) == r.base_code(repeat) && r.base_code(i + 1) == r.base_code(repeat + 1)) ++count;
		else if (r.base_code(i + 1) == r.base_code(repeat + 1) && r.base_code(i + 2) == r.base_code(repeat + 2)) { ++count; ++i; }
		else { count = 1; repeat = i; }
		if (count >= 8) return false;
	}
	return true;
}

struct tandem_t { bool forward, first_in_pair, supplementary; u16 contig; i32 start, end; u32 cigar[3]; u32 n_cigar; };
// internal tandem duplications that the aligner left soft-clipped (read_chimeric_alignments.cpp:216-336)
ARB_HD bool tandem_duplication(const annot_view& an, u32 max_itd_length, const rec_t* rp, tandem_t& t) {
	if (!rp) return false;
	const rec_t& r = *rp;
	const u32 min_clip = 12, min_dup = 9, max_dup = max_itd_length, max_mismatches = 1, max_non_template = 6, min_aligned = 15;
	u32 clip_len = 0, clip_pos = 0; bool clipped_start = true; int direction = +1; int win_start = 0, win_end = 0, ext_start = 0;
	const u32 first = r.cig(0), last = r.cig(r.n_cigar - 1);
	if ((first & 15) == C_S && (first >> 4) >= min_clip) {
		clip_len = first >> 4; clip_pos = 0; direction = -1;
		win_start = (int) ((i64) r.pos + min_dup - clip_len); win_end = (int) ((i64) r.pos + max_dup - clip_len); ext_start = (int) ((i64) r.pos - clip_len); clipped_start = true;
	}
	if ((last & 15) == C_S && (last >> 4) >= hd_max(min_clip, clip_len)) {
		clip_len = last >> 4; clip_pos = (u32) r.l_seq - clip_len; direction = +1;
		win_start = (int) ((i64) r.endpos() - max_dup); win_end = (int) ((i64) r.endpos() - min_dup); ext_start = r.endpos(); clipped_start = false;
	}
	if (clip_len == 0) return false;
	if ((u32) r.tid >= an.n_contigs || an.contig_len[r.tid] == 0) return false;
	const char* contig_seq = an.assembly + an.contig_seq_off[r.tid];
	const u64 contig_len = an.contig_len[r.tid];
	// unsigned comparison on purpose (the reference compares an int sum with a size_t)
	if ((u64) (u32) ((u32) win_end + max_dup + clip_len + 1u) >= contig_len || win_start <= (int) (max_dup + clip_len + 1)) return false;
	// the clipped bases as characters: clip(k)
	#define ARB_CLIP(k) nt16_char(r.base_code(clip_pos + (k)))
	// can the read simply be extended linearly? then it is no tandem duplication
	u32 ext_matches = 0;
	for (u32 k = 0; k < clip_len; ++k) {
		const i64 g = (i64) ext_start + k;
		if (g >= 0 && (u64) g < contig_len && contig_seq[g] == ARB_CLIP(k)) ++ext_matches;
	}
	if (1.0 * ext_matches / clip_len >= 0.7f) return false;
	// Quick rejection of a window: the 7th to 14th compared base (positions 6..13 in visiting order) sit in eight consecutive reference bytes. Two
	// mismatches among them end the exact loop below by its 14th step with at most 12 matches -- fewer than min_aligned, and matches + mismatches
	// stays below clip_len when clip_len > 14 -- so such a window cannot be accepted.
	const bool prefilter = clip_len > max_non_template + 8 && max_mismatches == 1 && min_aligned > max_non_template + 8 - 2;
	const u32 probe_at = direction == +1 ? max_non_template : clip_len - max_non_template - 8;
	char probe[8];
	if (prefilter) for (u32 k = 0; k < 8; ++k) probe[k] = ARB_CLIP(probe_at + k);
	for (int cp = win_start; cp <= win_end; ++cp) {
		if (prefilter) {
			u32 differ = 0;
			for (u32 k = 0; k < 8; ++k) differ += contig_seq[cp + probe_at + k] != probe[k];
			if (differ >= 2) continue;
		}
		u32 matches = 0, mismatches = 0;
		i64 t_start = (i64) contig_len; i64 t_end = -1;
		for (u32 i = 0; i < clip_len; ++i) {
			const int rp2 = direction == +1 ? (int) i : (int) (clip_len - 1 - i);
			if (contig_seq[cp + rp2] == ARB_CLIP(rp2)) {
				++matches;
				if (cp + rp2 < t_start) t_start = cp + rp2;
				if (cp + rp2 > t_end) t_end = cp + rp2;
			} else if (i >= max_non_template) { if (++mismatches > max_mismatches) break; }
		}
		if (matches >= min_aligned || matches + mismatches == clip_len) {
			t.forward = !r.reverse(); t.first_in_pair = r.flag & BF_READ1; t.contig = (u16) r.tid;
			t.supplementary = !(r.flag & BF_PAIRED) || (clipped_start && !r.reverse()) || (!clipped_start && r.reverse());
			t.start = (i32) t_start; t.end = (i32) t_end;
			u32 clip_left = clipped_start ? 0 : (u32) r.l_seq - clip_len, clip_right = clipped_start ? (u32) r.l_seq - clip_len : 0;
			if (t.start > cp) clip_left += t.start - cp;
			if (t.end < cp + (int) clip_len - 1) clip_right += cp + clip_len - 1 - t.end;
			t.n_cigar = 0;
			if (clip_left > 0) t.cigar[t.n_cigar++] = clip_left << 4 | C_S;
			t.cigar[t.n_cigar++] = (u32) (t.end - t.start + 1) << 4 | C_M;
			if (clip_right > 0) t.cigar[t.n_cigar++] = clip_right << 4 | C_S;
			return true;
		}
	}
	#undef ARB_CLIP
	return false;
}

// The fragments of one key ("<qname>,<HI>", and "<qname>,<HI>ITD" for tandem duplications) as the loop builds them. Counting (out.frags == NULL) only
// advances the tallies; writing puts fragments, alignments, names, CIGAR operations and sequences at the segment's bases plus the tallies.
struct rec_emit {
	arb_pool_fragment* frags; arb_pool_alignment* alns; char* names; u32* cigars; u8* seqs;
	u32 base[RS_N]; u32 n[RS_N];
	i32 id[2]; // fragment of the key / of the key's ITD, -1 before it is created
	u8 chimeric_file; // the fragments created now come from a -c file
	ARB_HD bool writing() const { return frags != 0; }
	// fragment(name, &created)
	ARB_HD u32 fragment(const rec_t& named, i64 hit_index, int itd, bool* created) {
		if (id[itd] >= 0) { if (created) *created = false; return (u32) id[itd]; }
		const u32 f = base[RS_FRAGS] + n[RS_FRAGS]++;
		char digits[21]; const u32 nd = rec_hit_digits(hit_index, digits);
		const u32 nn = named.name_len(), len = nn + 1 + nd + (itd ? 3 : 0);
		if (writing()) {
			char* d = names + base[RS_NAMES] + n[RS_NAMES];
			for (u32 x = 0; x < nn; ++x) d[x] = named.qname()[x];
			d[nn] = ',';
			for (u32 x = 0; x < nd; ++x) d[nn + 1 + x] = digits[x];
			if (itd) { d[nn + 1 + nd] = 'I'; d[nn + 2 + nd] = 'T'; d[nn + 3 + nd] = 'D'; }
			arb_pool_fragment& g = frags[f];
			g.name_off = base[RS_NAMES] + n[RS_NAMES]; g.name_len = len; g.head = g.tail = -1; g.count = 0; g.single_end = 0; g.duplicate = 0; g.chimeric_file = chimeric_file;
		}
		n[RS_NAMES] += len;
		id[itd] = (i32) f;
		if (created) *created = true;
		return f;
	}
	ARB_HD u64 store_seq(const rec_t& r) { // nt16 nibbles copied verbatim, 16-byte aligned, the rest of the last unit zero
		const u32 bytes = ((u32) r.l_seq + 1) / 2, units = (bytes + 15) / 16;
		const u64 off = (u64) (base[RS_UNITS] + n[RS_UNITS]) * 16;
		if (writing()) for (u32 u = 0; u < units; ++u) rec_put_u128(seqs + off + 16 * u, rec_get_u64(r.seq, 16 * u, bytes), rec_get_u64(r.seq, 16 * u + 8, bytes));
		n[RS_UNITS] += units;
		return off;
	}
	ARB_HD void push_cigar(u32 op) { if (writing()) cigars[base[RS_CIGARS] + n[RS_CIGARS]] = op; ++n[RS_CIGARS]; }
	ARB_HD void link(u32 f, arb_pool_alignment& a) {
		const i32 k = (i32) (base[RS_ALNS] + n[RS_ALNS]++);
		if (!writing()) return;
		a.next = -1; alns[k] = a;
		arb_pool_fragment& g = frags[f];
		if (g.tail >= 0) alns[g.tail].next = k; else g.head = k;
		g.tail = k; ++g.count;
	}
	// converts a record (or a part of it, for read-through alignments) into an alignment of `f`
	// clip: 0 whole record; 1 keep CIGAR ops from `op` on (clip the start); 2 keep ops up to `op` (clip the end)   (read_chimeric_alignments.cpp:50-91)
	ARB_HD void add_alignment(u32 f, const rec_t& r, bool supplementary, u32 op = 0, int clip = 0) {
		if (writing()) { arb_pool_fragment& g = frags[f]; g.single_end = !(r.flag & BF_PAIRED); g.duplicate = g.duplicate || (r.flag & BF_DUP); }
		arb_pool_alignment a; a.supplementary = supplementary; a.first_in_pair = (r.flag & BF_READ1) ? 1 : 0; a.forward = !r.reverse(); a.contig = (u16) r.tid;
		a.seq_off = 0; a.seq_len = 0;
		if (!supplementary) { a.seq_off = store_seq(r); a.seq_len = (u32) r.l_seq; }
		a.cigar_off = base[RS_CIGARS] + n[RS_CIGARS];
		if (clip == 1) {
			a.start = r.pos + r.ref_len(op); a.end = r.endpos() - 1;
			const u32 clip_type = (r.cig(0) & 15) == C_H ? C_H : C_S;
			push_cigar((u32) r.query_len(op) << 4 | clip_type);
			for (u32 k = op; k < r.n_cigar; ++k) push_cigar(r.cig(k));
		} else if (clip == 2) {
			a.start = r.pos; a.end = r.pos + r.ref_len(op + 1) - 1;
			const u32 clip_type = (r.cig(r.n_cigar - 1) & 15) == C_H ? C_H : C_S;
			for (u32 k = 0; k <= op; ++k) push_cigar(r.cig(k));
			push_cigar((u32) (r.l_seq - r.query_len(op + 1)) << 4 | clip_type);
		} else {
			a.start = r.pos; a.end = r.endpos() - 1;
			for (u32 k = 0; k < r.n_cigar; ++k) push_cigar(r.cig(k));
		}
		a.cigar_cnt = base[RS_CIGARS] + n[RS_CIGARS] - a.cigar_off;
		link(f, a);
	}
};

// coverage (read_stats.cpp:161-266): the reference's counters are 16 bits wide and saturate. Saturating increments commute -- the final value is
// min(increments, 65535) in any order -- so the writing pass adds plainly into 64-bit counts (which no sample can wrap) and rec_cov_pack_fn saturates.
ARB_HD void cov_increment(u64* counts, u64 w) { rec_atomic_add_u64(counts + w, 1); }
struct rec_cov_pack_fn { // word i: windows 2i (low half) and 2i + 1 (high half), as a plain little-endian u16 array
	const u64* counts; u32* words;
	ARB_HD void operator()(u32 i) const {
		const u64 a = counts[2 * (u64) i], b = counts[2 * (u64) i + 1];
		words[i] = (u32) (a < 0xFFFFu ? a : 0xFFFFu) | (u32) (b < 0xFFFFu ? b : 0xFFFFu) << 16;
	}
};
ARB_HD void add_coverage(const rec_cov_view& cov, const rec_t& m1, const rec_t* m2p, bool is_chimeric, bool flags_cleared) {
	const rec_t& m2 = m2p ? *m2p : m1;
	const u32 f1 = flags_cleared ? 0 : m1.flag;
	if ((u32) m1.tid >= cov.n_contigs || cov.n[m1.tid] == 0 || (u32) m2.tid >= cov.n_contigs || cov.n[m2.tid] == 0) return;
	if ((f1 & BF_PAIRED) && !(f1 & BF_PROPER)) is_chimeric = true; // the reference's soft-clip tests can never fire (bam_cigar_type() is 0..3)
	if (!is_chimeric) {
		if (!(f1 & BF_REVERSE) || !(f1 & BF_PAIRED)) cov.starts[cov.off[m1.tid] + m1.pos / 20] = 1; else cov.starts[cov.off[m2.tid] + m2.pos / 20] = 1;
	}
	i32 p1 = m1.pos, p2 = m2.pos, position = hd_min(p1, p2);
	int window = position / 20;
	u32 i1 = 0, i2 = 0;
	for (;;) {
		u32 c1 = 0, c2 = 0, l1 = 0, l2 = 0;
		if (i1 < m1.n_cigar) { c1 = m1.cig(i1); const u32 o = c1 & 15; l1 = (o == C_M || o == C_D || o == C_N || o == C_EQ || o == C_X) ? c1 >> 4 : 0; } else window = hd_max(window, p2 / 20);
		if (i2 < m2.n_cigar) { c2 = m2.cig(i2); const u32 o = c2 & 15; l2 = (o == C_M || o == C_D || o == C_N || o == C_EQ || o == C_X) ? c2 >> 4 : 0; } else window = hd_max(window, p1 / 20);
		u32 contig, c;
		if (i1 < m1.n_cigar && (p1 + (i32) l1 < p2 + (i32) l2 || i2 >= m2.n_cigar)) { ++i1; if (l1 == 0) continue; c = c1; contig = (u32) m1.tid; p1 += (i32) l1; position = p1; }
		else if (i2 < m2.n_cigar) { ++i2; if (l2 == 0) continue; c = c2; contig = (u32) m2.tid; p2 += (i32) l2; position = p2; }
		else break;
		const u32 o = c & 15;
		const bool consumes_query = o == C_M || o == C_I || o == C_S || o == C_EQ || o == C_X;
		if (consumes_query) {
			while (window <= position / 20) {
				if (position - window * 20 >= 10) cov_increment(cov.counts, cov.off[contig] + (u64) window);
				++window;
			}
		} else window = position / 20;
	}
	if (!is_chimeric) {
		if ((f1 & BF_REVERSE) || !(f1 & BF_PAIRED)) cov.ends[cov.off[m1.tid] + (p1 - 1) / 20] = 1; else cov.ends[cov.off[m2.tid] + (p2 - 1) / 20] = 1;
	}
}

// What the counting pass decided for a record that reached the searches, indexed by store position (the writing pass replays from it):
//   bits 0-1: the tandem duplication found in the record's / its mate's soft clip (REC_LOG_TANDEM_*),
//   bits 2-3: the read-through branch taken (REC_RT_*), bits 4-5: the forward / reverse mate spans an intron at the gene boundary,
//   bits 16-31 / 32-47: the CIGAR operation of that intron in the forward / reverse mate (an index below n_cigar, which is 16 bits wide).
enum { REC_LOG_TANDEM_RECORD = 1, REC_LOG_TANDEM_MATE = 2, REC_LOG_RT_SHIFT = 2, REC_LOG_F_INTRON = 16, REC_LOG_R_INTRON = 32 };
enum { REC_RT_NONE = 0, REC_RT_FORWARD_INTRON = 1, REC_RT_REVERSE_INTRON = 2, REC_RT_INSIDE = 3 };
ARB_HD u64 rec_log_read_through(u32 branch, bool f_intron, bool r_intron, u32 fop, u32 rop) {
	return (u64) branch << REC_LOG_RT_SHIFT | (f_intron ? REC_LOG_F_INTRON : 0) | (r_intron ? REC_LOG_R_INTRON : 0) | (u64) (fop & 0xFFFFu) << 16 | (u64) (rop & 0xFFFFu) << 32;
}

// the gene ids that a point query of the gene index returns (query_index with start == end): the item list of one region, or none
struct rec_genes { const u32* v; u32 n; };
ARB_HD rec_genes rec_genes_at(const region_index_view& ix, u32 contig, i32 pos) {
	rec_genes g = {0, 0};
	if (contig >= ix.n_contigs) return g;
	const u32 lo = ix.begin[contig], hi = ix.begin[contig + 1];
	const u32 r = region_find(ix, contig, lo, hi, pos);
	if (r < hi) { g.v = ix.items + ix.off[r]; g.n = ix.off[r + 1] - ix.off[r]; }
	return g;
}

// What the replay keeps per key while it walks the key's records
struct rec_key_state {
	i32 waiting, waiting_c; // the first mate of a proper pair waiting for the second, in the main file's / the -c file's loop (-1: none)
	u32 c_n, c_rec[3];      // the alignments of the key's -c fragment (store items of the first three)
	u8 c_single_end; bool c_judged, c_kept; // c_kept: the first malformed pass keeps the -c fragment (once c_judged)
};
// the CIGAR operations of a stored record, read where they lie (the store keeps them behind the name, 4-byte alignment not guaranteed)
struct rec_cigar_ops { const u8* raw; ARB_HD u32 operator[](u32 k) const { return rec_rd32(raw + 4 * k); } };

// One thread per segment (run of equal key hashes). CAP bounds the gene sets of the read-through test, as the reference's fixed-capacity sets do: a segment
// whose sets exceed 32 ids is left untouched and marked in `big` for a second launch with the reference's capacity (1024), where more is the reference's
// fatal error. The sets are read in place from the gene index; CAP only decides which launch a segment belongs to.
// Counting pass (write == false): the searches, their log, the segment's tallies. Writing pass: the pools, the coverage, the counters.
// CHIMERIC_FILE: a -c file precedes the main file (its steps are compiled into these launches only: the launches of a run without one keep their registers).
template <int CAP, bool CHIMERIC_FILE = false> struct rec_replay_fn {
	rec_store_view s; const u32* seg_begin; const u32* list /* segments of this launch, NULL: all */; u8* big;
	annot_view an; rec_params prm; rec_cov_view cov;
	u32* tally /* RS_N rows of `stride` entries, one per segment */; const u32* bases /* the rows after their exclusive scans */; u32 stride;
	arb_pool_fragment* frags; arb_pool_alignment* alns; char* names; u32* cigars; u8* seqs;
	u64* log /* per store position: what the searches decided */; u64* counters; u64* error; bool write;
	u32* chimeric /* counting pass with a -c file: the keys' -c fragments that the first malformed pass rejects / keeps */;

	// the decision of the read-through test (read_chimeric_alignments.cpp:93-193) as a log entry; returns false and marks the segment when a gene set exceeds CAP
	ARB_HD bool decide_read_through(u32 k, const rec_t* a, const rec_t* b, u64& decision) const {
		decision = 0;
		const rec_t* fm = a; const rec_t* rm = b;
		if (fm->reverse()) { const rec_t* t = fm; fm = rm; rm = t; }
		const region_index_view gix = gene_index(an);
		const rec_genes fg = fm ? rec_genes_at(gix, (u32) fm->tid, fm->pos) : rec_genes_at(gix, (u32) rm->tid, rm->pos);
		const rec_genes rg = rm ? rec_genes_at(gix, (u32) rm->tid, rm->endpos()) : rec_genes_at(gix, (u32) fm->tid, fm->endpos());
		if (fg.n > (u32) CAP || rg.n > (u32) CAP) {
			if (CAP >= 1024) rec_atomic_min_u64(error, s.pos[k] << 3 | REC_ERR_ANNOTATION);
			return false;
		}
		if (sets_intersect(fg.v, fg.n, rg.v, rg.n) || (fg.n == 0 && rg.n == 0)) return true;
		i32 fgs, fge, rgs, rge;
		gene_set_extent(an, fg.v, fg.n, fgs, fge); gene_set_extent(an, rg.v, rg.n, rgs, rge);
		if (fge == -1) fge = rgs - 1;
		if (rgs == -1) rgs = fge + 1;
		u32 fop = 0, rop = 0; i32 fpos = 0, rpos = 0;
		const bool f_intron = fm ? spanning_intron(*fm, fge, rgs, fop, fpos) : false;
		const bool r_intron = rm ? spanning_intron(*rm, fge, rgs, rop, rpos) : false;
		u32 branch = REC_RT_NONE;
		if (f_intron && (!r_intron || fpos < rm->l_seq - rpos)) branch = REC_RT_FORWARD_INTRON;
		else if (r_intron) branch = REC_RT_REVERSE_INTRON;
		else if (fm && rm && rm->pos >= rgs && fm->endpos() <= fge) branch = REC_RT_INSIDE;
		decision = rec_log_read_through(branch, f_intron, r_intron, fop, rop);
		return true;
	}
	// the read-through fragment that `decision` calls for; returns whether the record is a read-through one
	ARB_HD bool emit_read_through(rec_emit& e, i64 hit_index, const rec_t* a, const rec_t* b, u64 decision) const {
		const rec_t* fm = a; const rec_t* rm = b;
		if (fm->reverse()) { const rec_t* t = fm; fm = rm; rm = t; }
		const u32 branch = (u32) (decision >> REC_LOG_RT_SHIFT) & 3u, fop = (u32) (decision >> 16) & 0xFFFFu, rop = (u32) (decision >> 32) & 0xFFFFu;
		const bool f_intron = decision & REC_LOG_F_INTRON, r_intron = decision & REC_LOG_R_INTRON;
		const rec_t& named = *a;
		if (branch == REC_RT_NONE) return false;
		bool created; const u32 f = e.fragment(named, hit_index, 0, &created);
		if (branch == REC_RT_FORWARD_INTRON) {
			if (!created) return false;
			e.add_alignment(f, *fm, false, fop + 1, 1);
			e.add_alignment(f, *fm, true, fop - 1, 2);
			if (rm) { if (r_intron) e.add_alignment(f, *rm, false, rop + 1, 1); else e.add_alignment(f, *rm, false); }
		} else if (branch == REC_RT_REVERSE_INTRON) {
			if (!created) return false;
			e.add_alignment(f, *rm, true, rop + 1, 1);
			e.add_alignment(f, *rm, false, rop - 1, 2);
			if (fm) { if (f_intron) e.add_alignment(f, *fm, false, fop - 1, 2); else e.add_alignment(f, *fm, false); }
		} else if (created) { e.add_alignment(f, *fm, false); e.add_alignment(f, *rm, false); }
		return true;
	}

	// A -c record (read_chimeric_alignments.cpp:627-631, 657-681, separate_chimeric_bam_file without is_rna_bam_file): a secondary alignment (0x100) is
	// added as a supplementary one at once; mates are collated in the -c file's own slot and added as (this record, its waiting mate); single-end records
	// are added as they come. A mate still waiting after the key's last -c record is dropped. No search, no coverage.
	ARB_HD void chimeric_add(rec_emit& e, rec_key_state& st, u32 k, const rec_t& r, bool supplementary) const {
		e.add_alignment(e.fragment(r, s.hit[k], 0, 0), r, supplementary);
		if (st.c_n < 3) st.c_rec[st.c_n] = k;
		++st.c_n; st.c_single_end = !(r.flag & BF_PAIRED);
	}
	ARB_HD void process_chimeric(rec_emit& e, u32 k, const rec_t& r, rec_key_state& st) const {
		e.chimeric_file = 1;
		if (r.flag & BF_SECONDARY) chimeric_add(e, st, k, r, true);
		else if (r.flag & BF_PAIRED) {
			if (st.waiting_c < 0) { st.waiting_c = (i32) k; e.chimeric_file = 0; return; }
			const u32 mk = (u32) st.waiting_c; st.waiting_c = -1;
			rec_t mate; s.get(mk, mate);
			chimeric_add(e, st, k, r, false); chimeric_add(e, st, mk, mate, false);
		} else chimeric_add(e, st, k, r, false);
		e.chimeric_file = 0;
		counters[REC_CTR_CHIMERIC] = 1; // in both passes: when the main file has a fatal error, the counting pass alone tells whether the -c file had chimeric reads
	}
	// Does the first pass of remove_malformed_alignments (after the -c file) keep the key's -c fragment? The rule of the fragment table (ft_decide), on
	// slots made from the stored records: a -c alignment is an unclipped copy of its record.
	ARB_HD bool chimeric_fragment_kept(const rec_key_state& st) const {
		const bool single_end = st.c_single_end != 0;
		if (!ft_count_ok(single_end, st.c_n)) return false;
		ft_slot_t<rec_cigar_ops> m[3];
#pragma unroll
		for (u32 x = 0; x < 3; ++x) {
			if (x >= st.c_n) break;
			rec_t r; s.get(st.c_rec[x], r);
			const bool supplementary = r.flag & BF_SECONDARY;
			m[x].contig = (u16) r.tid; m[x].supplementary = supplementary; m[x].first_in_pair = (r.flag & BF_READ1) ? 1 : 0; m[x].forward = !r.reverse();
			m[x].start = r.pos; m[x].end = r.endpos() - 1; m[x].seq_len = supplementary ? 0 : (u32) r.l_seq; m[x].seq_off = 0;
			m[x].cnt = r.n_cigar; m[x].ops.raw = r.cigar_raw; m[x].n_set = 0;
		}
		return ft_decide(single_end, st.c_n, m) != 0;
	}

	// one record of a key, in file order (read_chimeric_alignments.cpp:611-749): the -c file's records first, then the main file's. With a -c file the main
	// file's loop adds no supplementary, discordant or SA-tagged alignment (it still counts coverage for them), and its read-through fragments are inserted
	// only where the map holds no fragment of the key: the -c fragment counts only if the first malformed pass kept it.
	ARB_HD bool process(rec_emit& e, u32 k, rec_key_state& st) const {
		rec_t r; s.get(k, r);
		if (CHIMERIC_FILE && s.from_chimeric_file(k)) { process_chimeric(e, k, r, st); return true; }
		if (CHIMERIC_FILE && !st.c_judged) {
			st.c_judged = true; st.c_kept = st.c_n > 0 && chimeric_fragment_kept(st);
			if (st.c_n > 0 && !st.c_kept) e.id[0] = -1; // erased: a read-through fragment may take its name (the build drops the rejected one)
		}
		const i64 hit_index = s.hit[k];
		if (r.flag & BF_SUPPLEMENTARY) {
			if (CHIMERIC_FILE) return true;
			if (clipped_at_correct_end(r)) e.add_alignment(e.fragment(r, hit_index, 0, 0), r, true);
			else if (write) rec_atomic_add_u64(&counters[REC_CTR_MALFORMED], 1);
			if (write) counters[REC_CTR_CHIMERIC] = 1;
			return true;
		}
		if ((r.flag & BF_PAIRED) && !(r.flag & BF_PROPER)) { // discordant mate
			if (!CHIMERIC_FILE) e.add_alignment(e.fragment(r, hit_index, 0, 0), r, false);
			if (write) {
				if (!CHIMERIC_FILE) counters[REC_CTR_CHIMERIC] = 1;
				if (!prm.external_duplicate_marking || !(r.flag & BF_DUP)) add_coverage(cov, r, 0, true, true); // all flag bits cleared (`flag &= !BAM_FPAIRED`)
			}
			return true;
		}
		rec_t mate; const rec_t* m = 0; u32 mk = 0;
		if (r.flag & BF_PAIRED) { // the first mate of a proper pair waits for the second
			if (st.waiting < 0) { st.waiting = (i32) k; return true; }
			mk = (u32) st.waiting; st.waiting = -1;
			s.get(mk, mate); m = &mate;
		}
		u64 decision = write ? log[k] : 0;
		tandem_t t;
		if (!write) {
			if (!clipped_sequence_is_adapter(r, m) && (!m || r.reverse() != m->reverse())) {
				if (tandem_duplication(an, prm.max_itd_length, &r, t)) decision = REC_LOG_TANDEM_RECORD;
				else if (tandem_duplication(an, prm.max_itd_length, m, t)) decision = REC_LOG_TANDEM_MATE;
			}
		} else if (decision & REC_LOG_TANDEM_RECORD) tandem_duplication(an, prm.max_itd_length, &r, t); // a hit is rare: its search runs again to rebuild it
		else if (decision & REC_LOG_TANDEM_MATE) tandem_duplication(an, prm.max_itd_length, m, t);
		const bool tandem_from_mate = decision & REC_LOG_TANDEM_MATE, is_tandem = decision & (REC_LOG_TANDEM_RECORD | REC_LOG_TANDEM_MATE);
		if (is_tandem) {
			const u32 f = e.fragment(r, hit_index, 1, 0);
			e.add_alignment(f, r, (!r.reverse()) == t.forward && !t.supplementary);
			if (m) e.add_alignment(f, *m, (!m->reverse()) == t.forward && !t.supplementary);
			arb_pool_alignment a; a.supplementary = t.supplementary; a.first_in_pair = t.first_in_pair; a.forward = t.forward; a.contig = t.contig; a.start = t.start; a.end = t.end;
			a.seq_off = 0; a.seq_len = 0;
			if (!t.supplementary) { const rec_t& src = tandem_from_mate ? *m : r; a.seq_off = e.store_seq(src); a.seq_len = (u32) src.l_seq; }
			a.cigar_off = e.base[RS_CIGARS] + e.n[RS_CIGARS]; for (u32 x = 0; x < t.n_cigar; ++x) e.push_cigar(t.cigar[x]); a.cigar_cnt = t.n_cigar;
			e.link(f, a);
		}
		bool is_read_through = false;
		if ((s.sa[k] && clipped_at_correct_end(r)) || (m && s.sa[mk] && clipped_at_correct_end(*m))) {
			if (!CHIMERIC_FILE) {
				const u32 f = e.fragment(r, hit_index, 0, 0);
				e.add_alignment(f, r, false);
				if (m) e.add_alignment(f, *m, false);
				if (write) counters[REC_CTR_CHIMERIC] = 1;
			}
		} else if (!is_tandem) {
			if (!write) {
				u64 rt;
				if (!decide_read_through(k, &r, m, rt)) return false;
				decision |= rt;
			}
			is_read_through = emit_read_through(e, hit_index, &r, m, decision);
			if (write && prm.viral[r.tid]) {
				if (pristine(r)) rec_atomic_add_u64(&counters[REC_CTR_VIRAL + r.tid], 1);
				if (m && pristine(*m)) rec_atomic_add_u64(&counters[REC_CTR_VIRAL + m->tid], 1);
			}
		}
		if (!write) log[k] = decision;
		if (write && (!prm.external_duplicate_marking || !(r.flag & BF_DUP))) add_coverage(cov, r, m, is_read_through, false);
		return true;
	}

	ARB_HD void operator()(u32 i) const {
		const u32 seg = list ? list[i] : i;
		if (!list && big[seg]) return; // left to the launch with the larger sets
		rec_emit e;
		e.frags = write ? frags : 0; e.alns = alns; e.names = names; e.cigars = cigars; e.seqs = seqs; e.chimeric_file = 0;
		for (u32 q = 0; q < RS_N; ++q) { e.base[q] = write ? bases[q * stride + seg] : 0; e.n[q] = 0; }
		const u32 lo = seg_begin[seg], hi = seg_begin[seg + 1];
		u32 c_rejected = 0, c_kept = 0;
		// Every key of the segment (keys with one hash: names compared exactly), in the order of their first records. Quadratic in the segment's length:
		// with 64-bit hashes a segment is one key's 2-4 records (keys sharing a hash are rare); only the ARB_KEY_HASH_BITS test hook makes segments long.
		for (u32 x = lo; x < hi; ++x) {
			const u32 kx = s.order[x];
			bool seen = false;
			for (u32 y = lo; y < x && !seen; ++y) seen = s.same_key(s.order[y], kx);
			if (seen) continue;
			e.id[0] = e.id[1] = -1;
			rec_key_state st = {-1, -1, 0, {0, 0, 0}, 0, false, false}; // mates still waiting at the end: dropped
			for (u32 y = x; y < hi; ++y) {
				const u32 ky = s.order[y];
				if (y != x && !s.same_key(kx, ky)) continue;
				if (!process(e, ky, st)) { big[seg] = 1; return; }
			}
			if (CHIMERIC_FILE && !write && st.c_n > 0) { // the first pass's verdict on the key's -c fragment, also for keys without main-file records
				const bool kept = st.c_judged ? st.c_kept : chimeric_fragment_kept(st);
				if (kept) ++c_kept; else ++c_rejected;
			}
		}
		if (!write) for (u32 q = 0; q < RS_N; ++q) tally[q * stride + seg] = e.n[q];
		if (CHIMERIC_FILE && !write) { if (c_rejected) atomic_add_u32(&chimeric[0], c_rejected); if (c_kept) atomic_add_u32(&chimeric[1], c_kept); } // the segment is complete
	}
};

} // namespace arb
