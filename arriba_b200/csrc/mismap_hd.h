// mismap_hd.h -- k-mer index of fused genes, gene homology and re-alignment of supporting reads ("mismappers").
//
// Reference behaviour: make_kmer_index (filter_mismappers.cpp:47-84), kmer_to_int (:33-45), align (:86-187), align_both_strands
// (:189-230), extend_split_read (:247-270), filter_mismappers (:272-359), is_homolog (filter_homologs.cpp:13-63).
// The reference's per-contig unordered_map<kmer, vector<position>> becomes one position array sorted by (contig, 8-mer, position)
// with a dense bucket-offset table (65,536 buckets per contig), so a lookup is two loads.
#pragma once
#include "model.h"
#include "annot_hd.h"
#include "prims.h"
#include "read_filters.h"
#include <math.h>

namespace arb {

ARB_HD u32 base2(char c) { return c == 'T' ? 0u : c == 'G' ? 1u : c == 'C' ? 2u : 3u; } // every other character (A, N, IUPAC) is 3
ARB_HD char complement_char(char c) { switch (c) { case 'A': return 'T'; case 'T': return 'A'; case 'C': return 'G'; case 'G': return 'C'; default: return c; } }

// A bucket holds the positions of one 8-mer on a whole contig (hundreds of entries once half of a chromosome is indexed), while a search only wants the
// hits at or after a lower bound inside one gene window. block_first answers that without a binary search over the bucket: the contig is cut into blocks
// of 2^block_shift bases, and block_first[(first block of the contig + b) << 16 | 8-mer] is the index of the bucket's first position >= b << block_shift
// (the bucket's end if there is none): one load, then a step or two forward.
struct kmer_index_view {
	const i32* pos;          // positions sorted by (contig, 8-mer, position)
	const u32* bucket_off;   // n_index_contigs * 65536 + 1
	u32 n_index_contigs;     // contigs >= this have no index (kmer_indices.size() in the reference)
	const u32* block_first; const u32* contig_block_base; u32 block_shift;
	ARB_HD void bucket(u32 contig, u32 kmer, u32& lo, u32& hi) const { const u64 b = (u64) contig * 65536 + kmer; lo = bucket_off[b]; hi = bucket_off[b + 1]; }
	// first entry of the bucket [lo, hi) of (contig, kmer) whose position is >= from (an empty index has no blocks, but then every bucket is empty)
	ARB_HD u32 first_at_or_after(u32 contig, u32 kmer, u32 lo, u32 hi, i32 from) const {
		if (from <= 0 || lo == hi) return lo;
		u32 h = block_first[((u64) contig_block_base[contig] + ((u32) from >> block_shift)) << 16 | kmer];
		while (h < hi && pos[h] < from) ++h;
		return h;
	}
};
// index construction: the block table
struct block_first_min_fn { // entry idx of the sorted index: the smallest index per (block, 8-mer)
	const u32* key /* contig << 16 | 8-mer */; const i32* pos; const u32* contig_block_base; u32 block_shift; u32* block_first;
	ARB_HD void operator()(u32 idx) const { const u32 contig = key[idx] >> 16, km = key[idx] & 0xffffu; atomic_min_u32(&block_first[((u64) contig_block_base[contig] + ((u32) pos[idx] >> block_shift)) << 16 | km], idx); }
};
struct block_first_sweep_fn { // thread per (contig, 8-mer): blocks without an entry point at the next later entry of the bucket
	const u32* bucket_off; const u32* contig_block_base; u32* block_first;
	ARB_HD void operator()(u32 t) const {
		const u32 contig = t >> 16, km = t & 0xffffu;
		u32 next = bucket_off[(u64) contig * 65536 + km + 1];
		for (u32 b = contig_block_base[contig + 1]; b-- > contig_block_base[contig]; ) { u32& v = block_first[(u64) b << 16 | km]; if (v == 0xFFFFFFFFu) v = next; else next = v; }
	}
};

// ---- index construction
struct interval_view { const u32* contig; const i32* start; const i32* end /* exclusive */; const u32* first /* prefix sum of lengths, n+1 */; u32 n; };
ARB_HD u32 interval_of(const interval_view& iv, u32 j) { u32 lo = 0, hi = iv.n; while (hi - lo > 1) { u32 mid = (lo + hi) >> 1; if (iv.first[mid] <= j) lo = mid; else hi = mid; } return lo; }
struct kmer_flag_fn { // candidate position j: is it indexed? (first base not 'N')
	interval_view iv; annot_view an; u32* flag;
	ARB_HD void operator()(u32 j) const {
		const u32 t = interval_of(iv, j); const i32 p = iv.start[t] + (i32) (j - iv.first[t]);
		flag[j] = an.assembly[an.contig_seq_off[iv.contig[t]] + (u32) p] != 'N';
	}
};
struct kmer_emit_fn { // key = contig << 16 | 8-mer
	interval_view iv; annot_view an; const u32* flag_scan; u32* key; u32* pos;
	ARB_HD void operator()(u32 j) const {
		if (flag_scan[j + 1] == flag_scan[j]) return;
		const u32 t = interval_of(iv, j); const i32 p = iv.start[t] + (i32) (j - iv.first[t]);
		const char* s = an.assembly + an.contig_seq_off[iv.contig[t]] + (u32) p;
		u32 k = 0;
		for (u32 b = 0; b < 8; ++b) k = k << 2 | base2(s[b]);
		key[flag_scan[j]] = iv.contig[t] << 16 | k; pos[flag_scan[j]] = (u32) p;
	}
};
struct bucket_count_fn { const u32* key; u32* count; ARB_HD void operator()(u32 j) const { atomic_add_u32(&count[key[j]], 1); } };

// ---- sequences to re-align: a slice of a stored read, optionally reverse-complemented
struct read_slice { const u8* nt16; u32 off; u32 len; bool rc; };

ARB_HD u32 lower_bound_i32(const i32* v, u32 lo, u32 hi, i32 x) { while (lo < hi) { u32 mid = lo + ((hi - lo) >> 1); if (v[mid] < x) lo = mid + 1; else hi = mid; } return lo; }

// complement of an nt16 code the way the reference complements characters (A<->T, C<->G, everything else unchanged; assembly.hpp:9-22)
ARB_HD u32 nt16_comp(u32 code) { return (u32) (0xFEDCBA9176523480ull >> (4 * code)) & 15u; }
// 2-bit code of a base for the 8-mer index: T=0 G=1 C=2, anything else 3 (filter_mismappers.cpp:33-45); table indexed by the nt16 code
ARB_HD u32 nt16_base2(u32 code) { return 0xFFFCFDEFu >> (2 * code) & 3u; }

// Everything one re-alignment keeps fixed across the searches of a (segment, gene, strand): the top-level search and its continuations.
struct realign_env {
	const u8* seq; u32 off, len; bool rc;        // the read slice
	const i32* pos; const u32* bucket;           // k-mer hits and the 65,536 bucket offsets of the window's contig
	const u32* block_first; u32 block_shift;     // the contig's part of the block table (kmer_index_view)
	const i32* splice; u32 n_splice;             // downstream splice sites of the gene
	i32 wstart, wend;                            // gene +- padding
	int min_score;
	const u32* g4; const char* ref;              // reference of the contig: packed nt16 codes, or characters when g4 == 0
};
// the index part of the env: hits, bucket offsets and block table of one (indexed) contig
ARB_HD void env_index(const kmer_index_view& ix, u32 contig, realign_env& env) {
	env.pos = ix.pos; env.bucket = ix.bucket_off + (u64) contig * 65536;
	env.block_first = ix.block_first + ((u64) ix.contig_block_base[contig] << 16); env.block_shift = ix.block_shift;
}
// first hit of the non-empty bucket [lo, hi) of `km` at or after gene_pos
ARB_HD u32 env_first_hit(const realign_env& env, u32 km, u32 lo, u32 hi, i32 gene_pos) {
	if (gene_pos <= 0) return lo;
	u32 h = env.block_first[(u64) ((u32) gene_pos >> env.block_shift) << 16 | km];
	while (h < hi && env.pos[h] < gene_pos) ++h;
	return h;
}
ARB_HD u32 env_code(const u8* seq, u32 off, u32 len, bool rc, u32 r) { // nt16 code of base r of the (possibly reverse-complemented) slice
	const u32 code = nt16_at(seq, rc ? off + len - 1 - r : off + r);
	return rc ? nt16_comp(code) : code;
}
ARB_HD bool env_ref_equals(const u32* g4, const char* ref, i32 g, u32 code) {
	return g4 ? (g4[(u32) g >> 3] >> (28 - 4 * ((u32) g & 7)) & 15u) == code : ref[g] == nt16_char(code);
}

// Work control of pass 2 and the task rounds. The reference's align() is a pure "does ANY placement reach min_score" search: the outcome is the OR over all
// (read position, k-mer hit) pairs and over the continuations they start (at a splice site, at the first mismatch), so the pairs may be visited in any order
// and by any number of threads.
//  * lanes/lane/counter: `lanes` threads of the same search deal its hits round-robin (realign_search);
//  * stop: set as soon as any lane (or any other item of the same fragment) found a placement.
//  * table: a continuation is not run by the thread that meets it. It is REGISTERED in a hash table under (item, segment, gene, strand, score, read position,
//    deletions left) with the smallest lower bound requested so far, and the caller goes on as if it had failed (valid: the answer is an OR). After the pass,
//    every entry whose bound went down becomes one task; a group of lanes deals that task's hits and registers the continuations IT meets. A continuation
//    only looks at hits at or above its bound, so the entry with the smallest bound answers for all the others: a read in a tandem repeat reaches the same
//    (score, read position) from thousands of hits, and that is one task instead of thousands of identical searches. A registration that finds no room
//    drops the continuation and marks the item incomplete: the driver re-runs the incomplete items with a larger table.
//  * memo: a continuation is a pure function of (score, read position, deletions left, lower bound of the hits) and it only ever looks at hits at or
//    above the lower bound. Once it has failed for a bound g it fails for every bound >= g. In a tandem repeat thousands of hits reach the same
//    (score, read position) with ascending bounds: the first one registers, the others are answered from a small per-thread table without the atomics.
struct realign_task { u32 item; u16 gene_k; u8 segment, rc; i32 score, read_pos, gene_pos, max_deletions; u32 item_slot; };
struct continuation_slot { u64 key; i32 want /* smallest lower bound requested */, done /* bound already turned into a task */; };
// key of a continuation, never 0: cooperative item (24 bits) | segment | strand | deletions left (2) | gene of the segment (16) | score + 512 (10) | read
// position (9). Every field fits: fewer than 2^24 items are re-aligned cooperatively, genes_cnt is a u16, and realign_can_start keeps the continuations of a
// read under 300 bases within scores -316 .. 300 and read positions below 300.
ARB_HD u64 continuation_key(const realign_task& t) {
	return 1ull << 63 | (u64) t.item_slot << 39 | (u64) t.segment << 38 | (u64) t.rc << 37 | (u64) (u32) t.max_deletions << 35 | (u64) t.gene_k << 19 | (u64) (u32) (t.score + 512) << 9 | (u64) (u32) t.read_pos;
}
ARB_HD void continuation_unpack(u64 key, realign_task& t) {
	t.item_slot = (u32) (key >> 39) & 0xFFFFFFu; t.segment = (u8) (key >> 38 & 1); t.rc = (u8) (key >> 37 & 1); t.max_deletions = (i32) (key >> 35 & 3); t.gene_k = (u16) (key >> 19 & 0xFFFF);
	t.score = (i32) (key >> 9 & 1023) - 512; t.read_pos = (i32) (key & 511);
}
// the registry of one attempt at the cooperative items: table_slots is a power of two; incomplete (per item slot) = a registration of the item did not fit
struct continuation_registry { continuation_slot* table; u32 table_slots; u32* overflow /* registrations that did not fit */; u8* incomplete; };
struct realign_memo { i32 score, read_pos, max_deletions, fail_from; };
struct realign_ctl {
	enum { MEMO_SLOTS = 16 };
	realign_memo memo[MEMO_SLOTS]; u32 memo_n, memo_next;
	ARB_HD void forget() { memo_n = 0; memo_next = 0; } // new gene window or strand: different function
	ARB_HD bool known_to_fail(int score, int read_pos, int max_deletions, int gene_pos) const {
		for (u32 k = 0; k < memo_n; ++k) if (memo[k].score == score && memo[k].read_pos == read_pos && memo[k].max_deletions == max_deletions) return gene_pos >= memo[k].fail_from;
		return false;
	}
	ARB_HD void remember_failure(int score, int read_pos, int max_deletions, int gene_pos) {
		for (u32 k = 0; k < memo_n; ++k) if (memo[k].score == score && memo[k].read_pos == read_pos && memo[k].max_deletions == max_deletions) { if (gene_pos < memo[k].fail_from) memo[k].fail_from = gene_pos; return; }
		const u32 slot = memo_n < MEMO_SLOTS ? memo_n++ : (memo_next++ % MEMO_SLOTS);
		memo[slot].score = score; memo[slot].read_pos = read_pos; memo[slot].max_deletions = max_deletions; memo[slot].fail_from = gene_pos;
	}
	u32 lanes, lane, counter;
	const volatile u8* stop;
	continuation_registry reg; realign_task proto; // proto: item / segment / gene / strand of the running search
	ARB_HD void spawn(int score, int read_pos, int gene_pos, int max_deletions) { // registers the continuation, or drops it and marks the item incomplete
		realign_task t = proto; t.score = score; t.read_pos = read_pos; t.max_deletions = max_deletions;
		const u64 key = continuation_key(t);
		u64 h = key * 0x9E3779B97F4A7C15ULL; h ^= h >> 29;
		for (u32 probe = 0; probe < 256; ++probe) {
			continuation_slot& s = reg.table[(h + probe) & (reg.table_slots - 1)];
			const u64 seen = atomic_cas_u64(&s.key, 0, key);
			if (seen == 0 || seen == key) { atomic_min_i32(&s.want, gene_pos); return; }
		}
		atomic_add_u32(reg.overflow, 1);
		reg.incomplete[proto.item_slot] = 1;
	}
	// the continuation sink of realign_extend
	ARB_HD void operator()(int score, int read_pos, int gene_pos, int max_deletions) {
		if (known_to_fail(score, read_pos, max_deletions, gene_pos)) return; // an identical continuation with a lower or equal bound is registered already
		spawn(score, read_pos, gene_pos, max_deletions);
		remember_failure(score, read_pos, max_deletions, gene_pos);
	}
};
ARB_HD realign_ctl registry_ctl(u32 lanes, u32 lane, const u8* stop, const continuation_registry& reg) { realign_ctl c; c.forget(); c.lanes = lanes; c.lane = lane; c.counter = 0; c.stop = stop; c.reg = reg; return c; }

struct gene_splice_view { const u32* off; const i32* sites; }; // per gene: sorted downstream splice sites (filter_mismappers.cpp:16-31)

// One of the two sequences of a work item that is re-aligned against the genes of the OTHER breakpoint (filter_mismappers.cpp:189-230, :296-333)
struct realign_segment {
	read_slice read; int read_length; bool same_contig; i32 aln_start, aln_end; const u32* genes; u32 n_genes; float min_align_fraction;
	ARB_HD int min_score() const {
#ifdef __CUDA_ARCH__
		return (int) ((double) __fmul_rn(min_align_fraction, (float) read.len) + 0.5);
#else
		volatile float prod = min_align_fraction * (float) read.len;
		return (int) ((double) prod + 0.5);
#endif
	}
};
// window, index and splice sites of gene k of the segment; false if the reference skips this gene (:204-214)
ARB_HD bool segment_env(const realign_segment& s, u32 k, int max_mate_gap, const annot_view& an, const kmer_index_view& ix, const gene_splice_view& sp, realign_env& env) {
	const u32 g = s.genes[k];
	const u32 contig = an.gene_contig[g];
	env.wstart = hd_max(an.gene_start[g] - max_mate_gap - s.read_length, 0);
	env.wend = hd_min(an.gene_end[g] + max_mate_gap + s.read_length, (i32) an.contig_len[contig] - 1);
	if (s.same_contig && ((s.aln_start >= env.wstart && s.aln_start <= env.wend) || (s.aln_end >= env.wstart && s.aln_end <= env.wend))) return false;
	if (contig >= ix.n_index_contigs) return false;
	env.seq = s.read.nt16; env.off = s.read.off; env.len = s.read.len; env.rc = s.read.rc;
	env_index(ix, contig, env);
	env.splice = sp.sites + sp.off[g]; env.n_splice = sp.off[g + 1] - sp.off[g];
	env.min_score = s.min_score();
	env.g4 = an.assembly4 ? an.assembly4 + an.contig_seq_off[contig] / 8 : 0; env.ref = an.assembly + an.contig_seq_off[contig];
	return true;
}

// test hook (arb_selftest_kmer_lookup): per query (contig, 8-mer, lower bound) the bucket [lo, hi) and the first hit at or after the bound, found twice:
// through kmer_index_view::first_at_or_after (gene homology) and through env_first_hit (re-alignment); out = lo, hi, hit, its position (~0 if none) x 2
struct kmer_lookup_fn {
	kmer_index_view ix; const u32* contig; const u32* kmer; const i32* from; u32* out;
	ARB_HD void operator()(u32 j) const {
		u32 lo, hi; ix.bucket(contig[j], kmer[j], lo, hi);
		const u32 h1 = ix.first_at_or_after(contig[j], kmer[j], lo, hi, from[j]);
		realign_env env; env_index(ix, contig[j], env);
		const u32 h2 = lo == hi ? lo : env_first_hit(env, kmer[j], lo, hi, from[j]);
		u32* o = out + 6 * (size_t) j;
		o[0] = lo; o[1] = hi; o[2] = h1; o[3] = h1 < hi ? (u32) ix.pos[h1] : ~0u; o[4] = h2; o[5] = h2 < hi ? (u32) ix.pos[h2] : ~0u;
	}
};

struct mismap_params { i32 max_mate_gap; float max_mismapper_fraction; };

// one work item = one (candidate, listed fragment) pair
// what pass 1 looked at, for the SURVEY.md section 8(d) byte budget of the re-alignment: sequences searched (segment x gene x strand), their bases, k-mer hits visited
struct realign_tally { u32 sequences, bases, hits; };
struct mismap_items {
	frag_view f; annot_view an; kmer_index_view ix; gene_splice_view sp; mismap_params p;
	const u32* item_cand; const u32* item_frag; const u8* item_kind /* 0 split read, 1 discordant */; const u16* cand_contig1; const u16* cand_contig2; const u8* cand_filter;
	u8* mismapper; // per fragment, set to 1 when any evaluation says "mis-mapped"
	unsigned long long* tallies; // 0, or 3 * TALLY_SLOTS counters (sequences, bases, hits), spread over slots to keep the atomics apart
	enum { TALLY_SLOTS = 1024 };
	ARB_HD bool skip(u32 j) const { return cand_filter[item_cand[j]] != F_none || f.filter[item_frag[j]] != F_none; }
	// segment 0 / 1 of item j: split read -> clipped part vs. the genes of the split read's anchor side, then mate1 (+ aligned part) vs. the genes of the
	// supplementary; discordant mates -> each mate vs. the genes of the other (filter_mismappers.cpp:296-333)
	ARB_HD realign_segment segment(u32 j, u32 x) const {
		const u32 cand = item_cand[j], i = item_frag[j];
		realign_segment s;
		s.same_contig = cand_contig1[cand] == cand_contig2[cand];
		s.read.rc = false;
		if (item_kind[j] == 0) {
			const u32 m = f.idx(i, MATE1), sr = f.idx(i, SPLIT_READ), u = f.idx(i, SUPPLEMENTARY);
			const u32 slen = f.seq_len[sr], mlen = f.seq_len[m];
			s.min_align_fraction = 0.8f;
			if (x == 0) {
				s.read.nt16 = f.sq(sr);
				if (f.fwd(sr)) { s.read.off = 0; s.read.len = hd_min(f.preclip(sr), slen); } else { const u32 post = hd_min(f.postclip(sr), slen); s.read.off = slen - post; s.read.len = post; }
				s.read_length = (int) slen; s.aln_start = f.start[u]; s.aln_end = f.end[u]; s.genes = f.genes + f.genes_off[sr]; s.n_genes = f.genes_cnt[sr];
			} else {
				s.read.nt16 = f.sq(m);
				if (f.fwd(sr)) { const u32 pre = hd_min(f.preclip(m), mlen); s.read.off = pre; s.read.len = mlen - pre; } else { const u32 mpost = hd_min(f.postclip(m), mlen); s.read.off = 0; s.read.len = mlen - mpost; }
				s.read_length = (int) mlen; s.aln_start = f.start[m]; s.aln_end = f.end[m]; s.genes = f.genes + f.genes_off[u]; s.n_genes = f.genes_cnt[u];
			}
		} else {
			const u32 a = f.idx(i, x == 0 ? MATE1 : MATE2), b = f.idx(i, x == 0 ? MATE2 : MATE1);
			const float clipped = ((float) f.preclip(a) + f.postclip(a)) / f.seq_len[a];
			s.min_align_fraction = hd_min(0.8f, 0.8f * (1 - clipped));
			s.read.nt16 = f.sq(a); s.read.off = 0; s.read.len = f.seq_len[a];
			s.read_length = (int) f.seq_len[a]; s.aln_start = f.start[a]; s.aln_end = f.end[a]; s.genes = f.genes + f.genes_off[b]; s.n_genes = f.genes_cnt[b];
		}
		return s;
	}
};

// ---- pass 1: a GROUP of lanes per item, continuations on a worklist -----------------------------------------------------------------------------------
// The search is an OR over (read position, k-mer hit) pairs and over the continuations they start (a continuation = the same search from a later read
// position with a lower bound on the hits). Read positions are independent of each other -- score and skipped bases at position p follow from p alone -- so
// the lanes of a group take the positions of a search in turn, and a continuation is not called but pushed on the group's small worklist (shared memory)
// and searched by the whole group later. No per-thread memo in local memory; the order of evaluation differs from the reference's, the result (an OR) does
// not. An item that overflows the worklist or the step budget goes to the cooperative pass 2.
struct realign_work { i32 gene_pos; i16 score; u16 read_pos; u16 gene_k; u8 segment, rc_deletions /* bit 7 strand, bits 0..6 deletions left */; };
struct realign_worklist { realign_work* tasks; u32* top; u32 capacity; };
ARB_HD u32 worklist_fetch_add(u32* p, u32 v) {
#ifdef __CUDA_ARCH__
	return atomicAdd(p, v);
#else
	const u32 old = *p; *p = old + v; return old;
#endif
}
ARB_HD bool realign_can_start(int score, int read_pos, int len, int min_score) { return read_pos + 8 < len && read_pos + min_score <= len + score + 16; } // filter_mismappers.cpp:90-94
struct worklist_push { // the continuation sink of pass 1: a continuation of `current` goes on the group's worklist
	const realign_worklist& wl; const realign_work& current;
	ARB_HD void operator()(int score, int read_pos, int gene_pos, int max_deletions) const {
		const u32 slot = worklist_fetch_add(wl.top, 1);
		if (slot >= wl.capacity) return; // noticed by the group when it reads `top` next: the item goes to pass 2
		realign_work t = current; t.score = (i16) score; t.read_pos = (u16) read_pos; t.gene_pos = gene_pos; t.rc_deletions = (u8) ((current.rc_deletions & 0x80u) | (u32) max_deletions);
		wl.tasks[slot] = t;
	}
};
// 8-mer (2 bits per base) of the read slice at position r, on the strand of the search
ARB_HD u32 env_kmer(const realign_env& env, u32 r) {
	if (!env.rc) return nt16_dense2(nt16_window(env.seq, 0x7fffffffu, (i32) (env.off + r)));
	// reverse strand: bases r..r+7 are the complements of the stored bases off+len-1-r .. off+len-8-r: bit reversal of the word reverses the order of the nibbles
	// and complements A/C/G/T/N; every other code keeps more than one bit and maps to 3 like the character it stands for
	return nt16_dense2(brev32(nt16_window(env.seq, 0x7fffffffu, (i32) (env.off + env.len - 8 - r))));
}
enum { REALIGN_UNDECIDED_NO = 0, REALIGN_FOUND = 1, REALIGN_EXHAUSTED = 2 };
// Eight bases of the read slice (on the strand of the search, from base r0) against eight reference bases from g0, in one XOR of packed words:
// bit 28 - 4j of `differs` is set where base r0 + j differs from reference base g0 + j. false = this stretch has to be compared base by base (no packed
// reference, or -- reverse strand -- an ambiguity code among the `cnt` bases in question: the reference complements A/C/G/T only, assembly.hpp:9-22, while
// the bit reversal that complements a whole word would turn R into Y).
ARB_HD bool env_differs8(const realign_env& env, int r0, int g0, int first, int cnt, u32& differs) { // bases first .. first + cnt - 1 of the window matter
	if (!env.g4 || g0 < 0) return false;
	u32 rw;
	if (!env.rc) rw = nt16_window(env.seq, 0x7fffffffu, (i32) env.off + r0);
	else {
		const u32 w0 = nt16_window(env.seq, 0x7fffffffu, (i32) (env.off + env.len) - 8 - r0); // stored bases, in stored order: window base j is nibble 7 - j of w0
		const u32 s2 = (w0 & 0x55555555u) + (w0 >> 1 & 0x55555555u), c4 = (s2 & 0x33333333u) + (s2 >> 2 & 0x33333333u); // bits set per nibble: 1 (A/C/G/T) or 4 (N) are fine
		const u32 odd = (c4 ^ (c4 >> 2)) & 0x11111111u;   // nibble count 1 -> 1, 4 -> 1, 0 / 2 -> 0, 3 -> 1 ...
		const u32 three = c4 & (c4 >> 1) & 0x11111111u;    // ... except 3
		const u32 simple = odd & ~three;                   // bit 4k: nibble k holds A, C, G, T or N
		const u32 wanted = (cnt >= 8 ? 0x11111111u : ((0x11111111u >> (32 - 4 * cnt)))) << (4 * first); // window bases first .. first+cnt-1 = nibbles first .. of w0 (reversed order)
		if ((simple & wanted) != wanted) return false;
		rw = brev32(w0);
	}
	const u32 x = rw ^ packed_window(env.g4, (u64) (u32) g0);
	differs = (x | x >> 1 | x >> 2 | x >> 3) & 0x11111111u;
	return true;
}
// The extension of one (read position, k-mer hit) pair of the search that starts at (score0, read_pos0, max_deletions) (filter_mismappers.cpp:86-187), in every
// pass: true as soon as the placement reaches min_score. A continuation it meets -- at a splice site, and one deletion at the first mismatch -- is not run
// here but handed to `sink(score, read_pos, gene_pos, max_deletions)` unless it would stop at once: pass 1 pushes it on the group's worklist, pass 2 and the
// task rounds register it (realign_ctl).
template <class Sink> ARB_HD bool realign_extend(const realign_env& env, int score0, int read_pos0, int max_deletions, int read_pos, int hit, Sink& sink, u32& steps) {
	const u8* const seq = env.seq; const u32 off = env.off; const bool rc = env.rc; const int len = (int) env.len;
	const i32 wstart = env.wstart, wend = env.wend; const int min_score = env.min_score;
	const u32* const g4 = env.g4; const char* const ref = env.ref;
	const bool leading = read_pos0 == 0; // every base before the seed was skipped: no penalty for them (local alignment start)
	const int skipped = read_pos - read_pos0, score = score0 - skipped;
	++steps;
	int ext = score + 8;
	if (leading) ext += skipped;
	if (ext >= min_score) return true;
	{ // extend to the left over the skipped bases, one mismatch allowed; eight bases per packed comparison where that is possible
		int r = read_pos - 1, gp = hit - 1; u32 mm = 0;
		const int r_stop = read_pos - skipped;
		bool open = true;
		while (open && r >= r_stop && gp >= wstart) {
			const int cnt = hd_min(8, hd_min(r - r_stop + 1, gp - wstart + 1)); // bases r, r-1, ... r-cnt+1 = window bases 7 .. 8-cnt of the window that starts at r - 7
			u32 differs;
			if (env_differs8(env, r - 7, gp - 7, 8 - cnt, cnt, differs)) {
				for (int j = 7; j > 7 - cnt; --j) {
					if (!(differs >> (28 - 4 * j) & 1u)) { ext += leading ? 1 : 2; if (ext >= min_score) return true; }
					else if (++mm > 1) { open = false; break; }
				}
				r -= cnt; gp -= cnt;
			} else {
				if (env_ref_equals(g4, ref, gp, env_code(seq, off, (u32) len, rc, (u32) r))) { ext += leading ? 1 : 2; if (ext >= min_score) return true; }
				else if (++mm > 1) break;
				--r; --gp;
			}
		}
	}
	{ // extend to the right; a spliced continuation at splice sites and one deletion at the first mismatch go to the sink
		int r = read_pos + 8, gp = hit + 8; u32 mm = 0, consecutive = 0;
		u32 ss = lower_bound_i32(env.splice, 0, env.n_splice, gp - 1);
		i32 next_site = ss < env.n_splice ? env.splice[ss] : 0x7fffffff;
		while (r < len && gp <= wend) {
			int cnt = hd_min(8, hd_min(len - r, wend - gp + 1));
			u32 differs;
			if (!env_differs8(env, r, gp, 0, cnt, differs)) { cnt = 1; differs = env_ref_equals(g4, ref, gp, env_code(seq, off, (u32) len, rc, (u32) r)) ? 0u : 0x10000000u; }
			for (int j = 0; j < cnt; ++j, ++r, ++gp) {
				++steps;
				if (gp - 1 >= next_site) {
					if (gp - 1 > next_site) { ++ss; next_site = ss < env.n_splice ? env.splice[ss] : 0x7fffffff; }
					if (gp - 1 == next_site && realign_can_start(ext, r, len, min_score)) sink(ext, r, gp, max_deletions);
				}
				if (!(differs >> (28 - 4 * j) & 1u)) { ++ext; if (ext >= min_score) return true; consecutive = 0; }
				else {
					if (++mm == 1 && max_deletions > 0 && len >= 30 && realign_can_start(ext, r, len, min_score)) sink(ext, r, gp, max_deletions - 1);
					--ext;
					if (++consecutive >= 4) return false;
				}
			}
		}
	}
	return false;
}
// One search (top level or continuation) by the lanes of a group: the lanes take the read positions in turn (score and skipped bases at a position follow
// from the position alone); a lane looks up its position's 8-mer, finds the first hit at or after the lower bound through the block table and extends
// every hit inside the window. Returns REALIGN_FOUND on the lane that reached min_score (the caller combines the lanes).
ARB_HD u32 realign_group(const lane_group& g, const realign_env& env, const realign_work& task, const realign_worklist& wl, u32& steps, u32& hits) {
	const int len = (int) env.len;
	const i32* const pos = env.pos; const u32* const bucket = env.bucket;
	const i32 wend = env.wend; const int min_score = env.min_score;
	const int read_pos0 = task.read_pos, score0 = task.score, gene_pos = task.gene_pos, max_deletions = task.rc_deletions & 0x7f;
	worklist_push sink = {wl, task};
	for (int read_pos = read_pos0 + (int) g.lane; ; read_pos += (int) g.lanes) {
		if (!realign_can_start(score0 - (read_pos - read_pos0), read_pos, len, min_score)) return REALIGN_UNDECIDED_NO; // the valid positions are a prefix
		const u32 km = env_kmer(env, (u32) read_pos);
		const u32 lo = bucket[km], hi = bucket[km + 1];
		if (lo == hi) continue;
		for (u32 h = env_first_hit(env, km, lo, hi, gene_pos); h < hi; ++h) {
			const int hit = pos[h];
			if (hit >= wend) break;
			++hits;
			if (realign_extend(env, score0, read_pos0, max_deletions, read_pos, hit, sink, steps)) return REALIGN_FOUND;
		}
	}
}
// One search (top level or continuation) in pass 2 and the task rounds: every lane walks the read positions, and the hits of each position are dealt
// round-robin to the `lanes` threads of the search, continuing the deal of the previous positions (ctl.counter) so that positions with few hits do not all
// fall to the first lanes. Continuations go to the registry.
ARB_HD bool realign_search(const realign_env& env, int score0, int read_pos0, int gene_pos, int max_deletions, realign_ctl& ctl) {
	const i32* const pos = env.pos;
	u32 steps = 0; // pass 1's budget; not counted here
	for (int read_pos = read_pos0; realign_can_start(score0 - (read_pos - read_pos0), read_pos, (int) env.len, env.min_score); ++read_pos) {
		const u32 km = env_kmer(env, (u32) read_pos);
		const u32 lo = env.bucket[km], hi = env.bucket[km + 1];
		if (lo == hi) continue;
		if (*ctl.stop) return false;
		u32 h = env_first_hit(env, km, lo, hi, gene_pos);
		const u32 n_hits = lower_bound_i32(pos, h, hi, env.wend) - h;
		h += (ctl.lane + ctl.lanes - ctl.counter % ctl.lanes) % ctl.lanes;
		ctl.counter += n_hits;
		for (; h < hi; h += ctl.lanes) {
			const int hit = pos[h];
			if (hit >= env.wend) break;
			if (realign_extend(env, score0, read_pos0, max_deletions, read_pos, hit, ctl, steps)) return true;
		}
	}
	return false;
}

// filter_mismappers.cpp:247-270: can the clipped segment simply be extended along the reference? The lanes of the group share the clipped bases.
ARB_HD bool extends_linearly_group(const lane_group& g, const frag_view& f, const annot_view& an, u32 a /* SPLIT_READ */) {
	const u8* seq = f.sq(a); const u32 len = f.seq_len[a];
	const char* ref = an.assembly + an.contig_seq_off[f.contig[a]]; const i32 clen = (i32) an.contig_len[f.contig[a]];
	int n; u32 matches = 0;
	if (f.fwd(a)) {
		const u32 pre = f.preclip(a);
		n = hd_min((int) pre, f.start[a]);
		for (int i = (int) g.lane; i < n; i += (int) g.lanes) if (nt16_char(nt16_at(seq, pre - n + i)) == ref[f.start[a] - n + i]) ++matches;
	} else {
		const u32 post = f.postclip(a);
		n = hd_min((int) post, clen - f.end[a] - 2);
		if (n < 0) n = (int) post; // clipped segment runs over the contig end: the reference compares the whole clipped segment (std::string::substr with a huge count)
		for (int i = (int) g.lane; i < n; i += (int) g.lanes) { const i32 gp = f.end[a] + 1 + i; if (gp < clen && nt16_char(nt16_at(seq, len - post + i)) == ref[gp]) ++matches; }
	}
	matches = g.sum(matches);
#ifdef __CUDA_ARCH__
	return (double) matches >= floor((double) __fmul_rn((float) (u32) n, 0.7f));
#else
	volatile float prod = (float) (u32) n * 0.7f;
	return (double) matches >= floor((double) prod);
#endif
}

// one item by a group: 0 = not mis-mapped, 1 = mis-mapped, 2 = gave up (worklist or budget), re-aligned cooperatively in pass 2
ARB_HD u32 evaluate_group(const lane_group& g, const mismap_items& it, u32 j, const realign_worklist& wl, int budget, realign_tally& tally) {
	if (g.lane == 0) *wl.top = 0;
	g.sync();
	if (it.item_kind[j] == 0 && extends_linearly_group(g, it.f, it.an, it.f.idx(it.item_frag[j], SPLIT_READ))) return REALIGN_FOUND;
	// top-level searches: both sequences of the item against every gene of the other breakpoint, both strands (filter_mismappers.cpp:189-230, :296-333)
	u32 n = 0; bool too_many = false;
	for (u32 x = 0; x < 2 && !too_many; ++x) {
		const realign_segment s = it.segment(j, x);
		if (s.read.len >= 300) continue;
		for (u32 k = 0; k < s.n_genes; ++k) {
			realign_env env;
			if (!segment_env(s, k, it.p.max_mate_gap, it.an, it.ix, it.sp, env)) continue;
			if (!realign_can_start(0, 0, (int) env.len, env.min_score)) continue;
			if (n + 2 > wl.capacity || k >= 0xFFFFu) { too_many = true; break; }
			tally.sequences += 2; tally.bases += 2 * env.len;
			if (g.lane == 0) {
				realign_work t; t.gene_pos = env.wstart; t.score = 0; t.read_pos = 0; t.gene_k = (u16) k; t.segment = (u8) x; t.rc_deletions = 1;
				wl.tasks[n] = t; t.rc_deletions = 0x81; wl.tasks[n + 1] = t;
			}
			n += 2;
		}
	}
	if (too_many) return REALIGN_EXHAUSTED;
	if (g.lane == 0) *wl.top = n;
	g.sync();
	u32 total_steps = 0;
	for (;;) {
		const u32 top = *(volatile u32*) wl.top;
		if (top == 0) return REALIGN_UNDECIDED_NO;
		if (top > wl.capacity) return REALIGN_EXHAUSTED; // a continuation did not fit
		const realign_work task = wl.tasks[top - 1];
		g.sync();
		if (g.lane == 0) *wl.top = top - 1;
		g.sync();
		const realign_segment s = it.segment(j, task.segment);
		realign_env env;
		segment_env(s, task.gene_k, it.p.max_mate_gap, it.an, it.ix, it.sp, env); // it was usable when the task was made
		if (task.rc_deletions & 0x80u) env.rc = !s.read.rc;
		u32 steps = 0;
		const u32 verdict = realign_group(g, env, task, wl, steps, tally.hits);
		if (g.any(verdict == REALIGN_FOUND)) return REALIGN_FOUND;
		total_steps += g.sum(steps);
		if (budget > 0 && total_steps > (u32) budget) return REALIGN_EXHAUSTED;
		g.sync();
	}
}

// pass 1, one lane per item (host build; the device runs k_mismap_items with groups of lanes)
struct mismap_item_group_fn {
	mismap_items it; int budget; u32* heavy; u32* n_heavy;
	ARB_HD void operator()(u32 j) const {
		if (it.skip(j)) return;
		const u32 i = it.item_frag[j];
		if (((const volatile u8*) it.mismapper)[i]) return;
		realign_work tasks[64]; u32 top = 0;
		realign_worklist wl = {tasks, &top, 64};
		lane_group g; g.lane = 0; g.lanes = 1; g.mask = 1;
		realign_tally tally = {0, 0, 0};
		const u32 verdict = evaluate_group(g, it, j, wl, budget, tally);
		if (it.tallies) { unsigned long long* t = it.tallies + 3 * (j % mismap_items::TALLY_SLOTS); t[0] += tally.sequences; t[1] += tally.bases; t[2] += tally.hits; }
		if (verdict == REALIGN_FOUND) it.mismapper[i] = 1;
		else if (verdict == REALIGN_EXHAUSTED) heavy[atomic_add_u32(n_heavy, 1)] = j;
	}
};
// pass 2: `lanes` threads per queued item share the top-level k-mer hits of both sequences of the item against every gene of the other breakpoint, both
// strands (filter_mismappers.cpp:189-230, :296-333; pass 1 has tried the linear extension); continuations go to the registry
struct mismap_heavy_fn {
	mismap_items it; const u32* heavy; u32 lanes; u32 first_slot; continuation_registry reg;
	ARB_HD void operator()(u32 t) const {
		const u32 slot = first_slot + t / lanes, j = heavy[slot], i = it.item_frag[j];
		realign_ctl ctl = registry_ctl(lanes, t % lanes, it.mismapper + i, reg); ctl.proto.item = j; ctl.proto.item_slot = slot;
		if (*ctl.stop) return;
		for (u32 x = 0; x < 2; ++x) {
			const realign_segment s = it.segment(j, x);
			if (s.read.len >= 300) continue;
			for (u32 k = 0; k < s.n_genes; ++k) {
				realign_env env;
				if (!segment_env(s, k, it.p.max_mate_gap, it.an, it.ix, it.sp, env)) continue;
				ctl.proto.segment = (u8) x; ctl.proto.gene_k = (u16) k;
				for (u32 strand = 0; strand < 2; ++strand) {
					env.rc = strand ? !s.read.rc : s.read.rc; ctl.proto.rc = (u8) strand; ctl.forget();
					if (realign_search(env, 0, 0, env.wstart, 1, ctl)) { it.mismapper[i] = 1; return; }
				}
			}
		}
	}
};
struct continuation_init_fn { continuation_slot* tables; ARB_HD void operator()(u32 k) const { tables[k].key = 0; tables[k].want = 0x7fffffff; tables[k].done = 0x7fffffff; } };
// between rounds: every registered continuation whose bound went down since it last ran becomes a task
struct continuation_collect_fn {
	continuation_slot* tables; u32 table_slots; const u32* heavy; const u32* item_frag; const u8* mismapper; realign_task* tasks; u32* n_tasks;
	ARB_HD void operator()(u32 k) const {
		continuation_slot& s = tables[k];
		if (s.key == 0 || s.want >= s.done) return;
		s.done = s.want;
		realign_task t; t.gene_pos = s.want;
		continuation_unpack(s.key, t);
		t.item = heavy[t.item_slot];
		if (mismapper[item_frag[t.item]]) return; // already decided
		tasks[append_slot(n_tasks)] = t;
	}
};
// task rounds: `lanes` threads per registered continuation
struct mismap_task_fn {
	mismap_items it; const realign_task* tasks; u32 lanes; continuation_registry reg;
	ARB_HD void operator()(u32 t) const {
		const realign_task task = tasks[t / lanes];
		const u32 i = it.item_frag[task.item];
		realign_ctl ctl = registry_ctl(lanes, t % lanes, it.mismapper + i, reg); ctl.proto = task;
		if (*ctl.stop) return;
		const realign_segment s = it.segment(task.item, task.segment);
		realign_env env;
		if (!segment_env(s, task.gene_k, it.p.max_mate_gap, it.an, it.ix, it.sp, env)) return;
		if (task.rc) env.rc = !s.read.rc;
		if (realign_search(env, task.score, task.read_pos, task.gene_pos, task.max_deletions, ctl)) it.mismapper[i] = 1;
	}
};
// after the rounds: the items a registration failed for whose fragment is still undecided, to be re-aligned again with a larger registry
struct incomplete_collect_fn {
	const u8* incomplete; const u32* heavy; const u32* item_frag; const u8* mismapper; u32* redo; u32* n_redo;
	ARB_HD void operator()(u32 slot) const { if (incomplete[slot] && !mismapper[item_frag[heavy[slot]]]) redo[append_slot(n_redo)] = heavy[slot]; }
};

struct mismap_apply_fn { const u8* mismapper; u8* filter; ARB_HD void operator()(u32 i) const { if (mismapper[i] && filter[i] == F_none) filter[i] = F_mismappers; } };

// filter_mismappers.cpp:232-244, 336-356: recount and discard candidates supported mostly by mis-mapped reads
struct mismap_count_fn {
	const u8* frag_filter; const u32* l1o; const u32* l1; const u32* l2o; const u32* l2; const u32* ldo; const u32* ld;
	u32* sr1; u32* sr2; u32* dm; u8* cand_filter; float max_fraction;
	ARB_HD void scan(const u32* off, const u32* list, u32 cand, u32& count, u32& mism, u32& total) const {
		for (u32 p = off[cand]; p < off[cand + 1]; ++p) {
			const u8 fl = frag_filter[list[p]];
			if (fl == F_none) ++total;
			else if (fl == F_mismappers) { ++total; ++mism; if (count > 0) --count; }
		}
	}
	ARB_HD void operator()(u32 cand) const {
		if (cand_filter[cand] != F_none) return;
		u32 mism = 0, total = 0, a = sr1[cand], b = sr2[cand], c = dm[cand];
		scan(l1o, l1, cand, a, mism, total); scan(l2o, l2, cand, b, mism, total); scan(ldo, ld, cand, c, mism, total);
		sr1[cand] = a; sr2[cand] = b; dm[cand] = c;
		mism &= 0xFFFF; total &= 0xFFFF; // the reference counts in unsigned short
#ifdef __CUDA_ARCH__
		const double limit = floor((double) __fmul_rn(max_fraction, (float) total));
#else
		volatile float prod = max_fraction * (float) total; const double limit = floor((double) prod);
#endif
		if (mism > 0 && (double) mism >= limit) cand_filter[cand] = F_mismappers;
	}
};

// work items of the re-alignment: every listed fragment of every unfiltered candidate
struct item_count_fn { const u8* cand_filter; const u32* l1o; const u32* l2o; const u32* ldo; u32* count; ARB_HD void operator()(u32 c) const { count[c] = cand_filter[c] != F_none ? 0 : (l1o[c + 1] - l1o[c]) + (l2o[c + 1] - l2o[c]) + (ldo[c + 1] - ldo[c]); } };
struct item_fill_fn {
	const u8* cand_filter; const u32* l1o; const u32* l1; const u32* l2o; const u32* l2; const u32* ldo; const u32* ld; const u32* item_off; u32* item_cand; u32* item_frag; u8* item_kind;
	ARB_HD void operator()(u32 c) const {
		if (cand_filter[c] != F_none) return;
		u32 w = item_off[c];
		for (u32 p = l1o[c]; p < l1o[c + 1]; ++p, ++w) { item_cand[w] = c; item_frag[w] = l1[p]; item_kind[w] = 0; }
		for (u32 p = l2o[c]; p < l2o[c + 1]; ++p, ++w) { item_cand[w] = c; item_frag[w] = l2[p]; item_kind[w] = 0; }
		for (u32 p = ldo[c]; p < ldo[c + 1]; ++p, ++w) { item_cand[w] = c; item_frag[w] = ld[p]; item_kind[w] = 1; }
	}
};

// ---- gene homology (filter_homologs.cpp:13-63): fraction of the small gene's 8-mers (stride 8) that occur, with 8 more matching bases, in the big gene
struct homolog_pair { // the comparison of one gene pair, set up once
	bool comparable; u32 sc, bc, len; i32 ss, se, bs, be, blen; bool rc; const char* sref; const char* bref; float threshold;
	ARB_HD char small_at(u32 i) const { return rc ? complement_char(sref[ss + (i32) (len - 1 - i)]) : sref[ss + (i32) i]; } // base i of the small gene's (possibly reverse-complemented) sequence
};
ARB_HD homolog_pair homolog_setup(const annot_view& an, const kmer_index_view& ix, u32 g1, u32 g2, float max_identity) {
	homolog_pair p; p.comparable = false;
	if (g1 == g2) return p;
	u32 sm = g1, bg = g2;
	if ((u32) (an.gene_end[sm] - an.gene_start[sm]) > (u32) (an.gene_end[bg] - an.gene_start[bg])) { sm = g2; bg = g1; }
	p.sc = an.gene_contig[sm]; p.bc = an.gene_contig[bg];
	p.ss = an.gene_start[sm]; p.se = an.gene_end[sm]; p.bs = an.gene_start[bg]; p.be = an.gene_end[bg];
	if (p.sc == p.bc && ((p.ss >= p.bs && p.ss <= p.be) || (p.se >= p.bs && p.se <= p.be))) return p;
	if (p.bc >= ix.n_index_contigs) return p;
	p.len = (u32) (p.se - p.ss);
	p.rc = an.gene_strand[sm] != an.gene_strand[bg];
	p.sref = an.assembly + an.contig_seq_off[p.sc]; p.bref = an.assembly + an.contig_seq_off[p.bc]; p.blen = (i32) an.contig_len[p.bc];
#ifdef __CUDA_ARCH__
	p.threshold = __fmul_rn((float) p.len, max_identity);
#else
	volatile float threshold_v = (float) p.len * max_identity; p.threshold = threshold_v;
#endif
	p.comparable = true;
	return p;
}
// does the 8-mer at `pos` of the small gene occur in the big gene followed by the same 8 bases? (filter_homologs.cpp:36-55)
ARB_HD bool homolog_position_matches(const homolog_pair& p, const kmer_index_view& ix, u32 pos) {
	u32 k = 0;
	for (u32 b = 0; b < 8; ++b) k = k << 2 | base2(p.small_at(pos + b));
	u32 lo, hi; ix.bucket(p.bc, k, lo, hi);
	for (u32 h = ix.first_at_or_after(p.bc, k, lo, hi, p.bs); h < hi && ix.pos[h] <= p.be; ++h) {
		const i32 hit = ix.pos[h];
		if (!(p.sc != p.bc || hit < p.ss || hit > p.se)) continue;
		bool same = true;
		for (u32 b = 0; b < 8 && same; ++b) { const i32 g = hit + 8 + (i32) b; const char x = g < p.blen ? p.bref[g] : '\0'; if (x != p.small_at(pos + 8 + b)) same = false; }
		if (same) return true;
	}
	return false;
}
ARB_HD bool genes_are_homologs(const annot_view& an, const kmer_index_view& ix, u32 g1, u32 g2, float max_identity) {
	const homolog_pair p = homolog_setup(an, ix, g1, g2, max_identity);
	if (!p.comparable) return false;
	u32 matching = 0;
	for (u32 pos = 0; pos + 16 < p.len; pos += 8) {
		if ((float) (matching * 8 + (p.len - pos)) < p.threshold) return false;
		if (homolog_position_matches(p, ix, pos)) { ++matching; if ((float) (matching * 8) >= p.threshold) return true; }
	}
	return false;
}
struct homolog_pairs_fn { annot_view an; kmer_index_view ix; const u32* ga; const u32* gb; u8* out; float max_identity; ARB_HD void operator()(u32 j) const { out[j] = genes_are_homologs(an, ix, ga[j], gb[j], max_identity); } };
// The same verdict from `lanes` threads per pair. The sequential loop above answers "does the number of matching positions, times 8, reach the threshold":
// its early `false` only fires when even a match at every remaining position could not reach it, its early `true` when the count has reached it. So the
// positions may be counted in any order: lane l takes positions 8 * (l + lanes * i), the counts are added up, one more thread per pair decides.
struct homolog_count_fn {
	annot_view an; kmer_index_view ix; const u32* ga; const u32* gb; u32* count; u32 lanes; float max_identity;
	ARB_HD void operator()(u32 t) const {
		const u32 j = t / lanes, lane = t % lanes;
		const homolog_pair p = homolog_setup(an, ix, ga[j], gb[j], max_identity);
		if (!p.comparable) return;
		u32 matching = 0;
		for (u32 pos = 8 * lane; pos + 16 < p.len; pos += 8 * lanes) if (homolog_position_matches(p, ix, pos)) ++matching;
		if (matching) atomic_add_u32(&count[j], matching);
	}
};
struct homolog_decide_fn {
	annot_view an; kmer_index_view ix; const u32* ga; const u32* gb; const u32* count; u8* out; float max_identity;
	ARB_HD void operator()(u32 j) const {
		const homolog_pair p = homolog_setup(an, ix, ga[j], gb[j], max_identity);
		out[j] = p.comparable && count[j] > 0 && (float) (count[j] * 8) >= p.threshold;
	}
};

} // namespace arb
