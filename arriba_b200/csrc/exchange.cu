// exchange.cu -- one sample on several GPUs: what a context exposes so that a transport (NCCL through torch.distributed in arriba_b200/sharded.py, any
// other in another launcher) can replicate and combine device-resident state, device to device. The library never calls a communication library itself.
//
// Design (SURVEY.md section 8e, DESIGN.md section 7): the fragment table is REPLICATED -- the rank that ingested the BAM broadcasts its resident columns
// over NVLink/NVSwitch (a few GB, milliseconds) -- and the WORK is sharded:
//   * find_fusions by contig pair: a rank only emits the breakpoint records of the fragments whose contig-pair component it owns (arb_set_work_partition),
//     so it finds exactly the candidates of those pairs, with GLOBAL fragment ids; one all-gather of the packed candidate tables follows and every rank
//     merges them into the table a single GPU would have built (candidates ordered by the fragment that created them, then by local id);
//   * filter_mismappers by work item: rank r re-aligns items r, r+W, ... and the per-fragment verdict bytes are combined by a MAX all-reduce
//     (filter_mismappers.cpp:232-244 counts verdicts, their order is irrelevant).
// Exchange groups (broadcast from the owning rank): the sender describes a group by a header of 64-bit words, the receiver sizes its buffers from it, both
// sides then list the same device buffers in the same order.
#include "engine.h"
#include "fusions_hd.h"

namespace arb {

enum { XG_CONTIGS = 0, XG_ANNOTATION = 1, XG_TABLE = 2, XG_MISMAP_STATE = 3, XG_COUNT = 4 };

template <class T> static void add_buf(std::vector<exchange_buffer>& out, dbuf<T>& b, u64 n) { exchange_buffer x = {(void*) b.ptr(), n * sizeof(T)}; out.push_back(x); }

void engine::exchange_header(int group, std::vector<u64>& h) {
	h.clear();
	h.push_back((u64) group);
	switch (group) {
		case XG_CONTIGS:
			if (!has_contigs) throw arb_error("exchange: no contig table to send");
			h.push_back(annot.n_contigs); h.push_back(annot.assembly_bytes); h.push_back(annot.assembly4_words); h.push_back(annot.assembly4_ok ? 1 : 0);
			break;
		case XG_ANNOTATION:
			if (!has_annotation) throw arb_error("exchange: no annotation to send");
			h.push_back(annot.n_genes); h.push_back(annot.n_exons); h.push_back(annot.n_contigs); h.push_back(annot.n_exon_regions); h.push_back(annot.n_exon_items);
			h.push_back(annot.n_gene_regions); h.push_back(annot.n_gene_items);
			break;
		case XG_TABLE:
			if (push_open) throw arb_error("exchange: the fragment table is not complete");
			h.push_back(frags.n); h.push_back(frags.max_seq_len); h.push_back(frags.canonical_seq_layout ? 1 : 0); h.push_back(frags.n_seq_bytes); h.push_back(push_cigar_ops);
			h.push_back(n_gene_entries); h.push_back(push_alignments); h.push_back(push_bases);
			break;
		case XG_MISMAP_STATE:
			h.push_back(cands.n); h.push_back(cands.n_list1); h.push_back(cands.n_list2); h.push_back(frags.n); h.push_back(kmer_indexed); h.push_back(kmer_index_contigs);
			h.push_back(annot.n_genes); h.push_back(n_splice_sites); h.push_back(has_splice_sites ? 1 : 0); h.push_back(kmer_block_shift); h.push_back(kmer_blocks);
			break;
		default: throw arb_error("exchange: unknown group");
	}
}

void engine::exchange_prepare(int group, const u64* h, u32 n_words) {
	if (n_words < 1 || (int) h[0] != group) throw arb_error("exchange: header does not belong to the group");
	auto need = [&](u32 k) { if (n_words < k) throw arb_error("exchange: truncated header"); };
	switch (group) {
		case XG_CONTIGS:
			need(5);
			annot.n_contigs = (u32) h[1]; annot.assembly_bytes = h[2]; annot.assembly4_words = h[3]; annot.assembly4_ok = h[4] != 0;
			annot.assembly.ensure(annot.assembly_bytes + 64); annot.assembly4.ensure(annot.assembly4_words);
			annot.contig_flags.ensure(annot.n_contigs); annot.contig_len.ensure(annot.n_contigs); annot.contig_seq_off.ensure(annot.n_contigs);
			break;
		case XG_ANNOTATION:
			need(8);
			annot.n_genes = (u32) h[1]; annot.n_exons = (u32) h[2]; annot.n_contigs = (u32) h[3]; annot.n_exon_regions = (u32) h[4]; annot.n_exon_items = (u32) h[5];
			annot.n_gene_regions = (u32) h[6]; annot.n_gene_items = (u32) h[7];
			annot.gene_contig.ensure(annot.n_genes); annot.gene_start.ensure(annot.n_genes); annot.gene_end.ensure(annot.n_genes); annot.gene_strand.ensure(annot.n_genes);
			annot.gene_exonic_length.ensure(annot.n_genes); annot.gene_flags.ensure(annot.n_genes);
			annot.exon_gene.ensure(annot.n_exons); annot.exon_start.ensure(annot.n_exons); annot.exon_end.ensure(annot.n_exons); annot.exon_cds_start.ensure(annot.n_exons);
			annot.exon_cds_end.ensure(annot.n_exons); annot.exon_next_start.ensure(annot.n_exons); annot.exon_flags.ensure(annot.n_exons);
			annot.exon_region_begin.ensure((size_t) annot.n_contigs + 1); annot.exon_region_end.ensure(annot.n_exon_regions); annot.exon_region_off.ensure((size_t) annot.n_exon_regions + 1);
			annot.exon_region_items.ensure(annot.n_exon_items);
			annot.gene_region_begin.ensure((size_t) annot.n_contigs + 1); annot.gene_region_end.ensure(annot.n_gene_regions); annot.gene_region_off.ensure((size_t) annot.n_gene_regions + 1);
			annot.gene_region_items.ensure(annot.n_gene_items);
			break;
		case XG_TABLE: {
			need(9);
			ex.sync(); // kernels of the previous sample may still read the buffers
			const u32 n = (u32) h[1]; const size_t A = 3 * (size_t) n;
			frags.n = n; frags.max_seq_len = (u32) h[2]; frags.canonical_seq_layout = h[3] != 0; frags.n_seq_bytes = h[4]; push_cigar_ops = h[5]; n_gene_entries = h[6];
			push_alignments = h[7]; push_bases = h[8];
			frags.n_aln.ensure(n); frags.fflags.ensure(n); frags.filter.ensure(n); frags.early.ensure(n); frags.swapped.ensure(n);
			frags.aflags.ensure(A); frags.contig.ensure(A); frags.start.ensure(A); frags.end.ensure(A); frags.cigar_off.ensure(A); frags.cigar_cnt.ensure(A);
			frags.seq_off.ensure(2 * (size_t) n); frags.seq_len.ensure(2 * (size_t) n); frags.genes_off.ensure(A); frags.genes_cnt.ensure(A);
			frags.cigar.ensure(push_cigar_ops + 1); frags.seq.ensure(frags.n_seq_bytes); frags.genes.ensure(n_gene_entries + 1);
			break;
		}
		case XG_MISMAP_STATE: {
			need(12);
			if ((u32) h[1] != cands.n || (u32) h[4] != frags.n) throw arb_error("exchange: re-alignment state of another candidate table / fragment table");
			cands.n_list1 = h[2]; cands.n_list2 = h[3];
			cands.list1.ensure(cands.n_list1); cands.list2.ensure(cands.n_list2);
			kmer_indexed = h[5]; kmer_index_contigs = (u32) h[6];
			kmer_pos.ensure(kmer_indexed); kmer_bucket_off.ensure((size_t) kmer_index_contigs * 65536 + 2);
			if ((u32) h[7] != annot.n_genes) throw arb_error("exchange: re-alignment state of another annotation");
			n_splice_sites = h[8];
			splice_off.ensure((size_t) annot.n_genes + 1); splice_sites.ensure(n_splice_sites);
			has_splice_sites = h[9] != 0;
			kmer_block_shift = (u32) h[10]; kmer_blocks = (u32) h[11];
			kmer_block_base.ensure((size_t) kmer_index_contigs + 1); kmer_block_first.ensure((u64) kmer_blocks << 16);
			break;
		}
		default: throw arb_error("exchange: unknown group");
	}
}

void engine::exchange_buffers(int group, std::vector<exchange_buffer>& out) {
	out.clear();
	switch (group) {
		case XG_CONTIGS:
			add_buf(out, annot.assembly, annot.assembly_bytes); add_buf(out, annot.assembly4, annot.assembly4_words);
			add_buf(out, annot.contig_flags, annot.n_contigs); add_buf(out, annot.contig_len, annot.n_contigs); add_buf(out, annot.contig_seq_off, annot.n_contigs);
			break;
		case XG_ANNOTATION:
			add_buf(out, annot.gene_contig, annot.n_genes); add_buf(out, annot.gene_start, annot.n_genes); add_buf(out, annot.gene_end, annot.n_genes); add_buf(out, annot.gene_strand, annot.n_genes);
			add_buf(out, annot.gene_exonic_length, annot.n_genes); add_buf(out, annot.gene_flags, annot.n_genes);
			add_buf(out, annot.exon_gene, annot.n_exons); add_buf(out, annot.exon_start, annot.n_exons); add_buf(out, annot.exon_end, annot.n_exons); add_buf(out, annot.exon_cds_start, annot.n_exons);
			add_buf(out, annot.exon_cds_end, annot.n_exons); add_buf(out, annot.exon_next_start, annot.n_exons); add_buf(out, annot.exon_flags, annot.n_exons);
			add_buf(out, annot.exon_region_begin, (u64) annot.n_contigs + 1); add_buf(out, annot.exon_region_end, annot.n_exon_regions); add_buf(out, annot.exon_region_off, (u64) annot.n_exon_regions + 1);
			add_buf(out, annot.exon_region_items, annot.n_exon_items);
			add_buf(out, annot.gene_region_begin, (u64) annot.n_contigs + 1); add_buf(out, annot.gene_region_end, annot.n_gene_regions); add_buf(out, annot.gene_region_off, (u64) annot.n_gene_regions + 1);
			add_buf(out, annot.gene_region_items, annot.n_gene_items);
			break;
		case XG_TABLE: {
			const u64 n = frags.n, A = 3 * n;
			add_buf(out, frags.n_aln, n); add_buf(out, frags.fflags, n); add_buf(out, frags.filter, n);
			add_buf(out, frags.aflags, A); add_buf(out, frags.contig, A); add_buf(out, frags.start, A); add_buf(out, frags.end, A); add_buf(out, frags.cigar_off, A); add_buf(out, frags.cigar_cnt, A);
			add_buf(out, frags.seq_off, 2 * n); add_buf(out, frags.seq_len, 2 * n); add_buf(out, frags.genes_off, A); add_buf(out, frags.genes_cnt, A);
			add_buf(out, frags.cigar, push_cigar_ops); add_buf(out, frags.seq, frags.n_seq_bytes); add_buf(out, frags.genes, n_gene_entries);
			break;
		}
		case XG_MISMAP_STATE: {
			const u64 C = cands.n;
			add_buf(out, cands.filter, C); add_buf(out, cands.split_reads1, C); add_buf(out, cands.split_reads2, C); add_buf(out, cands.discordant_mates, C);
			add_buf(out, cands.list1_off, C + 1); add_buf(out, cands.list1, cands.n_list1); add_buf(out, cands.list2_off, C + 1); add_buf(out, cands.list2, cands.n_list2);
			add_buf(out, frags.filter, frags.n);
			add_buf(out, kmer_pos, kmer_indexed); add_buf(out, kmer_bucket_off, (u64) kmer_index_contigs * 65536 + 2);
			add_buf(out, splice_off, (u64) annot.n_genes + 1); add_buf(out, splice_sites, n_splice_sites);
			add_buf(out, kmer_block_base, (u64) kmer_index_contigs + 1); add_buf(out, kmer_block_first, (u64) kmer_blocks << 16);
			break;
		}
		default: throw arb_error("exchange: unknown group");
	}
}

void engine::exchange_commit(int group) {
	switch (group) {
		case XG_CONTIGS:
			annot.h_contig_flags.resize(annot.n_contigs); annot.h_contig_len.resize(annot.n_contigs);
			annot.contig_flags.download(ex, annot.h_contig_flags.data(), annot.n_contigs); annot.contig_len.download(ex, annot.h_contig_len.data(), annot.n_contigs);
			has_contigs = true; table_n = 0;
			break;
		case XG_ANNOTATION:
			annot.h_gene_contig.resize(annot.n_genes); annot.h_gene_start.resize(annot.n_genes); annot.h_gene_end.resize(annot.n_genes); annot.h_gene_strand.resize(annot.n_genes); annot.h_gene_flags.resize(annot.n_genes);
			annot.gene_contig.download(ex, annot.h_gene_contig.data(), annot.n_genes); annot.gene_start.download(ex, annot.h_gene_start.data(), annot.n_genes);
			annot.gene_end.download(ex, annot.h_gene_end.data(), annot.n_genes); annot.gene_strand.download(ex, annot.h_gene_strand.data(), annot.n_genes);
			annot.gene_flags.download(ex, annot.h_gene_flags.data(), annot.n_genes);
			has_annotation = true;
			break;
		case XG_TABLE:
			frags.swapped.zero(ex, frags.n);
			push_open = true; // finish_push closes it
			finish_push(n_gene_entries);
			filters_done = false; cands.n = 0; cands.genomic_marked = false; has_tag_csr = false;
			ex.sync();
			break;
		case XG_MISMAP_STATE: ex.sync(); break;
		default: throw arb_error("exchange: unknown group");
	}
}

// ------------------------------------------------------------------------------------------- work partition of find_fusions
// owner of a fragment = owner of the contig pair its candidates live in (host/shard.cpp computes the pairs, links pairs that share duplicates and balances them)
struct owned_fn {
	frag_view f; const u32* keys; const u8* owner; u32 n_keys; u8 part; u8* owned;
	ARB_HD static u32 pair_key(u32 a, u32 b) { return a < b ? a << 16 | b : b << 16 | a; }
	ARB_HD void operator()(u32 i) const {
		const u32 key = f.n_aln[i] == 3 ? pair_key(f.contig[f.idx(i, 1)], f.contig[f.idx(i, 2)]) : pair_key(f.contig[f.idx(i, 0)], f.contig[f.idx(i, 1)]);
		u32 lo = 0, hi = n_keys;
		while (lo < hi) { const u32 mid = lo + ((hi - lo) >> 1); if (keys[mid] < key) lo = mid + 1; else hi = mid; }
		owned[i] = (lo < n_keys && keys[lo] == key && owner[lo] == part) ? 1 : 0;
	}
};

void engine::set_work_partition(const u32* keys, const u8* owner, u32 n_keys, int part, int parts) {
	work_part = part; work_parts = parts;
	if (parts <= 1) { work_owned.release(); return; }
	if (part < 0 || part >= parts || parts > 255) throw arb_error("arb_set_work_partition: invalid part");
	dbuf<u32> d_keys; dbuf<u8> d_owner;
	d_keys.upload(ex, keys, n_keys); d_owner.upload(ex, owner, n_keys);
	work_owned.ensure(frags.n);
	owned_fn fn = {frags.view(), d_keys.ptr(), d_owner.ptr(), n_keys, (u8) part, work_owned.ptr()};
	for_each(ex, frags.n, fn);
	ex.sync();
}

// ------------------------------------------------------------------------------------------- candidate tables: pack, all-gather (caller), merge
// blob = [u64 sizes[4] = {C, n_list1, n_list2, n_listd}] + sections, each aligned to 16 bytes, in the order of candidate_sections()
struct cand_section { void* p; u64 elem; int count_kind; }; // count_kind: 0 C, 1 C+1, 2 n_list1, 3 n_list2, 4 n_listd
static void candidate_sections(cand_store& c, std::vector<cand_section>& s) {
	s.clear();
	auto add = [&](void* p, u64 elem, int kind) { cand_section x = {p, elem, kind}; s.push_back(x); };
	add(c.gene1.ptr(), 4, 0); add(c.gene2.ptr(), 4, 0); add(c.contig1.ptr(), 2, 0); add(c.contig2.ptr(), 2, 0); add(c.bp1.ptr(), 4, 0); add(c.bp2.ptr(), 4, 0); add(c.dir1.ptr(), 1, 0); add(c.dir2.ptr(), 1, 0);
	add(c.split_reads1.ptr(), 4, 0); add(c.split_reads2.ptr(), 4, 0); add(c.discordant_mates.ptr(), 4, 0); add(c.filter.ptr(), 1, 0); add(c.bits.ptr(), 1, 0); add(c.bits2.ptr(), 1, 0);
	add(c.anchor1.ptr(), 4, 0); add(c.anchor2.ptr(), 4, 0); add(c.evalue.ptr(), 4, 0); add(c.first_frag.ptr(), 4, 0);
	add(c.list1_off.ptr(), 4, 1); add(c.list2_off.ptr(), 4, 1); add(c.listd_off.ptr(), 4, 1); add(c.list1.ptr(), 4, 2); add(c.list2.ptr(), 4, 3); add(c.listd.ptr(), 4, 4);
}
static u64 section_count(int kind, const u64 sizes[4]) { return kind == 0 ? sizes[0] : kind == 1 ? sizes[0] + 1 : sizes[kind - 1]; }
static u64 blob_bytes(const std::vector<cand_section>& s, const u64 sizes[4]) { u64 at = 64; for (size_t k = 0; k < s.size(); ++k) at += (s[k].elem * section_count(s[k].count_kind, sizes) + 15) & ~(u64) 15; return at; }

static void copy_dd(const exec_ctx& ex, void* dst, const void* src, u64 bytes) {
	if (!bytes) return;
#ifdef ARB_DEVICE_BUILD
	ARB_CUDA_CHECK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, ex.stream));
#else
	(void) ex; memcpy(dst, src, bytes);
#endif
}

void engine::candidates_export(void** blob, u64* bytes, u64 sizes[4]) {
	sizes[0] = cands.n; sizes[1] = cands.n_list1; sizes[2] = cands.n_list2; sizes[3] = cands.n_listd;
	std::vector<cand_section> s; candidate_sections(cands, s);
	const u64 total = blob_bytes(s, sizes);
	cand_blob.ensure(total);
	u64 at = 64;
	for (size_t k = 0; k < s.size(); ++k) { const u64 b = s[k].elem * section_count(s[k].count_kind, sizes); copy_dd(ex, cand_blob.ptr() + at, s[k].p, b); at += (b + 15) & ~(u64) 15; }
	ex.sync();
	*blob = cand_blob.ptr(); *bytes = total;
}

struct add_base_fn { u32* p; u32 base; ARB_HD void operator()(u32 i) const { p[i] += base; } };
struct iota_fn { u32* p; ARB_HD void operator()(u32 i) const { p[i] = i; } };
template <class T> struct permute_fn { const T* in; const u32* perm; T* out; ARB_HD void operator()(u32 k) const { out[k] = in[perm[k]]; } };
struct list_size_fn { const u32* off; const u32* src_cand_off; const u32* perm; u32* cnt; ARB_HD void operator()(u32 k) const { const u32 j = perm[k]; cnt[k] = off[src_cand_off[j] + 1] - off[src_cand_off[j]]; (void) 0; } };
// lists of the merged table: candidate k takes the list of its source candidate (source offsets are positions in the concatenated source lists)
struct list_copy_fn {
	const u32* src_begin; const u32* src_end; const u32* perm; const u32* out_off; const u32* src; u32* out;
	ARB_HD void operator()(u32 k) const { const u32 j = perm[k]; u32 w = out_off[k]; for (u32 p = src_begin[j]; p < src_end[j]; ++p, ++w) out[w] = src[p]; }
};
struct list_len_fn { const u32* b; const u32* e; const u32* perm; u32* cnt; ARB_HD void operator()(u32 k) const { const u32 j = perm[k]; cnt[k] = e[j] - b[j]; } };
struct span_fn { const u32* off; u32 base_cand; u32 base_list; u32* b; u32* e; ARB_HD void operator()(u32 j) const { b[base_cand + j] = base_list + off[j]; e[base_cand + j] = base_list + off[j + 1]; } };

static u32 bits_for_u32(u32 n) { u32 b = 1; while (b < 32 && ((u64) 1 << b) < n) ++b; return b; }

void engine::candidates_import(const void* all_blobs, u64 stride, const u64* sizes /* 4 per part */, u32 n_parts) {
	u64 C_total = 0, n_total[3] = {0, 0, 0};
	for (u32 r = 0; r < n_parts; ++r) { C_total += sizes[4 * r]; for (int q = 0; q < 3; ++q) n_total[q] += sizes[4 * r + 1 + q]; }
	if (C_total > 0xFFFFFFF0ull || n_total[0] > 0xFFFFFFF0ull || n_total[1] > 0xFFFFFFF0ull || n_total[2] > 0xFFFFFFF0ull) throw arb_error("more than 2^32 candidates or list entries");
	const u32 C = (u32) C_total;
	// concatenated source columns (part-major, local id ascending)
	cand_store src;
	src.gene1.ensure(C); src.gene2.ensure(C); src.contig1.ensure(C); src.contig2.ensure(C); src.bp1.ensure(C); src.bp2.ensure(C); src.dir1.ensure(C); src.dir2.ensure(C);
	src.split_reads1.ensure(C); src.split_reads2.ensure(C); src.discordant_mates.ensure(C); src.filter.ensure(C); src.bits.ensure(C); src.bits2.ensure(C);
	src.anchor1.ensure(C); src.anchor2.ensure(C); src.evalue.ensure(C); src.first_frag.ensure(C);
	src.list1.ensure(n_total[0]); src.list2.ensure(n_total[1]); src.listd.ensure(n_total[2]);
	dbuf<u32> b1(C), e1(C), b2(C), e2(C), bd(C), ed(C); // list spans of the source candidates in the concatenated lists
	std::vector<cand_section> dst_sections; candidate_sections(src, dst_sections);
	u64 cand_at = 0, list_at[3] = {0, 0, 0};
	for (u32 r = 0; r < n_parts; ++r) {
		const u64* sz = sizes + 4 * r;
		const char* blob = (const char*) all_blobs + stride * r;
		u64 at = 64;
		const u32* off_ptr[3] = {0, 0, 0};
		for (size_t k = 0; k < dst_sections.size(); ++k) {
			const cand_section& s = dst_sections[k];
			const u64 count = section_count(s.count_kind, sz), b = s.elem * count;
			if (s.count_kind == 0) copy_dd(ex, (char*) s.p + cand_at * s.elem, blob + at, b);
			else if (s.count_kind == 1) off_ptr[k - 18] = (const u32*) (blob + at); // the three offset arrays follow the 18 per-candidate columns
			else copy_dd(ex, (char*) s.p + list_at[s.count_kind - 2] * 4, blob + at, b);
			at += (b + 15) & ~(u64) 15;
		}
		if (sz[0]) {
			span_fn s1 = {off_ptr[0], (u32) cand_at, (u32) list_at[0], b1.ptr(), e1.ptr()}; for_each(ex, (u32) sz[0], s1);
			span_fn s2 = {off_ptr[1], (u32) cand_at, (u32) list_at[1], b2.ptr(), e2.ptr()}; for_each(ex, (u32) sz[0], s2);
			span_fn sd = {off_ptr[2], (u32) cand_at, (u32) list_at[2], bd.ptr(), ed.ptr()}; for_each(ex, (u32) sz[0], sd);
		}
		cand_at += sz[0]; for (int q = 0; q < 3; ++q) list_at[q] += sz[1 + q];
	}
	// order of first insertion: the fragment that created the candidate (name order), ties in local id order (same fragment => same part); stable sort
	dbuf<u32> key(C), perm(C), tk(C), tv(C);
	copy_dd(ex, key.ptr(), src.first_frag.ptr(), (u64) C * 4);
	iota_fn io = {perm.ptr()}; for_each(ex, C, io);
	radix_sort_pairs_u32(ex, key.ptr(), perm.ptr(), tk.ptr(), tv.ptr(), C, bits_for_u32(frags.n + 1));
	cands.n = C; cands.genomic_marked = false; has_tag_csr = false;
	cands.gene1.ensure(C); cands.gene2.ensure(C); cands.contig1.ensure(C); cands.contig2.ensure(C); cands.bp1.ensure(C); cands.bp2.ensure(C); cands.dir1.ensure(C); cands.dir2.ensure(C);
	cands.split_reads1.ensure(C); cands.split_reads2.ensure(C); cands.discordant_mates.ensure(C); cands.filter.ensure(C); cands.bits.ensure(C); cands.bits2.ensure(C);
	cands.anchor1.ensure(C); cands.anchor2.ensure(C); cands.evalue.ensure(C); cands.first_frag.ensure(C);
	cands.list1_off.ensure((size_t) C + 1); cands.list2_off.ensure((size_t) C + 1); cands.listd_off.ensure((size_t) C + 1);
#define ARB_PERMUTE(T, col) { permute_fn<T> pf = {src.col.ptr(), perm.ptr(), cands.col.ptr()}; for_each(ex, C, pf); }
	ARB_PERMUTE(u32, gene1) ARB_PERMUTE(u32, gene2) ARB_PERMUTE(u16, contig1) ARB_PERMUTE(u16, contig2) ARB_PERMUTE(i32, bp1) ARB_PERMUTE(i32, bp2) ARB_PERMUTE(u8, dir1) ARB_PERMUTE(u8, dir2)
	ARB_PERMUTE(u32, split_reads1) ARB_PERMUTE(u32, split_reads2) ARB_PERMUTE(u32, discordant_mates) ARB_PERMUTE(u8, filter) ARB_PERMUTE(u8, bits) ARB_PERMUTE(u8, bits2)
	ARB_PERMUTE(i32, anchor1) ARB_PERMUTE(i32, anchor2) ARB_PERMUTE(float, evalue) ARB_PERMUTE(u32, first_frag)
#undef ARB_PERMUTE
	cands.n_list1 = n_total[0]; cands.n_list2 = n_total[1]; cands.n_listd = n_total[2];
	cands.list1.ensure(n_total[0]); cands.list2.ensure(n_total[1]); cands.listd.ensure(n_total[2]);
	struct { dbuf<u32>* b; dbuf<u32>* e; dbuf<u32>* src_list; dbuf<u32>* off; dbuf<u32>* out; } lists[3] = {
		{&b1, &e1, &src.list1, &cands.list1_off, &cands.list1}, {&b2, &e2, &src.list2, &cands.list2_off, &cands.list2}, {&bd, &ed, &src.listd, &cands.listd_off, &cands.listd}};
	for (int q = 0; q < 3; ++q) {
		list_len_fn ll = {lists[q].b->ptr(), lists[q].e->ptr(), perm.ptr(), lists[q].off->ptr()};
		for_each(ex, C, ll);
		exclusive_scan_u32(ex, lists[q].off->ptr(), lists[q].off->ptr(), C);
		list_copy_fn lc = {lists[q].b->ptr(), lists[q].e->ptr(), perm.ptr(), lists[q].off->ptr(), lists[q].src_list->ptr(), lists[q].out->ptr()};
		for_each(ex, C, lc);
	}
	ex.sync();
}

// ------------------------------------------------------------------------------------------- mate swaps of the other parts' candidates
// find_fusions exchanges MATE1/MATE2 of the discordant mates it lists (fusions.cpp:414-421). A fragment is listed by candidates of one part only; the flags
// of all parts are combined by the caller (MAX all-reduce over swaps_buffer), swaps_apply then performs the exchanges this part has not done itself.
struct pending_swap_fn { const u8* all; const u8* mine; u32* need; ARB_HD void operator()(u32 i) const { need[i] = (all[i] && !mine[i]) ? 1u : 0u; } };
void engine::swaps_buffer(void** p, u64* bytes) {
	swap_union.ensure(frags.n);
	copy_dd(ex, swap_union.ptr(), frags.swapped.ptr(), frags.n);
	ex.sync();
	*p = swap_union.ptr(); *bytes = frags.n;
}
void engine::swaps_apply() {
	const u32 n = frags.n;
	dbuf<u32> need(n);
	pending_swap_fn pf = {swap_union.ptr(), frags.swapped.ptr(), need.ptr()};
	for_each(ex, n, pf);
	swap_mates_fn sm = {frags.view(), need.ptr(), frags.swapped.ptr()};
	for_each(ex, n, sm);
	ex.sync();
}

} // namespace arb
