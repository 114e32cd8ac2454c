// engine.h -- device-resident state of one arriba-b200 context and the stage drivers.
#pragma once
#include "model.h"
#include "prims.h"
#include "read_filters.h"
#include "../../include/arriba_b200.h"
#include <time.h>
#include <vector>
#include <string>

namespace arb {

// CUDA-event stopwatch on the context's stream (wall clock in the hostsim build)
struct stage_timer {
#ifdef ARB_DEVICE_BUILD
	cudaEvent_t a, b; cudaStream_t s;
	explicit stage_timer(const exec_ctx& ex): s(ex.stream) { ARB_CUDA_CHECK(cudaEventCreate(&a)); ARB_CUDA_CHECK(cudaEventCreate(&b)); ARB_CUDA_CHECK(cudaEventRecord(a, s)); }
	float stop() { float ms = 0; ARB_CUDA_CHECK(cudaEventRecord(b, s)); ARB_CUDA_CHECK(cudaEventSynchronize(b)); ARB_CUDA_CHECK(cudaEventElapsedTime(&ms, a, b)); return ms; }
	~stage_timer() { cudaEventDestroy(a); cudaEventDestroy(b); }
#else
	double t0;
	static double now() { timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return ts.tv_sec * 1e3 + ts.tv_nsec * 1e-6; }
	explicit stage_timer(const exec_ctx&): t0(now()) {}
	float stop() { return (float) (now() - t0); }
#endif
};


struct frag_store {
	u32 n; u32 max_seq_len; bool canonical_seq_layout; u64 n_seq_bytes;
	dbuf<u8> n_aln, fflags, filter, early, aflags, seq, swapped;
	dbuf<u16> contig, cigar_cnt, seq_len, genes_cnt;
	dbuf<i32> start, end;
	dbuf<u32> cigar_off, seq_off, genes_off, cigar, genes;
	frag_store(): n(0), max_seq_len(0), canonical_seq_layout(false), n_seq_bytes(0) {}
	frag_view view() const {
		frag_view v;
		v.n = n; v.n_aln = n_aln.ptr(); v.fflags = fflags.ptr(); v.filter = filter.ptr();
		v.contig = contig.ptr(); v.start = start.ptr(); v.end = end.ptr(); v.aflags = aflags.ptr();
		v.cigar_off = cigar_off.ptr(); v.cigar_cnt = cigar_cnt.ptr(); v.seq_off = seq_off.ptr(); v.seq_len = seq_len.ptr();
		v.genes_off = genes_off.ptr(); v.genes_cnt = genes_cnt.ptr(); v.cigar = cigar.ptr(); v.seq = seq.ptr(); v.genes = genes.ptr();
		return v;
	}
};

struct annot_store {
	u32 n_genes, n_exons, n_contigs;
	dbuf<u16> gene_contig; dbuf<i32> gene_start, gene_end, gene_exonic_length; dbuf<u8> gene_strand, gene_flags;
	dbuf<u32> exon_gene; dbuf<i32> exon_start, exon_end, exon_cds_start, exon_cds_end, exon_next_start; dbuf<u8> exon_flags;
	dbuf<u32> exon_region_begin, exon_region_off, exon_region_items, gene_region_begin, gene_region_off, gene_region_items;
	dbuf<i32> exon_region_end, gene_region_end;
	dbuf<u8> contig_flags; dbuf<u64> contig_seq_off; dbuf<u32> contig_len; dbuf<char> assembly; dbuf<u32> assembly4; bool assembly4_ok;
	std::vector<u8> h_contig_flags; std::vector<u32> h_contig_len;
	// host mirrors needed by host-side steps
	std::vector<u16> h_gene_contig; std::vector<i32> h_gene_start, h_gene_end; std::vector<u8> h_gene_strand, h_gene_flags;
	u64 assembly_bytes, assembly4_words; u32 n_exon_regions, n_exon_items, n_gene_regions, n_gene_items; // exact sizes of the buffers above (exchange.cu)
	annot_store(): n_genes(0), n_exons(0), n_contigs(0), assembly4_ok(false), assembly_bytes(0), assembly4_words(0), n_exon_regions(0), n_exon_items(0), n_gene_regions(0), n_gene_items(0) {}
	annot_view view() const {
		annot_view v;
		v.n_genes = n_genes; v.gene_contig = gene_contig.ptr(); v.gene_start = gene_start.ptr(); v.gene_end = gene_end.ptr();
		v.gene_strand = gene_strand.ptr(); v.gene_exonic_length = gene_exonic_length.ptr(); v.gene_flags = gene_flags.ptr();
		v.n_exons = n_exons; v.exon_gene = exon_gene.ptr(); v.exon_start = exon_start.ptr(); v.exon_end = exon_end.ptr();
		v.exon_cds_start = exon_cds_start.ptr(); v.exon_cds_end = exon_cds_end.ptr(); v.exon_next_start = exon_next_start.ptr(); v.exon_flags = exon_flags.ptr();
		v.n_contigs = n_contigs;
		v.exon_region_begin = exon_region_begin.ptr(); v.exon_region_end = exon_region_end.ptr(); v.exon_region_off = exon_region_off.ptr(); v.exon_region_items = exon_region_items.ptr();
		v.gene_region_begin = gene_region_begin.ptr(); v.gene_region_end = gene_region_end.ptr(); v.gene_region_off = gene_region_off.ptr(); v.gene_region_items = gene_region_items.ptr();
		v.exon_grid = 0; v.exon_grid_begin = 0; v.gene_grid = 0; v.gene_grid_begin = 0;
		v.contig_flags = contig_flags.ptr(); v.contig_seq_off = contig_seq_off.ptr(); v.contig_len = contig_len.ptr(); v.assembly = assembly.ptr(); v.assembly4 = assembly4_ok ? assembly4.ptr() : 0;
		return v;
	}
};

struct cand_store {
	u32 n; u64 n_list1, n_list2, n_listd;
	dbuf<u32> gene1, gene2, split_reads1, split_reads2, discordant_mates, list1_off, list2_off, listd_off, list1, list2, listd;
	dbuf<u16> contig1, contig2; dbuf<i32> bp1, bp2, anchor1, anchor2; dbuf<u8> dir1, dir2, filter, bits, bits2; dbuf<float> evalue;
	dbuf<u32> first_frag; // fragment whose record created the candidate (merge key of the sharded run)
	dbuf<i32> closest1, closest2; bool genomic_marked; // closest genomic breakpoints (-d), valid once mark_genomic_support has run on this table
	cand_store(): n(0), n_list1(0), n_list2(0), n_listd(0), genomic_marked(false) {}
};

struct exchange_buffer { void* p; u64 bytes; };

class engine {
public:
	scratch_set scratch; // scan / radix-sort scratch of this context (its device, its stream)
	exec_ctx ex;
	std::string last_error;
	arb_params params;
	frag_store frags;
	annot_store annot;
	cand_store cands;
	dbuf<u8> mismatch_table; u32 table_n, table_k;
	hash_index table;
	dbuf<u32> label_counts;
	bool has_contigs, has_annotation, filters_done;
	arb_timings timings;

	engine();
	~engine();
	void set_contigs(const arb_contigs& c);
	void set_annotation(const arb_annotation& a);
	void set_contig_flags(const u8* flags, u32 n);
	void set_params(const arb_params& p) { // the mismatch table is tabulated for one p-value cutoff: a new cutoff rebuilds it on the next run
		if (p.mismatch_pvalue_cutoff != params.mismatch_pvalue_cutoff) table_n = 0;
		params = p;
	}
	void push_chunk(const arb_soa_chunk& c) { push_chunk_begin(c); push_chunk_end(c); }
	void push_chunk_begin(const arb_soa_chunk& c); // everything but the annotation columns (aflags, gene sets), asynchronously on the copy stream
	void push_chunk_end(const arb_soa_chunk& c);   // the annotation columns; returns when the whole table is resident
	// device-side annotation of the resident chunk (annotate.cu): between the two passes the gene sets live in fixed rows + a pool
	u32 annotate_pass1(const u8* aflags, int strandedness); void get_dummy_genes(u16* contig, i32* start, i32* end); u64 annotate_pass2();
	void get_annotation_columns(u8* aflags, u32* genes_off, u16* genes_cnt, u32* genes);
	dbuf<u32> annot_rows, annot_pool, annot_ctl; dbuf<u16> annot_cnt; u32 annot_pool_cap, n_dummy; u64 n_gene_entries; dbuf<u16> dummy_contig; dbuf<i32> dummy_start, dummy_end;
	void finish_push(u64 n_gene_ids); u64 push_cigar_ops; dbuf<u64> chunk_stats;
	void adopt_table(const exec_ctx& cx, u64 n_cigar, u64 n_seq_bytes); // the columns in `frags` become the resident table (statistics, push_open)
	// the fragment table built from the fragment pools the record replay wrote (fragtable.cu)
	void fragment_table_build(u64 sizes[6]);
	void fragment_table_download(const arb_soa_chunk& columns, char* names, u64* name_off);
	dbuf<arb_pool_fragment> pool_frags; dbuf<arb_pool_alignment> pool_alns; dbuf<char> pool_names, frag_names; dbuf<u32> pool_cigars; dbuf<u8> pool_seqs;
	dbuf<u64> pool_base, frag_name_off; u32 pool_workers; u64 frag_name_bytes;
	u64 ft_chimeric[2] = {0, 0}; // fragments of a separate chimeric file that the first malformed pass rejects / keeps (the last replay's counting pass)
	// one sample on several GPUs (exchange.cu): replicated state travels as groups of device buffers, the work of find_fusions / filter_mismappers is divided
	void exchange_header(int group, std::vector<u64>& header); void exchange_prepare(int group, const u64* header, u32 n_words);
	void exchange_buffers(int group, std::vector<exchange_buffer>& out); void exchange_commit(int group);
	void set_work_partition(const u32* keys, const u8* owner, u32 n_keys, int part, int parts); int work_part, work_parts; dbuf<u8> work_owned;
	void candidates_export(void** blob, u64* bytes, u64 sizes[4]); void candidates_import(const void* all_blobs, u64 stride, const u64* sizes, u32 n_parts); dbuf<char> cand_blob;
	void swaps_buffer(void** p, u64* bytes); void swaps_apply(); dbuf<u8> swap_union;
	void filter_mismappers_part(i32 max_mate_gap, int part, int parts, void** verdicts, u64* bytes); u64 filter_mismappers_finish(); dbuf<u8> mismap_verdicts; u64 mismap_items_total; float mismap_ms_part;
	u64 n_splice_sites;
	exec_ctx copy_ex; bool push_open; // copy stream: H2D of a chunk overlaps with host work (annotation) and with kernels on `ex`
	void run_read_filters();
	void get_fragment_filters(u8* filter_out, u8* early_out);
	void set_fragment_filters(const u8* filter);
	void get_filter_counts(u32* counts);
	void find_fusions(i32 max_mate_gap);
	void get_candidates(arb_candidates& out);
	void get_slot_swaps(u8* out);
	void set_candidate_state(const u8* filter, const u32* s1, const u32* s2, const u32* dm, const float* ev);
	void get_candidate_state(u8* filter, u32* s1, u32* s2, u32* dm, float* ev);
	void set_candidate_lists(const u32* l1o, const u32* l1, const u32* l2o, const u32* l2);
	u32 merge_adjacent(i32 max_distance);
	void get_merge_log(u32* triples, u32 n);
	void estimate_evalues(const arb_evalue_inputs& in);
	void filter_relative_support(float cutoff); void filter_multimappers(); u32 filter_simple(int stage, float exonic_fraction, int min_support); void evalue_tallies(u32* out); u32 select_best();
	void replay_insertion_order(const u32* phase_start, const u64* phase_buckets, u32 n_phases, u32* order_out, u32* rank_out); dbuf<u32> order_rank;
	void partner_counts(i32* count_out); dbuf<u32> order_seq;
	// BAM record boundaries of an inflated chunk in device memory (bamscan.cu)
	void bam_scan(const u8* B, u64 bytes, u64 first, i32 n_ref, dbuf<u32>& rec_off, u64* consumed, u32* n_records, u32* malformed); dbuf<u8> bam_buf, bam_buf_next;
	// the record loop of the ingest (records.cu): the record store across chunks, then the replay by key into the fragment pools
	void records_begin(const u16* tid_to_contig, u32 n_tid, const u8* interesting, const u8* viral, const u64* n_windows, u32 n_contigs, u32 max_itd_length, bool external_duplicate_marking, u64 expected_bytes);
	void records_chunk(const u8* chunk, u64 bytes, u64 first, u64 chunk_pos, u64* n_records, u64* carry, u32* malformed, u64* error);
	void records_finish(u16* const* coverage, u8* const* starts, u8* const* ends, u64* counters, u64* error);
	u64 records_upload(const u8* chunk, u64 bytes);
	// stream input: the inflated chunk assembled on the device from the raw BGZF blocks (stage_hd.h); the next records_chunk / records_text_chunk with
	// chunk == NULL takes it
	void records_bgzf_stage(const u8* raw, u64 raw_bytes, const arb_bgzf_block* blocks, u32 n_blocks);
	dbuf<u8> rec_raw; dbuf<arb_bgzf_block> rec_stage_blocks; u64 rec_staged = 0; bool rec_stage_pending = false;
	void records_store(const dbuf<u8>& B, u64 buf_pos, u64 total, const u32* rec_off, u32 R, u64 seen, u64* error);
	// SAM text input (samscan.cu): lines staged as BAM records, then records_store
	void records_text_names(const char* names, const u64* name_off, u32 n);
	void records_text_chunk(const u8* chunk, u64 bytes, u64 first, u64 chunk_pos, bool last, u64* n_records, u64* carry, u64* error);
	dbuf<u8> sam_blob, sam_stage; dbuf<u64> sam_name_off; dbuf<u32> sam_name_tid; u32 sam_n_names = 0; u64 rec_text_staged = 0;
	dbuf<u8> rec_arena, rec_sa, rec_interesting, rec_viral, rec_cov_starts, rec_cov_ends; dbuf<u64> rec_at, rec_pos, rec_error, rec_counters, rec_cov_off; dbuf<i64> rec_hit;
	dbuf<u32> rec_hash_lo, rec_hash_hi, rec_cov_words, rec_cov_n; dbuf<u16> rec_tid;
	u64 rec_n, rec_arena_used, rec_carry, rec_carry_at, rec_expected_bytes, rec_cov_windows, rec_hash_mask; u32 rec_n_tid, rec_n_contigs, rec_max_itd; bool rec_external_dup, rec_open;
	std::vector<u8> rec_error_record; // the body of the record a chunk's error names
	// a separate chimeric file (-c) ahead of the main file: the file whose chunks follow, its references; positions of later files start behind it
	void records_source(bool chimeric_file, const u16* tid_to_contig, u32 n_tid, u64* first_position);
	bool rec_src_chimeric = false /* the chunks are the -c file's */, rec_has_chimeric = false /* a -c file was selected since arb_records_begin */;
	u64 rec_pos_base = 0 /* added to the positions of the current file */, rec_pos_end = 0 /* behind every position so far */, rec_chimeric_end = 0 /* positions below: -c records */;
	// rows of the discarded-fusions file (rows.cu)
	void set_row_texts(const arb_row_texts& t); void format_discarded_rows(const u8* confidence, u64* n_rows, u64* n_bytes); void get_row_text(char* out);
	dbuf<char> row_gene_name, row_gene_id, row_contig_name, row_filter_name, row_text; dbuf<u32> row_gene_name_off, row_gene_id_off, row_contig_name_off, row_filter_name_off; dbuf<i32> row_exon_prev, row_exon_next;
	u8 row_filters_by_name[ARB_N_FILTERS]; u32 row_max_itd_length; bool has_row_texts; u64 row_text_bytes; struct cand_state make_state_for_rows();
	// pileups and consensus sequences of the rows of fusions.tsv (consensus.cu)
	void build_consensus(const u32* rows, u32 n_rows, arb_consensus_info& info); void get_consensus(u32* seq_off, u32* pos_off, u32* clip_off, u8* verdict, u32* non_template, char* seq, i32* pos, char* clip);
	dbuf<u32> cons_seq_off, cons_pos_off, cons_clip_off, cons_non_template; dbuf<u8> cons_verdict; dbuf<char> cons_seq, cons_clip; dbuf<i32> cons_pos; u32 cons_rows; u64 cons_seq_bytes, cons_pos_count, cons_clip_bytes;
	dbuf<u32> merge_log; u32 merge_log_n;
	// filter_in_vitro on the device (events.cu): coverage windows of the sample, expression per gene
	void set_coverage(const u16* const* per_contig, const u64* n_windows, u32 n_contigs); void reads_by_gene(u32* out);
	void filter_in_vitro(const u32* reads, u32 n_genes, u32 threshold, const u64* pairs, u64 n_pairs); void spliced_support(const u32* reads, u32 n_genes, u32 threshold, u32* support_out);
	dbuf<u16> coverage_windows; dbuf<u64> coverage_off; dbuf<u32> coverage_n; u32 coverage_contigs;
	// k-mer index / re-alignment
	dbuf<i32> kmer_pos; dbuf<u32> kmer_bucket_off; u32 kmer_index_contigs; u64 kmer_indexed;
	dbuf<u32> kmer_block_first, kmer_block_base; u32 kmer_block_shift, kmer_blocks; struct kmer_index_view index_view(); // block table of the index (mismap_hd.h)
	u64 push_alignments, push_bases; u64 head_bytes, sequence_bytes; // column budgets of the two cascade launches for the resident chunk
	size_t cascade_smem_bytes; u32 cascade_resident_blocks; // launch shape of the sequence kernel on this context's device
	int device;
	int mismap_budget; u32 mismap_lanes, mismap_task_lanes, homolog_lanes; // work control of the re-alignment passes (mismap_hd.h, realign_ctl)
	dbuf<u32> splice_off; dbuf<i32> splice_sites; bool has_splice_sites;
	void set_splice_sites(const u32* off, const i32* sites);
	u64 build_kmer_index(const u32* contig, const i32* start, const i32* end, u32 n, u32 n_index_contigs);
	void homolog_pairs(const u32* ga, const u32* gb, u32 n, u8* out);
	u64 filter_mismappers(i32 max_mate_gap);
	void probe_mismatch_counts(u32* out); // test hook (arb_selftest_mismatch_counts)
	void probe_kmer_lookup(const u32* contig, const u32* kmer, const i32* from, u32 n, u32* out); // test hook (arb_selftest_kmer_lookup)
	// genomic breakpoints from whole-genome sequencing (genomic.cu): sorted records + key table, the search writes cands.closest1/2
	void set_genomic_breakpoints(u32 n, const u16* c1, const u16* c2, const u8* d1, const u8* d2, const i32* p1, const i32* p2);
	u32 mark_genomic_support(i32 max_distance, i32 max_itd_length); void get_genomic_support(i32* closest1, i32* closest2);
	dbuf<u64> genomic_key_table; dbuf<u32> genomic_key_begin; dbuf<i32> genomic_pos1, genomic_pos2; u32 genomic_n, genomic_keys, genomic_heavy; bool has_genomic_breakpoints;
	// rules of a blacklist (-b), known fusions (-k) or tags (-t) file (blacklist.cu): the rule columns in file order; the key tables are built per call (the
	// blacklist's depends on max_mate_gap)
	struct rule_set {
		dbuf<u8> type1, type2, strand1, strand2; dbuf<u16> contig1, contig2; dbuf<i32> start1, end1, start2, end2; dbuf<u32> gene1, gene2;
		u32 n; bool loaded;
		rule_set(): n(0), loaded(false) {}
	};
	void set_rules(rule_set& set, const char* who, u32 n, const u8* type1, const u8* type2, const u8* strand1, const u8* strand2, const u16* contig1, const u16* contig2,
	               const i32* start1, const i32* end1, const i32* start2, const i32* end2, const u32* gene1, const u32* gene2);
	rule_set blacklist_rules, known_rules, tag_rules;
	u32 filter_blacklist(u32 n_ids, const u32* ids, float evalue_cutoff, i32 max_mate_gap, u8* verdicts);
	u32 recover_known_fusions(u32 n_ids, const u32* ids, i32 max_mate_gap, u8* verdicts);
	void set_tags(const u32* rank, u32 n_tags, const char* chars, const u32* off); // after set_rules(tag_rules, ...): the tag rank of every rule and the tag texts
	u64 annotate_tags(u32 n_ids, const u32* ids, i32 max_mate_gap); void get_tags(u32* off, u32* ranks);
	dbuf<u32> tag_rank_of_rule, tag_text_off, tag_csr_off, tag_csr_rank; dbuf<char> tag_text; u32 n_tags, tag_csr_n; u64 tag_csr_pairs; bool has_tags, has_tag_csr;
	u32 blacklist_heavy, known_heavy, tags_heavy;
	// protein domains (-p, protein_domains.cu): the per-gene table of domains_hd.h, dropped when the annotation is replaced; the retained_protein_domains
	// column of the rows the host formats
	void set_protein_domains(u32 n, const u16* contig, const i32* start, const i32* end, const u32* gene, const u32* name_rank, u32 n_names, const char* chars, const u32* off);
	u64 retained_protein_domains(u32 n_ids, const u32* ids); void get_retained_protein_domains(u64* off, char* text);
	struct domain_view domain_tables(); void check_domain_error(const char* who);
	dbuf<u16> dom_contig; dbuf<i32> dom_start, dom_end; dbuf<u32> dom_mult, dom_name, dom_gene_off, dom_name_off, dom_error; dbuf<char> dom_name_chars, dom_text;
	std::vector<u64> dom_text_off; u32 dom_records; bool has_protein_domains;
	// gap filling of fusion transcript sequences (-I, fill_gaps.cu): the transcript table of the writer, and the filled sides of the last call
	void set_fill_transcripts(u32 n, const i32* first_exon, const i32* last_exon, const u32* contig, const i32* exon_next, const i32* exon_prev);
	u64 fill_gaps(u32 n_rows, const char* text, const u32* row_off, const i32* pos, const u32* pos_off, u32 n_jobs, const u32* row, const u32* transcript, const u8* flags);
	void get_filled(u32* off, char* chars, i32* pos);
	dbuf<i32> fill_first, fill_last, fill_next, fill_prev, fill_pos; dbuf<u32> fill_contig; dbuf<char> fill_chars; std::vector<u32> fill_off;
	u32 fill_transcript_count = 0; u64 fill_chars_total = 0; bool has_fill_transcripts = false;
private:
	read_filter_params make_filter_params();
	unsigned long genome_size() const;
};

void default_params(arb_params& p);

} // namespace arb
