// capi.cu -- the C ABI declared in include/arriba_b200.h: thin exception-to-status shims over arb::engine.
#include "engine.h"
#include <new>
#include <map>
#include <mutex>
#include <sys/mman.h>

using namespace arb;

struct arb_ctx { engine e; };
static std::string g_create_error;

// ---- page-locked host memory for the caller's columns -----------------------------------------------------------------------------------------------
// The host side builds its large columns in recycled blocks (host/ingest.h, host_block_get); in the CUDA library fresh blocks are page-locked, so that
// arb_push_chunk_begin/end copy them asynchronously at full PCIe speed.
namespace arb { namespace host { void set_host_block_backend(void* (*alloc)(size_t), void (*release)(void*)); } }
static int g_host_memory_device = -1;
#ifdef ARB_DEVICE_BUILD
// The blocks are mapped by the process, asked for 2 MiB pages (THP "madvise") and then registered with the driver: the ingest's record loop visits its
// workers' pools (hundreds of megabytes, page-locked so that they go to the device at full speed) all over, and on 4 KiB pages nearly every visit would
// also miss the TLB. Where the kernel grants no huge pages the block is page-locked all the same.
namespace { struct pinned_blocks { std::mutex lock; std::map<void*, std::pair<void*, size_t> > mapping; }; pinned_blocks& pinned() { static pinned_blocks* b = new pinned_blocks(); return *b; } }
static void* pinned_alloc(size_t bytes) {
	if (g_host_memory_device >= 0) { int cur = -1; if (cudaGetDevice(&cur) != cudaSuccess || cur != g_host_memory_device) { if (cudaSetDevice(g_host_memory_device) != cudaSuccess) { cudaGetLastError(); return NULL; } } }
	const size_t huge = (size_t) 2 << 20, len = ((bytes ? bytes : 1) + huge - 1) & ~(huge - 1);
	void* base = mmap(NULL, len + huge, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
	if (base == MAP_FAILED) return NULL;
	void* p = (void*) (((uintptr_t) base + huge - 1) & ~(uintptr_t) (huge - 1));
#ifdef MADV_HUGEPAGE
	madvise(p, len, MADV_HUGEPAGE);
#endif
	if (cudaHostRegister(p, len, cudaHostRegisterPortable) != cudaSuccess) { cudaGetLastError(); munmap(base, len + huge); return NULL; }
	std::lock_guard<std::mutex> g(pinned().lock);
	pinned().mapping[p] = std::make_pair(base, len + huge);
	return p;
}
static void pinned_free(void* p) {
	std::pair<void*, size_t> m(NULL, 0);
	{ std::lock_guard<std::mutex> g(pinned().lock); std::map<void*, std::pair<void*, size_t> >::iterator it = pinned().mapping.find(p); if (it == pinned().mapping.end()) return; m = it->second; pinned().mapping.erase(it); }
	cudaHostUnregister(p);
	munmap(m.first, m.second);
}
namespace { struct install_pinned_backend { install_pinned_backend() { arb::host::set_host_block_backend(pinned_alloc, pinned_free); } } g_install_pinned_backend; }
#endif

#ifdef ARB_DEVICE_BUILD
#define ARB_BIND_DEVICE(ctx) ARB_CUDA_CHECK(cudaSetDevice((ctx)->e.device));
#else
#define ARB_BIND_DEVICE(ctx)
#endif
#define ARB_API_BEGIN(ctx) if (!(ctx)) return 2; try { ARB_BIND_DEVICE(ctx)
#define ARB_API_END(ctx) } catch (const std::exception& x) { (ctx)->e.last_error = x.what(); return 1; } catch (...) { (ctx)->e.last_error = "unknown error"; return 1; } return 0;

extern "C" {

const char* arb_backend(void) {
#ifdef ARB_DEVICE_BUILD
	return "cuda-sm_90a";
#else
	return "hostsim-TEST-ONLY";
#endif
}

uint64_t arb_kernel_launches(void) { return stats().kernels; }

int arb_ctx_create(arb_ctx** out, int device) {
	if (!out) return 2;
	*out = NULL;
	try {
#ifdef ARB_DEVICE_BUILD
		int count = 0;
		cudaError_t e = cudaGetDeviceCount(&count);
		if (e != cudaSuccess || count == 0) throw arb_error(std::string("no usable CUDA device (") + cudaGetErrorString(e) + "); arriba-b200 has no CPU fallback");
		if (device < 0 || device >= count) throw arb_error("device index out of range");
		ARB_CUDA_CHECK(cudaSetDevice(device));
		cudaDeviceProp prop;
		ARB_CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
		if (prop.major != 9 || prop.minor != 0) throw arb_error(std::string("device '") + prop.name + "' is not sm_90 (Hopper); this build targets sm_90a only");
#else
		(void) device;
#endif
		*out = new arb_ctx();
		(*out)->e.device = device;
	} catch (const std::exception& x) { g_create_error = x.what(); return 1; }
	return 0;
}

void arb_ctx_destroy(arb_ctx* ctx) {
	if (!ctx) return;
#ifdef ARB_DEVICE_BUILD
	cudaSetDevice(ctx->e.device);
#endif
	delete ctx; // device blocks go back to the pool, not to the driver: the next context on this device reuses them
}
void arb_release_device_memory(void) { pool_trim(); }
void arb_set_host_memory_device(int device) { g_host_memory_device = device; }
const char* arb_last_error(arb_ctx* ctx) { return ctx ? ctx->e.last_error.c_str() : g_create_error.c_str(); }

void arb_default_params(arb_params* p) { if (p) default_params(*p); }
int arb_set_params(arb_ctx* ctx, const arb_params* p) { ARB_API_BEGIN(ctx) ctx->e.set_params(*p); ARB_API_END(ctx) }
int arb_set_contigs(arb_ctx* ctx, const arb_contigs* c) { ARB_API_BEGIN(ctx) ctx->e.set_contigs(*c); ARB_API_END(ctx) }
int arb_set_annotation(arb_ctx* ctx, const arb_annotation* a) { ARB_API_BEGIN(ctx) ctx->e.set_annotation(*a); ARB_API_END(ctx) }
int arb_set_contig_flags(arb_ctx* ctx, const uint8_t* flags, uint32_t n) { ARB_API_BEGIN(ctx) ctx->e.set_contig_flags(flags, n); ARB_API_END(ctx) }
int arb_push_chunk(arb_ctx* ctx, const arb_soa_chunk* c) { ARB_API_BEGIN(ctx) ctx->e.push_chunk(*c); ARB_API_END(ctx) }
int arb_push_chunk_begin(arb_ctx* ctx, const arb_soa_chunk* c) { ARB_API_BEGIN(ctx) ctx->e.push_chunk_begin(*c); ARB_API_END(ctx) }
int arb_push_chunk_end(arb_ctx* ctx, const arb_soa_chunk* c) { ARB_API_BEGIN(ctx) ctx->e.push_chunk_end(*c); ARB_API_END(ctx) }
int arb_fragment_table_build(arb_ctx* ctx, uint64_t sizes[6]) { ARB_API_BEGIN(ctx) ctx->e.fragment_table_build(sizes); ARB_API_END(ctx) }
int arb_fragment_table_download(arb_ctx* ctx, const arb_soa_chunk* columns, char* names, uint64_t* name_off) { ARB_API_BEGIN(ctx) ctx->e.fragment_table_download(*columns, names, name_off); ARB_API_END(ctx) }
int arb_records_begin(arb_ctx* ctx, const uint16_t* tid_to_contig, uint32_t n_tid, const uint8_t* interesting, const uint8_t* viral, const uint64_t* n_windows, uint32_t n_contigs,
                      uint32_t max_itd_length, int external_duplicate_marking, uint64_t expected_bytes) {
	ARB_API_BEGIN(ctx) std::vector<u64> w(n_windows, n_windows + n_contigs); ctx->e.records_begin(tid_to_contig, n_tid, interesting, viral, w.data(), n_contigs, max_itd_length, external_duplicate_marking != 0, expected_bytes); ARB_API_END(ctx)
}
int arb_records_chunk(arb_ctx* ctx, const uint8_t* chunk, uint64_t bytes, uint64_t first, uint64_t chunk_pos, uint64_t* n_records, uint64_t* carry, uint32_t* malformed, uint64_t* error) {
	ARB_API_BEGIN(ctx) u64 r = 0, c = 0, e = 0; ctx->e.records_chunk(chunk, bytes, first, chunk_pos, &r, &c, malformed, &e); *n_records = r; *carry = c; *error = e; ARB_API_END(ctx)
}
int arb_records_bgzf_stage(arb_ctx* ctx, const uint8_t* raw, uint64_t raw_bytes, const arb_bgzf_block* blocks, uint32_t n_blocks) {
	ARB_API_BEGIN(ctx) if (n_blocks && !blocks) throw arb_error("arb_records_bgzf_stage: no block table"); ctx->e.records_bgzf_stage(raw, raw_bytes, blocks, n_blocks); ARB_API_END(ctx)
}
int arb_records_source(arb_ctx* ctx, int chimeric_file, const uint16_t* tid_to_contig, uint32_t n_tid, uint64_t* first_position) {
	ARB_API_BEGIN(ctx) u64 f = 0; ctx->e.records_source(chimeric_file != 0, tid_to_contig, n_tid, &f); *first_position = f; ARB_API_END(ctx)
}
int arb_fragment_table_chimeric_file(arb_ctx* ctx, uint64_t counts[2]) { ARB_API_BEGIN(ctx) counts[0] = ctx->e.ft_chimeric[0]; counts[1] = ctx->e.ft_chimeric[1]; ARB_API_END(ctx) }
int arb_records_text_names(arb_ctx* ctx, const char* names, const uint64_t* name_off, uint32_t n_names) {
	ARB_API_BEGIN(ctx) std::vector<u64> off(name_off, name_off + n_names + 1); ctx->e.records_text_names(names, off.data(), n_names); ARB_API_END(ctx)
}
int arb_records_text_chunk(arb_ctx* ctx, const uint8_t* chunk, uint64_t bytes, uint64_t first, uint64_t chunk_pos, int last, uint64_t* n_records, uint64_t* carry, uint64_t* error) {
	ARB_API_BEGIN(ctx) u64 r = 0, c = 0, e = 0; ctx->e.records_text_chunk(chunk, bytes, first, chunk_pos, last != 0, &r, &c, &e); *n_records = r; *carry = c; *error = e; ARB_API_END(ctx)
}
int arb_records_error_record(arb_ctx* ctx, const uint8_t** body, uint64_t* bytes) {
	ARB_API_BEGIN(ctx) *body = ctx->e.rec_error_record.data(); *bytes = ctx->e.rec_error_record.size(); ARB_API_END(ctx)
}
int arb_records_finish(arb_ctx* ctx, uint16_t* const* coverage, uint8_t* const* starts, uint8_t* const* ends, uint64_t* counters, uint64_t* error) {
	ARB_API_BEGIN(ctx) u64 e = 0; ctx->e.records_finish(coverage, starts, ends, (u64*) counters, &e); *error = e; ARB_API_END(ctx)
}
int arb_annotate_pass1(arb_ctx* ctx, const uint8_t* aflags, int32_t strandedness, uint32_t* n_dummy) { ARB_API_BEGIN(ctx) const uint32_t k = ctx->e.annotate_pass1(aflags, strandedness); if (n_dummy) *n_dummy = k; ARB_API_END(ctx) }
int arb_get_dummy_genes(arb_ctx* ctx, uint16_t* contig, int32_t* start, int32_t* end) { ARB_API_BEGIN(ctx) ctx->e.get_dummy_genes(contig, start, end); ARB_API_END(ctx) }
int arb_annotate_pass2(arb_ctx* ctx, uint64_t* n_gene_ids) { ARB_API_BEGIN(ctx) const uint64_t k = ctx->e.annotate_pass2(); if (n_gene_ids) *n_gene_ids = k; ARB_API_END(ctx) }
int arb_get_annotation_columns(arb_ctx* ctx, uint8_t* aflags, uint32_t* genes_off, uint16_t* genes_cnt, uint32_t* genes) { ARB_API_BEGIN(ctx) ctx->e.get_annotation_columns(aflags, genes_off, genes_cnt, genes); ARB_API_END(ctx) }
int arb_run_read_filters(arb_ctx* ctx) { ARB_API_BEGIN(ctx) ctx->e.run_read_filters(); ARB_API_END(ctx) }
int arb_get_fragment_filters(arb_ctx* ctx, uint8_t* f, uint8_t* early) { ARB_API_BEGIN(ctx) ctx->e.get_fragment_filters(f, early); ARB_API_END(ctx) }
int arb_set_fragment_filters(arb_ctx* ctx, const uint8_t* f) { ARB_API_BEGIN(ctx) ctx->e.set_fragment_filters(f); ARB_API_END(ctx) }
int arb_get_filter_counts(arb_ctx* ctx, uint32_t counts[ARB_N_FILTERS]) { ARB_API_BEGIN(ctx) ctx->e.get_filter_counts(counts); ARB_API_END(ctx) }
int arb_find_fusions(arb_ctx* ctx, int32_t max_mate_gap) { ARB_API_BEGIN(ctx) ctx->e.find_fusions(max_mate_gap); ARB_API_END(ctx) }
int arb_candidates_size(arb_ctx* ctx, uint32_t* n, uint64_t* n1, uint64_t* n2, uint64_t* nd) {
	ARB_API_BEGIN(ctx)
	if (n) *n = ctx->e.cands.n; if (n1) *n1 = ctx->e.cands.n_list1; if (n2) *n2 = ctx->e.cands.n_list2; if (nd) *nd = ctx->e.cands.n_listd;
	ARB_API_END(ctx)
}
int arb_get_candidates(arb_ctx* ctx, arb_candidates* out) { ARB_API_BEGIN(ctx) ctx->e.get_candidates(*out); ARB_API_END(ctx) }
int arb_set_candidate_state(arb_ctx* ctx, const uint8_t* f, const uint32_t* s1, const uint32_t* s2, const uint32_t* dm, const float* ev) { ARB_API_BEGIN(ctx) ctx->e.set_candidate_state(f, s1, s2, dm, ev); ARB_API_END(ctx) }
int arb_get_candidate_filters(arb_ctx* ctx, uint8_t* f) { ARB_API_BEGIN(ctx) ctx->e.cands.filter.download(ctx->e.ex, f, ctx->e.cands.n); ARB_API_END(ctx) }
int arb_get_candidate_state(arb_ctx* ctx, uint8_t* f, uint32_t* s1, uint32_t* s2, uint32_t* dm, float* ev) { ARB_API_BEGIN(ctx) ctx->e.get_candidate_state(f, s1, s2, dm, ev); ARB_API_END(ctx) }
int arb_set_candidate_lists(arb_ctx* ctx, const uint32_t* l1o, const uint32_t* l1, const uint32_t* l2o, const uint32_t* l2) { ARB_API_BEGIN(ctx) ctx->e.set_candidate_lists(l1o, l1, l2o, l2); ARB_API_END(ctx) }
int arb_merge_adjacent(arb_ctx* ctx, int32_t max_distance, uint32_t* n) { ARB_API_BEGIN(ctx) uint32_t k = ctx->e.merge_adjacent(max_distance); if (n) *n = k; ARB_API_END(ctx) }
int arb_get_merge_log(arb_ctx* ctx, uint32_t* triples, uint32_t n) { ARB_API_BEGIN(ctx) ctx->e.get_merge_log(triples, n); ARB_API_END(ctx) }
int arb_estimate_evalues(arb_ctx* ctx, const arb_evalue_inputs* in) { ARB_API_BEGIN(ctx) ctx->e.estimate_evalues(*in); ARB_API_END(ctx) }
int arb_select_best(arb_ctx* ctx, uint32_t* remaining) { ARB_API_BEGIN(ctx) const uint32_t r = ctx->e.select_best(); if (remaining) *remaining = r; ARB_API_END(ctx) }
int arb_evalue_tallies(arb_ctx* ctx, uint32_t out[11]) { ARB_API_BEGIN(ctx) ctx->e.evalue_tallies(out); ARB_API_END(ctx) }
int arb_filter_simple(arb_ctx* ctx, int32_t stage, float exonic_fraction, int32_t min_support, uint32_t* remaining) { ARB_API_BEGIN(ctx) const uint32_t r = ctx->e.filter_simple(stage, exonic_fraction, min_support); if (remaining) *remaining = r; ARB_API_END(ctx) }
int arb_filter_relative_support(arb_ctx* ctx, float cutoff) { ARB_API_BEGIN(ctx) ctx->e.filter_relative_support(cutoff); ARB_API_END(ctx) }
int arb_set_coverage(arb_ctx* ctx, const uint16_t* const* cov, const uint64_t* n_windows, uint32_t n_contigs) { ARB_API_BEGIN(ctx) std::vector<u64> w(n_windows, n_windows + n_contigs); ctx->e.set_coverage(cov, w.data(), n_contigs); ARB_API_END(ctx) }
int arb_reads_by_gene(arb_ctx* ctx, uint32_t* out) { ARB_API_BEGIN(ctx) ctx->e.reads_by_gene(out); ARB_API_END(ctx) }
int arb_filter_in_vitro(arb_ctx* ctx, const uint32_t* reads, uint32_t n_genes, uint32_t threshold, const uint64_t* pairs, uint64_t n_pairs) { ARB_API_BEGIN(ctx) ctx->e.filter_in_vitro(reads, n_genes, threshold, (const u64*) pairs, n_pairs); ARB_API_END(ctx) }
int arb_spliced_support(arb_ctx* ctx, const uint32_t* reads, uint32_t n_genes, uint32_t threshold, uint32_t* out) { ARB_API_BEGIN(ctx) ctx->e.spliced_support(reads, n_genes, threshold, out); ARB_API_END(ctx) }
int arb_replay_insertion_order(arb_ctx* ctx, const uint32_t* phase_start, const uint64_t* phase_buckets, uint32_t n_phases, uint32_t* order_out, uint32_t* rank_out) { ARB_API_BEGIN(ctx) ctx->e.replay_insertion_order(phase_start, (const u64*) phase_buckets, n_phases, order_out, rank_out); ARB_API_END(ctx) }
int arb_partner_counts(arb_ctx* ctx, int32_t* out) { ARB_API_BEGIN(ctx) ctx->e.partner_counts(out); ARB_API_END(ctx) }
int arb_set_row_texts(arb_ctx* ctx, const arb_row_texts* t) { ARB_API_BEGIN(ctx) if (!t) throw arb_error("null tables"); ctx->e.set_row_texts(*t); ARB_API_END(ctx) }
int arb_format_discarded_rows(arb_ctx* ctx, const uint8_t* confidence, uint64_t* n_rows, uint64_t* n_bytes) { ARB_API_BEGIN(ctx) u64 r = 0, b = 0; ctx->e.format_discarded_rows(confidence, &r, &b); *n_rows = r; *n_bytes = b; ARB_API_END(ctx) }
int arb_get_row_text(arb_ctx* ctx, char* out) { ARB_API_BEGIN(ctx) ctx->e.get_row_text(out); ARB_API_END(ctx) }
int arb_build_consensus(arb_ctx* ctx, const uint32_t* candidates, uint32_t n_rows, arb_consensus_info* info) { ARB_API_BEGIN(ctx) ctx->e.build_consensus(candidates, n_rows, *info); ARB_API_END(ctx) }
int arb_get_consensus(arb_ctx* ctx, uint32_t* seq_off, uint32_t* pos_off, uint32_t* clip_off, uint8_t* verdict, uint32_t* non_template, char* seq, int32_t* pos, char* clip) {
	ARB_API_BEGIN(ctx) ctx->e.get_consensus(seq_off, pos_off, clip_off, verdict, non_template, seq, pos, clip); ARB_API_END(ctx)
}
int arb_filter_multimappers(arb_ctx* ctx) { ARB_API_BEGIN(ctx) ctx->e.filter_multimappers(); ARB_API_END(ctx) }
int arb_set_splice_sites(arb_ctx* ctx, const uint32_t* off, const int32_t* sites) { ARB_API_BEGIN(ctx) ctx->e.set_splice_sites(off, sites); ARB_API_END(ctx) }
int arb_build_kmer_index(arb_ctx* ctx, const uint32_t* contig, const int32_t* start, const int32_t* end, uint32_t n, uint32_t nc, uint64_t* n_indexed) { ARB_API_BEGIN(ctx) uint64_t k = ctx->e.build_kmer_index(contig, start, end, n, nc); if (n_indexed) *n_indexed = k; ARB_API_END(ctx) }
int arb_homolog_pairs(arb_ctx* ctx, const uint32_t* ga, const uint32_t* gb, uint32_t n, uint8_t* out) { ARB_API_BEGIN(ctx) ctx->e.homolog_pairs(ga, gb, n, out); ARB_API_END(ctx) }
int arb_filter_mismappers(arb_ctx* ctx, int32_t max_mate_gap, uint64_t* n) { ARB_API_BEGIN(ctx) uint64_t k = ctx->e.filter_mismappers(max_mate_gap); if (n) *n = k; ARB_API_END(ctx) }
int arb_exchange_header(arb_ctx* ctx, int group, uint64_t* header, uint32_t* n_words) {
	ARB_API_BEGIN(ctx) std::vector<u64> h; ctx->e.exchange_header(group, h); if (h.size() > 16) throw arb_error("exchange header too long"); for (size_t k = 0; k < h.size(); ++k) header[k] = h[k]; *n_words = (uint32_t) h.size(); ARB_API_END(ctx)
}
int arb_exchange_prepare(arb_ctx* ctx, int group, const uint64_t* header, uint32_t n_words) { ARB_API_BEGIN(ctx) ctx->e.exchange_prepare(group, header, n_words); ARB_API_END(ctx) }
int arb_exchange_buffers(arb_ctx* ctx, int group, void** ptrs, uint64_t* bytes, uint32_t* n) {
	ARB_API_BEGIN(ctx) std::vector<exchange_buffer> b; ctx->e.exchange_buffers(group, b); if (b.size() > *n) throw arb_error("arb_exchange_buffers: capacity too small"); for (size_t k = 0; k < b.size(); ++k) { ptrs[k] = b[k].p; bytes[k] = b[k].bytes; } *n = (uint32_t) b.size(); ARB_API_END(ctx)
}
int arb_exchange_commit(arb_ctx* ctx, int group) { ARB_API_BEGIN(ctx) ctx->e.exchange_commit(group); ARB_API_END(ctx) }
int arb_set_work_partition(arb_ctx* ctx, const uint32_t* keys, const uint8_t* owner, uint32_t n_keys, int part, int parts) { ARB_API_BEGIN(ctx) ctx->e.set_work_partition(keys, owner, n_keys, part, parts); ARB_API_END(ctx) }
int arb_candidates_export(arb_ctx* ctx, void** blob, uint64_t* bytes, uint64_t sizes[4]) { ARB_API_BEGIN(ctx) u64 s[4]; u64 b = 0; ctx->e.candidates_export(blob, &b, s); *bytes = b; for (int k = 0; k < 4; ++k) sizes[k] = s[k]; ARB_API_END(ctx) }
int arb_candidates_import(arb_ctx* ctx, const void* all_blobs, uint64_t stride, const uint64_t* sizes, uint32_t n_parts) { ARB_API_BEGIN(ctx) std::vector<u64> s(sizes, sizes + 4 * (size_t) n_parts); ctx->e.candidates_import(all_blobs, stride, s.data(), n_parts); ARB_API_END(ctx) }
int arb_swaps_buffer(arb_ctx* ctx, void** p, uint64_t* bytes) { ARB_API_BEGIN(ctx) u64 b = 0; ctx->e.swaps_buffer(p, &b); *bytes = b; ARB_API_END(ctx) }
int arb_swaps_apply(arb_ctx* ctx) { ARB_API_BEGIN(ctx) ctx->e.swaps_apply(); ARB_API_END(ctx) }
int arb_filter_mismappers_part(arb_ctx* ctx, int32_t max_mate_gap, int part, int parts, void** verdicts, uint64_t* bytes) { ARB_API_BEGIN(ctx) u64 b = 0; ctx->e.filter_mismappers_part(max_mate_gap, part, parts, verdicts, &b); *bytes = b; ARB_API_END(ctx) }
int arb_filter_mismappers_finish(arb_ctx* ctx, uint64_t* n) { ARB_API_BEGIN(ctx) const uint64_t k = ctx->e.filter_mismappers_finish(); if (n) *n = k; ARB_API_END(ctx) }
int arb_get_timings(arb_ctx* ctx, arb_timings* out) { ARB_API_BEGIN(ctx) *out = ctx->e.timings; ARB_API_END(ctx) }
int arb_selftest_mismatch_counts(arb_ctx* ctx, uint32_t* out) { ARB_API_BEGIN(ctx) ctx->e.probe_mismatch_counts(out); ARB_API_END(ctx) } // tests only, not declared in the public header
int arb_selftest_staged_chunk(arb_ctx* ctx, uint8_t* out, uint64_t n) { ARB_API_BEGIN(ctx) if (!ctx->e.rec_stage_pending || n > ctx->e.rec_carry + ctx->e.rec_staged) throw arb_error("no staged chunk of that size"); ctx->e.bam_buf.download(ctx->e.ex, out, n); ARB_API_END(ctx) } // tests only, as above: the chunk arb_records_bgzf_stage assembled, behind the carried record
int arb_selftest_kmer_lookup(arb_ctx* ctx, const uint32_t* contig, const uint32_t* kmer, const int32_t* from, uint32_t n, uint32_t* out) { ARB_API_BEGIN(ctx) ctx->e.probe_kmer_lookup(contig, kmer, from, n, out); ARB_API_END(ctx) } // tests only, as above
int arb_set_genomic_breakpoints(arb_ctx* ctx, uint32_t n, const uint16_t* c1, const uint16_t* c2, const uint8_t* d1, const uint8_t* d2, const int32_t* p1, const int32_t* p2) {
	ARB_API_BEGIN(ctx) ctx->e.set_genomic_breakpoints(n, c1, c2, d1, d2, p1, p2); ARB_API_END(ctx)
}
int arb_mark_genomic_support(arb_ctx* ctx, int32_t max_distance, int32_t max_itd_length, uint32_t* marked) { ARB_API_BEGIN(ctx) const uint32_t m = ctx->e.mark_genomic_support(max_distance, max_itd_length); if (marked) *marked = m; ARB_API_END(ctx) }
int arb_get_genomic_support(arb_ctx* ctx, int32_t* closest1, int32_t* closest2) { ARB_API_BEGIN(ctx) ctx->e.get_genomic_support(closest1, closest2); ARB_API_END(ctx) }
int arb_set_blacklist(arb_ctx* ctx, uint32_t n, const uint8_t* t1, const uint8_t* t2, const uint8_t* s1, const uint8_t* s2, const uint16_t* c1, const uint16_t* c2,
                      const int32_t* b1, const int32_t* e1, const int32_t* b2, const int32_t* e2, const uint32_t* g1, const uint32_t* g2) {
	ARB_API_BEGIN(ctx) ctx->e.set_rules(ctx->e.blacklist_rules, "arb_set_blacklist", n, t1, t2, s1, s2, c1, c2, b1, e1, b2, e2, g1, g2); ARB_API_END(ctx)
}
int arb_filter_blacklist(arb_ctx* ctx, uint32_t n_ids, const uint32_t* ids, float evalue_cutoff, int32_t max_mate_gap, uint8_t* verdicts, uint32_t* n_blacklisted) {
	ARB_API_BEGIN(ctx) const uint32_t b = ctx->e.filter_blacklist(n_ids, ids, evalue_cutoff, max_mate_gap, verdicts); if (n_blacklisted) *n_blacklisted = b; ARB_API_END(ctx)
}
int arb_set_known_fusions(arb_ctx* ctx, uint32_t n, const uint8_t* t1, const uint8_t* t2, const uint8_t* s1, const uint8_t* s2, const uint16_t* c1, const uint16_t* c2,
                          const int32_t* b1, const int32_t* e1, const int32_t* b2, const int32_t* e2, const uint32_t* g1, const uint32_t* g2) {
	ARB_API_BEGIN(ctx) ctx->e.set_rules(ctx->e.known_rules, "arb_set_known_fusions", n, t1, t2, s1, s2, c1, c2, b1, e1, b2, e2, g1, g2); ARB_API_END(ctx)
}
int arb_recover_known_fusions(arb_ctx* ctx, uint32_t n_ids, const uint32_t* ids, int32_t max_mate_gap, uint8_t* verdicts, uint32_t* n_rescued) {
	ARB_API_BEGIN(ctx) const uint32_t r = ctx->e.recover_known_fusions(n_ids, ids, max_mate_gap, verdicts); if (n_rescued) *n_rescued = r; ARB_API_END(ctx)
}
int arb_set_tags(arb_ctx* ctx, uint32_t n, const uint8_t* t1, const uint8_t* t2, const uint8_t* s1, const uint8_t* s2, const uint16_t* c1, const uint16_t* c2,
                 const int32_t* b1, const int32_t* e1, const int32_t* b2, const int32_t* e2, const uint32_t* g1, const uint32_t* g2,
                 const uint32_t* tag_rank, uint32_t n_tags, const char* tag_chars, const uint32_t* tag_off) {
	ARB_API_BEGIN(ctx) ctx->e.set_rules(ctx->e.tag_rules, "arb_set_tags", n, t1, t2, s1, s2, c1, c2, b1, e1, b2, e2, g1, g2); ctx->e.set_tags(tag_rank, n_tags, tag_chars, tag_off); ARB_API_END(ctx)
}
int arb_annotate_tags(arb_ctx* ctx, uint32_t n_ids, const uint32_t* ids, int32_t max_mate_gap, uint64_t* n_pairs) {
	ARB_API_BEGIN(ctx) const uint64_t p = ctx->e.annotate_tags(n_ids, ids, max_mate_gap); if (n_pairs) *n_pairs = p; ARB_API_END(ctx)
}
int arb_get_tags(arb_ctx* ctx, uint32_t* off, uint32_t* ranks) { ARB_API_BEGIN(ctx) ctx->e.get_tags(off, ranks); ARB_API_END(ctx) }
int arb_set_protein_domains(arb_ctx* ctx, uint32_t n, const uint16_t* contig, const int32_t* start, const int32_t* end, const uint32_t* gene, const uint32_t* name_rank,
                            uint32_t n_names, const char* name_chars, const uint32_t* name_off) {
	ARB_API_BEGIN(ctx) ctx->e.set_protein_domains(n, contig, start, end, gene, name_rank, n_names, name_chars, name_off); ARB_API_END(ctx)
}
int arb_retained_protein_domains(arb_ctx* ctx, uint32_t n_ids, const uint32_t* ids, uint64_t* n_bytes) {
	ARB_API_BEGIN(ctx) const uint64_t b = ctx->e.retained_protein_domains(n_ids, ids); if (n_bytes) *n_bytes = b; ARB_API_END(ctx)
}
int arb_get_retained_protein_domains(arb_ctx* ctx, uint64_t* off, char* text) { ARB_API_BEGIN(ctx) ctx->e.get_retained_protein_domains(off, text); ARB_API_END(ctx) }
int arb_set_fill_transcripts(arb_ctx* ctx, uint32_t n, const int32_t* first_exon, const int32_t* last_exon, const uint32_t* contig, const int32_t* exon_next, const int32_t* exon_prev) {
	ARB_API_BEGIN(ctx) ctx->e.set_fill_transcripts(n, first_exon, last_exon, contig, exon_next, exon_prev); ARB_API_END(ctx)
}
int arb_fill_gaps(arb_ctx* ctx, uint32_t n_rows, const char* text, const uint32_t* row_off, const int32_t* pos, const uint32_t* pos_off, uint32_t n_jobs, const uint32_t* row, const uint32_t* transcript,
                  const uint8_t* flags, uint64_t* n_chars) {
	ARB_API_BEGIN(ctx) const uint64_t n = ctx->e.fill_gaps(n_rows, text, row_off, pos, pos_off, n_jobs, row, transcript, flags); if (n_chars) *n_chars = n; ARB_API_END(ctx)
}
int arb_get_filled(arb_ctx* ctx, uint32_t* off, char* chars, int32_t* pos) { ARB_API_BEGIN(ctx) ctx->e.get_filled(off, chars, pos); ARB_API_END(ctx) }
int arb_get_slot_swaps(arb_ctx* ctx, uint8_t* out) { ARB_API_BEGIN(ctx) ctx->e.get_slot_swaps(out); ARB_API_END(ctx) }

} // extern "C"
