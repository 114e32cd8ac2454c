// host_capi.cpp -- C ABI of the whole-run driver (include/arriba_b200.h, "whole-run driver" section).
#include <malloc.h>
#include "pipeline.h"
#include "index_query.h"
#include <climits>
#include <cstring>
#include <stdexcept>

using namespace arb::host;

struct arb_pipeline { pipeline p; std::string error; };
static std::string g_pipeline_create_error;

#define PIPE_BEGIN(x) if (!(x)) return 2; try {
#define PIPE_END(x) } catch (const std::exception& e) { (x)->error = e.what(); return 1; } catch (...) { (x)->error = "unknown error"; return 1; } return 0;

extern "C" {

void arb_struct_sizes(uint32_t out[9]) {
	out[0] = sizeof(arb_contigs); out[1] = sizeof(arb_annotation); out[2] = sizeof(arb_params); out[3] = sizeof(arb_soa_chunk); out[4] = sizeof(arb_candidates);
	out[5] = sizeof(arb_evalue_inputs); out[6] = sizeof(arb_timings); out[7] = sizeof(arb_run_options); out[8] = sizeof(arb_run_stats);
}

void arb_default_run_options(arb_run_options* o) {
	if (!o) return;
	memset(o, 0, sizeof(*o));
	arb_default_params(&o->params);
	o->strandedness = 3; o->fragment_length = 200; o->threads = 1; o->device = 0;
	o->min_support = 2; o->min_anchor_length = 23; o->min_spliced_events = 4; o->high_expression_quantile = 0.998f; o->exonic_fraction = 0.33f;
	o->min_itd_allele_fraction = 0.07f; o->min_itd_support = 10; o->print_extra_info_for_discarded_fusions = 0; o->echo_progress = 0;
	o->top_viral_contigs = 5; o->viral_contig_min_covered_fraction = 0.05f;
	o->genomic_breakpoints_file = NULL; o->max_genomic_breakpoint_distance = 100000; o->blacklist_file = NULL; o->known_fusions_file = NULL; o->tags_file = NULL; o->protein_domains_file = NULL; o->chimeric_file = NULL;
}

// Dozens of host threads allocate and free at the same time (record parsing, annotation, row formatting). glibc gives every thread its own arena, but arenas
// hand memory back to the kernel and map new chunks all the time, and those calls serialise on the process's address-space lock: keep what was obtained.
static void tune_allocator() { // once per process, also when two threads create their first pipelines at the same moment (a local static's initialiser runs once)
	static const int done = (mallopt(M_TRIM_THRESHOLD, 1 << 30), mallopt(M_TOP_PAD, 64 << 20), mallopt(M_MMAP_THRESHOLD, 32 << 20), 1);
	(void) done;
}

void arb_release_host_memory(void) { arb::host::host_block_trim(); }

int arb_pipeline_create(arb_pipeline** out, const arb_run_options* o) {
	tune_allocator();
	if (!out || !o) return 2;
	*out = NULL;
	try {
		if (!o->bam_file || !o->gtf_file || !o->assembly_file) throw std::runtime_error("bam_file, gtf_file and assembly_file are mandatory");
		if (o->max_genomic_breakpoint_distance > INT_MAX) throw std::runtime_error("max_genomic_breakpoint_distance must not exceed INT_MAX"); // -D takes 0..INT_MAX (options.cpp:401-403)
		arb_set_host_memory_device(o->device); // the device whose context page-locks the recycled host blocks
		arb_pipeline* x = new arb_pipeline();
		run_options& r = x->p.opt;
		r.bam_file = o->bam_file; r.gtf_file = o->gtf_file; r.assembly_file = o->assembly_file;
		if (o->output_file) r.output_file = o->output_file;
		if (o->discarded_output_file) r.discarded_output_file = o->discarded_output_file;
		if (o->interesting_contigs) r.interesting_contigs = o->interesting_contigs;
		if (o->viral_contigs) r.viral_contigs = o->viral_contigs;
		r.min_support = o->min_support; r.min_anchor_length = o->min_anchor_length; r.min_spliced_events = o->min_spliced_events; r.high_expression_quantile = o->high_expression_quantile;
		r.exonic_fraction = o->exonic_fraction; r.min_itd_allele_fraction = o->min_itd_allele_fraction; r.min_itd_support = o->min_itd_support;
		r.print_extra_info_for_discarded_fusions = o->print_extra_info_for_discarded_fusions != 0; r.echo_progress = o->echo_progress != 0;
		r.top_viral_contigs = o->top_viral_contigs; r.viral_contig_min_covered_fraction = o->viral_contig_min_covered_fraction;
		if (o->genomic_breakpoints_file) r.genomic_breakpoints_file = o->genomic_breakpoints_file;
		r.max_genomic_breakpoint_distance = o->max_genomic_breakpoint_distance;
		if (o->blacklist_file) r.blacklist_file = o->blacklist_file;
		if (o->known_fusions_file) r.known_fusions_file = o->known_fusions_file;
		if (o->tags_file) r.tags_file = o->tags_file;
		if (o->protein_domains_file) r.protein_domains_file = o->protein_domains_file;
		if (o->chimeric_file) r.chimeric_file = o->chimeric_file;
		r.fill_sequence_gaps = o->fill_sequence_gaps != 0;
		r.params = o->params; r.strandedness = o->strandedness; r.fragment_length = o->fragment_length; r.threads = o->threads; r.device = o->device;
		*out = x;
	} catch (const std::exception& e) { g_pipeline_create_error = e.what(); return 1; }
	return 0;
}

void arb_pipeline_destroy(arb_pipeline* p) { delete p; }
const char* arb_pipeline_error(arb_pipeline* p) { return p ? p->error.c_str() : g_pipeline_create_error.c_str(); }

int arb_pipeline_step(arb_pipeline* x, int step) {
	PIPE_BEGIN(x)
	switch (step) {
		case ARB_STEP_LOAD_REFERENCE: x->p.load_reference(); break;
		case ARB_STEP_INGEST: x->p.ingest(); break;
		case ARB_STEP_ANNOTATE: x->p.annotate(); break;
		case ARB_STEP_UPLOAD: x->p.upload(); break;
		case ARB_STEP_READ_FILTERS: x->p.read_filters(); break;
		case ARB_STEP_FRAGMENT_LENGTH: x->p.fragment_length(); break;
		case ARB_STEP_FIND_FUSIONS: x->p.find_fusions(); break;
		default: throw std::runtime_error("unknown pipeline step");
	}
	PIPE_END(x)
}

int arb_pipeline_attach_device(arb_pipeline* x) { PIPE_BEGIN(x) x->p.attach_device(); PIPE_END(x) }
int arb_pipeline_work_partition(arb_pipeline* x, int parts, const uint32_t** keys, const uint8_t** owner, uint32_t* n_keys) {
	PIPE_BEGIN(x) x->p.work_partition(parts); *keys = x->p.partition_keys.data(); *owner = x->p.partition_owner.data(); *n_keys = (uint32_t) x->p.partition_keys.size(); PIPE_END(x)
}
int arb_pipeline_mismappers_begin(arb_pipeline* x, int* active) { PIPE_BEGIN(x) const bool a = x->p.mismappers_begin(); if (active) *active = a ? 1 : 0; PIPE_END(x) }
int arb_pipeline_mismappers_end(arb_pipeline* x) { PIPE_BEGIN(x) x->p.mismappers_end(); PIPE_END(x) }
int arb_pipeline_run(arb_pipeline* x) { PIPE_BEGIN(x) x->p.run_all(); PIPE_END(x) }
arb_ctx* arb_pipeline_ctx(arb_pipeline* x) { return x ? x->p.ctx : NULL; }

int arb_pipeline_stats(arb_pipeline* x, arb_run_stats* s) {
	PIPE_BEGIN(x)
	const pipeline& p = x->p;
	memset(s, 0, sizeof(*s));
	s->n_fragments = p.frags.n; s->n_records = p.istats.records; s->mapped_reads = p.istats.mapped_reads; s->malformed = p.istats.malformed;
	s->strandedness = p.strandedness; s->max_mate_gap = p.max_mate_gap; s->fragment_length_ok = p.fragment_length_ok;
	s->mate_gap_mean = p.mate_gap_mean; s->mate_gap_stddev = p.mate_gap_stddev; s->read_length_mean = p.read_length_mean;
	s->seconds[ARB_STEP_LOAD_REFERENCE] = p.t_reference; s->seconds[ARB_STEP_INGEST] = p.t_ingest; s->seconds[ARB_STEP_ANNOTATE] = p.t_annotate;
	s->seconds[ARB_STEP_UPLOAD] = p.t_upload; s->seconds[ARB_STEP_READ_FILTERS] = p.t_read_filters; s->seconds[ARB_STEP_FRAGMENT_LENGTH] = p.t_fragment_length;
	s->seconds[ARB_STEP_FIND_FUSIONS] = p.t_find_fusions;
	s->t_inflate = p.istats.t_inflate; s->t_parse = p.istats.t_parse; s->t_finalize = p.istats.t_finalize;
	for (int q = 0; q < 32 && q < EV_COUNT; ++q) s->event_seconds[q] = p.t_events[q];
	s->output_seconds = p.t_output; s->n_candidates = p.ev.n;
	s->chimeric_records = p.istats.chimeric_records; s->chimeric_malformed = p.istats.chimeric_malformed; s->chimeric_total = p.istats.chimeric_total;
	for (arb::u32 q = 0; q < p.ev.n; ++q) if (p.ev.filter[q] == 0) ++s->n_unfiltered_candidates;
	const arb::host::fragment_table& f = p.frags;
	s->h2d_bytes = f.n_aln.size() + f.fflags.size() + f.filter.size() + f.aflags.size() + 2 * (f.contig.size() + f.cigar_cnt.size() + f.seq_len.size() + f.genes_cnt.size()) +
	               4 * (f.start.size() + f.end.size() + f.cigar_off.size() + f.seq_off.size() + f.genes_off.size() + f.cigar.size() + f.genes.size()) + f.seq.size();
	PIPE_END(x)
}

int arb_pipeline_fragments(arb_pipeline* x, arb_soa_chunk* c, const char** names, const uint64_t** name_off) {
	PIPE_BEGIN(x)
	const arb::host::fragment_table& f = x->p.frags;
	c->n_fragments = f.n; c->n_aln = f.n_aln.data(); c->fflags = f.fflags.data(); c->filter = f.filter.data(); c->contig = f.contig.data(); c->start = f.start.data(); c->end = f.end.data();
	c->aflags = f.aflags.data(); c->cigar_off = f.cigar_off.data(); c->cigar_cnt = f.cigar_cnt.data(); c->seq_off = f.seq_off.data(); c->seq_len = f.seq_len.data();
	c->genes_off = f.genes_off.data(); c->genes_cnt = f.genes_cnt.data(); c->cigar = f.cigar.data(); c->n_cigar = f.cigar.size(); c->seq = f.seq.data(); c->n_seq_bytes = f.seq.size();
	c->genes = f.genes.data(); c->n_genes = f.genes.size();
	if (names) *names = f.names.data();
	if (name_off) *name_off = f.name_off.data();
	PIPE_END(x)
}

int arb_pipeline_genes(arb_pipeline* x, arb_annotation* a) {
	PIPE_BEGIN(x)
	refdata& r = x->p.ref;
	memset(a, 0, sizeof(*a));
	a->n_genes = (uint32_t) r.genes.size(); a->gene_contig = r.f_gene_contig.data(); a->gene_start = r.f_gene_start.data(); a->gene_end = r.f_gene_end.data();
	a->gene_strand = r.f_gene_strand.data(); a->gene_exonic_length = r.f_gene_exonic_length.data(); a->gene_flags = r.f_gene_flags.data();
	a->n_exons = (uint32_t) r.exons.size(); a->exon_gene = r.f_exon_gene.data(); a->exon_start = r.f_exon_start.data(); a->exon_end = r.f_exon_end.data();
	a->exon_cds_start = r.f_exon_cds_start.data(); a->exon_cds_end = r.f_exon_cds_end.data(); a->exon_next_start = r.f_exon_next_start.data(); a->exon_flags = r.f_exon_flags.data();
	a->n_contigs = (uint32_t) r.contig_ids.size();
	a->exon_region_begin = r.exon_index.begin.data(); a->exon_region_end = r.exon_index.end.data(); a->exon_region_off = r.exon_index.off.data(); a->exon_region_items = r.exon_index.items.data();
	a->gene_region_begin = r.gene_index.begin.data(); a->gene_region_end = r.gene_index.end.data(); a->gene_region_off = r.gene_index.off.data(); a->gene_region_items = r.gene_index.items.data();
	PIPE_END(x)
}

int arb_pipeline_coverage(arb_pipeline* x, uint32_t contig, const uint16_t** cov, const uint8_t** starts, const uint8_t** ends, uint64_t* n) {
	PIPE_BEGIN(x)
	const coverage_windows& c = x->p.coverage;
	if (contig >= c.coverage.size()) { *n = 0; *cov = NULL; *starts = NULL; *ends = NULL; }
	else { *n = c.coverage[contig].size(); *cov = c.coverage[contig].data(); *starts = c.starts[contig].data(); *ends = c.ends[contig].data(); }
	PIPE_END(x)
}

int arb_pipeline_write_output(arb_pipeline* x) { PIPE_BEGIN(x) x->p.write_output(); PIPE_END(x) }
int arb_pipeline_events(arb_pipeline* x, int last_stage) { PIPE_BEGIN(x) x->p.events_until(last_stage); PIPE_END(x) }

int arb_pipeline_candidates(arb_pipeline* x, arb_candidates* c, const uint32_t** order, const uint8_t** confidence, const uint8_t** labels) {
	PIPE_BEGIN(x)
	x->p.order_ready();
	event_table& e = x->p.ev;
	c->n = e.n; c->gene1 = e.gene1.data(); c->gene2 = e.gene2.data(); c->contig1 = e.contig1.data(); c->contig2 = e.contig2.data(); c->breakpoint1 = e.bp1.data(); c->breakpoint2 = e.bp2.data();
	c->direction1 = e.dir1.data(); c->direction2 = e.dir2.data(); c->split_reads1 = e.split_reads1.data(); c->split_reads2 = e.split_reads2.data(); c->discordant_mates = e.discordant_mates.data();
	c->filter = e.filter.data(); c->bits = e.bits.data(); c->bits2 = e.bits2.data(); c->anchor_start1 = e.anchor1.data(); c->anchor_start2 = e.anchor2.data(); c->evalue = e.evalue.data();
	c->list1_off = e.list1_off.data(); c->list2_off = e.list2_off.data(); c->listd_off = e.listd_off.data(); c->list1 = e.list1.data(); c->list2 = e.list2.data(); c->listd = e.listd.data();
	if (order) *order = e.order.data();
	if (confidence) *confidence = e.confidence.data();
	if (labels) *labels = x->p.labels.data();
	PIPE_END(x)
}

int arb_pipeline_genomic_support(arb_pipeline* x, const int32_t** closest1, const int32_t** closest2) {
	PIPE_BEGIN(x)
	const event_table& e = x->p.ev;
	*closest1 = e.closest1.empty() ? NULL : e.closest1.data(); *closest2 = e.closest2.empty() ? NULL : e.closest2.data();
	PIPE_END(x)
}

/* tests only (tests/test_prims.py), not part of the public header: the small-set-first front end of the annotation queries (index_query.h) against the plain
   query with a large set, on a hand-made index whose loci hold up to `crowd` records; returns the number of queries that differ */
int arb_selftest_index_query(uint32_t crowd) {
	using namespace arb;
	// regions (ends ascending): a crowded one, a second crowded one ending 1 bp later (range queries merge neighbours within 2 bp), then sparse ones
	std::vector<i32> end; std::vector<u32> off(1, 0), items;
	auto region = [&](i32 e, u32 first, u32 n) { end.push_back(e); for (u32 k = 0; k < n; ++k) items.push_back(first + k); off.push_back((u32) items.size()); };
	region(100, 0, crowd); region(101, crowd / 2, crowd); region(500, 5, 1); region(900, 7, 3); region(2000, 2 * crowd, 2);
	const u32 begin[2] = {0, (u32) end.size()};
	region_index_view ix; ix.begin = begin; ix.end = end.data(); ix.off = off.data(); ix.items = items.data(); ix.n_contigs = 1; ix.grid = NULL; ix.grid_begin = NULL;
	int differing = 0;
	const i32 points[] = {0, 50, 99, 100, 101, 102, 300, 498, 500, 501, 899, 900, 1500, 2000, 2001};
	for (size_t a = 0; a < sizeof(points) / sizeof(points[0]); ++a)
		for (size_t b = 0; b < sizeof(points) / sizeof(points[0]); ++b) {
			idset<4096> want; query_index(ix, 0, points[a], points[b], want);
			std::vector<u32> got;
			host::index_query<4096>(ix, 0, points[a], points[b], [&](const u32* v, u32 n) { got.assign(v, v + n); }, "overflow");
			if (want.overflow || got.size() != want.n || !std::equal(got.begin(), got.end(), want.v)) ++differing;
		}
	return differing;
}

} // extern "C"
