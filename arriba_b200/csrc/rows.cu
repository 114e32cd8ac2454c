// rows.cu -- driver of the device-side formatting of the discarded-fusions file (see rows_hd.h).
#include <cstdlib>
#include "engine.h"
#include "rows_hd.h"

namespace arb {

static void upload_pool(const exec_ctx& ex, dbuf<char>& chars, dbuf<u32>& off, const char* c, const u32* o, u32 n) {
	off.upload(ex, o, (size_t) n + 1);
	chars.ensure((size_t) o[n] + 1);
	if (o[n]) chars.upload(ex, c, o[n]);
}

void engine::set_row_texts(const arb_row_texts& t) {
	if (!has_annotation || t.n_genes != annot.n_genes || t.n_exons != annot.n_exons || t.n_contigs != annot.n_contigs) throw arb_error("arb_set_row_texts: the tables do not match the resident annotation");
	upload_pool(ex, row_gene_name, row_gene_name_off, t.gene_name, t.gene_name_off, t.n_genes);
	upload_pool(ex, row_gene_id, row_gene_id_off, t.gene_id, t.gene_id_off, t.n_genes);
	upload_pool(ex, row_contig_name, row_contig_name_off, t.contig_name, t.contig_name_off, t.n_contigs);
	upload_pool(ex, row_filter_name, row_filter_name_off, t.filter_name, t.filter_name_off, ARB_N_FILTERS);
	row_exon_prev.upload(ex, t.exon_prev, t.n_exons); row_exon_next.upload(ex, t.exon_next, t.n_exons);
	for (int k = 0; k < ARB_N_FILTERS; ++k) row_filters_by_name[k] = t.filters_by_name[k];
	row_max_itd_length = t.max_itd_length;
	ex.sync();
	has_row_texts = true;
}

// the rows of the candidates that are not F_none, in iteration order; the text stays on the device until arb_get_row_text
void engine::format_discarded_rows(const u8* confidence, u64* n_rows, u64* n_bytes) {
	if (!has_row_texts) throw arb_error("arb_format_discarded_rows: arb_set_row_texts must be called first");
	if (coverage_contigs == 0) throw arb_error("arb_format_discarded_rows: arb_set_coverage must be called first");
	const u32 C = cands.n;
	*n_rows = 0; *n_bytes = 0; row_text_bytes = 0;
	if (C == 0) return;
	if (order_seq.size() < C) throw arb_error("arb_format_discarded_rows: arb_replay_insertion_order must be called first");
	stage_timer t_all(ex);
	dbuf<u8> conf; conf.upload(ex, confidence, C);
	dbuf<u32> flag((size_t) C + 1), rows(C);
	row_select_fn sf = {order_seq.ptr(), cands.filter.ptr(), flag.ptr()};
	for_each(ex, C, sf);
	exclusive_scan_u32(ex, flag.ptr(), flag.ptr(), C);
	u32 R = 0; flag.download(ex, &R, 1, C);
	row_gather_fn gf = {order_seq.ptr(), flag.ptr(), rows.ptr()};
	for_each(ex, C, gf);
	row_formatter fm;
	fm.c = make_state_for_rows(); fm.f = frags.view(); fm.an = annot.view();
	fm.t.gene_name.chars = row_gene_name.ptr(); fm.t.gene_name.off = row_gene_name_off.ptr(); fm.t.gene_id.chars = row_gene_id.ptr(); fm.t.gene_id.off = row_gene_id_off.ptr();
	fm.t.contig_name.chars = row_contig_name.ptr(); fm.t.contig_name.off = row_contig_name_off.ptr(); fm.t.filter_name.chars = row_filter_name.ptr(); fm.t.filter_name.off = row_filter_name_off.ptr();
	fm.t.exon_prev = row_exon_prev.ptr(); fm.t.exon_next = row_exon_next.ptr(); fm.t.confidence = conf.ptr();
	fm.t.closest1 = cands.genomic_marked ? cands.closest1.ptr() : NULL; fm.t.closest2 = cands.genomic_marked ? cands.closest2.ptr() : NULL;
	fm.t.cov.windows = coverage_windows.ptr(); fm.t.cov.contig_off = coverage_off.ptr(); fm.t.cov.contig_windows = coverage_n.ptr(); fm.t.cov.n_contigs = coverage_contigs;
	const bool tags = has_tag_csr && tag_csr_n == C; // arb_annotate_tags ran on this candidate table
	fm.t.tag_text.chars = tags ? tag_text.ptr() : NULL; fm.t.tag_text.off = tags ? tag_text_off.ptr() : NULL;
	fm.t.tag_off = tags ? tag_csr_off.ptr() : NULL; fm.t.tag_rank = tags ? tag_csr_rank.ptr() : NULL;
	fm.t.domains = domain_tables();
	for (int k = 0; k < ARB_N_FILTERS; ++k) fm.t.filters_by_name[k] = row_filters_by_name[k];
	fm.t.max_itd_length = row_max_itd_length;
	fm.l1o = cands.list1_off.ptr(); fm.l1 = cands.list1.ptr(); fm.l2o = cands.list2_off.ptr(); fm.l2 = cands.list2.ptr(); fm.ldo = cands.listd_off.ptr(); fm.ld = cands.listd.ptr();
	// pass 1: row lengths, block by block (32-bit offsets inside a block of rows)
	u32 BLOCK = 1u << 21; // 2 M rows: even kilobyte rows stay below 2^32 bytes
	if (const char* e = getenv("ARB_ROW_BLOCK")) BLOCK = (u32) std::max(4L, atol(e)) / 4 * 4; // test hook: many blocks
	const u32 n_blocks = (R + BLOCK - 1) / BLOCK;
	const size_t STRIDE = (size_t) BLOCK + 4; // a block's lengths + its total, every block's array 16-byte aligned (the scan reads vectors)
	dbuf<u32> length(STRIDE * n_blocks + 4);
	std::vector<u64> base(n_blocks + 1, 0);
	for (u32 b = 0; b < n_blocks; ++b) {
		const u32 lo = b * BLOCK, n = std::min(BLOCK, R - lo);
		u32* len = length.ptr() + STRIDE * b; // n + 1 entries
		row_length_fn lf = {fm, rows.ptr() + lo, len};
		for_each(ex, n, lf);
		exclusive_scan_u32(ex, len, len, n);
		u32 total = 0; length.download(ex, &total, 1, STRIDE * b + n);
		base[b + 1] = base[b] + total;
	}
	if (has_protein_domains) check_domain_error("arb_format_discarded_rows");
	row_text.ensure(base[n_blocks] + 1);
	for (u32 b = 0; b < n_blocks; ++b) {
		const u32 lo = b * BLOCK, n = std::min(BLOCK, R - lo);
		row_write_fn wf = {fm, rows.ptr() + lo, length.ptr() + STRIDE * b, row_text.ptr() + base[b]};
		for_each(ex, n, wf);
	}
	row_text_bytes = base[n_blocks];
	timings.rows_ms = t_all.stop();
	ex.sync();
	*n_rows = R; *n_bytes = row_text_bytes;
}

void engine::get_row_text(char* out) { row_text.download(ex, out, row_text_bytes); }

} // namespace arb
