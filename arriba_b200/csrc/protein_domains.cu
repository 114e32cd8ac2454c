// protein_domains.cu -- driver of the protein domain tables (-p, see domains_hd.h) and of the retained_protein_domains column of the rows the host formats.
#include <cstdlib>
#include "engine.h"
#include "rows_hd.h"

namespace arb {

static u32 bits_for_values_below(u32 n) { u32 b = 1; while (b < 32 && ((u64) 1 << b) < n) ++b; return b; }

// the accepted records in file order: the distinct (contig, key) pairs of the index, the multiplicity of every record, and the kept records by (gene, name rank)
void engine::set_protein_domains(u32 n, const u16* contig, const i32* start, const i32* end, const u32* gene, const u32* name_rank, u32 n_names, const char* chars, const u32* off) {
	has_protein_domains = false;
	if (!has_annotation) throw arb_error("arb_set_protein_domains: no annotation");
	if (n == 0) throw arb_error("arb_set_protein_domains: no records");
	if (n >= (1u << 30)) throw arb_error("arb_set_protein_domains: too many records");
	for (u32 k = 0; k < n_names; ++k) if (off[k + 1] < off[k]) throw arb_error("arb_set_protein_domains: name offsets must not decrease");
	for (u32 i = 0; i < n; ++i) {
		if (gene[i] >= annot.n_genes) throw arb_error("arb_set_protein_domains: gene out of range in record " + std::to_string(i));
		if (name_rank[i] >= n_names) throw arb_error("arb_set_protein_domains: name rank out of range in record " + std::to_string(i));
		if (contig[i] >= n || contig[i] >= annot.n_contigs) throw arb_error("arb_set_protein_domains: contig out of range in record " + std::to_string(i) + " (it must be below the number of records)");
	}
	stage_timer t(ex);
	dbuf<u16> d_contig; dbuf<i32> d_start, d_end; dbuf<u32> d_gene, d_name;
	d_contig.upload(ex, contig, n); d_start.upload(ex, start, n); d_end.upload(ex, end, n); d_gene.upload(ex, gene, n); d_name.upload(ex, name_rank, n);
	// the index keys, sorted by (contig, key) and made distinct
	const u32 K = 2 * n;
	dbuf<u32> key(K), key_contig(K), key_tmp(K), contig_tmp(K), flag((size_t) K + 1);
	domain_keys_fn kf = {d_contig.ptr(), d_start.ptr(), d_end.ptr(), key.ptr(), key_contig.ptr()};
	for_each(ex, n, kf);
	radix_sort_pairs_u32(ex, key.ptr(), key_contig.ptr(), key_tmp.ptr(), contig_tmp.ptr(), K, 32);
	radix_sort_pairs_u32(ex, key_contig.ptr(), key.ptr(), contig_tmp.ptr(), key_tmp.ptr(), K, bits_for_values_below(annot.n_contigs));
	domain_distinct_fn df = {key_contig.ptr(), key.ptr(), flag.ptr()};
	for_each(ex, K, df);
	exclusive_scan_u32(ex, flag.ptr(), flag.ptr(), K);
	u32 n_keys = 0; flag.download(ex, &n_keys, 1, K);
	dbuf<u64> keys(n_keys);
	domain_compact_keys_fn cf = {key_contig.ptr(), key.ptr(), flag.ptr(), keys.ptr()};
	for_each(ex, K, cf);
	// multiplicities, then the records that count, by name rank and (stable) by gene
	dbuf<u32> mult(n), keep((size_t) n + 1);
	domain_mult_fn mf = {d_contig.ptr(), d_start.ptr(), d_end.ptr(), d_gene.ptr(), annot.gene_start.ptr(), annot.gene_end.ptr(), annot.gene_flags.ptr(), keys.ptr(), n_keys, mult.ptr(), keep.ptr()};
	for_each(ex, n, mf);
	exclusive_scan_u32(ex, keep.ptr(), keep.ptr(), n);
	u32 R = 0; keep.download(ex, &R, 1, n);
	dbuf<u32> sk(R), idx(R), sk_tmp(R), idx_tmp(R);
	domain_select_fn sf = {keep.ptr(), d_name.ptr(), sk.ptr(), idx.ptr()};
	for_each(ex, n, sf);
	if (R) radix_sort_pairs_u32(ex, sk.ptr(), idx.ptr(), sk_tmp.ptr(), idx_tmp.ptr(), R, bits_for_values_below(n_names));
	domain_gene_key_fn gk = {d_gene.ptr(), idx.ptr(), sk.ptr()};
	for_each(ex, R, gk);
	if (R) radix_sort_pairs_u32(ex, sk.ptr(), idx.ptr(), sk_tmp.ptr(), idx_tmp.ptr(), R, bits_for_values_below(annot.n_genes));
	dom_contig.ensure(R); dom_start.ensure(R); dom_end.ensure(R); dom_mult.ensure(R); dom_name.ensure(R); dom_gene_off.ensure((size_t) annot.n_genes + 1);
	domain_gather_fn gf = {idx.ptr(), d_contig.ptr(), d_start.ptr(), d_end.ptr(), mult.ptr(), d_name.ptr(), dom_contig.ptr(), dom_start.ptr(), dom_end.ptr(), dom_mult.ptr(), dom_name.ptr()};
	for_each(ex, R, gf);
	domain_gene_off_fn of = {sk.ptr(), R, dom_gene_off.ptr()};
	for_each(ex, annot.n_genes + 1, of);
	dom_name_off.upload(ex, off, (size_t) n_names + 1);
	dom_name_chars.ensure((size_t) off[n_names] + 1);
	if (off[n_names]) dom_name_chars.upload(ex, chars, off[n_names]);
	dom_error.ensure(1); dom_error.zero(ex, 1);
	timings.protein_domains_ms = t.stop();
	ex.sync();
	dom_records = n; has_protein_domains = true;
}

domain_view engine::domain_tables() {
	domain_view d;
	const bool on = has_protein_domains;
	d.gene_off = on ? dom_gene_off.ptr() : NULL;
	d.contig = dom_contig.ptr(); d.start = dom_start.ptr(); d.end = dom_end.ptr(); d.mult = dom_mult.ptr(); d.name = dom_name.ptr();
	d.name_chars = dom_name_chars.ptr(); d.name_off = dom_name_off.ptr(); d.n_records = dom_records; d.error = on ? dom_error.ptr() : NULL;
	return d;
}

void engine::check_domain_error(const char* who) {
	u32 e = 0; dom_error.download(ex, &e, 1);
	if (e) { dom_error.zero(ex, 1); ex.sync(); throw arb_error(std::string(who) + ": the lengths of a protein domain name sum to 0 (mod 2^32) while its retained bases do not: its percentage is undefined"); }
}

// the retained_protein_domains column of the candidates `ids`, one text per id; the texts stay here until arb_get_retained_protein_domains
u64 engine::retained_protein_domains(u32 n_ids, const u32* ids) {
	if (!has_protein_domains) throw arb_error("arb_retained_protein_domains: arb_set_protein_domains must be called first");
	const u32 C = cands.n;
	for (u32 i = 0; i < n_ids; ++i) if (ids[i] >= C) throw arb_error("arb_retained_protein_domains: candidate id out of range");
	dom_text_off.assign((size_t) n_ids + 1, 0);
	if (n_ids == 0) return 0;
	stage_timer t(ex);
	dbuf<u32> d_ids, length(n_ids);
	d_ids.upload(ex, ids, n_ids);
	row_formatter fm;
	fm.c = make_state_for_rows(); fm.an = annot.view(); fm.t.domains = domain_tables();
	domain_length_fn lf = {fm, d_ids.ptr(), length.ptr()};
	for_each(ex, n_ids, lf);
	std::vector<u32> len(n_ids); length.download(ex, len.data(), n_ids);
	check_domain_error("arb_retained_protein_domains");
	for (u32 i = 0; i < n_ids; ++i) dom_text_off[i + 1] = dom_text_off[i] + len[i];
	dbuf<u64> offset; offset.upload(ex, dom_text_off.data(), n_ids);
	dom_text.ensure(dom_text_off[n_ids] + 1);
	domain_write_fn wf = {fm, d_ids.ptr(), offset.ptr(), dom_text.ptr()};
	for_each(ex, n_ids, wf);
	timings.protein_domains_ms += t.stop();
	ex.sync();
	return dom_text_off[n_ids];
}

void engine::get_retained_protein_domains(u64* off, char* text) {
	for (size_t i = 0; i < dom_text_off.size(); ++i) off[i] = dom_text_off[i];
	if (!dom_text_off.empty()) dom_text.download(ex, text, dom_text_off.back());
}

} // namespace arb
