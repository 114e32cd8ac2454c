// events.cu -- drivers of the candidate-level device stages (see events_hd.h).
#include "engine.h"
#include "events_hd.h"

namespace arb {

static cand_state make_state(cand_store& c, u32* n1, u32* n2) {
	cand_state s;
	s.n = c.n; s.gene1 = c.gene1.ptr(); s.gene2 = c.gene2.ptr(); s.contig1 = c.contig1.ptr(); s.contig2 = c.contig2.ptr(); s.bp1 = c.bp1.ptr(); s.bp2 = c.bp2.ptr();
	s.dir1 = c.dir1.ptr(); s.dir2 = c.dir2.ptr(); s.bits = c.bits.ptr(); s.bits2 = c.bits2.ptr();
	s.split_reads1 = c.split_reads1.ptr(); s.split_reads2 = c.split_reads2.ptr(); s.discordant_mates = c.discordant_mates.ptr(); s.filter = c.filter.ptr(); s.evalue = c.evalue.ptr();
	s.n_list1 = n1; s.n_list2 = n2;
	return s;
}

cand_state engine::make_state_for_rows() { return make_state(cands, NULL, NULL); }

void engine::set_candidate_state(const u8* f, const u32* s1, const u32* s2, const u32* dm, const float* ev) {
	const u32 C = cands.n;
	cands.filter.upload(ex, f, C); cands.split_reads1.upload(ex, s1, C); cands.split_reads2.upload(ex, s2, C); cands.discordant_mates.upload(ex, dm, C); cands.evalue.upload(ex, ev, C);
	ex.sync();
}
void engine::get_candidate_state(u8* f, u32* s1, u32* s2, u32* dm, float* ev) {
	const u32 C = cands.n;
	cands.filter.download(ex, f, C); cands.split_reads1.download(ex, s1, C); cands.split_reads2.download(ex, s2, C); cands.discordant_mates.download(ex, dm, C); cands.evalue.download(ex, ev, C);
}
void engine::set_candidate_lists(const u32* l1o, const u32* l1, const u32* l2o, const u32* l2) {
	const u32 C = cands.n;
	cands.n_list1 = l1o[C]; cands.n_list2 = l2o[C];
	cands.list1_off.upload(ex, l1o, (size_t) C + 1); cands.list2_off.upload(ex, l2o, (size_t) C + 1);
	cands.list1.upload(ex, l1, cands.n_list1); cands.list2.upload(ex, l2, cands.n_list2);
	ex.sync();
}

struct list_size_fn { const u32* off; u32* n; ARB_HD void operator()(u32 k) const { n[k] = off[k + 1] - off[k]; } };
struct identity_fn { u32* p; ARB_HD void operator()(u32 k) const { p[k] = k; } };
struct gather_u32_fn { const u32* src; const u32* perm; u32* dst; ARB_HD void operator()(u32 k) const { dst[k] = src[perm[k]]; } };

u32 engine::merge_adjacent(i32 max_distance) {
	const u32 C = cands.n;
	merge_log_n = 0;
	if (C == 0) return 0;
	stage_timer t_all(ex);
	dbuf<u32> n1(C), n2(C), flag((size_t) C + 1);
	list_size_fn ls1 = {cands.list1_off.ptr(), n1.ptr()}, ls2 = {cands.list2_off.ptr(), n2.ptr()};
	for_each(ex, C, ls1); for_each(ex, C, ls2);
	cand_state s = make_state(cands, n1.ptr(), n2.ptr());
	merge_eligible_fn el = {s, params.max_itd_length, flag.ptr()};
	for_each(ex, C, el);
	exclusive_scan_u32(ex, flag.ptr(), flag.ptr(), C);
	u32 M = 0; flag.download(ex, &M, 1, C);
	if (M == 0) return 0;
	dbuf<u32> ids(M), key(M), perm(M), tk(M), tv(M), ids_sorted(M);
	merge_gather_fn mg = {flag.ptr(), ids.ptr()};
	for_each(ex, C, mg);
	// LSD over the four key fields; every pass sorts the current permutation of candidate ids (stable)
	for (int which = 0; which < 4; ++which) {
		merge_key_fn kf = {s, ids.ptr(), key.ptr(), which};
		for_each(ex, M, kf);
		const u32 bits = (which == 1 || which == 3) ? 16 : 32;
		radix_sort_pairs_u32(ex, key.ptr(), ids.ptr(), tk.ptr(), tv.ptr(), M, bits);
	}
	dbuf<u32> head((size_t) M + 1);
	merge_cluster_head_fn hf = {s, ids.ptr(), head.ptr(), max_distance};
	for_each(ex, M, hf);
	exclusive_scan_u32(ex, head.ptr(), head.ptr(), M);
	u32 K = 0; head.download(ex, &K, 1, M);
	dbuf<u32> cluster_start((size_t) K + 1), log_count(1);
	merge_cluster_start_fn cs = {head.ptr(), cluster_start.ptr(), M, K};
	for_each(ex, M, cs);
	const u32 capacity = 1u << 20;
	merge_log.ensure(3 * (size_t) capacity);
	log_count.zero(ex, 1);
	merge_cluster_fn mc = {s, ids.ptr(), cluster_start.ptr(), max_distance, params.max_itd_length, merge_log.ptr(), log_count.ptr(), capacity};
	for_each(ex, K, mc);
	u32 n_log = 0; log_count.download(ex, &n_log, 1);
	if (n_log > capacity) throw arb_error("merge_adjacent: more internal tandem duplication merges than the log can hold");
	merge_log_n = n_log;
	timings.merge_adjacent_ms = t_all.stop();
	return n_log;
}

void engine::get_merge_log(u32* triples, u32 n) { merge_log.download(ex, triples, 3 * (size_t) std::min(n, merge_log_n)); }

void engine::estimate_evalues(const arb_evalue_inputs& a) {
	const u32 C = cands.n;
	if (C == 0) return;
	if (a.n_genes != annot.n_genes) throw arb_error("arb_estimate_evalues: partner_count must have one entry per gene");
	dbuf<i32> pc; pc.upload(ex, a.partner_count, a.n_genes);
	dbuf<double> t_reads, t_intra, t_inter, t1000, t400, trt, tprox;
	t_reads.upload(ex, a.pow_reads, a.n_read_table); t_intra.upload(ex, a.pow_intragenic, a.n_read_table); t_inter.upload(ex, a.pow_intergenic, a.n_read_table);
	t1000.upload(ex, a.pow_spliced1000, 1000); t400.upload(ex, a.pow_spliced400, 400); trt.upload(ex, a.pow_read_through, 400000); tprox.upload(ex, a.pow_proximal, 400000);
	evalue_inputs in;
	in.partner_count = pc.ptr();
	in.spliced_breakpoints = a.spliced_breakpoints; in.exonic_breakpoints = a.exonic_breakpoints; in.intronic_breakpoints = a.intronic_breakpoints; in.exonic_intronic_breakpoints = a.exonic_intronic_breakpoints;
	in.intragenic_duplications = a.intragenic_duplications; in.intragenic_inversions = a.intragenic_inversions; in.spliced_same_gene = a.spliced_same_gene; in.spliced_different_genes = a.spliced_different_genes;
	in.read_through_fraction = a.read_through_fraction; in.mapped_reads = a.mapped_reads;
	in.pow_reads = t_reads.ptr(); in.pow_intragenic = t_intra.ptr(); in.pow_intergenic = t_inter.ptr(); in.n_read_table = a.n_read_table;
	in.pow_spliced1000 = t1000.ptr(); in.pow_spliced400 = t400.ptr(); in.pow_read_through = trt.ptr(); in.pow_proximal = tprox.ptr();
	in.read_through_penalty = a.read_through_penalty; in.cutoff = 0; in.apply_filter = 0;
	cand_state s = make_state(cands, NULL, NULL);
	evalue_fn fn = {s, annot.view(), in};
	stage_timer t_all(ex);
	for_each(ex, C, fn);
	timings.evalue_ms = t_all.stop();
	ex.sync();
}

void engine::filter_relative_support(float cutoff) {
	cand_state s = make_state(cands, NULL, NULL);
	relative_support_fn fn = {s, annot.view(), cutoff};
	for_each(ex, cands.n, fn);
	ex.sync();
}

u32 engine::select_best() {
	const u32 C = cands.n;
	if (C == 0) return 0;
	if (order_rank.size() < C) throw arb_error("arb_select_best: arb_replay_insertion_order must be called first");
	if (annot.n_genes >= (1u << 30)) throw arb_error("arb_select_best: too many genes");
	cand_state s = make_state(cands, NULL, NULL);
	dbuf<u32> flag((size_t) C + 1);
	select_eligible_fn el = {s, flag.ptr()};
	for_each(ex, C, el);
	exclusive_scan_u32(ex, flag.ptr(), flag.ptr(), C);
	u32 M = 0; flag.download(ex, &M, 1, C);
	if (M == 0) return 0;
	dbuf<u32> ids(M), key(M), tk(M), tv(M);
	merge_gather_fn mg = {flag.ptr(), ids.ptr()};
	for_each(ex, C, mg);
	u32 rank_bits = 1; while (rank_bits < 32 && ((u64) 1 << rank_bits) < C) ++rank_bits;
	u32 gene_bits = 1; while (gene_bits < 32 && ((u64) 1 << gene_bits) < annot.n_genes) ++gene_bits;
	for (int which = 0; which < 3; ++which) { // LSD: iteration rank, then the two words of the key
		select_key_fn kf = {s, order_rank.ptr(), ids.ptr(), key.ptr(), which};
		for_each(ex, M, kf);
		radix_sort_pairs_u32(ex, key.ptr(), ids.ptr(), tk.ptr(), tv.ptr(), M, which == 0 ? rank_bits : which == 1 ? gene_bits + 2 : gene_bits);
	}
	dbuf<u32> head((size_t) M + 1);
	select_head_fn hf = {s, ids.ptr(), head.ptr()};
	for_each(ex, M, hf);
	exclusive_scan_u32(ex, head.ptr(), head.ptr(), M);
	u32 G = 0; head.download(ex, &G, 1, M);
	dbuf<u32> group_start((size_t) G + 1);
	merge_cluster_start_fn cs = {head.ptr(), group_start.ptr(), M, G};
	for_each(ex, M, cs);
	select_group_fn gf = {s, ids.ptr(), group_start.ptr()};
	for_each(ex, G, gf);
	ex.sync();
	return G; // one candidate per group is left
}

void engine::evalue_tallies(u32* out) {
	dbuf<u32> tally(ET_COUNT); tally.zero(ex, ET_COUNT);
	dbuf<u8> with_fusion((size_t) annot.n_genes + 1), with_read_through((size_t) annot.n_genes + 1);
	with_fusion.zero(ex, annot.n_genes); with_read_through.zero(ex, annot.n_genes);
	evalue_tally_fn fn = {make_state(cands, NULL, NULL), annot.view(), tally.ptr(), with_fusion.ptr(), with_read_through.ptr()};
	for_each(ex, cands.n, fn);
	evalue_gene_tally_fn gf = {with_fusion.ptr(), with_read_through.ptr(), tally.ptr()};
	for_each(ex, annot.n_genes, gf);
	tally.download(ex, out, ET_COUNT);
}

u32 engine::filter_simple(int stage, float exonic_fraction, int min_support) {
	if (stage < SIMPLE_NON_CODING_NEIGHBORS || stage > SIMPLE_MIN_SUPPORT) throw arb_error("arb_filter_simple: unknown stage");
	dbuf<u32> remaining(1); remaining.zero(ex, 1);
	simple_filter_fn fn = {make_state(cands, NULL, NULL), annot.view(), stage, exonic_fraction, min_support, remaining.ptr()};
	for_each(ex, cands.n, fn);
	u32 r = 0; remaining.download(ex, &r, 1);
	return r;
}

// ------------------------------------------------------------------------------------------- filter_in_vitro and its inputs
void engine::set_coverage(const u16* const* per_contig, const u64* n_windows, u32 n_contigs) {
	std::vector<u64> off(n_contigs, 0); std::vector<u32> wins(n_contigs, 0);
	u64 total = 0;
	for (u32 c = 0; c < n_contigs; ++c) { off[c] = total; if (n_windows[c] > 0xFFFFFFFFull) throw arb_error("arb_set_coverage: contig too long"); wins[c] = (u32) n_windows[c]; total += n_windows[c]; }
	coverage_windows.ensure(total + 1);
	for (u32 c = 0; c < n_contigs; ++c) if (n_windows[c]) {
#ifdef ARB_DEVICE_BUILD
		ARB_CUDA_CHECK(cudaMemcpyAsync(coverage_windows.ptr() + off[c], per_contig[c], n_windows[c] * 2, cudaMemcpyHostToDevice, ex.stream));
#else
		memcpy(coverage_windows.ptr() + off[c], per_contig[c], n_windows[c] * 2);
#endif
	}
	coverage_off.upload(ex, off.data(), n_contigs); coverage_n.upload(ex, wins.data(), n_contigs);
	coverage_contigs = n_contigs;
	ex.sync();
}

void engine::reads_by_gene(u32* out) {
	dbuf<u32> reads(annot.n_genes); reads.zero(ex, annot.n_genes);
	reads_by_gene_fn fn = {frags.view(), reads.ptr()};
	for_each(ex, frags.n, fn);
	reads.download(ex, out, annot.n_genes);
}

void engine::filter_in_vitro(const u32* reads, u32 n_genes, u32 threshold, const u64* pairs, u64 n_pairs) {
	if (n_genes != annot.n_genes) throw arb_error("arb_filter_in_vitro: reads_by_gene must have one entry per gene");
	if (coverage_contigs == 0) throw arb_error("arb_filter_in_vitro: arb_set_coverage must be called first");
	const u32 C = cands.n;
	if (C == 0) return;
	dbuf<u32> d_reads; dbuf<u64> d_pairs;
	d_reads.upload(ex, reads, n_genes); d_pairs.upload(ex, pairs, n_pairs);
	stage_timer t_all(ex);
	coverage_view cov = {coverage_windows.ptr(), coverage_off.ptr(), coverage_n.ptr(), coverage_contigs};
	in_vitro_inputs in = {d_reads.ptr(), threshold, d_pairs.ptr(), n_pairs};
	in_vitro_fn fn = {make_state(cands, NULL, NULL), frags.view(), annot.view(), cov, in, cands.listd_off.ptr(), cands.listd.ptr()};
	for_each(ex, C, fn);
	timings.in_vitro_ms = t_all.stop();
	ex.sync();
}

void engine::spliced_support(const u32* reads, u32 n_genes, u32 threshold, u32* support_out) {
	if (n_genes != annot.n_genes) throw arb_error("arb_spliced_support: reads_by_gene must have one entry per gene");
	if (coverage_contigs == 0) throw arb_error("arb_spliced_support: arb_set_coverage must be called first");
	const u32 C = cands.n;
	if (C == 0) return;
	dbuf<u32> d_reads, d_support(C);
	d_reads.upload(ex, reads, n_genes);
	coverage_view cov = {coverage_windows.ptr(), coverage_off.ptr(), coverage_n.ptr(), coverage_contigs};
	spliced_support_fn fn = {make_state(cands, NULL, NULL), frags.view(), annot.view(), cov, d_reads.ptr(), threshold,
	                         cands.list1_off.ptr(), cands.list1.ptr(), cands.list2_off.ptr(), cands.list2.ptr(), cands.listd_off.ptr(), cands.listd.ptr(), d_support.ptr()};
	for_each(ex, C, fn);
	d_support.download(ex, support_out, C);
}

void engine::filter_multimappers() {
	const u32 C = cands.n, N = frags.n;
	if (C == 0 || N == 0) return;
	stage_timer t_all(ex);
	dbuf<u32> best(N); best.fill_bytes(ex, 0xFF, N);
	cand_state s = make_state(cands, NULL, NULL);
	multimapper_best_fn bf = {s, annot.view(), frags.view(), cands.list1_off.ptr(), cands.list1.ptr(), cands.list2_off.ptr(), cands.list2.ptr(), cands.listd_off.ptr(), cands.listd.ptr(), best.ptr()};
	for_each(ex, C, bf);
	multimapper_cluster_fn cf = {s, annot.view(), frags.view(), best.ptr()};
	for_each(ex, N, cf);
	multimapper_recount_fn rf = {s, frags.view(), cands.list1_off.ptr(), cands.list1.ptr(), cands.list2_off.ptr(), cands.list2.ptr(), cands.listd_off.ptr(), cands.listd.ptr()};
	for_each(ex, C, rf);
	timings.multimappers_ms = t_all.stop();
	ex.sync();
}

// phases: candidates [phase_start[j], phase_start[j + 1]) are inserted while the map has phase_buckets[j] buckets (phase_start[n_phases] = n candidates)
void engine::replay_insertion_order(const u32* phase_start, const u64* phase_buckets, u32 n_phases, u32* order_out, u32* rank_out) {
	const u32 C = cands.n;
	if (C == 0) return;
	if (n_phases == 0 || phase_start[0] != 0 || phase_start[n_phases] != C) throw arb_error("arb_replay_insertion_order: the phases must cover all candidates");
	stage_timer t_all(ex);
	dbuf<u64> code(C);
	order_code_fn cf = {make_state(cands, NULL, NULL), code.ptr()};
	for_each(ex, C, cf);
	dbuf<u32> seq(C), bucket(C), key(C), val(C), tk(C), tv(C), first;
	for (u32 j = 0; j < n_phases; ++j) {
		const u32 from = phase_start[j], m = phase_start[j + 1]; const u64 B = phase_buckets[j];
		if (m < from || B == 0 || B > 0xFFFFFFF0ull) throw arb_error("arb_replay_insertion_order: malformed phase");
		if (m == from) continue;
		order_append_fn ap = {seq.ptr(), from}; for_each(ex, m - from, ap); // the list so far is seq[0, from)
		first.ensure(B); first.fill_bytes(ex, 0xFF, B);
		order_bucket_fn bf = {seq.ptr(), code.ptr(), B, bucket.ptr(), first.ptr()};
		for_each(ex, m, bf);
		order_key_fn kf = {seq.ptr(), bucket.ptr(), first.ptr(), m, key.ptr(), val.ptr()};
		for_each(ex, m, kf);
		u32 bits = 1; while (bits < 32 && ((u64) 1 << bits) < m) ++bits;
		radix_sort_pairs_u32(ex, key.ptr(), val.ptr(), tk.ptr(), tv.ptr(), m, bits);
		seq.swap(val);
	}
	order_rank.ensure(C);
	order_rank_fn rf = {seq.ptr(), order_rank.ptr()};
	for_each(ex, C, rf);
	timings.order_ms = t_all.stop();
	seq.download(ex, order_out, C); order_rank.download(ex, rank_out, C);
	order_seq.swap(seq); // kept for the stages that visit candidates in this order on the device
}

// a gene's count = its distinct partners that have no more partners than the gene itself (filter_relative_support.cpp:19-60)
void engine::partner_counts(i32* count_out) {
	const u32 C = cands.n, G = annot.n_genes;
	for (u32 g = 0; g < G; ++g) count_out[g] = 0;
	if (C == 0) return;
	if (order_rank.size() < C) throw arb_error("arb_partner_counts: arb_replay_insertion_order must be called first");
	stage_timer t_all(ex);
	cand_state s = make_state(cands, NULL, NULL);
	dbuf<u32> flag((size_t) C + 1);
	partner_eligible_fn el = {s, flag.ptr()};
	for_each(ex, C, el);
	exclusive_scan_u32(ex, flag.ptr(), flag.ptr(), C);
	u32 E = 0; flag.download(ex, &E, 1, C);
	if (E == 0) return;
	if (E > 0x7FFFFFF0u) throw arb_error("too many candidates");
	const u32 M = 2 * E;
	dbuf<u32> occ(M), key(M), tk(M), tv(M);
	partner_emit_fn em = {s, flag.ptr(), occ.ptr()};
	for_each(ex, C, em);
	u32 cbits = 1; while (cbits < 32 && ((u64) 1 << cbits) < C) ++cbits;
	u32 gbits = 1; while (gbits < 32 && ((u64) 1 << gbits) < G) ++gbits;
	const u32 bits[4] = {cbits, 32, 32, gbits};
	for (int which = 0; which < 4; ++which) { // LSD over (gene, breakpoint1, breakpoint2, rank): every pass sorts the current order of the occurrences (stable)
		partner_key_fn kf = {s, order_rank.ptr(), occ.ptr(), key.ptr(), which};
		for_each(ex, M, kf);
		radix_sort_pairs_u32(ex, key.ptr(), occ.ptr(), tk.ptr(), tv.ptr(), M, bits[which]);
	}
	dbuf<u32> head((size_t) M + 1);
	partner_head_fn hf = {s, occ.ptr(), head.ptr()};
	for_each(ex, M, hf);
	exclusive_scan_u32(ex, head.ptr(), head.ptr(), M);
	u32 P = 0; head.download(ex, &P, 1, M);
	dbuf<u32> pg(P), pp(P), uflag(P), n_partners(G), count(G);
	partner_pair_fn pf = {s, occ.ptr(), head.ptr(), pg.ptr(), pp.ptr()};
	for_each(ex, M, pf);
	// pairs by (gene, partner): stable sort by partner, then by gene (the group heads are in gene order already, the partners inside a gene are not)
	radix_sort_pairs_u32(ex, pp.ptr(), pg.ptr(), tk.ptr(), tv.ptr(), P, gbits);
	radix_sort_pairs_u32(ex, pg.ptr(), pp.ptr(), tk.ptr(), tv.ptr(), P, gbits);
	n_partners.zero(ex, G); count.zero(ex, G);
	partner_unique_fn uf = {pg.ptr(), pp.ptr(), uflag.ptr(), n_partners.ptr()};
	for_each(ex, P, uf);
	partner_count_fn cf = {pg.ptr(), pp.ptr(), uflag.ptr(), n_partners.ptr(), count.ptr()};
	for_each(ex, P, cf);
	timings.partners_ms = t_all.stop();
	count.download(ex, (u32*) count_out, G);
}

} // namespace arb
