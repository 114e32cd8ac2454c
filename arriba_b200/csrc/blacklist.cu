// blacklist.cu -- drivers of the three rule-file searches (see blacklist_hd.h): the blacklist filter (-b), the rescue of known fusions (-k) and the tags (-t).
#include <cstdlib>
#include "engine.h"
#include "blacklist_hd.h"

namespace arb {

static const u32 RULE_LANES = 32, RULE_THREADS = 256;

#ifdef ARB_DEVICE_BUILD
template <class Test> __global__ void __launch_bounds__(RULE_THREADS) k_rule_search_groups(rule_search<Test> s, const u32* heavy, u32 n_heavy) {
	const u32 q = blockIdx.x * (RULE_THREADS / RULE_LANES) + threadIdx.x / RULE_LANES;
	if (q >= n_heavy) return;
	lane_group g; g.lane = threadIdx.x % RULE_LANES; g.lanes = RULE_LANES; g.mask = 0xFFFFFFFFu;
	rule_search_group(g, s, heavy[q]);
}
__global__ void __launch_bounds__(RULE_THREADS) k_tag_groups(tag_search s, const u32* heavy, u32 n_heavy) {
	const u32 q = blockIdx.x * (RULE_THREADS / RULE_LANES) + threadIdx.x / RULE_LANES;
	if (q >= n_heavy) return;
	lane_group g; g.lane = threadIdx.x % RULE_LANES; g.lanes = RULE_LANES; g.mask = 0xFFFFFFFFu;
	tag_group(g, s, heavy[q]);
}
#endif

static u32 bits_for(u32 n) { u32 b = 1; while (b < 32 && ((u64) 1 << b) < n) ++b; return b; }

// lists up to this length are walked by the candidate's own thread; ARB_BLACKLIST_SHORT_LIST (test hook) sends shorter ones to the lane groups too
static u32 short_list_length() {
	u32 n = 64;
	if (const char* e = getenv("ARB_BLACKLIST_SHORT_LIST")) n = (u32) atol(e);
	return n;
}

// the rules in file order, as parsed by the caller
void engine::set_rules(rule_set& set, const char* who, u32 n, const u8* type1, const u8* type2, const u8* strand1, const u8* strand2, const u16* contig1, const u16* contig2,
                       const i32* start1, const i32* end1, const i32* start2, const i32* end2, const u32* gene1, const u32* gene2) {
	for (u32 k = 0; k < n; ++k)
		if (type1[k] > ARB_RULE_NOT_BOTH_SPLICED || type2[k] > ARB_RULE_NOT_BOTH_SPLICED) throw arb_error(std::string(who) + ": unknown item type in rule " + std::to_string(k));
	set.n = n;
	set.type1.upload(ex, type1, n); set.type2.upload(ex, type2, n); set.strand1.upload(ex, strand1, n); set.strand2.upload(ex, strand2, n);
	set.contig1.upload(ex, contig1, n); set.contig2.upload(ex, contig2, n); set.start1.upload(ex, start1, n); set.end1.upload(ex, end1, n);
	set.start2.upload(ex, start2, n); set.end2.upload(ex, end2, n); set.gene1.upload(ex, gene1, n); set.gene2.upload(ex, gene2, n);
	ex.sync();
	set.loaded = true;
}

static rule_columns columns_of(engine::rule_set& set) {
	rule_columns r;
	r.n = set.n;
	r.type[0] = set.type1.ptr(); r.type[1] = set.type2.ptr(); r.strand[0] = set.strand1.ptr(); r.strand[1] = set.strand2.ptr();
	r.contig[0] = set.contig1.ptr(); r.contig[1] = set.contig2.ptr(); r.start[0] = set.start1.ptr(); r.start[1] = set.start2.ptr();
	r.end[0] = set.end1.ptr(); r.end[1] = set.end2.ptr(); r.gene[0] = set.gene1.ptr(); r.gene[1] = set.gene2.ptr();
	return r;
}

// key table of a rule set: the (contig, bin) keys of every rule's positional items, each widened by `widen`, sorted, one entry per distinct key
struct rule_keys {
	dbuf<u32> rule_of, table_key, table_begin; u32 n_keys;
	rule_key_table view() const { rule_key_table t; t.n_keys = n_keys; t.key = table_key.ptr(); t.begin = table_begin.ptr(); t.rules = rule_of.ptr(); return t; }
};
static void build_rule_keys(const exec_ctx& ex, const rule_columns& r, i32 widen, u32 n_contigs, const char* who, rule_keys& out) {
	const u32 R = r.n;
	dbuf<u32> offset((size_t) R + 1); dbuf<unsigned long long> total(1);
	total.zero(ex, 1);
	u64 K = 0;
	if (R) {
		rule_key_count_fn cnt = {r, widen, offset.ptr(), total.ptr()};
		for_each(ex, R, cnt);
		unsigned long long k = 0; total.download(ex, &k, 1); K = k;
	}
	if (K >= ((u64) 1 << 31)) throw arb_error(std::string(who) + ": the rules span " + std::to_string((unsigned long long) K) + " (contig, 100 kb bin) keys, more than 2^31");
	dbuf<u32> key((size_t) K), key_tmp((size_t) K + 1), rule_tmp((size_t) K), head((size_t) K);
	out.rule_of.alloc((size_t) K); out.table_key.alloc((size_t) K); out.table_begin.alloc((size_t) K + 1);
	out.n_keys = 0;
	if (!K) return;
	exclusive_scan_u32(ex, offset.ptr(), offset.ptr(), R);
	rule_key_fill_fn fill = {r, widen, offset.ptr(), key.ptr(), out.rule_of.ptr()};
	for_each(ex, R, fill);
	radix_sort_pairs_u32(ex, key.ptr(), out.rule_of.ptr(), key_tmp.ptr(), rule_tmp.ptr(), (u32) K, 16 + bits_for(n_contigs + 1));
	rule_key_head_fn hf = {key.ptr(), head.ptr()};
	for_each(ex, (u32) K, hf);
	exclusive_scan_u32(ex, head.ptr(), key_tmp.ptr(), (u32) K); // slot of every head; the number of distinct keys lands at [K]
	rule_key_table_fn tf = {key.ptr(), head.ptr(), key_tmp.ptr(), out.table_key.ptr(), out.table_begin.ptr(), (u32) K};
	for_each(ex, (u32) K, tf);
	key_tmp.download(ex, &out.n_keys, 1, (size_t) K);
}

// one verdict byte per id: the thread pass, then the lane groups for the candidates it queued; returns the number of queued candidates
template <class Test> static u32 run_rule_search(const exec_ctx& ex, rule_search<Test>& s, const u32* host_ids, u32 n_ids, dbuf<u8>& verdict) {
	dbuf<u32> heavy(n_ids), n_heavy(1);
	n_heavy.zero(ex, 1);
	s.short_list = short_list_length();
	s.heavy = heavy.ptr(); s.n_heavy = n_heavy.ptr();
	if (!s.b.t.n_keys) { verdict.zero(ex, n_ids); return 0; } // no rule has a positional item that could share a bin
	for_each(ex, n_ids, s);
	u32 H = 0; n_heavy.download(ex, &H, 1);
#ifdef ARB_DEVICE_BUILD
	(void) host_ids;
	if (H) {
		const u32 per_block = RULE_THREADS / RULE_LANES;
		k_rule_search_groups<Test><<<(H + per_block - 1) / per_block, RULE_THREADS, 0, ex.stream>>>(s, heavy.ptr(), H);
		ARB_CUDA_CHECK(cudaGetLastError());
		++stats().kernels;
	}
#else
	// the stand-in plays the lanes of a group one after the other and ORs their findings like __any_sync does
	std::vector<u32> queue = heavy.to_host(ex, H);
	hostsim_visit(H, [&](u32 q) {
		const u32 i = queue[q];
		bool any = false;
		for (u32 lane = 0; lane < RULE_LANES; ++lane) any = s.lane_walk(host_ids[i], lane, RULE_LANES) || any;
		verdict.ptr()[i] = any ? 1 : 0;
	});
	if (H) ++stats().kernels;
#endif
	return H;
}

static void check_ids(const char* who, u32 n_ids, const u32* ids, u32 C) {
	for (u32 i = 0; i < n_ids; ++i) if (ids[i] >= C) throw arb_error(std::string(who) + ": candidate id out of range");
}

u32 engine::filter_blacklist(u32 n_ids, const u32* ids, float evalue_cutoff, i32 max_mate_gap, u8* verdicts) {
	if (!blacklist_rules.loaded) throw arb_error("arb_filter_blacklist: arb_set_blacklist must be called first");
	if (!has_annotation) throw arb_error("arb_filter_blacklist: no annotation");
	if (max_mate_gap < 0) throw arb_error("arb_filter_blacklist: max_mate_gap must not be negative");
	check_ids("arb_filter_blacklist", n_ids, ids, cands.n);
	blacklist_heavy = 0;
	if (n_ids == 0) { timings.blacklist_ms = 0; return 0; }
	stage_timer t(ex);
	const rule_columns r = columns_of(blacklist_rules);
	rule_keys keys;
	build_rule_keys(ex, r, max_mate_gap, annot.n_contigs, "arb_filter_blacklist", keys);
	dbuf<u32> d_ids(n_ids); dbuf<u8> verdict(n_ids);
	d_ids.upload(ex, ids, n_ids);
	blacklist_search s;
	s.b.c = make_state_for_rows(); s.b.an = annot.view(); s.b.t = keys.view();
	s.test.r = r; s.test.c = s.b.c; s.test.an = s.b.an; s.test.max_mate_gap = max_mate_gap; s.test.evalue_cutoff = evalue_cutoff;
	s.ids = d_ids.ptr(); s.verdict = verdict.ptr();
	blacklist_heavy = run_rule_search(ex, s, ids, n_ids, verdict);
	verdict.download(ex, verdicts, n_ids);
	timings.blacklist_ms = t.stop();
	u32 blacklisted = 0;
	for (u32 i = 0; i < n_ids; ++i) blacklisted += verdicts[i] != 0;
	return blacklisted;
}

u32 engine::recover_known_fusions(u32 n_ids, const u32* ids, i32 max_mate_gap, u8* verdicts) {
	if (!known_rules.loaded) throw arb_error("arb_recover_known_fusions: arb_set_known_fusions must be called first");
	if (!has_annotation) throw arb_error("arb_recover_known_fusions: no annotation");
	if (coverage_contigs == 0) throw arb_error("arb_recover_known_fusions: arb_set_coverage must be called first");
	if (max_mate_gap < 0) throw arb_error("arb_recover_known_fusions: max_mate_gap must not be negative");
	check_ids("arb_recover_known_fusions", n_ids, ids, cands.n);
	known_heavy = 0;
	if (n_ids == 0) { timings.known_fusions_ms = 0; return 0; }
	stage_timer t(ex);
	const rule_columns r = columns_of(known_rules);
	rule_keys keys;
	build_rule_keys(ex, r, 0, annot.n_contigs, "arb_recover_known_fusions", keys);
	dbuf<u32> d_ids(n_ids); dbuf<u8> verdict(n_ids);
	d_ids.upload(ex, ids, n_ids);
	dbuf<u8> supported(cands.n);
	known_fusion_search s;
	s.b.c = make_state_for_rows(); s.b.an = annot.view(); s.b.t = keys.view();
	known_support_fn sf = {s.b.c, s.b.an, {coverage_windows.ptr(), coverage_off.ptr(), coverage_n.ptr(), coverage_contigs}, d_ids.ptr(), supported.ptr()};
	for_each(ex, n_ids, sf);
	s.test.m.r = r; s.test.m.c = s.b.c; s.test.m.an = s.b.an; s.test.m.max_mate_gap = max_mate_gap; s.test.m.evalue_cutoff = 0; s.test.supported = supported.ptr();
	s.ids = d_ids.ptr(); s.verdict = verdict.ptr();
	known_heavy = run_rule_search(ex, s, ids, n_ids, verdict);
	verdict.download(ex, verdicts, n_ids);
	timings.known_fusions_ms = t.stop();
	u32 rescued = 0;
	for (u32 i = 0; i < n_ids; ++i) rescued += verdicts[i] != 0;
	return rescued;
}

void engine::set_tags(const u32* rank, u32 n, const char* chars, const u32* off) {
	if (!tag_rules.loaded) throw arb_error("arb_set_tags: no rules");
	for (u32 k = 0; k < tag_rules.n; ++k) if (rank[k] >= n) throw arb_error("arb_set_tags: tag rank out of range in rule " + std::to_string(k));
	for (u32 k = 0; k < n; ++k) if (off[k + 1] < off[k]) throw arb_error("arb_set_tags: tag offsets must not decrease");
	tag_rank_of_rule.upload(ex, rank, tag_rules.n);
	tag_text_off.upload(ex, off, (size_t) n + 1);
	tag_text.ensure((size_t) off[n] + 1);
	if (off[n]) tag_text.upload(ex, chars, off[n]);
	ex.sync();
	n_tags = n; has_tags = true; has_tag_csr = false;
}

// the distinct tags of every row in `ids`, as ranks in ascending order: a CSR over all candidates (rows not in `ids` have none) that stays on the device
u64 engine::annotate_tags(u32 n_ids, const u32* ids, i32 max_mate_gap) {
	if (!has_tags) throw arb_error("arb_annotate_tags: arb_set_tags must be called first");
	if (!has_annotation) throw arb_error("arb_annotate_tags: no annotation");
	if (max_mate_gap < 0) throw arb_error("arb_annotate_tags: max_mate_gap must not be negative");
	const u32 C = cands.n;
	check_ids("arb_annotate_tags", n_ids, ids, C);
	stage_timer t(ex);
	tags_heavy = 0; timings.tags_pairs = 0; timings.tags_match_ms = timings.tags_sort_ms = 0;
	tag_csr_off.alloc((size_t) C + 1); tag_csr_off.zero(ex, (size_t) C + 1);
	tag_csr_pairs = 0; tag_csr_n = C; has_tag_csr = true;
	const rule_columns r = columns_of(tag_rules);
	rule_keys keys;
	build_rule_keys(ex, r, 0, annot.n_contigs, "arb_annotate_tags", keys);
	if (n_ids == 0 || keys.n_keys == 0) { tag_csr_rank.alloc(1); timings.tags_match_ms = timings.tags_ms = t.stop(); return 0; }
	dbuf<u32> d_ids(n_ids), count((size_t) n_ids + 1), heavy(n_ids), n_heavy(1); dbuf<u8> heavy_mark(n_ids); dbuf<unsigned long long> total(1);
	d_ids.upload(ex, ids, n_ids);
	n_heavy.zero(ex, 1); total.zero(ex, 1);
	tag_search s;
	s.b.c = make_state_for_rows(); s.b.an = annot.view(); s.b.t = keys.view();
	s.m.r = r; s.m.c = s.b.c; s.m.an = s.b.an; s.m.max_mate_gap = max_mate_gap; s.m.evalue_cutoff = 0;
	s.rank = tag_rank_of_rule.ptr(); s.ids = d_ids.ptr(); s.short_list = short_list_length();
	s.heavy_mark = heavy_mark.ptr(); s.heavy = heavy.ptr(); s.n_heavy = n_heavy.ptr();
	s.count = count.ptr(); s.offset = NULL; s.out_rank = NULL; s.out_cand = NULL; s.total = total.ptr();
	// pass 1: matches per row
	for_each(ex, n_ids, s);
	u32 H = 0; n_heavy.download(ex, &H, 1);
	tags_heavy = H;
	std::vector<u32> queue;
#ifdef ARB_DEVICE_BUILD
	const u32 per_block = RULE_THREADS / RULE_LANES, blocks = (H + per_block - 1) / per_block;
	if (H) { k_tag_groups<<<blocks, RULE_THREADS, 0, ex.stream>>>(s, heavy.ptr(), H); ARB_CUDA_CHECK(cudaGetLastError()); ++stats().kernels; }
#else
	// the stand-in plays the lanes of a group one after the other and adds up their counts like the ballots do
	queue = heavy.to_host(ex, H);
	hostsim_visit(H, [&](u32 q) {
		const u32 i = queue[q]; u32 n = 0;
		for (u32 lane = 0; lane < RULE_LANES; ++lane) n += s.lane_walk(ids[i], lane, RULE_LANES, 0);
		count.ptr()[i] = n; s.add_total(n);
	});
	if (H) ++stats().kernels;
#endif
	// every (row, matching rule) pair, a rule counted once per bin of the row it is listed under: the pairs are indexed in 32 bits
	unsigned long long all = 0; total.download(ex, &all, 1);
	if (all >= (1ull << 31)) throw arb_error("arb_annotate_tags: the rows and the tag rules make " + std::to_string(all) + " (row, rule) pairs, more than 2^31");
	exclusive_scan_u32(ex, count.ptr(), count.ptr(), n_ids);
	const u32 P = (u32) all;
	timings.tags_pairs = P;
	if (P == 0) { tag_csr_rank.alloc(1); timings.tags_match_ms = timings.tags_ms = t.stop(); return 0; }
	// pass 2: (rank, candidate) pairs at the row offsets
	dbuf<u32> rank(P), cand(P), rank_tmp(P), cand_tmp((size_t) P + 1), head(P);
	s.offset = count.ptr(); s.out_rank = rank.ptr(); s.out_cand = cand.ptr();
	for_each(ex, n_ids, s);
#ifdef ARB_DEVICE_BUILD
	if (H) { k_tag_groups<<<blocks, RULE_THREADS, 0, ex.stream>>>(s, heavy.ptr(), H); ARB_CUDA_CHECK(cudaGetLastError()); ++stats().kernels; }
#else
	{
		const std::vector<u32> offs = count.to_host(ex, n_ids);
		hostsim_visit(H, [&](u32 q) {
			const u32 i = queue[q]; u32 at = offs[i];
			for (u32 lane = 0; lane < RULE_LANES; ++lane) at += s.lane_walk(ids[i], lane, RULE_LANES, at);
		});
		if (H) ++stats().kernels;
	}
#endif
	timings.tags_match_ms = t.stop();
	stage_timer t_sort(ex);
	// sorted by (candidate, rank): two stable passes, rank first; then one entry per distinct pair, counted per candidate
	radix_sort_pairs_u32(ex, rank.ptr(), cand.ptr(), rank_tmp.ptr(), cand_tmp.ptr(), P, bits_for(n_tags));
	radix_sort_pairs_u32(ex, cand.ptr(), rank.ptr(), cand_tmp.ptr(), rank_tmp.ptr(), P, bits_for(C));
	tag_head_fn hf = {cand.ptr(), rank.ptr(), head.ptr()};
	for_each(ex, P, hf);
	exclusive_scan_u32(ex, head.ptr(), cand_tmp.ptr(), P);
	u32 D = 0; cand_tmp.download(ex, &D, 1, P);
	tag_csr_rank.alloc(D);
	tag_compact_fn cf = {cand.ptr(), rank.ptr(), head.ptr(), cand_tmp.ptr(), tag_csr_rank.ptr(), tag_csr_off.ptr()};
	for_each(ex, P, cf);
	exclusive_scan_u32(ex, tag_csr_off.ptr(), tag_csr_off.ptr(), C);
	tag_csr_pairs = D;
	timings.tags_sort_ms = t_sort.stop();
	timings.tags_ms = timings.tags_match_ms + timings.tags_sort_ms;
	return D;
}

void engine::get_tags(u32* off, u32* ranks) {
	if (!has_tag_csr || tag_csr_n != cands.n) throw arb_error("arb_get_tags: arb_annotate_tags must be called first");
	tag_csr_off.download(ex, off, (size_t) tag_csr_n + 1);
	if (tag_csr_pairs) tag_csr_rank.download(ex, ranks, tag_csr_pairs);
}

} // namespace arb
