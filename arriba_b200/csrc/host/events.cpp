// events.cpp -- event-level stages (everything after find_fusions, arriba.cpp:415-589). Stages named in the hot path
// (merge_adjacent, e-value / relative_support, k-mer index, homologs, mismappers) run on the device through the C ABI; the
// cheap O(#candidates) predicates and recoveries run here, visiting candidates in the reference's iteration order.
// Each function cites the reference file it reproduces.
#include "pipeline.h"
#include "../annot_hd.h"
#include "index_query.h"
#include <algorithm>
#include <atomic>
#include <climits>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <set>
#include <sstream>
#include <stdexcept>
#include <tuple>
#include <thread>
#include <chrono>
#include <unordered_map>

namespace arb { namespace host {

// candidates are independent in the predicate loops below (each writes only its own row): run slices on the host threads
template <class F> static void parallel_rows(int threads, size_t n, F f) {
	if (threads <= 1 || n < 4096) { for (size_t k = 0; k < n; ++k) f((u32) k); return; }
	std::vector<std::thread> pool; std::vector<std::string> errors(threads);
	// rows cost very different amounts (a candidate with thousands of supporting reads next to thousands with one): blocks of rows are drawn from a counter
	const size_t BLOCK = 2048; std::atomic<size_t> next(0);
	for (int t = 0; t < threads; ++t) pool.emplace_back([&, t]() {
		try { for (;;) { const size_t lo = next.fetch_add(BLOCK); if (lo >= n) break; const size_t hi = std::min(n, lo + BLOCK); for (size_t k = lo; k < hi; ++k) f((u32) k); } }
		catch (const std::exception& x) { errors[t] = x.what(); next.store(n); }
	});
	for (size_t t = 0; t < pool.size(); ++t) pool[t].join();
	for (int t = 0; t < threads; ++t) if (!errors[t].empty()) throw std::runtime_error(errors[t]);
}

// sort on the host threads: slices sorted concurrently, then rounds of pairwise merges between the vector and a spare buffer; every merge is cut into
// independent pieces by output rank, so all threads work down to the last round. For plain-data elements (the spare buffer is raw storage).
template <class V, class Less> static void parallel_sort(V& v, Less less, int threads) {
	typedef typename V::value_type T;
	const size_t n = v.size();
	if (threads <= 1 || n < 8192) { std::sort(v.begin(), v.end(), less); return; }
	const int parts = std::min(threads, 256);
	std::vector<size_t> cut(parts + 1); for (int t = 0; t <= parts; ++t) cut[t] = n * t / parts;
	{ std::vector<std::thread> pool; for (int t = 0; t < parts; ++t) pool.emplace_back([&, t]() { std::sort(v.begin() + cut[t], v.begin() + cut[t + 1], less); }); for (size_t t = 0; t < pool.size(); ++t) pool[t].join(); }
	T* const spare = (T*) malloc(n * sizeof(T));
	if (!spare) throw std::bad_alloc();
	T* src = v.data(); T* dst = spare;
	// how many elements of A precede output rank r of merge(A, B); equal elements take A first
	auto split = [&](const T* A, size_t nA, const T* B, size_t nB, size_t r) {
		size_t lo = r > nB ? r - nB : 0, hi = std::min(r, nA);
		while (lo < hi) { const size_t i = lo + (hi - lo) / 2, j = r - i; if (j == 0 || less(B[j - 1], A[i])) hi = i; else lo = i + 1; }
		return lo;
	};
	for (int width = 1; width < parts; width *= 2) {
		std::vector<std::thread> pool;
		for (int t = 0; t < parts; t += 2 * width) {
			const size_t a = cut[t], m = cut[std::min(parts, t + width)], b = cut[std::min(parts, t + 2 * width)];
			const int pieces = std::min(parts - t, 2 * width);
			for (int k = 0; k < pieces; ++k) pool.emplace_back([&, a, m, b, k, pieces]() {
				const T* A = src + a; const T* B = src + m; const size_t nA = m - a, nB = b - m;
				const size_t r0 = (b - a) * k / pieces, r1 = (b - a) * (k + 1) / pieces;
				const size_t i0 = split(A, nA, B, nB, r0), i1 = split(A, nA, B, nB, r1);
				std::merge(A + i0, A + i1, B + (r0 - i0), B + (r1 - i1), dst + a + r0, less);
			});
		}
		for (size_t k = 0; k < pool.size(); ++k) pool[k].join();
		std::swap(src, dst);
	}
	if (src != v.data()) {
		std::vector<std::thread> pool;
		for (int t = 0; t < parts; ++t) pool.emplace_back([&, t]() { std::copy(src + cut[t], src + cut[t + 1], v.data() + cut[t]); });
		for (size_t t = 0; t < pool.size(); ++t) pool[t].join();
	}
	free(spare);
}

static void check(arb_ctx* ctx, int rc, const char* what) { if (rc != 0) throw std::runtime_error(std::string(what) + ": " + arb_last_error(ctx)); }

// ------------------------------------------------------------------------------------------- iteration order
// The reference inserts the candidates, in the order the device numbers them, into a std::unordered_map and later ITERATES it. The order is computed on the
// device from the resident candidate keys (csrc/events_hd.h, "iteration order"); the host contributes what only its C++ library knows: when the table grows and
// to how many buckets (the library's own policy object, asked exactly like unordered_map::insert asks it).
void pipeline::replay_iteration_order() {
	const u32 n = ev.n;
	ev.order.assign(n, 0); ev.rank_of.assign(n, 0);
	if (n == 0) return;
	std::vector<u32> phase_start; std::vector<uint64_t> phase_buckets;
	std::__detail::_Prime_rehash_policy policy;
	size_t n_buckets = 1;
	phase_start.push_back(0); phase_buckets.push_back(1);
	for (size_t k = 0; k < n; ) {
		const std::pair<bool, size_t> grow = policy._M_need_rehash(n_buckets, k, 1);
		if (grow.first) {
			n_buckets = grow.second;
			if (phase_start.back() == k) phase_buckets.back() = n_buckets; else { phase_start.push_back((u32) k); phase_buckets.push_back(n_buckets); }
		}
		// the policy answers "no" without changing its state until the element count passes its next threshold
		const size_t next = policy._M_next_resize;
		k = std::max(k + 1, std::min<size_t>(next, n));
	}
	phase_start.push_back(n);
	check(ctx, arb_replay_insertion_order(ctx, phase_start.data(), phase_buckets.data(), (uint32_t) phase_buckets.size(), ev.order.data(), ev.rank_of.data()), "arb_replay_insertion_order");
}

// ------------------------------------------------------------------------------------------- helpers on (table, reference)
static inline bool overlaps_both(const event_table& e, const refdata& r, u32 k, int which = 0) { // common.hpp:260-264
	if (which == 1) return e.bp1[k] >= r.genes[e.gene2[k]].start && e.bp1[k] <= r.genes[e.gene2[k]].end;
	if (which == 2) return e.bp2[k] >= r.genes[e.gene1[k]].start && e.bp2[k] <= r.genes[e.gene1[k]].end;
	return overlaps_both(e, r, k, 1) || overlaps_both(e, r, k, 2);
}
static inline bool both_spliced(const event_table& e, const refdata& r, u32 k) { // common.hpp:280-284
	return e.spliced1(k) && e.spliced2(k) && ((r.genes[e.gene1[k]].forward == r.genes[e.gene2[k]].forward && e.dir1[k] != e.dir2[k]) || (r.genes[e.gene1[k]].forward != r.genes[e.gene2[k]].forward && e.dir1[k] == e.dir2[k]));
}
static inline bool is_intragenic(const event_table& e, const refdata& r, u32 k) { // common.hpp:275-279
	const gene_rec& g1 = r.genes[e.gene1[k]]; const gene_rec& g2 = r.genes[e.gene2[k]];
	return e.gene1[k] == e.gene2[k] || (e.bp1[k] >= g2.start - 10000 && e.bp1[k] <= g2.end + 10000 && e.bp2[k] >= g1.start - 10000 && e.bp2[k] <= g1.end + 10000);
}
static u32 count_unfiltered(const event_table& e) { u32 c = 0; for (u32 k = 0; k < e.n; ++k) if (e.filter[k] == F_none) ++c; return c; }

void pipeline::log_remaining(const char* what) { std::ostringstream s; s << what << " (remaining=" << count_unfiltered(ev) << ")"; say(s.str()); }

// ------------------------------------------------------------------------------------------- device <-> host state
void pipeline::fetch_candidates() {
	stage_laps laps("fetch");
	uint32_t n; uint64_t n1, n2, nd;
	check(ctx, arb_candidates_size(ctx, &n, &n1, &n2, &nd), "arb_candidates_size");
	laps.lap("sizes");
	event_table& e = ev;
	e.n = n;
	e.gene1.resize(n); e.gene2.resize(n); e.contig1.resize(n); e.contig2.resize(n); e.bp1.resize(n); e.bp2.resize(n); e.dir1.resize(n); e.dir2.resize(n);
	e.split_reads1.resize(n); e.split_reads2.resize(n); e.discordant_mates.resize(n); e.filter.resize(n); e.bits.resize(n); e.bits2.resize(n);
	e.anchor1.resize(n); e.anchor2.resize(n); e.evalue.resize(n); e.confidence.assign(n, 0); e.closest1.clear(); e.closest2.clear();
	e.list1_off.resize((size_t) n + 1); e.list2_off.resize((size_t) n + 1); e.listd_off.resize((size_t) n + 1);
	e.list1.resize(n1 + 1); e.list2.resize(n2 + 1); e.listd.resize(nd + 1);
	arb_candidates c;
	c.n = n; c.gene1 = e.gene1.data(); c.gene2 = e.gene2.data(); c.contig1 = e.contig1.data(); c.contig2 = e.contig2.data(); c.breakpoint1 = e.bp1.data(); c.breakpoint2 = e.bp2.data();
	c.direction1 = e.dir1.data(); c.direction2 = e.dir2.data(); c.split_reads1 = e.split_reads1.data(); c.split_reads2 = e.split_reads2.data(); c.discordant_mates = e.discordant_mates.data();
	c.filter = e.filter.data(); c.bits = e.bits.data(); c.bits2 = e.bits2.data(); c.anchor_start1 = e.anchor1.data(); c.anchor_start2 = e.anchor2.data(); c.evalue = e.evalue.data();
	c.list1_off = e.list1_off.data(); c.list2_off = e.list2_off.data(); c.listd_off = e.listd_off.data(); c.list1 = e.list1.data(); c.list2 = e.list2.data(); c.listd = e.listd.data();
	laps.lap("host columns sized");
	check(ctx, arb_get_candidates(ctx, &c), "arb_get_candidates");
	laps.lap("device -> host");
	e.list1.resize(n1); e.list2.resize(n2); e.listd.resize(nd);
	replay_iteration_order(); // needs the candidate keys only, which no later stage changes
	laps.lap("iteration order (device)");
	// mirror the canonical mate order the device established for listed discordant mates (fusions.cpp:414-421)
	std::vector<u8> swapped(frags.n);
	check(ctx, arb_get_slot_swaps(ctx, swapped.data()), "arb_get_slot_swaps");
	const size_t N = frags.n;
	parallel_rows(threads, N, [&](u32 i) {
		if (!swapped[i]) return;
		const size_t a = i, b = N + i;
		std::swap(frags.contig[a], frags.contig[b]); std::swap(frags.start[a], frags.start[b]); std::swap(frags.end[a], frags.end[b]); std::swap(frags.aflags[a], frags.aflags[b]);
		std::swap(frags.cigar_off[a], frags.cigar_off[b]); std::swap(frags.cigar_cnt[a], frags.cigar_cnt[b]); std::swap(frags.seq_off[a], frags.seq_off[b]); std::swap(frags.seq_len[a], frags.seq_len[b]);
		std::swap(frags.genes_off[a], frags.genes_off[b]); std::swap(frags.genes_cnt[a], frags.genes_cnt[b]);
	});
	check(ctx, arb_get_fragment_filters(ctx, labels.data(), NULL), "arb_get_fragment_filters");
	laps.lap("mate swaps + labels");
	std::ostringstream s; s << "Finding fusions and counting supporting reads (total=" << count_unfiltered(e) << ")"; say(s.str());
}

void pipeline::order_ready() {} // the order is complete when fetch_candidates returns

void pipeline::push_candidate_state() {
	check(ctx, arb_set_candidate_state(ctx, ev.filter.data(), ev.split_reads1.data(), ev.split_reads2.data(), ev.discordant_mates.data(), ev.evalue.data()), "arb_set_candidate_state");
}
void pipeline::pull_candidate_state() {
	check(ctx, arb_get_candidate_state(ctx, ev.filter.data(), ev.split_reads1.data(), ev.split_reads2.data(), ev.discordant_mates.data(), ev.evalue.data()), "arb_get_candidate_state");
}

// ------------------------------------------------------------------------------------------- merge_adjacent (device) + ITD list concatenation
void pipeline::merge_adjacent() {
	push_candidate_state();
	uint32_t n_log = 0;
	check(ctx, arb_merge_adjacent(ctx, 5, &n_log), "arb_merge_adjacent"); // max_distance 5 (arriba.cpp:422)
	pull_candidate_state();
	if (n_log > 0) { // internal tandem duplications: the absorbed candidates' read lists are appended, in the order the reference merges
		std::vector<u32> triples(3 * (size_t) n_log);
		check(ctx, arb_get_merge_log(ctx, triples.data(), n_log), "arb_get_merge_log");
		struct entry { u32 winner, loser, pos, seq; };
		std::vector<entry> es(n_log);
		for (u32 k = 0; k < n_log; ++k) { es[k].winner = triples[3 * k]; es[k].loser = triples[3 * k + 1]; es[k].pos = triples[3 * k + 2]; es[k].seq = k; }
		// a winner's entries were logged by one thread in order; winners are replayed by sorted position
		std::stable_sort(es.begin(), es.end(), [](const entry& a, const entry& b) { return a.pos != b.pos ? a.pos < b.pos : a.seq < b.seq; });
		// only the handful of candidates that take part get a list of their own; the table is then rewritten in long runs of untouched candidates
		std::map<u32, std::pair<std::vector<u32>, std::vector<u32> > > own;
		auto materialise = [&](u32 k) -> std::pair<std::vector<u32>, std::vector<u32> >& {
			std::map<u32, std::pair<std::vector<u32>, std::vector<u32> > >::iterator it = own.find(k);
			if (it != own.end()) return it->second;
			std::pair<std::vector<u32>, std::vector<u32> >& l = own[k];
			l.first.assign(ev.list1.begin() + ev.list1_off[k], ev.list1.begin() + ev.list1_off[k + 1]); l.second.assign(ev.list2.begin() + ev.list2_off[k], ev.list2.begin() + ev.list2_off[k + 1]);
			return l;
		};
		for (size_t k = 0; k < es.size(); ++k) {
			std::pair<std::vector<u32>, std::vector<u32> >& w = materialise(es[k].winner); const std::pair<std::vector<u32>, std::vector<u32> > l = materialise(es[k].loser); // a copy: winner and loser are different candidates, but the map may re-balance
			w.first.insert(w.first.end(), l.first.begin(), l.first.end());
			w.second.insert(w.second.end(), l.second.begin(), l.second.end());
		}
		size_t grow1 = 0, grow2 = 0;
		for (std::map<u32, std::pair<std::vector<u32>, std::vector<u32> > >::iterator it = own.begin(); it != own.end(); ++it) { grow1 += it->second.first.size(); grow2 += it->second.second.size(); }
		column<u32> o1((size_t) ev.n + 1), o2((size_t) ev.n + 1), n1, n2;
		n1.reserve(ev.list1.size() + grow1); n2.reserve(ev.list2.size() + grow2);
		o1[0] = o2[0] = 0;
		u32 from = 0;
		auto copy_run = [&](u32 to) { // candidates [from, to) keep their lists
			if (to <= from) return;
			const u32 d1 = (u32) n1.size() - ev.list1_off[from], d2 = (u32) n2.size() - ev.list2_off[from];
			n1.insert(n1.end(), ev.list1.begin() + ev.list1_off[from], ev.list1.begin() + ev.list1_off[to]); n2.insert(n2.end(), ev.list2.begin() + ev.list2_off[from], ev.list2.begin() + ev.list2_off[to]);
			for (u32 k = from; k < to; ++k) { o1[k + 1] = ev.list1_off[k + 1] + d1; o2[k + 1] = ev.list2_off[k + 1] + d2; }
		};
		for (std::map<u32, std::pair<std::vector<u32>, std::vector<u32> > >::iterator it = own.begin(); it != own.end(); ++it) {
			const u32 k = it->first;
			copy_run(k);
			n1.insert(n1.end(), it->second.first.begin(), it->second.first.end()); n2.insert(n2.end(), it->second.second.begin(), it->second.second.end());
			o1[k + 1] = (u32) n1.size(); o2[k + 1] = (u32) n2.size();
			from = k + 1;
		}
		copy_run(ev.n);
		ev.list1.swap(n1); ev.list2.swap(n2); ev.list1_off.swap(o1); ev.list2_off.swap(o2);
		check(ctx, arb_set_candidate_lists(ctx, ev.list1_off.data(), ev.list1.data(), ev.list2_off.data(), ev.list2.data()), "arb_set_candidate_lists");
	}
	log_remaining("Merging adjacent fusion breakpoints");
}

// ------------------------------------------------------------------------------------------- multimappers (filter_multimappers.cpp), on the device
void pipeline::filter_multimappers() { // csrc/events_hd.h: multimapper_best_fn, multimapper_cluster_fn, multimapper_recount_fn
	check(ctx, arb_set_fragment_filters(ctx, labels.data()), "arb_set_fragment_filters");
	push_candidate_state();
	check(ctx, arb_filter_multimappers(ctx), "arb_filter_multimappers");
	pull_candidate_state();
	check(ctx, arb_get_fragment_filters(ctx, labels.data(), NULL), "arb_get_fragment_filters");
	log_remaining("Filtering multi-mapping fusions by alignment score and read support");
}

// ------------------------------------------------------------------------------------------- e-value (filter_relative_support.cpp)
void pipeline::estimate_evalues() {
	event_table& e = ev;
	stage_laps laps("evalue");
	order_ready(); // first stage that visits candidates in the reference's order
	laps.lap("iteration order joined");
	// global statistics (filter_relative_support.cpp:19-127). Fusion partners of every gene (:19-60): counted on the device over the resident candidate
	// state and the iteration order it already holds (csrc/events_hd.h, "fusion partners per gene")
	push_candidate_state();
	std::vector<i32> partner_count(ref.genes.size(), 0);
	check(ctx, arb_partner_counts(ctx, partner_count.data()), "arb_partner_counts");
	laps.lap("partner counts (device)");
	arb_evalue_inputs in; memset(&in, 0, sizeof(in));
	uint32_t tally[11]; // breakpoint locations, intragenic duplications / inversions, spliced pairs, genes with (read-through) fusions, most supporting reads: csrc/events_hd.h, evalue_tally_fn
	check(ctx, arb_evalue_tallies(ctx, tally), "arb_evalue_tallies");
	u32 spliced = tally[0], exonic = tally[1], intronic = tally[2], mixed = tally[3], dups = tally[4], invs = tally[5], same = tally[6], diff = tally[7];
	if (spliced + exonic + intronic + mixed < 100 || spliced == 0 || exonic == 0 || intronic == 0 || mixed == 0) { spliced = 10; exonic = 65; intronic = 10; mixed = 15; }
	if (invs + dups < 100) { invs = 1; dups = 1; }
	if (same + diff < 100) { same = 0; diff = 100; }
	const size_t genes_with_fusions = tally[8], genes_with_read_through = tally[9];
	const float rt_fraction = genes_with_fusions == 0 ? 0 : 1.0 * genes_with_read_through / genes_with_fusions;
	// pow() tables over the integer domains of the reference's expressions (filter_relative_support.cpp:143-205), same libm
	const u32 max_reads = tally[10];
	std::vector<double> t_reads(max_reads + 2), t_intra(max_reads + 2), t_inter(max_reads + 2), t_s1000(1000), t_s400(400);
	// the two distance tables (400,000 entries each) do not depend on the sample: filled once per process, on all threads
	static std::vector<double> t_rt, t_prox; static std::once_flag distance_tables;
	std::call_once(distance_tables, [&]() {
		t_rt.resize(400000); t_prox.resize(400000);
		const int T = std::max(1, threads); std::vector<std::thread> pool;
		for (int t = 0; t < T; ++t) pool.emplace_back([&, t]() { for (int d = 400000 / T * t; d < (t + 1 == T ? 400000 : 400000 / T * (t + 1)); ++d) { t_rt[d] = pow(std::max(1, d) / 400000.0, -0.63); t_prox[d] = pow(std::max(1, d) / 400000.0, -1.53); } });
		for (size_t t = 0; t < pool.size(); ++t) pool[t].join();
	});
	for (unsigned int nr = 0; nr < t_reads.size(); ++nr) { t_reads[nr] = pow(0.02, nr - 2); t_intra[nr] = pow(nr - 0.42, -2.11) * pow(10, -1.11); t_inter[nr] = pow(nr - 0.73, -2.28) * pow(10, -1.75); }
	for (int d = 0; d < 1000; ++d) t_s1000[d] = pow(std::max(400, d) / 1000.0, -2);
	for (int d = 0; d < 400; ++d) t_s400[d] = pow(std::max(1, d) / 400.0, -4.58);
	in.partner_count = partner_count.data(); in.n_genes = (uint32_t) partner_count.size();
	in.spliced_breakpoints = spliced; in.exonic_breakpoints = exonic; in.intronic_breakpoints = intronic; in.exonic_intronic_breakpoints = mixed;
	in.intragenic_duplications = dups; in.intragenic_inversions = invs; in.spliced_same_gene = same; in.spliced_different_genes = diff;
	in.read_through_fraction = rt_fraction; in.mapped_reads = istats.mapped_reads;
	in.pow_reads = t_reads.data(); in.pow_intragenic = t_intra.data(); in.pow_intergenic = t_inter.data(); in.n_read_table = (uint32_t) t_reads.size();
	in.pow_spliced1000 = t_s1000.data(); in.pow_spliced400 = t_s400.data(); in.pow_read_through = t_rt.data(); in.pow_proximal = t_prox.data();
	in.read_through_penalty = 1 + pow((rt_fraction - 0.25) * 20, 2);
	laps.lap("tallies + pow tables");
	push_candidate_state();
	check(ctx, arb_estimate_evalues(ctx, &in), "arb_estimate_evalues");
	pull_candidate_state();
	laps.lap("device + state copies");
	say("Estimating expected number of fusions by random chance (e-value)");
}

void pipeline::filter_relative_support() {
	push_candidate_state();
	check(ctx, arb_filter_relative_support(ctx, opt.params.evalue_cutoff), "arb_filter_relative_support");
	pull_candidate_state();
	log_remaining("Filtering fusions with an e-value >=cutoff");
}

// ------------------------------------------------------------------------------------------- cheap predicates
// the three predicates between the e-value and its cutoff look at one candidate each: on the device (csrc/events_hd.h, simple_filter_fn); only the filter column travels
static void simple_stage(pipeline& p, int stage, const char* what) {
	p.push_candidate_state();
	uint32_t remaining = 0;
	check(p.ctx, arb_filter_simple(p.ctx, stage, p.opt.exonic_fraction, p.opt.min_support, &remaining), "arb_filter_simple");
	check(p.ctx, arb_get_candidate_filters(p.ctx, p.ev.filter.data()), "arb_get_candidate_filters");
	std::ostringstream s; s << what << " (remaining=" << remaining << ")"; p.say(s.str());
}
void pipeline::filter_non_coding_neighbors() { simple_stage(*this, 0, "Filtering fusions with both breakpoints in adjacent non-coding/intergenic regions"); } // filter_non_coding_neighbors.cpp
void pipeline::filter_intragenic_both_exonic() { simple_stage(*this, 1, "Filtering intragenic fusions with both breakpoints in exonic regions"); } // filter_intragenic_both_exonic.cpp
void pipeline::filter_min_support() { simple_stage(*this, 2, "Filtering fusions with <2 supporting reads"); } // filter_min_support.cpp

void pipeline::recover_internal_tandem_duplication() { // recover_internal_tandem_duplication.cpp
	const annot_view an = ref.host_view();
	const unsigned int max_itd_length = opt.params.max_itd_length, min_supporting_reads = opt.min_itd_support, subsampling_threshold = opt.params.subsampling_threshold;
	const float min_fraction_of_coverage = opt.min_itd_allele_fraction; // -z, -Z
	unsigned int duplicates = 0;
	for (u32 i = 0; i < frags.n; ++i) if (labels[i] == F_duplicates) ++duplicates;
	const float duplication_rate = 1.0 * duplicates / frags.n;
	auto recoverable = [](u8 f) { return f == F_hairpin || f == F_inconsistently_clipped || f == F_mismatches; };
	for (size_t q = 0; q < ev.order.size(); ++q) {
		const u32 k = ev.order[q];
		const u8 fl = ev.filter[k];
		if (fl != F_relative_support && fl != F_intragenic_exonic && fl != F_hairpin && fl != F_inconsistently_clipped && fl != F_mismatches) continue;
		if (!(ev.gene1[k] == ev.gene2[k] && ev.exonic1(k) && ev.exonic2(k) && ev.dir1[k] == UPSTREAM && ev.dir2[k] == DOWNSTREAM && ref.genes[ev.gene1[k]].is_protein_coding &&
		      ((unsigned int) ev.bp2[k] - (unsigned int) ev.bp1[k]) < max_itd_length)) continue;
		idset<4096> exons;
		query_index(exon_index(an), ev.contig1[k], ev.bp1[k], ev.bp2[k], exons); if (exons.overflow) throw std::runtime_error("too many overlapping annotation records at one locus");
		bool coding = false;
		for (u32 x = 0; x < exons.n; ++x) {
			const exon_rec& ex = ref.exons[exons.v[x]];
			if (ex.gene == ev.gene1[k] && ex.cds_start <= ev.bp1[k] + 7 && ex.cds_end + 7 >= ev.bp1[k] && ex.cds_start <= ev.bp2[k] + 7 && ex.cds_end + 7 >= ev.bp2[k]) coding = true;
		}
		if (!coding) continue;
		const int cov1 = coverage.get_coverage(ev.contig1[k], ev.bp1[k], ev.dir1[k] == UPSTREAM ? DOWNSTREAM : UPSTREAM);
		const int cov2 = coverage.get_coverage(ev.contig2[k], ev.bp2[k], ev.dir2[k] == UPSTREAM ? DOWNSTREAM : UPSTREAM);
		unsigned int split_reads = 0;
		for (u32 p = ev.list1_off[k]; p < ev.list1_off[k + 1]; ++p) if (labels[ev.list1[p]] == F_none || recoverable(labels[ev.list1[p]])) ++split_reads;
		for (u32 p = ev.list2_off[k]; p < ev.list2_off[k + 1]; ++p) if (labels[ev.list2[p]] == F_none || recoverable(labels[ev.list2[p]])) ++split_reads;
		if (split_reads >= min_supporting_reads && (1.0 * split_reads / std::max(cov1, cov2) / (1 - duplication_rate) > min_fraction_of_coverage || split_reads >= subsampling_threshold)) {
			ev.filter[k] = F_none;
			for (u32 p = ev.list1_off[k]; p < ev.list1_off[k + 1]; ++p) if (recoverable(labels[ev.list1[p]])) { labels[ev.list1[p]] = F_none; ++ev.split_reads1[k]; }
			for (u32 p = ev.list2_off[k]; p < ev.list2_off[k + 1]; ++p) if (recoverable(labels[ev.list2[p]])) { labels[ev.list2[p]] = F_none; ++ev.split_reads2[k]; }
		}
	}
	log_remaining("Searching for internal tandem duplications");
}

void pipeline::filter_both_intronic() { // filter_both_intronic.cpp
	const u32 N = frags.n;
	auto has_exonic = [&](const column<u32>& list, u32 lo, u32 hi) {
		for (u32 p = lo; p < hi; ++p) { const u32 i = list[p]; if (labels[i] != F_none) continue; for (u32 s = 0; s < frags.n_aln[i]; ++s) if (frags.aflags[(size_t) s * N + i] & AF_EXONIC) return true; }
		return false;
	};
	parallel_rows(threads, ev.n, [&](u32 k) {
		if (ev.filter[k] != F_none) return;
		if ((ref.contig_flags[ev.contig1[k]] & CF_VIRAL) || (ref.contig_flags[ev.contig2[k]] & CF_VIRAL)) return;
		if (!has_exonic(ev.list1, ev.list1_off[k], ev.list1_off[k + 1]) && !has_exonic(ev.list2, ev.list2_off[k], ev.list2_off[k + 1]) && !has_exonic(ev.listd, ev.listd_off[k], ev.listd_off[k + 1])) ev.filter[k] = F_intronic;
	});
	log_remaining("Filtering fusions with both breakpoints in intronic/intergenic regions");
}

// chimeric read count per gene and the expression quantile (filter_in_vitro.cpp:48-83)
void pipeline::find_top_expressed_genes(std::vector<u32>& reads_by_gene, std::vector<u8>& present, unsigned int& threshold, float quantile_f) {
	const u32 N = frags.n;
	const size_t G = ref.genes.size();
	reads_by_gene.assign(G, 0); present.assign(G, 0);
	check(ctx, arb_reads_by_gene(ctx, reads_by_gene.data()), "arb_reads_by_gene"); // counted on the device over the resident gene sets (csrc/events_hd.h, reads_by_gene_fn)
	for (size_t g = 0; g < G; ++g) present[g] = reads_by_gene[g] > 0;
	std::vector<u32> genes;
	for (u32 g = 0; g < present.size(); ++g) if (present[g]) genes.push_back(g);
	threshold = 0;
	if (genes.empty()) return;
	unsigned int q = static_cast<int>(floor(quantile_f * genes.size()));
	if (q >= genes.size()) q = genes.size() - 1;
	// the q-th element under (reads, id) ordering is unique, whatever nth_element's internal order
	std::nth_element(genes.begin(), genes.begin() + q, genes.end(), [&](u32 x, u32 y) { return reads_by_gene[x] != reads_by_gene[y] ? reads_by_gene[x] < reads_by_gene[y] : x < y; });
	threshold = reads_by_gene[genes[q]];
}

void pipeline::filter_in_vitro() { // filter_in_vitro.cpp:85-228
	stage_laps laps("in_vitro");
	std::vector<u64> exonic_breakpoints; // one (gene, partner) key per exonic, unspliced breakpoint pair, sorted: a count is the width of an equal range
	for (u32 k = 0; k < ev.n; ++k)
		if (ev.gene1[k] != ev.gene2[k] && !ev.spliced1(k) && !ev.spliced2(k) && ev.exonic1(k) && ev.exonic2(k) && ev.n_list1(k) + ev.n_list2(k) > 0 && ev.filter[k] != F_merge_adjacent && ev.filter[k] != F_uninteresting_contigs) {
			exonic_breakpoints.push_back((u64) ev.gene1[k] << 32 | ev.gene2[k]); exonic_breakpoints.push_back((u64) ev.gene2[k] << 32 | ev.gene1[k]);
		}
	parallel_sort(exonic_breakpoints, [](u64 a, u64 b) { return a < b; }, threads);
	laps.lap("exonic breakpoint pairs");
	std::vector<u32> reads_by_gene; std::vector<u8> present; unsigned int threshold;
	find_top_expressed_genes(reads_by_gene, present, threshold, opt.high_expression_quantile); // -Q
	laps.lap("top expressed genes");
	// the verdicts: one thread per candidate on the device (csrc/events_hd.h, in_vitro_fn) -- every candidate walks its discordant mates, which lie all over
	// the fragment table
	ensure_coverage_on_device();
	check(ctx, arb_set_fragment_filters(ctx, labels.data()), "arb_set_fragment_filters");
	push_candidate_state();
	check(ctx, arb_filter_in_vitro(ctx, reads_by_gene.data(), (uint32_t) reads_by_gene.size(), threshold, (const uint64_t*) exonic_breakpoints.data(), exonic_breakpoints.size()), "arb_filter_in_vitro");
	check(ctx, arb_get_candidate_filters(ctx, ev.filter.data()), "arb_get_candidate_filters");
	laps.lap("candidates");
	log_remaining("Filtering in vitro-generated fusions");
}

void pipeline::ensure_coverage_on_device() {
	if (coverage_on_device) return;
	std::vector<const u16*> cov(coverage.coverage.size(), (const u16*) NULL); std::vector<uint64_t> windows(coverage.coverage.size(), 0);
	for (size_t c = 0; c < coverage.coverage.size(); ++c) { cov[c] = coverage.coverage[c].data(); windows[c] = coverage.coverage[c].size(); }
	check(ctx, arb_set_coverage(ctx, cov.data(), windows.data(), (uint32_t) cov.size()), "arb_set_coverage");
	coverage_on_device = true;
}

void pipeline::recover_both_spliced() { // recover_both_spliced.cpp:64-182
	const unsigned int max_fusions_to_recover = 200;
	std::vector<u32> reads_by_gene; std::vector<u8> present; unsigned int threshold;
	find_top_expressed_genes(reads_by_gene, present, threshold, 0.998f); // fixed quantile (arriba.cpp:492)
	stage_laps laps("spliced");
	// spliced support of every candidate that may back another one up (recover_both_spliced.cpp:104-118); a pure function of the candidate: host threads
	const u32 NOT_ELIGIBLE = 0xFFFFFFFFu;
	column<u32> support(ev.n); // page-locked, written in full by the device
	ensure_coverage_on_device();
	check(ctx, arb_set_fragment_filters(ctx, labels.data()), "arb_set_fragment_filters");
	push_candidate_state();
	check(ctx, arb_spliced_support(ctx, reads_by_gene.data(), (uint32_t) reads_by_gene.size(), threshold, support.data()), "arb_spliced_support"); // csrc/events_hd.h, spliced_support_fn
	// group them by (gene1, gene2, direction1, direction2): sorted keys instead of the reference's map of vectors (only sums over a group are taken)
	auto key_of = [&](u32 k, bool flip) { return (u64) ev.gene1[k] << 34 | (u64) ev.gene2[k] << 4 | (u64) ((ev.dir1[k] != 0) != flip) << 1 | (u64) ((ev.dir2[k] != 0) != flip); };
	if (ref.genes.size() >= (1u << 30)) throw std::runtime_error("too many genes");
	std::vector<std::pair<u64, u32> > grouped;
	{ // the eligible candidates, collected by all threads (the sort below orders them by (key, candidate) whatever the order here)
		const int T = std::max(1, std::min(threads, (int) (ev.n / 65536 + 1)));
		std::vector<std::vector<std::pair<u64, u32> > > part(T);
		std::vector<std::thread> pool;
		for (int t = 0; t < T; ++t) pool.emplace_back([&, t]() { for (u32 k = (u32) ((u64) ev.n * t / T); k < (u32) ((u64) ev.n * (t + 1) / T); ++k) if (support[k] != NOT_ELIGIBLE) part[t].push_back(std::make_pair(key_of(k, false), k)); });
		for (size_t t = 0; t < pool.size(); ++t) pool[t].join();
		size_t total = 0; for (int t = 0; t < T; ++t) total += part[t].size();
		grouped.reserve(total);
		for (int t = 0; t < T; ++t) grouped.insert(grouped.end(), part[t].begin(), part[t].end());
	}
	laps.lap("support of eligible candidates");
	parallel_sort(grouped, [](const std::pair<u64, u32>& a, const std::pair<u64, u32>& b) { return a < b; }, threads);
	laps.lap("grouped by gene pair");
	auto group_of = [&](u64 key, size_t& lo, size_t& hi) {
		lo = std::lower_bound(grouped.begin(), grouped.end(), std::make_pair(key, (u32) 0)) - grouped.begin();
		hi = lo; while (hi < grouped.size() && grouped[hi].first == key) ++hi;
	};
	// reads that back each discarded, both-spliced candidate up (recover_both_spliced.cpp:123-160); independent per candidate
	std::vector<u32> backing(ev.n, 0);
	parallel_rows(threads, ev.n, [&](u32 k) {
		const u8 fl = ev.filter[k];
		if (fl == F_none) return;
		if (!both_spliced(ev, ref, k)) return;
		if (ev.gene1[k] == ev.gene2[k] || overlaps_both(ev, ref, k)) return;
		if (ev.is_read_through(k)) return;
		if (fl != F_relative_support && fl != F_min_support && fl != F_in_vitro) return;
		unsigned int sum = 0;
		size_t lo, hi;
		group_of(key_of(k, false), lo, hi);
		for (size_t x = lo; x < hi; ++x) sum += support[grouped[x].second];
		group_of(key_of(k, true), lo, hi); // the reciprocal orientation
		for (size_t x = lo; x < hi; ++x) {
			const u32 o = grouped[x].second;
			if (ev.is_read_through(o)) continue;
			if (both_spliced(ev, ref, o) || (((ev.dir1[k] == DOWNSTREAM) != (ev.bp1[k] > ev.bp1[o])) && ((ev.dir2[k] == DOWNSTREAM) != (ev.bp2[k] > ev.bp2[o])))) sum += support[o];
		}
		backing[k] = sum;
	});
	laps.lap("backing per candidate");
	// at most ~200 candidates are recovered: raise the read threshold until fewer would be (recover_both_spliced.cpp:162-175), then recover
	std::map<unsigned int, unsigned int> recovered_by_reads;
	for (u32 k = 0; k < ev.n; ++k) if (backing[k] >= 2) ++recovered_by_reads[ev.supporting_reads(k)];
	unsigned int min_supporting_reads = 1, would = 0;
	for (std::map<unsigned int, unsigned int>::reverse_iterator it = recovered_by_reads.rbegin(); it != recovered_by_reads.rend(); ++it) { would += it->second; if (would >= max_fusions_to_recover) { min_supporting_reads = it->first + 1; break; } }
	for (u32 k = 0; k < ev.n; ++k) if (backing[k] >= 2) {
		const unsigned int proximal = (ev.contig1[k] == ev.contig2[k] && std::abs(ev.bp1[k] - ev.bp2[k]) < 1000000) ? 1 : 0;
		if (ev.supporting_reads(k) >= min_supporting_reads + proximal) ev.filter[k] = F_none;
	}
	log_remaining("Searching for fusions with spliced split reads");
}

void pipeline::select_best() { // select_best.cpp, on the device (csrc/events_hd.h, select_group_fn): stable sorts by (gene pair + directions, iteration rank), one sequential scan per group
	push_candidate_state();
	uint32_t remaining = 0;
	check(ctx, arb_select_best(ctx, &remaining), "arb_select_best");
	check(ctx, arb_get_candidate_filters(ctx, ev.filter.data()), "arb_get_candidate_filters");
	std::ostringstream s; s << "Selecting best breakpoints from genes with multiple breakpoints (remaining=" << remaining << ")"; say(s.str());
}

void pipeline::filter_marginal_read_through() { // filter_marginal_read_through.cpp
	const float margin = 0.01f, min_vaf = 0.07f;
	for (u32 k = 0; k < ev.n; ++k) {
		if (!(ev.filter[k] == F_none && ev.is_read_through(k))) continue;
		const gene_rec& g1 = ref.genes[ev.gene1[k]]; const gene_rec& g2 = ref.genes[ev.gene2[k]];
		double donor = 1, acceptor = 1;
		if (!g1.is_dummy && g1.forward && ev.dir1[k] == DOWNSTREAM) donor = 1.0 * (ev.bp1[k] - g1.start) / (g1.end - g1.start);
		else if (!g2.is_dummy && !g2.forward && ev.dir2[k] == UPSTREAM) donor = 1.0 * (g2.end - ev.bp2[k]) / (g2.end - g2.start);
		else if (!g1.is_dummy && !g1.forward && ev.dir1[k] == DOWNSTREAM) acceptor = 1.0 * (ev.bp1[k] - g1.start) / (g1.end - g1.start);
		else if (!g2.is_dummy && g2.forward && ev.dir2[k] == UPSTREAM) acceptor = 1.0 * (g2.end - ev.bp2[k]) / (g2.end - g2.start);
		else continue;
		const int cov1 = coverage.get_coverage(ev.contig1[k], ev.bp1[k], ev.dir1[k] == UPSTREAM ? DOWNSTREAM : UPSTREAM);
		const int cov2 = coverage.get_coverage(ev.contig2[k], ev.bp2[k], ev.dir2[k] == UPSTREAM ? DOWNSTREAM : UPSTREAM);
		if (donor > 1 - margin && acceptor > 1 - margin && ev.supporting_reads(k) < min_vaf * std::max(cov1, cov2)) ev.filter[k] = F_marginal_read_through;
	}
	log_remaining("Filtering read-through fusions with breakpoints near the gene boundary");
}

void pipeline::recover_many_spliced() { // recover_many_spliced.cpp
	const unsigned int min_spliced_events = opt.min_spliced_events; // -M
	auto eligible_filter = [](u8 f) { return f == F_inconsistently_clipped || f == F_relative_support || f == F_min_support || f == F_select_best; };
	// distinct (breakpoint1 / 10, breakpoint2 / 10) pairs per gene pair: sorted tuples instead of the reference's map of sets (only the set sizes are used)
	struct event { u32 gene1, gene2; i32 b1, b2; };
	std::vector<event> events;
	for (u32 k = 0; k < ev.n; ++k)
		if ((ev.spliced1(k) || ev.spliced2(k)) && ev.gene1[k] != ev.gene2[k] && (ev.filter[k] == F_none || eligible_filter(ev.filter[k])) && !ev.is_read_through(k) && !overlaps_both(ev, ref, k)) {
			const event x = {ev.gene1[k], ev.gene2[k], ev.bp1[k] / 10, ev.bp2[k] / 10}; events.push_back(x);
		}
	auto before = [](const event& a, const event& b) { return a.gene1 != b.gene1 ? a.gene1 < b.gene1 : a.gene2 != b.gene2 ? a.gene2 < b.gene2 : a.b1 != b.b1 ? a.b1 < b.b1 : a.b2 < b.b2; };
	parallel_sort(events, before, threads);
	std::vector<std::pair<u64, u32> > pair_events; // (gene1 << 32 | gene2, distinct events), ascending
	for (size_t x = 0; x < events.size(); ++x) {
		if (x > 0 && !before(events[x - 1], events[x])) continue; // the same event again
		const u64 key = (u64) events[x].gene1 << 32 | events[x].gene2;
		if (pair_events.empty() || pair_events.back().first != key) pair_events.push_back(std::make_pair(key, 0u));
		++pair_events.back().second;
	}
	auto events_of = [&](u32 g1, u32 g2) { const u64 key = (u64) g1 << 32 | g2; std::vector<std::pair<u64, u32> >::const_iterator it = std::lower_bound(pair_events.begin(), pair_events.end(), std::make_pair(key, 0u)); return it != pair_events.end() && it->first == key ? it->second : 0u; };
	parallel_rows(threads, ev.n, [&](u32 k) {
		if (ev.filter[k] == F_none || !eligible_filter(ev.filter[k]) || !(ev.spliced1(k) || ev.spliced2(k))) return;
		if (ev.is_read_through(k) || ev.gene1[k] == ev.gene2[k] || overlaps_both(ev, ref, k)) return;
		if (events_of(ev.gene1[k], ev.gene2[k]) >= min_spliced_events) ev.filter[k] = F_none;
	});
	log_remaining("Searching for fusions with >=4 spliced events");
}

void pipeline::filter_short_anchor() { // filter_short_anchor.cpp
	const unsigned int min_length = opt.min_anchor_length; // -A
	for (u32 k = 0; k < ev.n; ++k) {
		if (ev.filter[k] != F_none) continue;
		if (!(ev.spliced1(k) && ev.spliced2(k)) && ((unsigned int) std::abs(ev.anchor1[k] - ev.bp1[k]) < min_length || (unsigned int) std::abs(ev.anchor2[k] - ev.bp2[k]) < min_length)) ev.filter[k] = F_short_anchor;
	}
	log_remaining("Filtering fusions with anchors <=23nt");
}

float pipeline::intronic_fraction(u32 gene) { // filter_end_to_end.cpp:9-25
	const gene_rec& g = ref.genes[gene];
	const region_index& ix = ref.exon_index;
	unsigned int intronic = 0; i32 previous = g.start;
	const u32 lo = ix.begin[g.contig], hi = ix.begin[g.contig + 1];
	for (u32 r = (u32) (std::lower_bound(ix.end.begin() + lo, ix.end.begin() + hi, g.start) - ix.end.begin()); r < hi && ix.end[r] <= g.end; ++r)
		for (u32 x = ix.off[r]; x < ix.off[r + 1]; ++x) {
			const exon_rec& ex = ref.exons[ix.items[x]];
			if (ex.gene != gene) continue;
			if (previous < ex.start) intronic += ex.start - previous;
			if (previous < ex.end) previous = ex.end + 1;
			break;
		}
	return ((float) intronic) / (g.end - g.start + 1);
}

void pipeline::filter_end_to_end() { // filter_end_to_end.cpp:27-78
	for (u32 k = 0; k < ev.n; ++k) {
		if (ev.filter[k] != F_none) continue;
		if ((ref.contig_flags[ev.contig1[k]] & CF_VIRAL) || (ref.contig_flags[ev.contig2[k]] & CF_VIRAL)) continue;
		if (!ev.is_read_through(k) && ev.gene1[k] != ev.gene2[k] && (ev.spliced1(k) || ev.spliced2(k))) continue;
		const u32 s1 = ev.split_reads1[k], s2 = ev.split_reads2[k], d = ev.discordant_mates[k];
		if (!(d + s1 == 0 || d + s2 == 0 || s1 + s2 == 0 || (overlaps_both(ev, ref, k) && (s1 == 0 || s2 == 0)))) continue;
		const gene_rec& g1 = ref.genes[ev.gene1[k]]; const gene_rec& g2 = ref.genes[ev.gene2[k]];
		if (!((g1.is_dummy || (g1.forward && ev.dir1[k] == UPSTREAM) || (!g1.forward && ev.dir1[k] == DOWNSTREAM)) && (g2.is_dummy || (g2.forward && ev.dir2[k] == UPSTREAM) || (!g2.forward && ev.dir2[k] == DOWNSTREAM)))) continue;
		if (d < 10 || (ev.contig1[k] == ev.contig2[k] && std::abs(ev.bp1[k] - ev.bp2[k]) < 1000000) ||
		    (ev.exonic1(k) && ev.exonic2(k) && intronic_fraction(ev.gene1[k]) > 0.66f && intronic_fraction(ev.gene2[k]) > 0.66f)) ev.filter[k] = F_end_to_end;
	}
	log_remaining("Filtering end-to-end fusions with low support");
}

void pipeline::filter_no_coverage() { // filter_no_coverage.cpp
	const annot_view an = ref.host_view();
	const int scan_range = 200;
	for (u32 k = 0; k < ev.n; ++k) {
		if (ev.filter[k] != F_none) continue;
		const u32 s1 = ev.split_reads1[k], s2 = ev.split_reads2[k], d = ev.discordant_mates[k];
		if (!ev.is_read_through(k)) {
			if (s1 + s2 != 0 && s1 + d != 0 && s2 + d != 0) continue;
			if (ev.spliced1(k) || ev.spliced2(k)) continue;
		} else if (ev.spliced1(k) && ev.spliced2(k)) continue;
		bool discard = false;
		for (int side = 1; side <= 2 && !discard; ++side) {
			const u16 contig = side == 1 ? ev.contig1[k] : ev.contig2[k]; const i32 bp = side == 1 ? ev.bp1[k] : ev.bp2[k];
			const u32 gene = side == 1 ? ev.gene1[k] : ev.gene2[k]; const u32 dir = side == 1 ? ev.dir1[k] : ev.dir2[k]; const i32 anchor = side == 1 ? ev.anchor1[k] : ev.anchor2[k];
			idset<4096> exons; query_index(exon_index(an), contig, bp, bp, exons); if (exons.overflow) throw std::runtime_error("too many overlapping annotation records at one locus");
			bool terminal = false;
			for (u32 x = 0; x < exons.n && !terminal; ++x) { const exon_rec& ex = ref.exons[exons.v[x]]; if (ex.gene == gene && (ex.prev == -1 || ex.next == -1)) terminal = true; }
			if (terminal) continue;
			i32 start, end;
			if (dir == UPSTREAM) { start = bp; if (s1 + s2 == 0) start -= scan_range; end = std::max(bp + scan_range, anchor); }
			else { start = std::min(bp - scan_range, anchor); end = bp; if (s1 + s2 == 0) end += scan_range; }
			if ((dir == UPSTREAM && !coverage.fragment_starts_here(contig, start, end)) || (dir == DOWNSTREAM && !coverage.fragment_ends_here(contig, start, end))) discard = true;
		}
		if (discard) ev.filter[k] = F_no_coverage;
	}
	log_remaining("Filtering fusions with no coverage around the breakpoints");
}

void pipeline::recover_isoforms() { // recover_isoforms.cpp
	typedef std::tuple<u32, u32, bool, bool> pair_key;
	std::map<pair_key, u32> fused; // last unfiltered candidate in iteration order wins
	for (u32 k = 0; k < ev.n; ++k) if (ev.filter[k] == F_none) { // the one with the highest rank in the iteration order
		const std::pair<std::map<pair_key, u32>::iterator, bool> ins = fused.insert(std::make_pair(pair_key(ev.gene1[k], ev.gene2[k], (bool) ev.dir1[k], (bool) ev.dir2[k]), k));
		if (!ins.second && ev.rank_of[k] > ev.rank_of[ins.first->second]) ins.first->second = k;
	}
	for (u32 k = 0; k < ev.n; ++k) { // a verdict per candidate, independent of the others (`fused` and the breakpoints it points at do not change)
		const u8 fl = ev.filter[k];
		if (fl == F_none) continue;
		if (fl == F_merge_adjacent || fl == F_blacklist || fl == F_end_to_end || fl == F_duplicates || ev.gene1[k] == ev.gene2[k]) continue;
		if (!(ev.spliced1(k) && ev.spliced2(k))) continue;
		std::map<pair_key, u32>::iterator it = fused.find(pair_key(ev.gene1[k], ev.gene2[k], (bool) ev.dir1[k], (bool) ev.dir2[k]));
		if (it != fused.end() && (std::abs(ev.bp1[it->second] - ev.bp1[k]) > 2 || std::abs(ev.bp2[it->second] - ev.bp2[k]) > 2)) ev.filter[k] = F_none;
	}
	log_remaining("Searching for additional isoforms");
}

// ------------------------------------------------------------------------------------------- k-mer index, homologs, mismappers (device)
void pipeline::make_kmer_index() { // windows of make_kmer_index (filter_mismappers.cpp:47-84); the device enumerates and sorts the positions
	const annot_view an = ref.host_view();
	std::vector<u8> wanted(ref.genes.size(), 0);
	for (u32 k = 0; k < ev.n; ++k) if (ev.filter[k] == F_none && ev.gene1[k] != ev.gene2[k]) { wanted[ev.gene1[k]] = 1; wanted[ev.gene2[k]] = 1; }
	int padding = max_mate_gap + 2 * read_length_mean; // int + float -> float -> int (arriba.cpp:552)
	if (padding < 0) padding = 0;
	struct iv { u32 contig; i32 start, end; };
	std::vector<iv> ivs; u32 n_index_contigs = 0;
	for (u32 g = 0; g < ref.genes.size(); ++g) if (wanted[g]) {
		const gene_rec& G = ref.genes[g];
		if (!ref.has_sequence(G.contig)) throw std::runtime_error("no sequence for a contig with fused genes");
		const i32 gs = std::max(G.start - padding, 0), ge = std::min(G.end + padding, (i32) ref.seq_len[G.contig] - 1);
		n_index_contigs = std::max(n_index_contigs, (u32) G.contig + 1);
		if (gs + 8 < ge) { iv x = {G.contig, gs, ge - 8}; ivs.push_back(x); } // positions pos with pos + 8 < gene_end
	}
	std::sort(ivs.begin(), ivs.end(), [](const iv& a, const iv& b) { return a.contig != b.contig ? a.contig < b.contig : a.start < b.start; });
	std::vector<u32> c; std::vector<i32> s, t;
	for (size_t k = 0; k < ivs.size(); ++k) {
		if (!c.empty() && c.back() == ivs[k].contig && ivs[k].start <= t.back()) { t.back() = std::max(t.back(), ivs[k].end); continue; }
		c.push_back(ivs[k].contig); s.push_back(ivs[k].start); t.push_back(ivs[k].end);
	}
	// downstream splice sites per gene (filter_mismappers.cpp:16-31)
	if (!splice_sites_ready) {
		std::vector<u32> off(ref.genes.size() + 1, 0); std::vector<i32> sites;
		const region_index& ix = ref.exon_index;
		for (u32 g = 0; g < ref.genes.size(); ++g) {
			const gene_rec& G = ref.genes[g];
			const u32 lo = ix.begin[G.contig], hi = ix.begin[G.contig + 1];
			for (u32 r = (u32) (std::lower_bound(ix.end.begin() + lo, ix.end.begin() + hi, G.start) - ix.end.begin()); r < hi && ix.end[r] <= G.end; ++r)
				if (is_breakpoint_spliced(an, g, DOWNSTREAM, ix.end[r])) sites.push_back(ix.end[r]);
			off[g + 1] = (u32) sites.size();
		}
		if (sites.empty()) sites.push_back(0);
		check(ctx, arb_set_splice_sites(ctx, off.data(), sites.data()), "arb_set_splice_sites");
		splice_sites_ready = true;
	}
	uint64_t n_indexed = 0;
	if (c.empty()) { c.push_back(0); s.push_back(0); t.push_back(0); check(ctx, arb_build_kmer_index(ctx, c.data(), s.data(), t.data(), 0, n_index_contigs, &n_indexed), "arb_build_kmer_index"); }
	else check(ctx, arb_build_kmer_index(ctx, c.data(), s.data(), t.data(), (uint32_t) c.size(), n_index_contigs, &n_indexed), "arb_build_kmer_index");
	say("Indexing gene sequences");
}

void pipeline::filter_homologs() { // filter_homologs.cpp:65-141; is_homolog() itself is evaluated on the device in two batches
	stage_laps laps("homologs");
	// remaining candidates in the reference's list order: push_front over the iteration order = reverse iteration order
	std::vector<u32> rem;
	for (u32 k = 0; k < ev.n; ++k) if (ev.filter[k] == F_none) rem.push_back(k);
	std::sort(rem.begin(), rem.end(), [&](u32 a, u32 b) { return ev.rank_of[a] > ev.rank_of[b]; });
	// batch 1: the two genes of every remaining candidate
	std::vector<u32> ga, gb; std::vector<u8> res;
	for (size_t x = 0; x < rem.size(); ++x) { ga.push_back(ev.gene1[rem[x]]); gb.push_back(ev.gene2[rem[x]]); }
	res.resize(ga.size() + 1);
	if (!ga.empty()) check(ctx, arb_homolog_pairs(ctx, ga.data(), gb.data(), (uint32_t) ga.size(), res.data()), "arb_homolog_pairs");
	std::vector<u8> self_homolog(res.begin(), res.begin() + ga.size());
	laps.lap("own gene pairs (device)");
	// batch 2: partner genes of candidates that share a gene (a superset of what the sequential pass will ask for)
	auto partner_genes = [&](u32 f, u32 o, u32& h1, u32& h2) { // which genes would be compared for the pair (f, o)?  (filter_homologs.cpp:97-113)
		if (ev.gene1[f] == ev.gene1[o] && ev.bp2[f] != ev.bp2[o]) { h1 = ev.gene2[f]; h2 = ev.gene2[o]; return true; }
		if (ev.gene1[f] == ev.gene2[o] && ev.bp2[f] != ev.bp1[o]) { h1 = ev.gene2[f]; h2 = ev.gene1[o]; return true; }
		if (ev.gene2[f] == ev.gene1[o] && ev.bp1[f] != ev.bp2[o]) { h1 = ev.gene1[f]; h2 = ev.gene2[o]; return true; }
		if (ev.gene2[f] == ev.gene2[o] && ev.bp1[f] != ev.bp1[o]) { h1 = ev.gene1[f]; h2 = ev.gene1[o]; return true; }
		return false;
	};
	std::vector<std::vector<u32> > by_gene(ref.genes.size()); // positions in rem, ascending
	for (size_t x = 0; x < rem.size(); ++x) { by_gene[ev.gene1[rem[x]]].push_back((u32) x); if (ev.gene2[rem[x]] != ev.gene1[rem[x]]) by_gene[ev.gene2[rem[x]]].push_back((u32) x); }
	// the distinct gene pairs: collected as 64-bit keys, sorted, made unique (a tree map took most of this stage's time)
	std::vector<u64> pair_keys; ga.clear(); gb.clear();
	for (size_t x = 0; x < rem.size(); ++x) {
		if (self_homolog[x]) continue;
		const u32 f = rem[x];
		for (int side = 0; side < 2; ++side) {
			const std::vector<u32>& v = by_gene[side == 0 ? ev.gene1[f] : ev.gene2[f]];
			for (size_t y = 0; y < v.size(); ++y) {
				if (v[y] <= x) continue;
				u32 h1, h2;
				if (!partner_genes(f, rem[v[y]], h1, h2)) continue;
				pair_keys.push_back((u64) h1 << 32 | h2);
			}
			if (ev.gene1[f] == ev.gene2[f]) break;
		}
	}
	parallel_sort(pair_keys, [](u64 a, u64 b) { return a < b; }, threads);
	pair_keys.erase(std::unique(pair_keys.begin(), pair_keys.end()), pair_keys.end());
	for (size_t k = 0; k < pair_keys.size(); ++k) { ga.push_back((u32) (pair_keys[k] >> 32)); gb.push_back((u32) pair_keys[k]); }
	auto pair_index_of = [&](u32 h1, u32 h2) { return (size_t) (std::lower_bound(pair_keys.begin(), pair_keys.end(), (u64) h1 << 32 | h2) - pair_keys.begin()); };
	laps.lap("gene pairs of candidates that share a gene");
	res.assign(ga.size() + 1, 0);
	if (!ga.empty()) check(ctx, arb_homolog_pairs(ctx, ga.data(), gb.data(), (uint32_t) ga.size(), res.data()), "arb_homolog_pairs");
	laps.lap("identity of the pairs (device)");
	// sequential resolution, exactly in list order
	for (size_t x = 0; x < rem.size(); ++x) {
		const u32 f = rem[x];
		if (ev.filter[f] != F_none) continue;
		if (self_homolog[x]) { ev.filter[f] = F_homologs; continue; }
		// later candidates that share a gene with f, in list order
		std::vector<u32> later;
		for (int side = 0; side < 2; ++side) { const std::vector<u32>& v = by_gene[side == 0 ? ev.gene1[f] : ev.gene2[f]]; for (size_t y = 0; y < v.size(); ++y) if (v[y] > x) later.push_back(v[y]); if (ev.gene1[f] == ev.gene2[f]) break; }
		std::sort(later.begin(), later.end()); later.erase(std::unique(later.begin(), later.end()), later.end());
		for (size_t y = 0; y < later.size(); ++y) {
			const u32 o = rem[later[y]];
			if (ev.filter[o] != F_none) continue;
			u32 h1, h2;
			if (!partner_genes(f, o, h1, h2)) continue;
			const unsigned int a1 = (ev.split_reads1[f] > 0) + (ev.split_reads2[f] > 0) + (ev.discordant_mates[f] > 0), a2 = (ev.split_reads1[o] > 0) + (ev.split_reads2[o] > 0) + (ev.discordant_mates[o] > 0);
			if (!res[pair_index_of(h1, h2)]) continue;
			if (a1 > a2 || (a1 == a2 && ev.supporting_reads(f) > ev.supporting_reads(o)) || (a1 == a2 && ev.supporting_reads(f) == ev.supporting_reads(o) && ev.evalue[f] <= ev.evalue[o])) ev.filter[o] = F_homologs;
			else { ev.filter[f] = F_homologs; break; }
		}
	}
	log_remaining("Filtering genes with >=30% identity");
}

void pipeline::filter_mismappers() { // filter_mismappers.cpp:272-359, on the device
	check(ctx, arb_set_fragment_filters(ctx, labels.data()), "arb_set_fragment_filters");
	push_candidate_state();
	uint64_t n_items = 0;
	check(ctx, arb_filter_mismappers(ctx, max_mate_gap, &n_items), "arb_filter_mismappers");
	pull_candidate_state();
	check(ctx, arb_get_fragment_filters(ctx, labels.data(), NULL), "arb_get_fragment_filters");
	log_remaining("Re-aligning chimeric reads to filter fusions with >=80% mis-mappers");
}

// ------------------------------------------------------------------------------------------- genomic support (-d)
void pipeline::mark_genomic_support() { // filter_genomic_support.cpp:80-220: the file is read here, the search runs on the device (csrc/genomic_hd.h)
	genomic_records g;
	read_genomic_breakpoints(opt.genomic_breakpoints_file, ref.contig_ids, g);
	check(ctx, arb_set_genomic_breakpoints(ctx, (uint32_t) g.pos1.size(), g.contig1.data(), g.contig2.data(), g.dir1.data(), g.dir2.data(), g.pos1.data(), g.pos2.data()), "arb_set_genomic_breakpoints");
	uint32_t marked = 0;
	check(ctx, arb_mark_genomic_support(ctx, (int32_t) opt.max_genomic_breakpoint_distance, (int32_t) opt.params.max_itd_length, &marked), "arb_mark_genomic_support");
	ev.closest1.resize(ev.n); ev.closest2.resize(ev.n);
	check(ctx, arb_get_genomic_support(ctx, ev.closest1.data(), ev.closest2.data()), "arb_get_genomic_support");
	std::ostringstream s; s << "Marking fusions with support from whole-genome sequencing in '" << opt.genomic_breakpoints_file << "' (marked=" << marked << ")"; say(s.str());
}

void pipeline::filter_no_genomic_support() { // filter_genomic_support.cpp:404-419; viral = the -v patterns, not the per-sample verdicts
	for (u32 k = 0; k < ev.n; ++k)
		if (ev.filter[k] == F_none && !ev.genomic_support(k) && ev.confidence[k] == 0 && !(ref.contig_flags[ev.contig1[k]] & CF_VIRAL) && !(ref.contig_flags[ev.contig2[k]] & CF_VIRAL))
			ev.filter[k] = F_no_genomic_support;
	log_remaining("Filtering low-confidence events with no support from WGS");
}

void pipeline::recover_genomic_support() { // filter_genomic_support.cpp:421-444
	for (u32 k = 0; k < ev.n; ++k) {
		const u8 f = ev.filter[k];
		if (f != F_none && ev.genomic_support(k) && (f == F_end_to_end || f == F_intronic || f == F_mismappers || f == F_no_coverage || f == F_in_vitro || f == F_relative_support)) ev.filter[k] = F_none;
	}
	log_remaining("Searching for fusions with support from WGS");
}

// ------------------------------------------------------------------------------------------- blacklist (-b)
// filter_blacklisted_ranges.cpp:232-300: the eligible set is fixed first, then the file is read (its warnings follow those of -d) and the rules are matched on the
// device (csrc/blacklist_hd.h). The device reads the split-read / discordant-mate counts and e-values it holds: estimate_evalues (EV_EVALUE, always run) left the
// host's there and no later stage changes them on the host; breakpoints, directions, genes and the spliced / strand bits never change after find_fusions.
void pipeline::filter_blacklist() {
	std::vector<u32> ids;
	for (u32 k = 0; k < ev.n; ++k) if (ev.filter[k] == F_none || ev.genomic_support(k)) ids.push_back(k); // :238-239
	fusion_rules r;
	read_fusion_rules(opt.blacklist_file, ref, RULES_BLACKLIST, max_mate_gap, r);
	const uint32_t n = (uint32_t) r.size();
	check(ctx, arb_set_blacklist(ctx, n, r.type1.data(), r.type2.data(), r.strand1.data(), r.strand2.data(), r.contig1.data(), r.contig2.data(),
	                             r.start1.data(), r.end1.data(), r.start2.data(), r.end2.data(), r.gene1.data(), r.gene2.data()), "arb_set_blacklist");
	std::vector<u8> verdict(ids.size());
	uint32_t blacklisted = 0;
	check(ctx, arb_filter_blacklist(ctx, (uint32_t) ids.size(), ids.data(), opt.params.evalue_cutoff, max_mate_gap, verdict.data(), &blacklisted), "arb_filter_blacklist");
	for (size_t x = 0; x < ids.size(); ++x) if (verdict[x]) ev.filter[ids[x]] = F_blacklist; // overwrites an earlier filter of a candidate with genomic support
	log_remaining(("Filtering blacklisted fusions in '" + opt.blacklist_file + "'").c_str());
}

// ------------------------------------------------------------------------------------------- known fusions (-k)
// recover_known_fusions.cpp:14-100, right after filter_both_intronic: candidates that min_support or relative_support removed come back if a rule of the file
// matches them (csrc/blacklist_hd.h). The device reads the support counts, the spliced bits and the coverage windows, so the host's state goes up first.
void pipeline::recover_known_fusions() {
	fusion_rules r;
	read_fusion_rules(opt.known_fusions_file, ref, RULES_KNOWN_FUSIONS, max_mate_gap, r);
	std::vector<u32> ids;
	for (u32 k = 0; k < ev.n; ++k)
		if ((ev.filter[k] == F_relative_support || ev.filter[k] == F_min_support) && ev.gene1[k] != ev.gene2[k]) ids.push_back(k); // :43-50
	const uint32_t n = (uint32_t) r.size();
	check(ctx, arb_set_known_fusions(ctx, n, r.type1.data(), r.type2.data(), r.strand1.data(), r.strand2.data(), r.contig1.data(), r.contig2.data(),
	                                 r.start1.data(), r.end1.data(), r.start2.data(), r.end2.data(), r.gene1.data(), r.gene2.data()), "arb_set_known_fusions");
	if (!ids.empty()) {
		ensure_coverage_on_device();
		push_candidate_state();
		std::vector<u8> verdict(ids.size());
		uint32_t rescued = 0;
		check(ctx, arb_recover_known_fusions(ctx, (uint32_t) ids.size(), ids.data(), max_mate_gap, verdict.data(), &rescued), "arb_recover_known_fusions");
		for (size_t x = 0; x < ids.size(); ++x) if (verdict[x]) ev.filter[ids[x]] = F_none;
	}
	log_remaining(("Searching for known fusions in '" + opt.known_fusions_file + "'").c_str());
}

// ------------------------------------------------------------------------------------------- tags (-t)
// load_tags (annotate_tags.cpp:11-43) and annotate_tags (:45-83) for every row that is written: the rows of fusions.tsv and, with a discarded file, all others.
// The device keeps the tags of every candidate for the rows it formats; the host keeps a copy for the rows it formats itself.
void pipeline::annotate_tags() {
	say("Loading tags from '" + opt.tags_file + "'");
	fusion_rules r;
	read_fusion_rules(opt.tags_file, ref, RULES_TAGS, max_mate_gap, r);
	std::vector<u32> rank;
	rank_tags(r, tag_names, rank);
	std::vector<char> chars; std::vector<u32> off(1, 0);
	for (size_t t = 0; t < tag_names.size(); ++t) { chars.insert(chars.end(), tag_names[t].begin(), tag_names[t].end()); off.push_back((u32) chars.size()); }
	chars.push_back(0); rank.push_back(0);
	const uint32_t n = (uint32_t) r.size();
	check(ctx, arb_set_tags(ctx, n, r.type1.data(), r.type2.data(), r.strand1.data(), r.strand2.data(), r.contig1.data(), r.contig2.data(), r.start1.data(), r.end1.data(),
	                        r.start2.data(), r.end2.data(), r.gene1.data(), r.gene2.data(), rank.data(), (uint32_t) tag_names.size(), chars.data(), off.data()), "arb_set_tags");
	const bool all = !opt.discarded_output_file.empty();
	std::vector<u32> ids;
	for (u32 k = 0; k < ev.n; ++k) if (all || ev.filter[k] == F_none) ids.push_back(k);
	push_candidate_state();
	uint64_t pairs = 0;
	if (arb_annotate_tags(ctx, (uint32_t) ids.size(), ids.data(), max_mate_gap, &pairs) != 0) throw std::runtime_error("tags '" + opt.tags_file + "': " + arb_last_error(ctx));
	tag_off.assign((size_t) ev.n + 1, 0); tag_ranks.assign(pairs ? pairs : 1, 0);
	check(ctx, arb_get_tags(ctx, tag_off.data(), tag_ranks.data()), "arb_get_tags");
	tags_loaded = true;
}

// the tags column of candidate k (annotate_tags.cpp:72-82)
std::string pipeline::tags_of(u32 k) const {
	if (!tags_loaded || tag_off[k] == tag_off[k + 1]) return ".";
	std::string out;
	for (u32 x = tag_off[k]; x < tag_off[k + 1]; ++x) { if (x > tag_off[k]) out += ','; out += tag_names[tag_ranks[x]]; }
	return out;
}

// ------------------------------------------------------------------------------------------- protein domains (-p)
// load_protein_domains (annotate_protein_domains.cpp:33-121): the records go to the device, which keeps the reference's index as a table per gene and fills
// the retained_protein_domains column of the rows it formats (arb_format_discarded_rows) and, here, of the rows the host formats: those of fusions.tsv and,
// with -X, the discarded ones.
void pipeline::load_protein_domains() {
	say("Loading protein domains from '" + opt.protein_domains_file + "'");
	protein_domain_records r;
	read_protein_domains(opt.protein_domains_file, ref, r);
	std::vector<char> chars; std::vector<u32> off(1, 0);
	for (size_t x = 0; x < r.names.size(); ++x) { chars.insert(chars.end(), r.names[x].begin(), r.names[x].end()); off.push_back((u32) chars.size()); }
	chars.push_back(0);
	check(ctx, arb_set_protein_domains(ctx, (uint32_t) r.contig.size(), r.contig.data(), r.start.data(), r.end.data(), r.gene.data(), r.name_rank.data(),
	                                   (uint32_t) r.names.size(), chars.data(), off.data()), "arb_set_protein_domains");
	const bool fusions = !opt.output_file.empty(), extra = !opt.discarded_output_file.empty() && opt.print_extra_info_for_discarded_fusions;
	std::vector<u32> ids;
	for (u32 k = 0; k < ev.n; ++k) if (ev.filter[k] == F_none ? fusions : extra) ids.push_back(k);
	uint64_t bytes = 0;
	if (arb_retained_protein_domains(ctx, (uint32_t) ids.size(), ids.data(), &bytes) != 0)
		throw std::runtime_error("protein domains '" + opt.protein_domains_file + "': " + arb_last_error(ctx));
	std::vector<u64> text_off(ids.size() + 1);
	domain_text.assign(bytes + 1, 0);
	check(ctx, arb_get_retained_protein_domains(ctx, text_off.data(), domain_text.data()), "arb_get_retained_protein_domains");
	domain_off.assign((size_t) ev.n + 1, 0); // ids ascend: the texts lie in candidate order
	for (size_t x = 0; x < ids.size(); ++x) domain_off[ids[x] + 1] = text_off[x + 1] - text_off[x];
	for (u32 k = 0; k < ev.n; ++k) domain_off[k + 1] += domain_off[k];
	domains_loaded = true;
}

// the retained_protein_domains column of candidate k, as the device formatted it
std::string pipeline::domains_of(u32 k) const {
	if (!domains_loaded || domain_off[k] == domain_off[k + 1]) return ".";
	return std::string(domain_text.data() + domain_off[k], domain_off[k + 1] - domain_off[k]);
}

void pipeline::assign_confidence() { // filter_genomic_support.cpp:222-402
	// the candidates of every gene (only counted below, so their order does not matter): one CSR table instead of a vector per gene
	struct gene_list { const u32* p; size_t n; size_t size() const { return n; } u32 operator[](size_t x) const { return p[x]; } };
	std::vector<u32> by_gene_off(ref.genes.size() + 1, 0), by_gene_items(2 * (size_t) ev.n);
	{ // counting sort by gene on all threads: a histogram per slice of the table, offsets by (gene, slice), every slice fills its own places
		const size_t G = ref.genes.size();
		const int T = std::max(1, std::min(std::min(threads, 16), (int) (ev.n / 65536 + 1))); // a histogram of G counters per slice
		std::vector<std::vector<u32> > count(T, std::vector<u32>(G, 0));
		auto slice = [&](int t, u32& lo, u32& hi) { lo = (u32) ((u64) ev.n * t / T); hi = (u32) ((u64) ev.n * (t + 1) / T); };
		{ std::vector<std::thread> pool; for (int t = 0; t < T; ++t) pool.emplace_back([&, t]() { u32 lo, hi; slice(t, lo, hi); std::vector<u32>& c = count[t]; for (u32 k = lo; k < hi; ++k) { ++c[ev.gene1[k]]; ++c[ev.gene2[k]]; } }); for (size_t t = 0; t < pool.size(); ++t) pool[t].join(); }
		u32 at = 0;
		for (size_t g = 0; g < G; ++g) { by_gene_off[g] = at; for (int t = 0; t < T; ++t) { const u32 c = count[t][g]; count[t][g] = at; at += c; } }
		by_gene_off[G] = at;
		{ std::vector<std::thread> pool; for (int t = 0; t < T; ++t) pool.emplace_back([&, t]() { u32 lo, hi; slice(t, lo, hi); std::vector<u32>& c = count[t]; for (u32 k = lo; k < hi; ++k) { by_gene_items[c[ev.gene1[k]]++] = k; by_gene_items[c[ev.gene2[k]]++] = k; } }); for (size_t t = 0; t < pool.size(); ++t) pool[t].join(); }
	}
	auto by_gene = [&](u32 g) { gene_list l = {by_gene_items.data() + by_gene_off[g], by_gene_off[g + 1] - by_gene_off[g]}; return l; };
	enum { LOW = 0, MEDIUM = 1, HIGH = 2 };
	parallel_rows(threads, ev.n, [&](u32 k) {
		if (ev.filter[k] != F_none) { ev.confidence[k] = LOW; return; } // before the coverage is looked up: nearly all candidates are filtered by now
		const int cov1 = coverage.get_coverage(ev.contig1[k], ev.bp1[k], ev.dir1[k] == UPSTREAM ? DOWNSTREAM : UPSTREAM);
		const int cov2 = coverage.get_coverage(ev.contig2[k], ev.bp2[k], ev.dir2[k] == UPSTREAM ? DOWNSTREAM : UPSTREAM);
		const float coverage_fraction = ((float) (ev.n_list1(k) + ev.n_list2(k) + ev.n_listd(k))) / std::max(1, std::max(cov1, cov2));
		int conf = HIGH;
		const u32 s1 = ev.split_reads1[k], s2 = ev.split_reads2[k], d = ev.discordant_mates[k], sup = s1 + s2 + d;
		if (ev.evalue[k] > 0.3 || sup < 2) conf = LOW;
		else if (ev.is_read_through(k)) {
			conf = LOW;
			if (((s1 > 0 && s2 > 0) || (s1 > 0 && d > 0) || (s2 > 0 && d > 0)) && sup >= 10) conf = (s1 + s2 >= 10 && coverage_fraction > 0.07) ? HIGH : MEDIUM;
			else {
				unsigned int deletions = 0;
				for (int side = 0; side < 2; ++side) {
					const gene_list v = by_gene(side == 0 ? ev.gene1[k] : ev.gene2[k]);
					for (size_t x = 0; x < v.size(); ++x) {
						const u32 o = v[x];
						if (ev.filter[o] == F_none && ev.split_reads1[o] + ev.split_reads2[o] > 0 && ev.dir1[o] == DOWNSTREAM && ev.dir2[o] == UPSTREAM &&
						    ((ev.gene1[o] == ev.gene1[k] && ev.gene2[o] != ev.gene2[k]) || (ev.gene1[o] != ev.gene1[k] && ev.gene2[o] == ev.gene2[k])) &&
						    (ev.bp1[o] != ev.bp1[k] || ev.bp2[o] != ev.bp2[k]) && ev.bp2[o] > ev.bp1[k] && ev.bp1[o] < ev.bp2[k]) ++deletions;
					}
				}
				if (deletions >= 1) conf = MEDIUM;
			}
		} else if (overlaps_both(ev, ref, k) || ev.gene1[k] == ev.gene2[k]) {
			conf = LOW;
			if (s1 + s2 > 0) {
				if (!ev.exonic1(k) && !ev.exonic2(k)) conf = (s1 > 0 && s2 > 0) ? HIGH : MEDIUM;
				else if (!ev.exonic1(k) || !ev.exonic2(k)) conf = (s1 > 3 && s2 > 3) ? HIGH : MEDIUM;
			}
		}
		if (conf == LOW && ev.gene1[k] == ev.gene2[k] && ev.exonic1(k) && ev.exonic2(k) && !ev.spliced1(k) && !ev.spliced2(k) && ev.bp2[k] - ev.bp1[k] < 100 && s1 > 0 && s2 > 0 && s1 + s2 >= 10 &&
		    coverage_fraction > 0.15 && ev.dir1[k] == UPSTREAM && ev.dir2[k] == DOWNSTREAM) conf = MEDIUM;
		if (conf < HIGH && ev.spliced1(k) && ev.spliced2(k) && !ev.is_read_through(k) && ev.gene1[k] != ev.gene2[k]) {
			unsigned int n_spliced = 0;
			for (int side = 0; side < 2; ++side) {
				const gene_list v = by_gene(side == 0 ? ev.gene1[k] : ev.gene2[k]);
				for (size_t x = 0; x < v.size(); ++x) { const u32 o = v[x]; if (ev.gene1[o] == ev.gene1[k] && ev.gene2[o] == ev.gene2[k] && ev.spliced1(o) && ev.spliced2(o) && (std::abs(ev.bp1[o] - ev.bp1[k]) > 2 || std::abs(ev.bp2[o] - ev.bp2[k]) > 2)) ++n_spliced; }
			}
			if (n_spliced > 0) ++conf;
		}
		if (ev.gene1[k] != ev.gene2[k] && conf > LOW && !ev.spliced1(k) && !ev.spliced2(k)) --conf;
		if (s1 > 20 && s2 > 20 && sup > 60) conf = HIGH;
		if (conf > LOW) {
			if (s1 + s2 == 0 || s1 + d == 0 || s2 + d == 0) --conf;
			else if ((s1 + s2) * 20 < d) --conf;
			else if (ev.evalue[k] > 0.2 || coverage_fraction < 0.01) conf = MEDIUM;
		}
		if (conf < HIGH && ev.genomic_support(k)) { // a supporting structural variant (-d)
			const i32 g1 = ev.closest1[k], g2 = ev.closest2[k];
			if ((ev.evalue[k] < 0.3 && sup >= 2) || (ev.spliced1(k) && ev.spliced2(k) && ev.gene1[k] != ev.gene2[k]) || std::abs(ev.bp1[k] - g1) + std::abs(ev.bp2[k] - g2) < 20000 ||
			    ev.contig1[k] != ev.contig2[k] || (std::abs(ev.bp2[k] - ev.bp1[k]) > 1000000 && ev.gene1[k] != ev.gene2[k])) ++conf;
		}
		ev.confidence[k] = (u8) conf;
	});
	say("Assigning confidence scores to events");
}

}} // namespace

// tests only (tests/test_prims.py), not part of the public header: parallel_sort against std::sort on pseudo-random records with many equal keys;
// returns 0 when the two orders are identical (the comparison is total, so there is exactly one sorted order)
extern "C" int arb_selftest_host_sort(uint32_t n, int threads, uint32_t seed) {
	struct rec { uint32_t key, rank; };
	std::vector<rec> a(n);
	uint64_t x = seed * 2654435761ull + 1;
	for (uint32_t i = 0; i < n; ++i) { x = x * 6364136223846793005ull + 1442695040888963407ull; a[i].key = (uint32_t) (x >> 40) % (n / 4 + 1); a[i].rank = i; }
	std::vector<rec> b(a);
	auto less = [](const rec& p, const rec& q) { return p.key != q.key ? p.key < q.key : p.rank < q.rank; };
	arb::host::parallel_sort(a, less, threads);
	std::sort(b.begin(), b.end(), less);
	for (uint32_t i = 0; i < n; ++i) if (a[i].key != b[i].key || a[i].rank != b[i].rank) return 1;
	return 0;
}
