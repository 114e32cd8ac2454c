// domains_hd.h -- the protein domains of a GFF3 file (-p) as the device holds them, and the functors that build those tables.
//
// Behavioural contract: make_annotation_index (annotation.t.hpp:25-45) over the accepted records and annotate_retained_protein_domains
// (annotate_protein_domains.cpp:123-161). The index has a key at start - 1 and at end of every record on its contig; the set at key k holds every record d with
// d.start <= k <= d.end. A row side walks the keys inside its gene and counts every record of that gene once per key, so a record d of gene G counts
//   m(d) = |{keys k on d.contig : max(d.start, G.start) <= k <= min(d.end, G.end)}|
// times, whatever the breakpoint. m is computed once per record (sorted, distinct (contig, key) pairs and two binary searches); the records with m > 0 go into
// a table per gene, ordered by name rank, and a row side needs one walk over its gene's part of that table (row_formatter::domain_side, rows_hd.h).
// Only records of protein-coding genes are kept: annotate_retained_protein_domains returns nothing for the others.
#pragma once
#include "model.h"

namespace arb {

struct domain_view {
	const u32* gene_off;                 // n_genes + 1: the records of gene g at [gene_off[g], gene_off[g + 1]); NULL: no protein domains loaded
	const u16* contig; const i32* start; const i32* end; const u32* mult; const u32* name; // by (gene, name rank); mult = m(d) above
	const char* name_chars; const u32* name_off; // name k = name_chars[name_off[k], name_off[k + 1])
	u32 n_records;                       // accepted records: the size of the reference's index (a side on a contig >= n_records has none)
	u32* error;                          // set to 1 when a name's length sums to 0 (mod 2^32) while its retained bases do not
};

ARB_HD u64 domain_key(u32 contig, i32 key) { return (u64) contig << 32 | (u64) ((u32) key ^ 0x80000000u); } // (contig, signed key) in ascending order

// the two index keys of every record: biased key + contig, sorted by the caller (key first, then contig: both passes stable)
struct domain_keys_fn {
	const u16* contig; const i32* start; const i32* end; u32* key; u32* key_contig;
	ARB_HD void operator()(u32 i) const {
		key[2 * i] = (u32) ((i32) ((u32) start[i] - 1u)) ^ 0x80000000u; key[2 * i + 1] = (u32) end[i] ^ 0x80000000u;
		key_contig[2 * i] = key_contig[2 * i + 1] = contig[i];
	}
};
struct domain_distinct_fn { // flag[i] = 1 for the first of equal (contig, key) pairs
	const u32* key_contig; const u32* key; u32* flag;
	ARB_HD void operator()(u32 i) const { flag[i] = i == 0 || key_contig[i] != key_contig[i - 1] || key[i] != key[i - 1] ? 1u : 0u; }
};
struct domain_compact_keys_fn {
	const u32* key_contig; const u32* key; const u32* flag_scan; u64* out;
	ARB_HD void operator()(u32 i) const { if (flag_scan[i + 1] != flag_scan[i]) out[flag_scan[i]] = (u64) key_contig[i] << 32 | (u64) key[i]; }
};

ARB_HD u32 lower_bound_u64(const u64* a, u32 n, u64 v) { u32 lo = 0, hi = n; while (lo < hi) { const u32 mid = (lo + hi) / 2; if (a[mid] < v) lo = mid + 1; else hi = mid; } return lo; }

// m(d) for every record, and whether it is kept (m > 0 and a protein-coding gene)
struct domain_mult_fn {
	const u16* contig; const i32* start; const i32* end; const u32* gene; const i32* gene_start; const i32* gene_end; const u8* gene_flags;
	const u64* keys; u32 n_keys; u32* mult; u32* keep;
	ARB_HD void operator()(u32 i) const {
		const u32 g = gene[i];
		const i32 lo = start[i] > gene_start[g] ? start[i] : gene_start[g], hi = end[i] < gene_end[g] ? end[i] : gene_end[g];
		u32 m = 0;
		if (lo <= hi && (gene_flags[g] & GF_CODING)) m = lower_bound_u64(keys, n_keys, domain_key(contig[i], hi) + 1) - lower_bound_u64(keys, n_keys, domain_key(contig[i], lo));
		mult[i] = m; keep[i] = m != 0 ? 1u : 0u;
	}
};
struct domain_select_fn { // the kept records, in file order, with their name rank as the first sort key
	const u32* keep_scan; const u32* name_rank; u32* key; u32* idx;
	ARB_HD void operator()(u32 i) const { if (keep_scan[i + 1] != keep_scan[i]) { key[keep_scan[i]] = name_rank[i]; idx[keep_scan[i]] = i; } }
};
struct domain_gene_key_fn { const u32* gene; const u32* idx; u32* key; ARB_HD void operator()(u32 x) const { key[x] = gene[idx[x]]; } };
struct domain_gather_fn {
	const u32* idx; const u16* contig; const i32* start; const i32* end; const u32* mult; const u32* name_rank;
	u16* o_contig; i32* o_start; i32* o_end; u32* o_mult; u32* o_name;
	ARB_HD void operator()(u32 x) const { const u32 i = idx[x]; o_contig[x] = contig[i]; o_start[x] = start[i]; o_end[x] = end[i]; o_mult[x] = mult[i]; o_name[x] = name_rank[i]; }
};
struct domain_gene_off_fn { // gene_off[g] = first record of a gene >= g (records sorted by gene)
	const u32* gene_sorted; u32 n; u32* gene_off;
	ARB_HD void operator()(u32 g) const { u32 lo = 0, hi = n; while (lo < hi) { const u32 mid = (lo + hi) / 2; if (gene_sorted[mid] < g) lo = mid + 1; else hi = mid; } gene_off[g] = lo; }
};

} // namespace arb
