// rows_hd.h -- the rows of the discarded-fusions file, formatted on the device from resident columns.
//
// Behavioural contract: write_fusions_to_file (output_fusions.cpp:1043-1261) for rows WITHOUT transcript / peptide / read identifiers (the file written by
// -O unless -X is given): gene names (:498-545, dummy genes print their annotated neighbours with distances), strands, breakpoints, sites (:635-709), type
// (:547-633), supporting read counts, coverage, confidence, gene ids, directions, and the filters column (:1187-1213: the candidate's own filter and, with
// counts, the filters of its supporting reads, names in alphabetical order). The surviving fusions (fusions.tsv) additionally carry a consensus transcript
// assembled from read pileups and stay with the host (csrc/host/output.cpp).
// One thread per row, two runs of the same code: the first with a counting writer (row lengths -> exclusive scan -> offsets), the second writes the bytes.
#pragma once
#include "model.h"
#include "annot_hd.h"
#include "events_hd.h"
#include "domains_hd.h"

namespace arb {

struct text_pool { const char* chars; const u32* off; }; // string k = chars[off[k], off[k + 1])

struct row_tables { // what the rows need besides the candidate state, the fragment labels and the annotation
	text_pool gene_name, gene_id, contig_name, filter_name;
	const i32* exon_prev; const i32* exon_next;   // neighbours in the transcript (-1: none)
	const u8* confidence;                          // per candidate
	const i32* closest1; const i32* closest2;      // closest genomic breakpoints per candidate (-d), NULL: none marked
	coverage_view cov;
	text_pool tag_text; const u32* tag_off; const u32* tag_rank; // -t: distinct tags by rank, and the ranks of every candidate's tags (CSR); NULL: no tags
	domain_view domains;                           // -p: the protein domains per gene (domains_hd.h); gene_off NULL: none
	u8 filters_by_name[ARB_N_FILTERS];             // filter ids in alphabetical order of their names
	u32 max_itd_length;
};

struct count_writer { u32 n; ARB_HD void put(char) { ++n; } ARB_HD void write(const char*, u32 len) { n += len; } };
struct memory_writer { char* p; ARB_HD void put(char c) { *p++ = c; } ARB_HD void write(const char* s, u32 len) { for (u32 k = 0; k < len; ++k) p[k] = s[k]; p += len; } };
template <class W> ARB_HD void put_text(W& w, const char* s) { while (*s) w.put(*s++); }
template <class W> ARB_HD void put_pool(W& w, const text_pool& t, u32 k) { w.write(t.chars + t.off[k], t.off[k + 1] - t.off[k]); }
template <class W> ARB_HD void put_int(W& w, long long v) {
	char buf[24]; int n = 0;
	unsigned long long u = v < 0 ? 0ull - (unsigned long long) v : (unsigned long long) v;
	do { buf[n++] = (char) ('0' + (int) (u % 10)); u /= 10; } while (u);
	if (v < 0) w.put('-');
	while (n > 0) w.put(buf[--n]);
}

struct row_formatter {
	cand_state c; frag_view f; annot_view an; row_tables t;
	const u32* l1o; const u32* l1; const u32* l2o; const u32* l2; const u32* ldo; const u32* ld;

	ARB_HD bool dummy(u32 g) const { return an.gene_flags[g] & GF_DUMMY; }
	ARB_HD bool coding(u32 g) const { return an.gene_flags[g] & GF_CODING; }
	ARB_HD bool forward(u32 g) const { return an.gene_strand[g] != 0; }

	template <class W> ARB_HD void gene_name(W& w, u32 gene, u32 contig, i32 bp) const { // output_fusions.cpp:498-545
		if (!dummy(gene)) { put_pool(w, t.gene_name, gene); return; }
		const u32 lo = an.gene_region_begin[contig], hi = an.gene_region_begin[contig + 1];
		const u32 hit = region_lower_bound(an.gene_region_end, lo, hi, bp);
		bool any = false;
		i64 up = (i64) hit - 1;
		while (up >= (i64) lo && !annotated((u32) up)) --up;
		if (up >= (i64) lo) for (u32 x = an.gene_region_off[up]; x < an.gene_region_off[up + 1]; ++x) {
			const u32 g = an.gene_region_items[x];
			if (dummy(g)) continue;
			if (any) w.put(',');
			put_pool(w, t.gene_name, g); w.put('('); put_int(w, (long long) (bp - an.gene_end[g])); w.put(')'); any = true;
		}
		u32 down = hit;
		while (down < hi && !annotated(down)) ++down;
		if (down < hi) for (u32 x = an.gene_region_off[down]; x < an.gene_region_off[down + 1]; ++x) {
			const u32 g = an.gene_region_items[x];
			if (dummy(g)) continue;
			if (any) w.put(',');
			put_pool(w, t.gene_name, g); w.put('('); put_int(w, (long long) (an.gene_start[g] - bp)); w.put(')'); any = true;
		}
		if (!any) w.put('.');
	}
	ARB_HD bool annotated(u32 r) const { return an.gene_region_off[r + 1] > an.gene_region_off[r] && !dummy(an.gene_region_items[an.gene_region_off[r]]); }

	template <class W> ARB_HD void fusion_type(W& w, u32 k) const { // output_fusions.cpp:547-633
		const u32 g1 = c.gene1[k], g2 = c.gene2[k], d1 = c.dir1[k], d2 = c.dir2[k];
		const bool dm = dummy(g1) || dummy(g2), f1 = forward(g1), f2 = forward(g2);
		if (c.contig1[k] != c.contig2[k]) {
			if (dm || (d1 == d2 && f1 != f2) || (d1 != d2 && f1 == f2)) { put_text(w, "translocation"); return; }
			if (((d1 == UPSTREAM && f1) || (d1 == DOWNSTREAM && !f1)) && ((d2 == UPSTREAM && f2) || (d2 == DOWNSTREAM && !f2))) { put_text(w, "translocation/3'-3'"); return; }
			put_text(w, "translocation/5'-5'"); return;
		}
		const bool rt = c.bp2[k] - c.bp1[k] < 400000 && d1 == DOWNSTREAM && d2 == UPSTREAM; // is_read_through on one contig (common.hpp:265-269)
		if (d1 == DOWNSTREAM && d2 == UPSTREAM) {
			if (dm || f1 == f2) { put_text(w, rt ? "deletion/read-through" : "deletion"); return; }
			if (f1 || !f2) { put_text(w, rt ? "deletion/read-through/5'-5'" : "deletion/5'-5'"); return; }
			put_text(w, rt ? "deletion/read-through/3'-3'" : "deletion/3'-3'"); return;
		}
		if (d1 == d2) { if (dm || f1 != f2) { put_text(w, "inversion"); return; } put_text(w, (d1 == UPSTREAM && !f1) ? "inversion/5'-5'" : "inversion/3'-3'"); return; }
		if (dm || f1 == f2) {
			const u8 bits = c.bits[k];
			if (g1 == g2 && (bits & CB_SPLICED1) && (bits & CB_SPLICED2)) { put_text(w, "duplication/non-canonical_splicing"); return; }
			if (g1 == g2 && ((u32) c.bp2[k] - (u32) c.bp1[k]) < t.max_itd_length && d1 == UPSTREAM && d2 == DOWNSTREAM) { put_text(w, "duplication/ITD"); return; }
			put_text(w, "duplication"); return;
		}
		put_text(w, !f1 ? "duplication/5'-5'" : "duplication/3'-3'");
	}

	template <class W> ARB_HD void genomic_breakpoint(W& w, u32 contig, i32 bp, i32 genomic) const { // output_fusions.cpp:1195-1205
		if (genomic < 0) { w.put('.'); return; }
		put_pool(w, t.contig_name, contig); w.put(':'); put_int(w, (long long) genomic + 1); w.put('(');
		put_int(w, bp < genomic ? (long long) genomic - bp : (long long) bp - genomic); w.put(')');
	}
	template <class W> ARB_HD void strand_column(W& w, bool strand, u32 gene, bool ambiguous) const { w.put(dummy(gene) ? '.' : (forward(gene) ? '+' : '-')); w.put('/'); w.put(ambiguous ? '.' : (strand ? '+' : '-')); }

	// 0 intergenic, 1 intron, 2 3'UTR, 3 5'UTR, 4 exon, 5 UTR, 6 CDS; bit 3: + "/splice-site"   (output_fusions.cpp:635-709)
	ARB_HD u32 site(u32 gene, bool spliced, bool exonic, u32 contig, i32 bp) const {
		if (dummy(gene) || bp < an.gene_start[gene] || bp > an.gene_end[gene]) return 0;
		if (!exonic) return 1;
		bool overlapping = false, utr = true; u32 end3 = 0, end5 = 0;
		const bool fwd = forward(gene), pc = coding(gene);
		if (contig < an.n_contigs) {
			const u32 lo = an.exon_region_begin[contig], hi = an.exon_region_begin[contig + 1];
			const u32 r = region_lower_bound(an.exon_region_end, lo, hi, bp);
			if (r < hi) for (u32 x = an.exon_region_off[r]; x < an.exon_region_off[r + 1]; ++x) {
				const u32 e = an.exon_region_items[x];
				if (an.exon_gene[e] != gene) continue;
				overlapping = true;
				const i32 cs = an.exon_cds_start[e], ce = an.exon_cds_end[e];
				if (cs <= bp && ce >= bp) utr = false;
				if (utr && pc) {
					if (cs != -1 && cs > bp) { if (fwd) ++end5; else ++end3; }
					else if (ce != -1 && ce < bp) { if (!fwd) ++end5; else ++end3; }
					else {
						i32 nx = t.exon_next[e]; while (nx >= 0 && an.exon_cds_start[nx] == -1) nx = t.exon_next[nx];
						i32 pv = t.exon_prev[e]; while (pv >= 0 && an.exon_cds_start[pv] == -1) pv = t.exon_prev[pv];
						if (pv >= 0 || nx >= 0) { if ((nx < 0) != (!fwd)) ++end3; else ++end5; }
					}
				}
			}
		}
		u32 s;
		if (!overlapping) s = 1;
		else if (pc) { if (utr) s = end3 > end5 ? 2u : end3 < end5 ? 3u : end3 + end5 == 0 ? 4u : 5u; else s = 6; }
		else s = 4;
		if (spliced && s != 1) s |= 8u;
		return s;
	}
	template <class W> ARB_HD void put_site(W& w, u32 s) const {
		switch (s & 7u) { case 0: put_text(w, "intergenic"); break; case 1: put_text(w, "intron"); break; case 2: put_text(w, "3'UTR"); break; case 3: put_text(w, "5'UTR"); break;
		                  case 4: put_text(w, "exon"); break; case 5: put_text(w, "UTR"); break; default: put_text(w, "CDS"); break; }
		if (s & 8u) put_text(w, "/splice-site");
	}

	ARB_HD void tally(const u32* off, const u32* list, u32 k, u32* count, u64& present) const {
		for (u32 p = off[k]; p < off[k + 1]; ++p) { const u8 l = f.filter[list[p]]; if (l != F_none && l < ARB_N_FILTERS) { present |= (u64) 1 << l; ++count[l]; } }
	}

	template <class W> ARB_HD void tags(W& w, u32 k) const { // annotate_tags.cpp:72-82: the distinct tags joined by ',', in bytewise order
		if (!t.tag_off || t.tag_off[k] == t.tag_off[k + 1]) { w.put('.'); return; }
		for (u32 x = t.tag_off[k]; x < t.tag_off[k + 1]; ++x) { if (x > t.tag_off[k]) w.put(','); put_pool(w, t.tag_text, t.tag_rank[x]); }
	}

	// annotate_retained_protein_domains (annotate_protein_domains.cpp:123-161) for one side: its gene's records on its contig, per name (bytewise order) the
	// lengths and the retained bases, each record counted mult times; "name(P%)" for every name with retained bases, joined by ','. Sums wrap like unsigned int.
	template <class W> ARB_HD void domain_side(W& w, u32 gene, u32 contig, i32 bp, u32 dir, bool strand, bool ambiguous) const {
		const domain_view& d = t.domains;
		if (!coding(gene) || ambiguous || strand != forward(gene) || contig >= d.n_records) return;
		bool any = false;
		for (u32 x = d.gene_off[gene], last = d.gene_off[gene + 1]; x < last; ) {
			const u32 name = d.name[x]; u32 length = 0, retained = 0;
			for (; x < last && d.name[x] == name; ++x) {
				if (d.contig[x] != contig) continue;
				const i32 s = d.start[x], e = d.end[x]; const u32 m = d.mult[x];
				u32 r = 0;
				if (dir == UPSTREAM && e >= bp) r = (u32) e - (u32) (s > bp ? s : bp) + 1u;
				else if (dir == DOWNSTREAM && s <= bp) r = (u32) (e < bp ? e : bp) - (u32) s + 1u;
				length += m * ((u32) e - (u32) s + 1u); retained += m * r;
			}
			if (retained == 0) continue;
			if (length == 0 && d.error) *d.error = 1u; // the reference divides by zero; the caller stops the run
			if (any) w.put(',');
			put_pool(w, text_pool{d.name_chars, d.name_off}, name); w.put('('); put_int(w, (long long) (length ? retained * 100u / length : 0u)); w.put('%'); w.put(')');
			any = true;
		}
	}
	// the retained_protein_domains column of candidate k (output_fusions.cpp:1183-1190): "p5|p3" if a side has any, else "."
	template <class W> ARB_HD void retained_protein_domains(W& w, u32 k) const {
		if (!t.domains.gene_off) { w.put('.'); return; }
		const u8 bits = c.bits[k];
		const bool ambiguous = bits & CB_PSTRANDS_AMBIGUOUS, first = bits & CB_TSTART_GENE1;
		const u32 g5 = first ? c.gene1[k] : c.gene2[k], g3 = first ? c.gene2[k] : c.gene1[k], c5 = first ? c.contig1[k] : c.contig2[k], c3 = first ? c.contig2[k] : c.contig1[k];
		const u32 d5 = first ? c.dir1[k] : c.dir2[k], d3 = first ? c.dir2[k] : c.dir1[k];
		const i32 b5 = first ? c.bp1[k] : c.bp2[k], b3 = first ? c.bp2[k] : c.bp1[k];
		const bool st1 = bits & CB_PSTRAND1, st2 = bits & CB_PSTRAND2, st5 = first ? st1 : st2, st3 = first ? st2 : st1;
		count_writer n5 = {0}, n3 = {0};
		domain_side(n5, g5, c5, b5, d5, st5, ambiguous); domain_side(n3, g3, c3, b3, d3, st3, ambiguous);
		if (n5.n + n3.n == 0) { w.put('.'); return; }
		both_sides(w, n5.n + n3.n + 1, g5, c5, b5, d5, st5, g3, c3, b3, d3, st3, ambiguous);
	}
	template <class W> ARB_HD void both_sides(W& w, u32, u32 g5, u32 c5, i32 b5, u32 d5, bool st5, u32 g3, u32 c3, i32 b3, u32 d3, bool st3, bool ambiguous) const {
		domain_side(w, g5, c5, b5, d5, st5, ambiguous); w.put('|'); domain_side(w, g3, c3, b3, d3, st3, ambiguous);
	}
	ARB_HD void both_sides(count_writer& w, u32 n, u32, u32, i32, u32, bool, u32, u32, i32, u32, bool, bool) const { w.n += n; } // the length is known already

	template <class W> ARB_HD void row(W& w, u32 k) const {
		const u8 bits = c.bits[k];
		u32 site5 = site(c.gene1[k], bits & CB_SPLICED1, bits & CB_EXONIC1, c.contig1[k], c.bp1[k]), site3 = site(c.gene2[k], bits & CB_SPLICED2, bits & CB_EXONIC2, c.contig2[k], c.bp2[k]);
		u32 g5 = c.gene1[k], g3 = c.gene2[k], c5 = c.contig1[k], c3 = c.contig2[k], d5 = c.dir1[k], d3 = c.dir2[k], s5 = c.split_reads1[k], s3 = c.split_reads2[k];
		i32 b5 = c.bp1[k], b3 = c.bp2[k]; bool st5 = bits & CB_PSTRAND1, st3 = bits & CB_PSTRAND2;
		i32 gb5 = t.closest1 ? t.closest1[k] : -1, gb3 = t.closest2 ? t.closest2[k] : -1;
		const bool ambiguous = bits & CB_PSTRANDS_AMBIGUOUS;
		if (!(bits & CB_TSTART_GENE1)) { u32 x = g5; g5 = g3; g3 = x; x = c5; c5 = c3; c3 = x; x = d5; d5 = d3; d3 = x; x = s5; s5 = s3; s3 = x; i32 y = b5; b5 = b3; b3 = y; const bool z = st5; st5 = st3; st3 = z; x = site5; site5 = site3; site3 = x; y = gb5; gb5 = gb3; gb3 = y; }
		const int cov5 = t.cov.get(c5, b5, d5 == UPSTREAM ? DOWNSTREAM : UPSTREAM), cov3 = t.cov.get(c3, b3, d3 == UPSTREAM ? DOWNSTREAM : UPSTREAM);
		gene_name(w, g5, c5, b5); w.put('\t'); gene_name(w, g3, c3, b3); w.put('\t'); strand_column(w, st5, g5, ambiguous); w.put('\t'); strand_column(w, st3, g3, ambiguous); w.put('\t');
		put_pool(w, t.contig_name, c5); w.put(':'); put_int(w, (long long) b5 + 1); w.put('\t'); put_pool(w, t.contig_name, c3); w.put(':'); put_int(w, (long long) b3 + 1); w.put('\t');
		put_site(w, site5); w.put('\t'); put_site(w, site3); w.put('\t'); fusion_type(w, k); w.put('\t');
		put_int(w, s5); w.put('\t'); put_int(w, s3); w.put('\t'); put_int(w, c.discordant_mates[k]); w.put('\t');
		if (cov5 >= 0) put_int(w, cov5); else w.put('.');
		w.put('\t');
		if (cov3 >= 0) put_int(w, cov3); else w.put('.');
		w.put('\t');
		switch (t.confidence[k] & 3) { case 0: put_text(w, "low"); break; case 1: put_text(w, "medium"); break; default: put_text(w, "high"); break; }
		put_text(w, "\t.\t"); // reading frame
		tags(w, k);
		w.put('\t');
		retained_protein_domains(w, k);
		w.put('\t');
		genomic_breakpoint(w, c5, b5, gb5); w.put('\t'); genomic_breakpoint(w, c3, b3, gb3);
		u32 count[ARB_N_FILTERS]; u64 present = 0;
		for (u32 x = 0; x < ARB_N_FILTERS; ++x) count[x] = 0;
		if (c.filter[k] != F_none) present |= (u64) 1 << c.filter[k];
		tally(l1o, l1, k, count, present); tally(l2o, l2, k, count, present); tally(ldo, ld, k, count, present);
		w.put('\t');
		if (dummy(g5)) w.put('.'); else put_pool(w, t.gene_id, g5);
		w.put('\t');
		if (dummy(g3)) w.put('.'); else put_pool(w, t.gene_id, g3);
		put_text(w, "\t.\t.\t"); // transcript ids
		put_text(w, d5 == UPSTREAM ? "upstream" : "downstream"); w.put('\t'); put_text(w, d3 == UPSTREAM ? "upstream" : "downstream"); w.put('\t');
		bool any = false;
		for (u32 x = 0; x < ARB_N_FILTERS; ++x) {
			const u32 fl = t.filters_by_name[x];
			if (fl == F_none || !(present >> fl & 1)) continue;
			if (any) w.put(',');
			put_pool(w, t.filter_name, fl);
			if (count[fl] != 0) { w.put('('); put_int(w, count[fl]); w.put(')'); }
			any = true;
		}
		if (!any) w.put('.');
		put_text(w, "\t.\t.\t.\n"); // fusion transcript, peptide sequence, read identifiers
	}
};

struct row_select_fn { const u32* order; const u8* filter; u32* flag; ARB_HD void operator()(u32 q) const { flag[q] = filter[order[q]] != F_none ? 1u : 0u; } };
struct row_gather_fn { const u32* order; const u32* flag_scan; u32* rows; ARB_HD void operator()(u32 q) const { if (flag_scan[q + 1] != flag_scan[q]) rows[flag_scan[q]] = order[q]; } };
struct row_length_fn { row_formatter fm; const u32* rows; u32* length; ARB_HD void operator()(u32 x) const { count_writer w = {0}; fm.row(w, rows[x]); length[x] = w.n; } };
// rows are written in blocks of a few million (a 10 M-fragment sample already has 0.8 GB of discarded rows: 32-bit offsets only inside a block)
struct row_write_fn { row_formatter fm; const u32* rows; const u32* offset; char* text; ARB_HD void operator()(u32 x) const { memory_writer w = {text + offset[x]}; fm.row(w, rows[x]); } };
// the retained_protein_domains column alone, for the rows the host formats (arb_retained_protein_domains)
struct domain_length_fn { row_formatter fm; const u32* ids; u32* length; ARB_HD void operator()(u32 x) const { count_writer w = {0}; fm.retained_protein_domains(w, ids[x]); length[x] = w.n; } };
struct domain_write_fn { row_formatter fm; const u32* ids; const u64* offset; char* text; ARB_HD void operator()(u32 x) const { memory_writer w = {text + offset[x]}; fm.retained_protein_domains(w, ids[x]); } };

} // namespace arb
