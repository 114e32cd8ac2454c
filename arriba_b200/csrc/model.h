// model.h -- structure-of-arrays data model of the hot path (device-resident; views are POD and passed by value to kernels).
//
// Replaces the reference's pointer-based containers:
//   chimeric_alignments_t = std::map<string, mates_t>   (common.hpp:191-220)  -> frag_view  (fragments in NAME ORDER: index == name rank)
//   gene/exon annotation lists + interval indices        (common.hpp:108-181)  -> annot_view
//   fusions_t = unordered_map<tuple, fusion_t>            (common.hpp:237-286)  -> cand_view  (candidate table + CSR supporting lists)
#pragma once
#include "hd.h"

namespace arb {

// per-alignment flag bits (aflags)
enum { AF_SUPPLEMENTARY = 1, AF_FIRST_IN_PAIR = 2, AF_EXONIC = 4, AF_FORWARD = 8, AF_PRED_FORWARD = 16, AF_PRED_AMBIGUOUS = 32 };
// per-fragment flag bits (fflags)
enum { FF_SINGLE_END = 1, FF_MULTIMAPPER = 2, FF_DUPLICATE = 4, FF_SAME_NAME_AS_PREVIOUS = 8 /* same read name (up to the last comma) as the fragment before it */ };
// slot meaning after ingest normalisation (common.hpp:208-211)
enum { MATE1 = 0, MATE2 = 1, SPLIT_READ = 1, SUPPLEMENTARY = 2 };

struct frag_view {
	u32 n;               // fragments
	// per fragment
	u8* n_aln;           // 2 (discordant mates) or 3 (split read)
	u8* fflags;
	u8* filter;          // filter_id that discarded the fragment (F_none = kept)
	// per alignment slot: index = slot * n + fragment
	u16* contig;
	i32* start;          // 0-based
	i32* end;            // 0-based inclusive
	u8* aflags;
	u32* cigar_off;      // into cigar[]
	u16* cigar_cnt;
	u32* seq_off;        // slots 0,1 only; in units of 16 bytes into seq[]
	u16* seq_len;        // bases
	u32* genes_off;      // into genes[]
	u16* genes_cnt;
	// pools
	u32* cigar;          // BAM-encoded ops
	u8* seq;             // nt16, 4 bit per base, BAM nibble order, each sequence 16-byte aligned
	u32* genes;          // gene ids, each set sorted ascending by gene id (== creation order)

	ARB_HD u32 idx(u32 frag, u32 slot) const { return slot * n + frag; }
	ARB_HD bool fwd(u32 a) const { return aflags[a] & AF_FORWARD; }
	ARB_HD const u32* cig(u32 a) const { return cigar + cigar_off[a]; }
	ARB_HD const u8* sq(u32 a) const { return seq + (size_t) seq_off[a] * 16; }
	ARB_HD u32 preclip(u32 a) const { u32 c = cigar[cigar_off[a]]; return cig_is_clip(c) ? cig_len(c) : 0; }
	ARB_HD u32 postclip(u32 a) const { u32 c = cigar[cigar_off[a] + cigar_cnt[a] - 1]; return cig_is_clip(c) ? cig_len(c) : 0; }
};

struct annot_view {
	// genes (id == index)
	u32 n_genes;
	u16* gene_contig; i32* gene_start; i32* gene_end; u8* gene_strand /*1 = forward*/; i32* gene_exonic_length; u8* gene_flags; // bit0 dummy, bit1 protein coding
	// exons (index == creation order)
	u32 n_exons;
	u32* exon_gene; i32* exon_start; i32* exon_end; i32* exon_cds_start; i32* exon_cds_end; i32* exon_next_start; u8* exon_flags; // bit0 has previous exon, bit1 has next exon
	// disjoint-region interval indices (annotation.t.hpp:25-45 semantics): region r covers (end[r-1], end[r]] on its contig
	u32 n_contigs;
	u32* exon_region_begin;  // per contig, n_contigs+1
	i32* exon_region_end; u32* exon_region_off; u32* exon_region_items;   // items: exon ids ascending
	u32* gene_region_begin;
	i32* gene_region_end; u32* gene_region_off; u32* gene_region_items;   // items: gene ids ascending
	const u32* exon_grid; const u32* exon_grid_begin; const u32* gene_grid; const u32* gene_grid_begin; // host-side search accelerators (annot_hd.h region_find); 0 on the device
	// contig properties
	u8* contig_flags;        // bit0 interesting, bit1 viral
	u64* contig_seq_off;     // offset of the contig's sequence in assembly[]; 0 if the sequence is not loaded (then contig_len is 0)
	u32* contig_len;
	const char* assembly;    // upper-cased reference bases, 1 byte per base
	const u32* assembly4;    // the same bases as nt16 codes, 8 per word (first base in the top nibble), same base offsets; 0 if a character outside the nt16 alphabet occurs
};
enum { GF_DUMMY = 1, GF_CODING = 2, EF_HAS_PREV = 1, EF_HAS_NEXT = 2, CF_INTERESTING = 1, CF_VIRAL = 2,
       CF_VIRAL_LOW_EXPRESSION = 4, CF_VIRAL_FOCAL_COVERAGE = 8 }; // per-sample verdicts of the two viral-contig heuristics (host/viral.cpp)

enum { UPSTREAM = 1, DOWNSTREAM = 0 }; // direction_t (common.hpp:229-231)

// candidate table ("fusions"), one row per distinct (gene1,gene2,contig1,contig2,bp1,bp2,dir1,dir2)
struct cand_view {
	u32 n;
	u32* gene1; u32* gene2; u16* contig1; u16* contig2; i32* bp1; i32* bp2; u8* dir1; u8* dir2;
	u32* split_reads1; u32* split_reads2; u32* discordant_mates;
	u8* filter; u8* bits;       // bits: see CB_*
	i32* anchor1; i32* anchor2;
	float* evalue;
	u64* first_seen;            // (name rank << 16 | i_gene1 << 8 | i_gene2): order of first insertion in the reference's hash map
	// CSR lists of supporting fragments (name rank), each in name order
	u32* list1_off; u32* list2_off; u32* listd_off;
	u32* list1; u32* list2; u32* listd;
};
enum { CB_EXONIC1 = 1, CB_EXONIC2 = 2, CB_SPLICED1 = 4, CB_SPLICED2 = 8, CB_PSTRAND1 = 16, CB_PSTRAND2 = 32, CB_PSTRANDS_AMBIGUOUS = 64,
       CB_TSTART_GENE1 = 128 };

} // namespace arb
