// refdata.h -- host-side reference data: contig table, assembly, gene/exon annotation and the flattened interval indices
// that are uploaded to the device (model.h: annot_view).
//
// Behaviour follows the reference loaders: load_assembly (assembly.cpp:28-58), read_annotation_gtf (annotation.cpp:161-377),
// make_annotation_index (annotation.t.hpp:25-45), is_interesting_contig / removeChr (common.hpp:74-107),
// exonic length (arriba.cpp:166-184). Identity/ordering rule: the reference orders gene and exon sets by list-node address;
// here the order is creation order (GTF order, dummy genes last), which is what the oracle's deterministic allocator yields.
#pragma once
#include <map>
#include <string>
#include <vector>
#include "../model.h"

namespace arb { namespace host {

std::string remove_chr(std::string contig);
bool contig_matches(std::string contig, const std::string& patterns);

struct gene_rec {
	u16 contig; i32 start, end; bool forward; std::string gene_id, name; i32 exonic_length; bool is_dummy, is_protein_coding;
};
struct transcript_rec { u32 id; std::string name; i32 first_exon, last_exon; u32 coding_length; };
struct exon_rec {
	u16 contig; i32 start, end; bool forward; u32 gene; u32 transcript; i32 prev, next; i32 cds_start, cds_end;
};

struct region_index { // disjoint regions per contig; region r covers (end[r-1], end[r]]
	std::vector<u32> begin; std::vector<i32> end; std::vector<u32> off; std::vector<u32> items;
	std::vector<u32> grid, grid_begin; // annot_hd.h region_find
};

struct refdata {
	// contigs (id = order of first appearance: assembly, then GTF, then BAM header)
	std::map<std::string, u16> contig_ids;           // key: name without "chr"
	std::vector<std::string> original_names;
	std::vector<u64> seq_off; std::vector<u32> seq_len; // into assembly (seq_len 0 = not loaded)
	std::vector<char> assembly;                      // upper-cased, contigs 64-byte aligned
	std::vector<gene_rec> genes; std::vector<transcript_rec> transcripts; std::vector<exon_rec> exons;
	std::map<std::string, u32> gene_by_name;
	region_index exon_index, gene_index;
	std::vector<u8> contig_flags;

	u16 contig_id(const std::string& name_without_chr); // inserts if new
	bool has_sequence(u32 contig) const { return contig < seq_len.size() && seq_len[contig] > 0; }
	const char* sequence(u32 contig) const { return assembly.data() + seq_off[contig]; }

	void load_assembly(const std::string& fasta_path, const std::string& interesting_contigs);
	void load_gtf(const std::string& gtf_path);
	void build_exon_index();
	void build_gene_index();
	void compute_exonic_lengths();
	void set_contig_flags(const std::string& interesting, const std::string& viral);
	// flattened columns (rebuilt by flatten()); annot_view over host memory for host-side use of annot_hd.h
	std::vector<u16> f_gene_contig; std::vector<i32> f_gene_start, f_gene_end, f_gene_exonic_length; std::vector<u8> f_gene_strand, f_gene_flags;
	std::vector<u32> f_exon_gene; std::vector<i32> f_exon_start, f_exon_end, f_exon_cds_start, f_exon_cds_end, f_exon_next_start; std::vector<u8> f_exon_flags;
	std::vector<u64> f_seq_off;
	void flatten();
	annot_view host_view();
};

std::vector<std::string> read_lines_autodecompress(const std::string& path, std::string& storage);
void read_whole_file(const std::string& path, std::string& out);

// the line at `at` of a file read whole, without its '\n' and a trailing '\r' (autodecompress_file_t::getline, read_compressed_file.cpp:47-63); false at the end
bool next_line(const std::string& text, size_t& at, std::string& line);

// tsv_stream_t (read_compressed_file.cpp:65-89): fields split at every delimiter, a missing field fails
struct tsv_fields {
	const std::string& s; char delimiter; size_t at; bool failed;
	explicit tsv_fields(const std::string& line, char d = '\t'): s(line), delimiter(d), at(0), failed(false) {}
	std::string next() {
		if (at >= s.size()) { failed = true; return std::string(); }
		const size_t start = at; at = s.find(delimiter, start);
		std::string out = s.substr(start, at - start);
		if (at < s.size()) ++at;
		return out;
	}
};

// str_to_int (common.hpp:316-321): a long that fits is truncated to int
bool str_to_int(const std::string& text, i32& v);

}} // namespace
