// protein_domains.cpp -- the protein domains of a GFF3 file (-p), read like load_protein_domains does (annotate_protein_domains.cpp:14-121). The accepted
// records go to the device (arb_set_protein_domains), which builds the reference's index from them and fills the retained_protein_domains column (domains_hd.h).
#include <algorithm>
#include <iostream>
#include <set>
#include <stdexcept>
#include <unordered_map>
#include "events.h"

namespace arb { namespace host {

namespace {

std::string strip_ensembl_version_number(const std::string& id) { // annotation.hpp:27-33
	size_t dot;
	if (id.compare(0, 3, "ENS") == 0 && (dot = id.find_last_of('.')) < id.size()) return id.substr(0, dot);
	return id;
}

// get_gff3_attribute (:14-31): a plain substring search for "<name>=", the value up to the next ';'
bool gff3_attribute(const std::string& attributes, const std::string& name, std::string& value) {
	size_t start = attributes.find(name + "=");
	if (start >= attributes.size()) { std::cerr << "WARNING: failed to extract " << name << " from line in GFF3 file: " << attributes << std::endl; return false; }
	start += name.size() + 1;
	size_t end = attributes.find(';', start);
	if (end >= attributes.size()) end = attributes.size();
	value = attributes.substr(start, end - start);
	return true;
}

bool hex_digit(char c) { return (c >= '0' && c <= '9') || (c >= 'a' && c <= 'f') || (c >= 'A' && c <= 'F'); }
int hex_value(char c) { return c <= '9' ? c - '0' : c <= 'F' ? c - 'A' + 10 : c - 'a' + 10; }

// :71-89: "%XX" decoded where both X are hex digits (the next '%' is searched from pos + 1 of the decoded text), then every byte outside '!'..'~' (char is
// signed: bytes >= 0x80 too), ',' and '|' become '_'
void decode_name(std::string& name) {
	for (size_t pos = name.find('%'); pos < name.size(); pos = name.find('%', pos + 1))
		if (pos + 2 < name.size() && hex_digit(name[pos + 1]) && hex_digit(name[pos + 2]))
			name = name.substr(0, pos) + (char) (hex_value(name[pos + 1]) * 16 + hex_value(name[pos + 2])) + name.substr(pos + 3);
	for (size_t pos = 0; pos < name.size(); ++pos)
		if ((signed char) name[pos] < '!' || (signed char) name[pos] > '~' || name[pos] == ',' || name[pos] == '|') name[pos] = '_';
}

} // namespace

void read_protein_domains(const std::string& path, const refdata& ref, protein_domain_records& out) {
	out = protein_domain_records();
	std::unordered_map<std::string, u32> gene_by_id; // every gene in annotation order, dummy genes included (their ID is empty): the last one wins
	for (size_t g = 0; g < ref.genes.size(); ++g) gene_by_id[strip_ensembl_version_number(ref.genes[g].gene_id)] = (u32) g;
	std::string text;
	read_whole_file(path, text);
	std::set<std::string> unknown_genes;
	std::vector<std::string> names;
	std::vector<size_t> line_of;
	size_t at = 0, line_no = 0; std::string line;
	while (next_line(text, at, line)) {
		++line_no;
		if (line.empty() || line[0] == '#') continue;
		tsv_fields f(line);
		const std::string contig = f.next(); f.next(); f.next();
		i32 start = 0, end = 0;
		const bool start_ok = str_to_int(f.next(), start), end_ok = str_to_int(f.next(), end);
		f.next();
		const std::string strand = f.next(); f.next();
		const std::string attributes = f.next(); // further columns are ignored
		if (f.failed || !start_ok || !end_ok || contig.empty() || strand.empty() || attributes.empty()) { std::cerr << "WARNING: failed to parse line in GFF3 file: " << line << std::endl; continue; }
		std::string gene_name, gene_id, name;
		if (!gff3_attribute(attributes, "gene_name", gene_name) || !gff3_attribute(attributes, "gene_id", gene_id) || !gff3_attribute(attributes, "Name", name)) continue;
		const std::map<std::string, u16>::const_iterator c = ref.contig_ids.find(remove_chr(contig));
		if (c == ref.contig_ids.end()) { std::cerr << "WARNING: unknown contig: " << contig << std::endl; continue; }
		decode_name(name);
		u32 gene;
		const std::unordered_map<std::string, u32>::const_iterator by_id = gene_by_id.find(strip_ensembl_version_number(gene_id));
		if (by_id != gene_by_id.end()) gene = by_id->second;
		else {
			const std::map<std::string, u32>::const_iterator by_name = ref.gene_by_name.find(gene_name);
			if (by_name == ref.gene_by_name.end()) {
				if (unknown_genes.insert(gene_name + " " + gene_id).second) std::cerr << "WARNING: unknown gene: " << gene_name << " " << gene_id << std::endl;
				continue;
			}
			gene = by_name->second;
		}
		out.contig.push_back(c->second); out.start.push_back((i32) ((u32) start - 1u)); out.end.push_back((i32) ((u32) end - 1u)); out.gene.push_back(gene);
		names.push_back(name); line_of.push_back(line_no);
	}
	if (out.contig.empty()) throw std::runtime_error("failed to parse GFF3 file");
	// the reference's index has one entry per record, not per contig (annotation.t.hpp:26): a record on a contig whose id is not below the number of records is
	// written past its end
	for (size_t r = 0; r < out.contig.size(); ++r)
		if (out.contig[r] >= out.contig.size())
			throw std::runtime_error("protein domains '" + path + "', line " + std::to_string((unsigned long long) line_of[r]) + ": the contig (" + ref.original_names[out.contig[r]] +
			                         ") has an id that is not below the number of accepted records (" + std::to_string((unsigned long long) out.contig.size()) + "); the reference's index has no entry for it");
	out.names = names;
	std::sort(out.names.begin(), out.names.end());
	out.names.erase(std::unique(out.names.begin(), out.names.end()), out.names.end());
	out.name_rank.resize(names.size());
	for (size_t r = 0; r < names.size(); ++r) out.name_rank[r] = (u32) (std::lower_bound(out.names.begin(), out.names.end(), names[r]) - out.names.begin());
}

}} // namespace
