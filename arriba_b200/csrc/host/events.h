// events.h -- host image of the candidate table ("fusions") and the event-level stages that stay on the host.
//
// The reference keeps candidates in an unordered_map whose ITERATION ORDER several stages depend on
// (estimate_expected_fusions' first-come partner sets, select_best's tie rules, recover_isoforms' last-wins map,
// the unsorted discarded file; SURVEY.md section 7 "hard parts" 2b). The device numbers candidates by first insertion;
// replay_iteration_order() inserts the same keys, in that order, into a libstdc++ unordered_map with the reference's
// hash (common.hpp:295-314) and reads the iteration order back, so every host loop below visits candidates exactly
// like the reference does.
#pragma once
#include <string>
#include <vector>
#include "refdata.h"
#include "ingest.h"

namespace arb { namespace host {

struct event_table {
	u32 n;
	// column<T>: resize() does not touch new elements (they are all written by the device-to-host copies that follow)
	column<u32> gene1, gene2, split_reads1, split_reads2, discordant_mates;
	column<u16> contig1, contig2;
	column<i32> bp1, bp2, anchor1, anchor2;
	column<u8> dir1, dir2, filter, bits, bits2, confidence;
	column<float> evalue;
	column<u32> list1_off, list2_off, listd_off, list1, list2, listd; // CSR, fragment indices in name order
	std::vector<u32> order; // order[k] = candidate visited k-th by the reference's loops
	std::vector<u32> rank_of; // inverse of `order`
	std::vector<i32> closest1, closest2; // closest genomic breakpoints (-d), -1 = none; empty without -d
	event_table(): n(0) {}

	bool exonic1(u32 k) const { return bits[k] & CB_EXONIC1; }
	bool exonic2(u32 k) const { return bits[k] & CB_EXONIC2; }
	bool spliced1(u32 k) const { return bits[k] & CB_SPLICED1; }
	bool spliced2(u32 k) const { return bits[k] & CB_SPLICED2; }
	u32 supporting_reads(u32 k) const { return split_reads1[k] + split_reads2[k] + discordant_mates[k]; }
	u32 n_list1(u32 k) const { return list1_off[k + 1] - list1_off[k]; }
	u32 n_list2(u32 k) const { return list2_off[k + 1] - list2_off[k]; }
	u32 n_listd(u32 k) const { return listd_off[k + 1] - listd_off[k]; }
	bool is_read_through(u32 k) const { return contig1[k] == contig2[k] && bp2[k] - bp1[k] < 400000 && dir1[k] == DOWNSTREAM && dir2[k] == UPSTREAM; } // common.hpp:265-269
	bool genomic_support(u32 k) const { return !closest1.empty() && closest1[k] >= 0; }
};

// genomic breakpoints of a -d file (genomic_breakpoints.cpp), normalised so that (contig1, pos1) <= (contig2, pos2), in file order; directions 1 = upstream.
// Lines that are neither format print the reference's WARNING on stderr.
struct genomic_records { std::vector<u16> contig1, contig2; std::vector<u8> dir1, dir2; std::vector<i32> pos1, pos2; };
void read_genomic_breakpoints(const std::string& path, const std::map<std::string, u16>& contigs, genomic_records& out);

// rules of a blacklist file (blacklist.cpp), in file order: the two items of every line that parse_blacklist_item accepted, one column per field (type: ARB_RULE_*,
// strand: ARB_RULE_STRAND_*, coordinates 0-based; gene: the gene of a GENE item). Lines it rejects print the reference's WARNING on stderr. A file of known
// fusions (-k) and a tags file (-t) have the same format; a tags file adds the tag of every rule, sanitised.
struct fusion_rules {
	std::vector<u8> type1, type2, strand1, strand2; std::vector<u16> contig1, contig2; std::vector<i32> start1, end1, start2, end2; std::vector<u32> gene1, gene2;
	std::vector<std::string> tag;
	size_t size() const { return type1.size(); }
};
enum rule_file { RULES_BLACKLIST = 0, RULES_KNOWN_FUSIONS = 1, RULES_TAGS = 2 };
void read_fusion_rules(const std::string& path, const refdata& ref, rule_file kind, i32 max_mate_gap, fusion_rules& out);
void rank_tags(const fusion_rules& r, std::vector<std::string>& distinct, std::vector<u32>& rank);

// protein domains of a GFF3 file (protein_domains.cpp), the accepted records in file order: contig, 0-based start and end, gene, and the rank of the decoded
// name among the distinct names (bytewise order). Lines it rejects print the reference's WARNING on stderr; no accepted line, or a record the reference's index
// cannot hold (contig id >= number of records), stops the run.
struct protein_domain_records { std::vector<u16> contig; std::vector<i32> start, end; std::vector<u32> gene, name_rank; std::vector<std::string> names; };
void read_protein_domains(const std::string& path, const refdata& ref, protein_domain_records& out);

}} // namespace
