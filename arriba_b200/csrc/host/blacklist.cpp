// blacklist.cpp -- the rules of a blacklist file (-b), read like filter_blacklisted_ranges does (filter_blacklisted_ranges.cpp:17-120, :252-268): two columns
// per line, each a gene name, a position or a range (contig:start-end, optionally with a strand prefix and a trailing '*' on the contig), or in column 2 a keyword.
// Files of known fusions (-k, recover_known_fusions.cpp:21-38) and tags (-t, annotate_tags.cpp:11-43) have the same two columns without keywords; a tags
// file has a third column, the tag.
// The rules go to the device in file order (arb_set_blacklist / arb_set_known_fusions / arb_set_tags), which matches them to the candidates (csrc/blacklist_hd.h).
#include <algorithm>
#include <climits>
#include <iostream>
#include <stdexcept>
#include "events.h"
#include "../../../include/arriba_b200.h"

namespace arb { namespace host {

namespace {

struct rule_item { u8 type, strand; u16 contig; i32 start, end; u32 gene; };

struct rule_reader {
	const refdata& ref; const std::string& path; const char* kind; size_t line_no; const std::string* line;

	[[noreturn]] void undefined(const std::string& why) const {
		throw std::runtime_error(std::string(kind) + " '" + path + "', line " + std::to_string((unsigned long long) line_no) + ": " + why + ": " + *line);
	}

	// parse_range (:17-80); every failure but an unmatched wildcard prints the same warning, with the text as the reference holds it by then (last ':' a tab)
	bool parse_range(std::string range, rule_item& item) const {
		const size_t colon = range.find_last_of(':');
		if (colon < range.size()) range[colon] = '\t';
		tsv_fields f(range);
		std::string contig_name = f.next(); const std::string position = f.next();
		if (f.failed || contig_name.empty() || position.empty()) { std::cerr << "WARNING: unknown gene or malformed range: " << range << std::endl; return false; }
		item.strand = ARB_RULE_STRAND_NONE;
		if (contig_name[0] == '+') { item.strand = ARB_RULE_STRAND_FORWARD; contig_name = contig_name.substr(1); }
		else if (contig_name[0] == '-') { item.strand = ARB_RULE_STRAND_REVERSE; contig_name = contig_name.substr(1); }
		contig_name = remove_chr(contig_name);
		std::map<std::string, u16>::const_iterator contig;
		if (contig_name.size() >= 2 && contig_name[contig_name.size() - 1] == '*') { // the first contig at or after the prefix, if the prefix matches it
			contig_name.resize(contig_name.size() - 1);
			contig = ref.contig_ids.lower_bound(contig_name);
			if (contig == ref.contig_ids.end()) undefined("the contig prefix '" + contig_name + "*' sorts after every contig name"); // the reference dereferences end()
			if (contig->first.compare(0, contig_name.size(), contig_name) != 0) return false; // silently
		} else {
			contig = ref.contig_ids.find(contig_name);
			if (contig == ref.contig_ids.end()) { std::cerr << "WARNING: unknown gene or malformed range: " << range << std::endl; return false; }
		}
		item.contig = contig->second;
		tsv_fields p(position, '-');
		bool ok;
		if (position.find('-') < position.size()) {
			const std::string a = p.next(), b = p.next();
			ok = str_to_int(a, item.start); ok = str_to_int(b, item.end) && ok && !p.failed;
			item.end = (i32) ((u32) item.end - 1u);
		} else {
			ok = str_to_int(p.next(), item.start);
			item.end = (i32) ((u32) item.start - 1u);
		}
		item.start = (i32) ((u32) item.start - 1u); // 0-based
		if (!ok) { std::cerr << "WARNING: unknown gene or malformed range: " << range << std::endl; return false; }
		return true;
	}

	// parse_blacklist_item (:83-120)
	bool parse_item(const std::string& text, rule_item& item, bool allow_keyword) const {
		item.type = ARB_RULE_ANY; item.strand = ARB_RULE_STRAND_NONE; item.contig = 0; item.start = item.end = 0; item.gene = 0;
		if (text.empty()) { std::cerr << "WARNING: encountered a line with an empty column => skipped" << std::endl; return false; }
		if (allow_keyword) {
			static const char* KEYWORDS[] = {"any", "split_read_donor", "split_read_acceptor", "split_read_any", "discordant_mates", "read_through", "low_support", "filter_spliced", "not_both_spliced"};
			for (u8 k = 0; k < 9; ++k) if (text == KEYWORDS[k]) { item.type = (u8) (ARB_RULE_ANY + k); return true; }
		}
		const std::map<std::string, u32>::const_iterator gene = ref.gene_by_name.find(text); // the last gene of a name (annotation.cpp:373-375)
		if (gene != ref.gene_by_name.end()) {
			const gene_rec& g = ref.genes[gene->second];
			item.type = ARB_RULE_GENE; item.gene = gene->second; item.contig = g.contig; item.start = g.start; item.end = g.end;
			return true;
		}
		if (!parse_range(text, item)) return false;
		item.type = item.start == item.end ? ARB_RULE_POSITION : ARB_RULE_RANGE;
		return true;
	}

	// the bins of a positional item (:272-275) must be computable in int: start - widen and end + widen + 99999 (get_genome_bins_from_range)
	void check_bins(const rule_item& item, i32 widen) const {
		if (item.type != ARB_RULE_POSITION && item.type != ARB_RULE_RANGE && item.type != ARB_RULE_GENE) return;
		if ((i64) item.start - widen < INT_MIN || (i64) item.end + widen + 99999 > INT_MAX) {
			if (widen) undefined("the coordinates widened by the maximum mate gap (" + std::to_string(widen) + ") overflow int");
			undefined("the coordinates overflow int");
		}
	}
};

} // namespace

// kind BLACKLIST: keywords in column 2, bins widened by max_mate_gap (filter_blacklisted_ranges.cpp:252-275); KNOWN_FUSIONS: no keywords, bins not widened
// (recover_known_fusions.cpp:23-37); TAGS: the same plus the third column, checked before the items and sanitised (annotate_tags.cpp:14-33)
void read_fusion_rules(const std::string& path, const refdata& ref, rule_file kind, i32 max_mate_gap, fusion_rules& out) {
	static const char* KIND[] = {"blacklist", "known fusions", "tags"};
	std::string text;
	read_whole_file(path, text);
	out = fusion_rules();
	rule_reader r = {ref, path, KIND[kind], 0, NULL};
	const i32 widen = kind == RULES_BLACKLIST ? max_mate_gap : 0;
	size_t at = 0; std::string line;
	while (next_line(text, at, line)) {
		++r.line_no; r.line = &line;
		if (line.empty() || line[0] == '#') continue;
		tsv_fields f(line);
		const std::string range1 = f.next(), range2 = f.next(); // further columns are ignored
		std::string tag;
		if (kind == RULES_TAGS) {
			tag = f.next();
			if (tag.empty()) { std::cerr << "WARNING: encountered a line with an empty tag => skipped" << std::endl; continue; }
		}
		rule_item a, b;
		if (!r.parse_item(range1, a, false) || !r.parse_item(range2, b, kind == RULES_BLACKLIST)) continue; // column 2 is parsed only if column 1 was
		r.check_bins(a, widen); r.check_bins(b, widen);
		out.type1.push_back(a.type); out.type2.push_back(b.type); out.strand1.push_back(a.strand); out.strand2.push_back(b.strand);
		out.contig1.push_back(a.contig); out.contig2.push_back(b.contig); out.start1.push_back(a.start); out.end1.push_back(a.end);
		out.start2.push_back(b.start); out.end2.push_back(b.end); out.gene1.push_back(a.gene); out.gene2.push_back(b.gene);
		if (kind == RULES_TAGS) {
			for (size_t x = 0; x < tag.size(); ++x) if ((signed char) tag[x] < '!' || (signed char) tag[x] > '~' || tag[x] == ',') tag[x] = '_'; // char is signed: bytes >= 0x80 too
			out.tag.push_back(tag);
		}
	}
}

// the distinct tags in bytewise order (std::set<std::string>, annotate_tags.cpp:55) and the rank of every rule's tag among them
void rank_tags(const fusion_rules& r, std::vector<std::string>& distinct, std::vector<u32>& rank) {
	distinct = r.tag;
	std::sort(distinct.begin(), distinct.end());
	distinct.erase(std::unique(distinct.begin(), distinct.end()), distinct.end());
	rank.resize(r.tag.size());
	for (size_t k = 0; k < r.tag.size(); ++k) rank[k] = (u32) (std::lower_bound(distinct.begin(), distinct.end(), r.tag[k]) - distinct.begin());
}

}} // namespace
