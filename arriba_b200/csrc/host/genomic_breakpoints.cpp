// genomic_breakpoints.cpp -- the file of genomic breakpoints from whole-genome sequencing (-d), read like mark_genomic_support does
// (filter_genomic_support.cpp:80-167): Arriba's four-column format or a VCF (BND in bracket notation, DEL / DUP / INV with END), one record per line.
// The records go to the device in file order (arb_set_genomic_breakpoints), which sorts them and searches them per candidate (csrc/genomic_hd.h).
#include <iostream>
#include "events.h"

namespace arb { namespace host {

// parse_breakpoint (:15-35): contig up to the LAST colon, without "chr", known to the run; position made 0-based
static bool parse_breakpoint(std::string bp, const std::map<std::string, u16>& contigs, u16& contig, i32& position) {
	const size_t colon = bp.find_last_of(':');
	if (colon < bp.size()) bp[colon] = '\t';
	tsv_fields f(bp);
	const std::map<std::string, u16>::const_iterator it = contigs.find(remove_chr(f.next()));
	if (it == contigs.end()) return false;
	contig = it->second;
	const std::string pos = f.next();
	if (f.failed || !str_to_int(pos, position)) return false;
	position = (i32) ((u32) position - 1u);
	return true;
}

static bool parse_direction(const std::string& s, u8& direction) { // :37-46
	if (s == "upstream" || s == "-") { direction = UPSTREAM; return true; }
	if (s == "downstream" || s == "+") { direction = DOWNSTREAM; return true; }
	return false;
}

static bool parse_vcf_info(const std::string& info, const std::string& field, std::string& value) { // :48-60
	size_t start;
	if (info.substr(0, field.size() + 1) == field + "=") start = field.size() + 1;
	else {
		start = info.find(";" + field + "=");
		if (start >= info.size()) return false;
		start += field.size() + 2;
	}
	value = info.substr(start, info.find(';', start) - start);
	return true;
}

void read_genomic_breakpoints(const std::string& path, const std::map<std::string, u16>& contigs, genomic_records& out) {
	std::string text;
	read_whole_file(path, text);
	out = genomic_records();
	auto add = [&](u16 c1, u16 c2, u8 d1, u8 d2, i32 p1, i32 p2) {
		out.contig1.push_back(c1); out.contig2.push_back(c2); out.dir1.push_back(d1); out.dir2.push_back(d2); out.pos1.push_back(p1); out.pos2.push_back(p2);
	};
	size_t at = 0; std::string line;
	while (next_line(text, at, line)) {
		if (line.empty() || line[0] == '#') continue;

		u16 c1 = 0, c2 = 0; i32 p1 = 0, p2 = 0; u8 d1 = 0, d2 = 0;
		std::string sv_type;
		tsv_fields f(line);
		const std::string bp1 = f.next(), bp2 = f.next(), dir1 = f.next(), dir2 = f.next();
		if (!(parse_breakpoint(bp1, contigs, c1, p1) && parse_breakpoint(bp2, contigs, c2, p2) && parse_direction(dir1, d1) && parse_direction(dir2, d2))) {
			// not the four-column format: VCF
			tsv_fields v(line);
			const std::string chrom = v.next(), pos = v.next(); v.next(); v.next();
			const std::string alt = v.next(); v.next();
			const std::string filter = v.next(), info = v.next();
			bool ok = parse_vcf_info(info, "SVTYPE", sv_type);
			std::string mate;
			if (ok && sv_type == "BND") {
				const size_t open = alt.find('['), close = alt.find(']');
				const char bracket = open < close ? '[' : ']';
				const size_t b1 = std::min(open, close), b2 = alt.find(bracket, b1 + 1);
				if (b1 >= alt.size() || b2 >= alt.size()) {
					if (!alt.empty() && (alt[0] == '.' || alt[alt.size() - 1] == '.')) continue; // single breakend: skipped silently
					ok = false;
				} else {
					d1 = b1 == 0 ? UPSTREAM : DOWNSTREAM;
					d2 = bracket == '[' ? UPSTREAM : DOWNSTREAM;
					mate = alt.substr(b1 + 1, b2 - b1 - 1);
				}
			} else if (ok) {
				std::string end;
				ok = parse_vcf_info(info, "END", end);
				mate = chrom + ":" + end;
				if (sv_type == "INV") { d1 = DOWNSTREAM; d2 = DOWNSTREAM; }
				else if (sv_type == "DEL") { d1 = DOWNSTREAM; d2 = UPSTREAM; }
				else if (sv_type == "DUP") { d1 = UPSTREAM; d2 = DOWNSTREAM; }
				else ok = false;
			}
			if (ok) ok = parse_breakpoint(chrom + ":" + pos, contigs, c1, p1) && parse_breakpoint(mate, contigs, c2, p2);
			if (!ok) { std::cerr << "WARNING: failed to parse line: " << line << std::endl; continue; }
			if (filter != "PASS") continue;
		}
		if (c2 < c1 || (c2 == c1 && p2 < p1)) { std::swap(c1, c2); std::swap(p1, p2); std::swap(d1, d2); } // index by the smaller coordinate
		add(c1, c2, d1, d2, p1, p2);
		if (sv_type == "INV") add(c1, c2, UPSTREAM, UPSTREAM, p1, p2); // an inversion is two breakpoint pairs
	}
}

}} // namespace
