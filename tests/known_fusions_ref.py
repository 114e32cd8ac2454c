"""Plain reference of known fusions (-k) and tags (-t): a literal Python transcription of recover_known_fusions (recover_known_fusions.cpp:14-100) and of
load_tags / annotate_tags (annotate_tags.cpp), on top of the item parser and item test of blacklist_ref.py. Shares no code with the product."""
import gzip
from blacklist_ref import parse_item, matches, _bins, _tsv, POSITION, RANGE, GENE

F_RELATIVE_SUPPORT, F_MIN_SUPPORT = 12, 17
CB_SPLICED1, CB_SPLICED2, CB_TSTART_GENE1 = 4, 8, 128
UPSTREAM, DOWNSTREAM = 1, 0


def read_rules(path, contigs, gene_by_name, gene_contig, gene_start, gene_end, tags=False):
    """Returns (list of (item1, item2, tag) in file order, warning lines). Items parsed without keywords; with tags, the empty-tag check comes first."""
    raw = gzip.open(path, "rb").read() if path.endswith(".gz") else open(path, "rb").read()
    lines = raw.decode("latin-1").split("\n")
    if lines and lines[-1] == "":
        lines.pop()
    sorted_names = sorted(contigs)
    rules, warnings = [], []
    for line in lines:
        if line.endswith("\r"):
            line = line[:-1]
        if not line or line[0] == "#":
            continue
        f = _tsv(line) + ["", "", ""]
        tag = None
        if tags:
            tag = f[2]
            if tag == "":
                warnings.append("WARNING: encountered a line with an empty tag => skipped"); continue
        a = parse_item(f[0], False, contigs, sorted_names, gene_by_name, gene_contig, gene_start, gene_end, warnings)
        if a is None:
            continue
        b = parse_item(f[1], False, contigs, sorted_names, gene_by_name, gene_contig, gene_start, gene_end, warnings)
        if b is None:
            continue
        if tags:  # char is signed: every byte >= 0x80 is below '!'
            tag = "".join("_" if ord(ch) < 0x21 or ord(ch) > 0x7E or ch == "," else ch for ch in tag)
        rules.append((a, b, tag))
    return rules, warnings


def _index(rules):
    """rules by bin of their items, NOT widened by max_mate_gap"""
    index = {}
    for r in rules:
        for bn in _bins(r[0]["contig"], r[0]["start"], r[0]["end"]) + _bins(r[1]["contig"], r[1]["start"], r[1]["end"]):
            index.setdefault(bn, []).append(r)
    return index


def _cand_bins(c, k, gene_start, gene_end):
    return (_bins(int(c["contig1"][k]), int(c["breakpoint1"][k]), int(c["breakpoint1"][k])) + _bins(int(c["contig2"][k]), int(c["breakpoint2"][k]), int(c["breakpoint2"][k]))
            + _bins(int(c["contig1"][k]), int(gene_start[c["gene1"][k]]), int(gene_end[c["gene1"][k]]))
            + _bins(int(c["contig2"][k]), int(gene_start[c["gene2"][k]]), int(gene_end[c["gene2"][k]])))


def coverage_get(windows, contig, position, direction):
    """coverage_t::get_coverage (read_stats.cpp:295-306); windows: list of per-contig arrays of 20 bp windows"""
    if contig >= len(windows) or len(windows[contig]) == 0:
        return -1
    if direction == UPSTREAM:
        return 0 if position < 20 else int(windows[contig][position // 20 - 1])
    return int(windows[contig][position // 20 + 1])


def _both_spliced(c, k, gene_strand):
    bits = int(c["bits"][k])
    s1, s2 = int(gene_strand[c["gene1"][k]]), int(gene_strand[c["gene2"][k]])
    d1, d2 = int(c["direction1"][k]), int(c["direction2"][k])
    return bool(bits & CB_SPLICED1) and bool(bits & CB_SPLICED2) and ((s1 == s2 and d1 != d2) or (s1 != s2 and d1 == d2))


def rescued(rules, c, genes, max_mate_gap, windows):
    """c: candidate columns as the stage sees them (after intronic). Returns {candidate: how}, how in "positions", "reads", "spliced"."""
    gs, ge = genes["gene_start"], genes["gene_end"]
    index = _index(rules)
    out = {}
    for k in range(len(c["breakpoint1"])):
        if int(c["filter"][k]) not in (F_RELATIVE_SUPPORT, F_MIN_SUPPORT) or int(c["gene1"][k]) == int(c["gene2"][k]):
            continue
        c1, c2, b1, b2 = int(c["contig1"][k]), int(c["contig2"][k]), int(c["breakpoint1"][k]), int(c["breakpoint2"][k])
        g5 = 1 if int(c["bits"][k]) & CB_TSTART_GENE1 else 2
        g3 = 3 - g5
        for bn in _cand_bins(c, k, gs, ge):
            for a, b, _ in index.get(bn, []):
                m = lambda it, w: matches(it, c, k, w, max_mate_gap, 0.0, gs, ge)
                found = m(a, g5) and m(b, g3)
                if not found and int(c["bits2"][k]) and not (c1 == c2 and abs(b2 - b1) < 1000000):
                    found = m(a, g3) and m(b, g5)
                if not found:
                    continue
                support = int(c["split_reads1"][k]) + int(c["split_reads2"][k]) + int(c["discordant_mates"][k])
                cov = (coverage_get(windows, c1, b1, DOWNSTREAM if int(c["direction1"][k]) == UPSTREAM else UPSTREAM)
                       + coverage_get(windows, c2, b2, DOWNSTREAM if int(c["direction2"][k]) == UPSTREAM else UPSTREAM))
                if a["type"] == POSITION and b["type"] == POSITION:
                    out.setdefault(k, "positions")
                elif support >= 2:
                    out.setdefault(k, "reads")
                elif _both_spliced(c, k, genes["gene_strand"]) and cov < 200 and (c1 != c2 or abs(b2 - b1) > 1000000):
                    out.setdefault(k, "spliced")
    return out


def tags_of(rules, c, genes, max_mate_gap, ids):
    """{candidate: sorted list of distinct tags} for the candidates in ids (annotate_tags.cpp:45-83: directional, no swapped order)"""
    gs, ge = genes["gene_start"], genes["gene_end"]
    index = _index(rules)
    out = {}
    for k in ids:
        g5 = 1 if int(c["bits"][k]) & CB_TSTART_GENE1 else 2
        g3 = 3 - g5
        found = set()
        for bn in _cand_bins(c, k, gs, ge):
            for a, b, tag in index.get(bn, []):
                if matches(a, c, k, g5, max_mate_gap, 0.0, gs, ge) and matches(b, c, k, g3, max_mate_gap, 0.0, gs, ge):
                    found.add(tag)
        out[k] = sorted(found)
    return out


def rule_columns(rules):
    """the columns of Context.set_blacklist / set_known_fusions / set_tags"""
    cols = {k: [] for k in ("type1", "type2", "strand1", "strand2", "contig1", "contig2", "start1", "end1", "start2", "end2", "gene1", "gene2")}
    for r in rules:
        for w, it in ((1, r[0]), (2, r[1])):
            cols["type%d" % w].append(it["type"]); cols["strand%d" % w].append({None: 0, "+": 1, "-": 2}[it.get("strand")])
            cols["contig%d" % w].append(it["contig"]); cols["start%d" % w].append(it["start"]); cols["end%d" % w].append(it["end"]); cols["gene%d" % w].append(it.get("gene", 0))
    return cols


__all__ = ["read_rules", "rescued", "tags_of", "rule_columns", "coverage_get", "POSITION", "RANGE", "GENE"]
