"""Writer of blacklist files (-b) built from a world's own candidates: every rule type and keyword, positions at and around the breakpoints, ranges at the
0.5 gene-overlap threshold in each branch of overlapping_fraction, strands, wildcards, bin edges, long ranges, and the malformed lines the reference has rules for."""
import gzip
import random

UPSTREAM, DOWNSTREAM = 1, 0
KEYWORDS = ["any", "split_read_donor", "split_read_acceptor", "split_read_any", "discordant_mates", "read_through", "low_support", "filter_spliced", "not_both_spliced"]


def gene_names(gtf_path, genes, contig_ids):
    """Name of every gene of the run (None for dummy genes): the GTF's genes in order of first appearance, keyed like the loader keys them (gene_id without
    its version, contig, strand), named by the first exon's gene_name (else gene_id), lined up with the run's genes by contig and extent."""
    order, ext = [], {}
    for line in open(gtf_path):
        if line.startswith("#"):
            continue
        f = line.rstrip("\n").split("\t")
        if len(f) < 9 or f[2] != "exon":
            continue
        attrs = {}
        for a in f[8].split(";"):
            a = a.strip()
            if " " in a:
                k, v = a.split(" ", 1); attrs.setdefault(k, v.strip('"'))
        if "gene_id" not in attrs:
            continue
        c = contig_ids.get(f[0][3:] if f[0].startswith("chr") else f[0])
        key = (attrs["gene_id"].split(".")[0], c, f[6] == "+")
        if key not in ext:
            order.append(key); ext[key] = [attrs.get("gene_name", attrs["gene_id"]), int(f[3]) - 1, int(f[4]) - 1]
        else:
            ext[key][1] = min(ext[key][1], int(f[3]) - 1); ext[key][2] = max(ext[key][2], int(f[4]) - 1)
    names = [None] * len(genes["gene_start"]); g = 0
    real = [x for x in range(len(names)) if not genes["gene_flags"][x] & 1]
    for key in order:
        if g < len(real) and (key[1], ext[key][1], ext[key][2]) == (int(genes["gene_contig"][real[g]]), int(genes["gene_start"][real[g]]), int(genes["gene_end"][real[g]])):
            names[real[g]] = ext[key][0]; g += 1
    return names


def gene_by_name(names):
    out = {}
    for g, n in enumerate(names):
        if n is not None:
            out[n] = g  # the last gene of a name wins (annotation.cpp:373-375)
    return out


def _name(contig_names, c, rng):
    n = contig_names[c]
    bare = n[3:] if n.startswith("chr") else n
    return rng.choice([bare, "chr" + bare]) if bare not in ("M", "MT") else rng.choice(["M", "chrM", "MT"])


def rule_lines(cand, genes, names, contig_names, rng, max_mate_gap, n_candidates=250):
    """cand: Pipeline.candidates() after many_spliced; genes: Pipeline.genes(); names: gene_names()."""
    n = len(cand["breakpoint1"])
    gs, ge = genes["gene_start"], genes["gene_end"]
    lines = ["# blacklist written from the world's candidates", ""]
    pick = rng.sample(range(n), min(n, n_candidates))

    def pos(c, p, strand=""):
        return "%s%s:%d" % (strand, _name(contig_names, c, rng), p + 1)

    def rng_text(c, s, e, strand=""):
        return "%s%s:%d-%d" % (strand, _name(contig_names, c, rng), s + 1, e + 1)

    def side(k, w):
        return int(cand["contig%d" % w][k]), int(cand["breakpoint%d" % w][k]), int(cand["direction%d" % w][k]), int(cand["gene%d" % w][k])

    def any_item(k, w):  # something on side w of candidate k that matches it
        c, b, d, g = side(k, w)
        choice = rng.random()
        if choice < 0.4:
            return pos(c, b)
        if choice < 0.6 and names[g] is not None:
            return names[g]
        if choice < 0.8:
            return rng_text(c, int(gs[g]) - rng.randint(0, 50), int(ge[g]) + rng.randint(0, 50))
        return rng.choice(KEYWORDS)

    for k in pick:
        c1, b1, d1, g1 = side(k, 1); c2, b2, d2, g2 = side(k, 2)
        # positions at the breakpoints, with every keyword and in both column orders
        lines.append("%s\t%s" % (pos(c1, b1), rng.choice(KEYWORDS + [pos(c2, b2)])))
        lines.append("%s\t%s" % (pos(c2, b2), pos(c1, b1)))
        lines.append("%s\t%s" % (any_item(k, 2), any_item(k, 1)) if rng.random() < 0.5 else "%s\t%s" % (any_item(k, 1), any_item(k, 2)))
        # candidates with only discordant mates: the max_mate_gap window, in the direction the mates point, and one past it
        if int(cand["split_reads1"][k]) + int(cand["split_reads2"][k]) == 0:
            for w in (1, 2):
                c, b, d, g = side(k, w)
                for off in (max_mate_gap, max_mate_gap + 1, -max_mate_gap, -max_mate_gap - 1, 1, -1):
                    other = pos(c2, b2) if w == 1 else pos(c1, b1)
                    lines.append("%s\t%s" % (pos(c, b + off), rng.choice(["any", "discordant_mates", other])))
        # ranges at the 0.5 overlap of the gene in each branch of overlapping_fraction
        for w in (1, 2):
            c, b, d, g = side(k, w)
            s, e = int(gs[g]), int(ge[g]); L = e - s + 1
            if L < 8:
                continue
            h = L // 2
            for dd in (-1, 0, 1):
                lines.append("%s\tany" % rng_text(c, s - 3, e + 3))                              # range holds the gene
                lines.append("%s\tany" % rng_text(c, s + 1, s + 1 + h + dd))                    # gene holds the range (no "+ 1")
                lines.append("%s\tany" % rng_text(c, s - 10, s + h + dd))                       # gene starts inside
                lines.append("%s\tany" % rng_text(c, e - h - dd, e + 10))                       # gene ends inside
        # strands, matching and not, on the breakpoint
        for strand in ("+", "-"):
            lines.append("%s\t%s" % (pos(c1, b1, strand), rng.choice(["any", pos(c2, b2, strand)])))
            lines.append("%s\tany" % rng_text(c1, int(gs[g1]) - 5, int(ge[g1]) + 5, strand))
        # wildcard contigs: a prefix that picks the first contig at or after it, and one that matches nothing
        bare = contig_names[c1][3:] if contig_names[c1].startswith("chr") else contig_names[c1]
        lines.append("%s*:%d\t%s" % (bare[:1], b1 + 1, rng.choice(["any", pos(c2, b2)])))
        lines.append("%s*:%d\tany" % (bare, b1 + 1))
        lines.append("0*:%d\tany" % (b1 + 1))
        # bin edges: multiples of 100000 near the breakpoint, and ranges that reach below 0
        edge = (b1 // 100000) * 100000
        for p in (edge - 1, edge, edge + 1, edge + 99999, edge + 100000):
            if p >= 0:
                lines.append("%s\t%s" % (pos(c1, p), rng.choice(["any", "split_read_any", pos(c2, b2)])))
        lines.append("%s\t%s" % (rng_text(c1, -1, rng.randint(0, 5)), "any"))
        # ranges over many bins
        lines.append("%s\t%s" % (rng_text(c1, max(0, b1 - 2000000), b1 + 2000000), rng.choice(["low_support", "read_through", "not_both_spliced", "filter_spliced"])))
    # keywords in column 1, malformed lines, comments, blank lines, extra columns
    c0 = int(cand["contig1"][pick[0]]) if pick else 0
    nm = contig_names[c0]
    lines += ["any\t%s:100" % nm, "read_through\tany", "\t%s:100" % nm, "%s:100\t" % nm, "%s:100" % nm, "nocolon\tany", "%s:12x\tany" % nm,
              "%s:100-\tany" % nm, "%s:-5\tany" % nm, "%s:500-100\tany" % nm, "%s:100-200\tany\textra\tcolumns" % nm, "unknown_contig:100\tany",
              "%s:\tany" % nm, ":100\tany", "+%s:100-200\t-%s:300" % (nm, nm), "no_such_gene\tany", "# comment\tany", ""]
    rng.shuffle(lines)
    return lines


def write(path, lines, crlf=False):
    data = ("\r\n" if crlf else "\n").join(lines) + "\n"
    if path.endswith(".gz"):
        with gzip.open(path, "wb") as f:
            f.write(data.encode())
    else:
        with open(path, "w", newline="") as f:
            f.write(data)


def dense_lines(cand, genes, contig_names, rng, n_rules, max_mate_gap):
    """n_rules rules concentrated on a few candidates' bins: rule lists of thousands of entries, most of which do not match."""
    eligible = [k for k in range(len(cand["breakpoint1"])) if cand["filter"][k] == 0] or list(range(len(cand["breakpoint1"])))
    hot = rng.sample(eligible, min(len(eligible), 16))
    lines = []
    for x in range(n_rules):
        k = hot[x % len(hot)]
        c1, b1 = int(cand["contig1"][k]), int(cand["breakpoint1"][k]); c2, b2 = int(cand["contig2"][k]), int(cand["breakpoint2"][k])
        p = b1 + rng.randint(-60000, 60000) if rng.random() >= 0.002 else b1  # a few rules hit the breakpoint
        second = "%s:%d" % (contig_names[c2], b2 + 1) if rng.random() < 0.3 else "%s:%d" % (contig_names[c2], max(1, b2 + rng.randint(1, 90000)))
        lines.append("%s:%d\t%s" % (contig_names[c1], max(1, p + 1), second))
    return lines
