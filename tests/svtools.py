"""Writer of structural-variant files (-d) built from a world's candidates: genomic breakpoints at and around the candidates' breakpoints and at the
edges of the distance window, in Arriba's four-column format and in every VCF form the reference reads, with the malformed and skipped lines it has rules for."""
import gzip
import random

UPSTREAM, DOWNSTREAM = 1, 0


def _name(contig_names, c, rng):
    n = contig_names[c]
    bare = n[3:] if n.startswith("chr") else n
    return rng.choice([bare, "chr" + bare])


def _four_column(names, c1, p1, d1, c2, p2, d2, rng):
    word = rng.choice([("upstream", "downstream"), ("-", "+")])
    dirs = [word[0] if d == UPSTREAM else word[1] for d in (d1, d2)]
    a = "%s:%d" % (_name(names, c1, rng), p1 + 1); b = "%s:%d" % (_name(names, c2, rng), p2 + 1)
    if rng.random() < 0.5:  # the same pair in the other column order
        a, b = b, a; dirs.reverse()
    return "\t".join([a, b] + dirs + (["extra"] if rng.random() < 0.1 else []))


def _bnd(names, c1, p1, d1, c2, p2, d2, rng, filt="PASS"):
    mate = "%s:%d" % (_name(names, c2, rng), p2 + 1)
    alt = {(UPSTREAM, UPSTREAM): "[%s[N", (UPSTREAM, DOWNSTREAM): "]%s]N", (DOWNSTREAM, UPSTREAM): "N[%s[", (DOWNSTREAM, DOWNSTREAM): "N]%s]"}[(d1, d2)] % mate
    return "\t".join([_name(names, c1, rng), str(p1 + 1), "bnd%d" % rng.randrange(1 << 30), "N", alt, ".", filt, "SVTYPE=BND;MATEID=x"])


def _vcf_end(names, c, p1, p2, sv, rng, filt="PASS"):
    info = rng.choice(["SVTYPE=%s;END=%d" % (sv, p2 + 1), "END=%d;SVTYPE=%s;SVLEN=3" % (p2 + 1, sv)])
    return "\t".join([_name(names, c, rng), str(p1 + 1), ".", "N", "<%s>" % sv, ".", filt, info])


def sv_lines(cand, gene_start, gene_end, gene_dummy, contig_names, rng, max_distance=100000, n_candidates=300):
    """cand: arrays contig1, contig2, breakpoint1, breakpoint2, direction1, direction2, gene1, gene2."""
    n = len(cand["breakpoint1"])
    pick = rng.sample(range(n), min(n, n_candidates))
    lines = ["##fileformat=VCFv4.2", "#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO", ""]

    def around(k, side):
        bp = int(cand["breakpoint%d" % side][k]); g = int(cand["gene%d" % side][k]); d = int(cand["direction%d" % side][k])
        out = [bp, bp - 4, bp + 4, bp - 5, bp + 5, bp - 6, bp + 6]
        edge = (bp if gene_dummy[g] else int(gene_start[g])) - max_distance if d == UPSTREAM else (bp if gene_dummy[g] else int(gene_end[g])) + max_distance
        out += [edge - 1, edge, edge + 1, 0, -1, -3, bp - 50, bp + 50, bp - 1000, bp + 1000]
        return out

    for k in pick:
        c1, c2 = int(cand["contig1"][k]), int(cand["contig2"][k]); d1, d2 = int(cand["direction1"][k]), int(cand["direction2"][k])
        b1, b2 = int(cand["breakpoint1"][k]), int(cand["breakpoint2"][k])
        firsts, seconds = around(k, 1), around(k, 2)
        for _ in range(rng.randint(2, 6)):
            p1, p2 = rng.choice(firsts), rng.choice(seconds)
            form = rng.random()
            if form < 0.55:
                lines.append(_four_column(contig_names, c1, p1, d1, c2, p2, d2, rng))
            elif form < 0.8:
                lines.append(_bnd(contig_names, c1, p1, d1, c2, p2, d2, rng, filt="PASS" if rng.random() < 0.9 else "LowQual"))
            elif c1 == c2:
                sv = {(DOWNSTREAM, UPSTREAM): "DEL", (UPSTREAM, DOWNSTREAM): "DUP"}.get((d1, d2), "INV")
                lines.append(_vcf_end(contig_names, c1, p1, p2, sv, rng, filt="PASS" if rng.random() < 0.9 else "q10"))
            else:
                lines.append(_bnd(contig_names, c2, p2, d2, c1, p1, d1, rng))  # the mate's record of the pair
        # ties: the same distance sum within one position1 and across position1 keys, several position2 values under one position1
        for dd in (3, 7):
            lines.append(_four_column(contig_names, c1, b1 - dd, d1, c2, b2 + dd, d2, rng))
            lines.append(_four_column(contig_names, c1, b1 + dd, d1, c2, b2 - dd, d2, rng))
            lines.append(_four_column(contig_names, c1, b1 - dd, d1, c2, b2 - dd, d2, rng))
        # between and outside the breakpoints of deletions, duplications and inversions
        if c1 == c2:
            mid = (b1 + b2) // 2
            for p1, p2 in ((mid, mid + 1), (b1 - 20, b2 + 20), (b1 + 20, b2 - 20), (b1 + 2, b2 - 2)):
                lines.append(_four_column(contig_names, c1, p1, d1, c2, p2, d2, rng))
    # single breakends, unknown contigs, a contig name with a colon, malformed lines, VCF lines the reference cannot use
    c0 = int(cand["contig1"][pick[0]]) if pick else 0
    lines += ["\t".join([_name(contig_names, c0, rng), "100", ".", "N", "N.", ".", "PASS", "SVTYPE=BND"]),
              "\t".join([_name(contig_names, c0, rng), "100", ".", "N", ".N", ".", "LowQual", "SVTYPE=BND"]),
              "unknown_contig:100\t%s:200\t+\t-" % contig_names[c0], "chrUn:weird:5\t%s:200\t-\t+" % contig_names[c0],
              "this line is garbage", "%s:12x\t%s:200\t+\t-" % (contig_names[c0], contig_names[c0]), "%s:100\t%s:200\tleft\t-" % (contig_names[c0], contig_names[c0]),
              "\t".join([contig_names[c0], "100", ".", "N", "<INS>", ".", "PASS", "SVTYPE=INS;END=300"]),
              "\t".join([contig_names[c0], "100", ".", "N", "<DEL>", ".", "PASS", "SVTYPE=DEL"]),
              "\t".join([contig_names[c0], "100", ".", "N", "N[%s:300" % contig_names[c0], ".", "PASS", "SVTYPE=BND"]),
              "\t".join([contig_names[c0], "100", ".", "N", "<DEL>", ".", "PASS", "NOTSVTYPE=DEL;END=300"]),
              "\t".join(["unknown_contig", "100", ".", "N", "<DEL>", ".", "PASS", "SVTYPE=DEL;END=300"]),
              "# a comment", ""]
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


def dense_lines(cand, gene_start, gene_end, contig_names, rng, n_records):
    """n_records breakpoint pairs concentrated on the keys of a few candidates with long genes: ranges of thousands of records per candidate."""
    n = len(cand["breakpoint1"])
    span = lambda k: int(gene_end[cand["gene1"][k]]) - int(gene_start[cand["gene1"][k]])
    heavy = sorted(range(n), key=span, reverse=True)[:8]
    lines = []
    for x in range(n_records):
        k = heavy[x % len(heavy)]
        c1, c2 = int(cand["contig1"][k]), int(cand["contig2"][k]); d1, d2 = int(cand["direction1"][k]), int(cand["direction2"][k])
        b1, b2 = int(cand["breakpoint1"][k]), int(cand["breakpoint2"][k])
        p1 = b1 + rng.randint(-120000, 120000) // rng.choice([1, 1, 7, 97])
        p2 = b2 + rng.randint(-120000, 120000) // rng.choice([1, 1, 7, 97])
        if rng.random() < 0.001:
            p2 = -rng.randint(1, 5)  # negative coordinates in some ranges
        lines.append("%s:%d\t%s:%d\t%s\t%s" % (contig_names[c1], p1 + 1, contig_names[c2], p2 + 1, "-" if d1 == UPSTREAM else "+", "-" if d2 == UPSTREAM else "+"))
    return lines
