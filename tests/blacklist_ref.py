"""Plain reference of the blacklist filter (-b): a literal Python transcription of filter_blacklisted_ranges (filter_blacklisted_ranges.cpp:17-300), with the
candidate bins as a dict of sets, the rules read line by line and blacklisted candidates erased from the sets. Shares no code with the product."""
import bisect
import gzip

UPSTREAM, DOWNSTREAM = 1, 0
RANGE, POSITION, GENE, ANY, SPLIT_READ_DONOR, SPLIT_READ_ACCEPTOR, SPLIT_READ_ANY, DISCORDANT_MATES, READ_THROUGH, LOW_SUPPORT, FILTER_SPLICED, NOT_BOTH_SPLICED = range(12)
KEYWORDS = {"any": ANY, "split_read_donor": SPLIT_READ_DONOR, "split_read_acceptor": SPLIT_READ_ACCEPTOR, "split_read_any": SPLIT_READ_ANY,
            "discordant_mates": DISCORDANT_MATES, "read_through": READ_THROUGH, "low_support": LOW_SUPPORT, "filter_spliced": FILTER_SPLICED,
            "not_both_spliced": NOT_BOTH_SPLICED}
CB_SPLICED1, CB_SPLICED2, CB_PSTRAND1, CB_PSTRAND2, CB_PSTRANDS_AMBIGUOUS = 4, 8, 16, 32, 64
F_NONE = 0


def _i32(x):
    x = int(x) & 0xFFFFFFFF
    return x - (1 << 32) if x >= 1 << 31 else x


def _str_to_int(s):  # common.hpp:316-321
    if not s or s[0] == " ":
        return None
    t = s.lstrip(" \t\n\v\f\r")
    body = t[1:] if t[:1] in ("+", "-") else t
    if not body or not body.isdigit() or not body.isascii():
        return None
    v = int(t)
    if v >= (1 << 63) - 1 or v <= -(1 << 63):
        return None
    return _i32(v)


def _remove_chr(c):
    if c.startswith("chr"):
        c = c[3:]
    return "MT" if c == "M" else c


def _tsv(s, d="\t"):
    """tsv_stream_t: list of fields; reading past the last one fails."""
    out, pos = [], 0
    while pos < len(s):
        e = s.find(d, pos)
        if e < 0:
            out.append(s[pos:]); pos = len(s)
        else:
            out.append(s[pos:e]); pos = e + 1
    return out


class Undefined(Exception):
    pass


def parse_range(rng, contigs, sorted_names, warnings):
    """parse_range (:17-80) -> dict or None"""
    i = rng.rfind(":")
    if i >= 0:
        rng = rng[:i] + "\t" + rng[i + 1:]
    f = _tsv(rng)
    if len(f) < 2 or not f[0] or not f[1]:
        warnings.append("WARNING: unknown gene or malformed range: " + rng); return None
    name, pos = f[0], f[1]
    item = {"strand": None}
    if name[0] == "+":
        item["strand"] = "+"; name = name[1:]
    elif name[0] == "-":
        item["strand"] = "-"; name = name[1:]
    name = _remove_chr(name)
    if len(name) >= 2 and name[-1] == "*":
        prefix = name[:-1]
        j = bisect.bisect_left(sorted_names, prefix)
        if j == len(sorted_names):
            raise Undefined(rng)
        if not sorted_names[j].startswith(prefix):
            return None
        item["contig"] = contigs[sorted_names[j]]
    else:
        if name not in contigs:
            warnings.append("WARNING: unknown gene or malformed range: " + rng); return None
        item["contig"] = contigs[name]
    p = _tsv(pos, "-")
    if "-" in pos:
        a = _str_to_int(p[0]) if len(p) > 0 else None
        b = _str_to_int(p[1]) if len(p) > 1 else None
        if a is None or b is None:
            warnings.append("WARNING: unknown gene or malformed range: " + rng); return None
        item["start"], item["end"] = _i32(a - 1), _i32(b - 1)
    else:
        a = _str_to_int(p[0])
        if a is None:
            warnings.append("WARNING: unknown gene or malformed range: " + rng); return None
        item["start"] = item["end"] = _i32(a - 1)
    return item


def parse_item(text, allow_keyword, contigs, sorted_names, gene_by_name, gene_contig, gene_start, gene_end, warnings):
    """parse_blacklist_item (:83-120) -> dict or None"""
    if text == "":
        warnings.append("WARNING: encountered a line with an empty column => skipped"); return None
    if allow_keyword and text in KEYWORDS:
        return {"type": KEYWORDS[text]}
    if text in gene_by_name:
        g = gene_by_name[text]
        return {"type": GENE, "gene": g, "contig": int(gene_contig[g]), "start": int(gene_start[g]), "end": int(gene_end[g]), "strand": None}
    item = parse_range(text, contigs, sorted_names, warnings)
    if item is None:
        return None
    item["type"] = POSITION if item["start"] == item["end"] else RANGE
    return item


def read_rules(path, contigs, gene_by_name, gene_contig, gene_start, gene_end):
    """contigs: name without chr -> id. Returns (list of (item1, item2) in file order, warning lines)."""
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
        f = _tsv(line) + ["", ""]
        a = parse_item(f[0], False, contigs, sorted_names, gene_by_name, gene_contig, gene_start, gene_end, warnings)
        if a is None:
            continue
        b = parse_item(f[1], True, contigs, sorted_names, gene_by_name, gene_contig, gene_start, gene_end, warnings)
        if b is None:
            continue
        rules.append((a, b))
    return rules, warnings


def _bins(contig, start, end):  # get_genome_bins_from_range (:226-230), C division
    q = lambda x: x // 100000 if x >= 0 else -((-x) // 100000)
    return [(contig, b * 100000) for b in range(q(start), q(end + 100000 - 1) + 1)]


def _f32(x):
    import numpy as np
    return float(np.float32(x))


def overlapping_fraction(s1, e1, s2, e2):
    if s1 >= s2 and e1 <= e2:
        return 1.0
    if s1 < s2 and e1 > e2:
        return _f32(1.0 * (e2 - s2) / (e1 - s1 + 1))
    if s1 >= s2 and s1 <= e2:
        return _f32(1.0 * (e2 - s1) / (e1 - s1 + 1))
    if e1 >= s2 and e1 <= e2:
        return _f32(1.0 * (e1 - s2) / (e1 - s1 + 1))
    return 0.0


def matches(item, c, k, which, max_mate_gap, evalue_cutoff, gene_start, gene_end):
    """matches_blacklist_item (:138-223); c: candidate columns"""
    t = item["type"]
    sr1, sr2, dm = int(c["split_reads1"][k]), int(c["split_reads2"][k]), int(c["discordant_mates"][k])
    bits = int(c["bits"][k]); spliced1, spliced2 = bool(bits & CB_SPLICED1), bool(bits & CB_SPLICED2)
    ev = float(c["evalue"][k])
    if t == ANY:
        return True
    if t == SPLIT_READ_DONOR:
        return (which == 1 and dm + sr1 == 0) or (which == 2 and dm + sr2 == 0)
    if t == SPLIT_READ_ACCEPTOR:
        return (which == 1 and dm + sr2 == 0) or (which == 2 and dm + sr1 == 0)
    if t == SPLIT_READ_ANY:
        return dm == 0
    if t == DISCORDANT_MATES:
        return sr1 + sr2 == 0
    if t == READ_THROUGH:
        return (int(c["contig1"][k]) == int(c["contig2"][k]) and int(c["breakpoint2"][k]) - int(c["breakpoint1"][k]) < 400000
                and int(c["direction1"][k]) == DOWNSTREAM and int(c["direction2"][k]) == UPSTREAM)
    if t == LOW_SUPPORT:
        return ev > evalue_cutoff
    if t == FILTER_SPLICED:
        return ev > evalue_cutoff and spliced1 and spliced2
    if t == NOT_BOTH_SPLICED:
        return not spliced1 or not spliced2
    if t == GENE:
        return int(c["gene%d" % which][k]) == item["gene"]
    if int(c["contig%d" % which][k]) != item["contig"]:
        return False
    if item["strand"] is not None and not (bits & CB_PSTRANDS_AMBIGUOUS):
        forward = bool(bits & (CB_PSTRAND1 if which == 1 else CB_PSTRAND2))
        if forward != (item["strand"] == "+"):
            return False
    if t == RANGE:
        g = int(c["gene%d" % which][k])
        return overlapping_fraction(int(gene_start[g]), int(gene_end[g]), item["start"], item["end"]) > 0.5
    bp = int(c["breakpoint%d" % which][k])
    if bp == item["start"]:
        return True
    if sr1 + sr2 == 0:
        d = int(c["direction%d" % which][k])
        if (d == DOWNSTREAM and bp <= item["start"] and bp >= item["start"] - max_mate_gap) or (d == UPSTREAM and bp >= item["start"] and bp <= item["start"] + max_mate_gap):
            return True
    return False


def blacklisted(rules, c, gene_start, gene_end, evalue_cutoff, max_mate_gap, closest1=None):
    """c: candidate columns (Pipeline.candidates()) as the stage sees them. Returns the set of blacklisted candidates."""
    index = {}
    n = len(c["breakpoint1"])
    for k in range(n):
        if int(c["filter"][k]) != F_NONE and (closest1 is None or int(closest1[k]) < 0):
            continue
        bins = (_bins(int(c["contig1"][k]), int(c["breakpoint1"][k]), int(c["breakpoint1"][k])) + _bins(int(c["contig2"][k]), int(c["breakpoint2"][k]), int(c["breakpoint2"][k]))
                + _bins(int(c["contig1"][k]), int(gene_start[c["gene1"][k]]), int(gene_end[c["gene1"][k]]))
                + _bins(int(c["contig2"][k]), int(gene_start[c["gene2"][k]]), int(gene_end[c["gene2"][k]])))
        for b in bins:
            index.setdefault(b, set()).add(k)
    out = set()
    for a, b in rules:
        bins = []
        for it in (a, b):
            if it["type"] in (POSITION, RANGE, GENE):
                bins += _bins(it["contig"], it["start"] - max_mate_gap, it["end"] + max_mate_gap)
        for bn in bins:
            members = index.get(bn)
            if not members:
                continue
            for k in sorted(members):
                m = lambda it, w: matches(it, c, k, w, max_mate_gap, evalue_cutoff, gene_start, gene_end)
                if (m(a, 1) and m(b, 2)) or (m(a, 2) and m(b, 1)):
                    out.add(k); members.discard(k)
    return out
