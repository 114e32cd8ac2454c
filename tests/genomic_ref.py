"""Plain reference of the genomic-support marking (-d): a literal Python transcription of mark_genomic_support (filter_genomic_support.cpp:80-219),
map walk, DOWNSTREAM quirk and negative-coordinate rule included. Shares no code with the product."""
import bisect
import gzip

UPSTREAM, DOWNSTREAM = 1, 0


def _i32(x):
    x = int(x) & 0xFFFFFFFF
    return x - (1 << 32) if x >= 1 << 31 else x


def _str_to_int(s):  # common.hpp:316-321 (strtol: leading whitespace and a sign, then digits only)
    t = s.lstrip(" \t\n\v\f\r") if s and s[0] != " " else None
    if not t:
        return None
    body = t[1:] if t[0] in "+-" else t
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


def _fields(line):
    return line.split("\t")


def _breakpoint(bp, contigs):
    i = bp.rfind(":")
    if i < 0:
        return None
    name, pos = bp[:i], bp[i + 1:]
    name = _remove_chr(name)
    if name not in contigs:
        return None
    p = _str_to_int(pos)
    return None if p is None else (contigs[name], _i32(p - 1))


def _direction(s):
    return UPSTREAM if s in ("upstream", "-") else DOWNSTREAM if s in ("downstream", "+") else None


def _info(info, field):
    if info.startswith(field + "="):
        start = len(field) + 1
    else:
        start = info.find(";" + field + "=")
        if start < 0:
            return None
        start += len(field) + 2
    end = info.find(";", start)
    return info[start:] if end < 0 else info[start:end]


def read_records(path, contigs):
    """contigs: name without chr -> id. Returns (records in file order as (c1, c2, d1, d2, p1, p2), warning lines)."""
    raw = gzip.open(path, "rb").read() if path.endswith(".gz") else open(path, "rb").read()
    text = raw.decode("latin-1")
    lines = text.split("\n")
    if lines and lines[-1] == "":
        lines.pop()
    recs, warnings = [], []
    for line in lines:
        if line.endswith("\r"):
            line = line[:-1]
        if not line or line[0] == "#":
            continue
        f = _fields(line) + [""] * 8
        a, b, d1, d2 = _breakpoint(f[0], contigs), _breakpoint(f[1], contigs), _direction(f[2]), _direction(f[3])
        sv = ""
        if a is None or b is None or d1 is None or d2 is None:
            chrom, pos, alt, filt, info = f[0], f[1], f[4], f[6], f[7]
            sv = _info(info, "SVTYPE")
            ok = sv is not None
            mate = None
            if ok and sv == "BND":
                o, c = alt.find("["), alt.find("]")
                o = len(alt) + 1 if o < 0 else o; c = len(alt) + 1 if c < 0 else c
                bracket = "[" if o < c else "]"
                p1 = min(o, c)
                p2 = alt.find(bracket, p1 + 1) if p1 < len(alt) else -1
                if p1 >= len(alt) or p2 < 0:
                    if alt and (alt[0] == "." or alt[-1] == "."):
                        continue
                    ok = False
                else:
                    d1 = UPSTREAM if p1 == 0 else DOWNSTREAM
                    d2 = UPSTREAM if bracket == "[" else DOWNSTREAM
                    mate = alt[p1 + 1:p2]
            elif ok:
                end = _info(info, "END")
                ok = end is not None
                mate = chrom + ":" + (end or "")
                if sv == "INV":
                    d1, d2 = DOWNSTREAM, DOWNSTREAM
                elif sv == "DEL":
                    d1, d2 = DOWNSTREAM, UPSTREAM
                elif sv == "DUP":
                    d1, d2 = UPSTREAM, DOWNSTREAM
                else:
                    ok = False
            if ok:
                a, b = _breakpoint(chrom + ":" + pos, contigs), _breakpoint(mate, contigs)
                ok = a is not None and b is not None
            if not ok:
                warnings.append("WARNING: failed to parse line: " + line)
                continue
            if filt != "PASS":
                continue
        (c1, q1), (c2, q2) = a, b
        if c2 < c1 or (c2 == c1 and q2 < q1):
            c1, c2, q1, q2, d1, d2 = c2, c1, q2, q1, d2, d1
        recs.append((c1, c2, d1, d2, q1, q2))
        if sv == "INV":
            recs.append((c1, c2, UPSTREAM, UPSTREAM, q1, q2))
    return recs, warnings


def mark(records, cand, gene_start, gene_end, gene_dummy, max_distance=100000, max_itd_length=100):
    """cand: dict of arrays contig1, contig2, breakpoint1, breakpoint2, direction1, direction2, gene1, gene2. Returns (closest1, closest2) lists."""
    index = {}
    for c1, c2, d1, d2, p1, p2 in records:
        index.setdefault((c1, c2, d1, d2), {}).setdefault(p1, []).append(p2)
    index = {k: (sorted(v), v) for k, v in index.items()}
    gene_start = [int(x) for x in gene_start]; gene_end = [int(x) for x in gene_end]; gene_dummy = [bool(x) for x in gene_dummy]

    def close_enough(direction, g, bp, gene):
        if direction == UPSTREAM:
            distal = _i32((bp if gene_dummy[gene] else gene_start[gene]) - max_distance)
            return g >= distal and g <= _i32(bp + 5)
        distal = _i32((bp if gene_dummy[gene] else gene_end[gene]) + max_distance)
        return g <= distal and g >= _i32(bp - 5)

    out1, out2 = [], []
    for k in range(len(cand["breakpoint1"])):
        c1, c2 = int(cand["contig1"][k]), int(cand["contig2"][k])
        d1, d2 = int(cand["direction1"][k]), int(cand["direction2"][k])
        b1, b2 = int(cand["breakpoint1"][k]), int(cand["breakpoint2"][k])
        g1, g2 = int(cand["gene1"][k]), int(cand["gene2"][k])
        best1 = best2 = -1
        entry = index.get((c1, c2, d1, d2))
        if entry is not None:
            keys, lists = entry
            it = bisect.bisect_left(keys, _i32(b1 + (5 if d1 == UPSTREAM else -5)))
            if d1 == UPSTREAM:
                it = it - 1 if it > 0 else None
            elif it == len(keys):
                it = None
            while it is not None and close_enough(d1, keys[it], b1, g1):
                key = keys[it]
                for p2 in lists[key]:
                    itd = g1 == g2 and ((b2 - b1) & 0xFFFFFFFF) < max_itd_length and d1 == UPSTREAM and d2 == DOWNSTREAM
                    if close_enough(d2, p2, b2, g2) and (
                            c1 != c2 or
                            (d1 == UPSTREAM and d2 == DOWNSTREAM and (not itd or (_i32(b1 - key) < max_itd_length and _i32(p2 - b2) < max_itd_length))) or
                            (d1 == DOWNSTREAM and d2 == UPSTREAM and key < b2 and p2 > b1) or
                            (d1 == UPSTREAM and d2 == UPSTREAM and p2 > b1) or
                            (d1 == DOWNSTREAM and d2 == DOWNSTREAM and key < b2)):
                        dist = lambda x, y: _i32(abs(_i32(x - b1)) + abs(_i32(b2 - y)))
                        if best1 < 0 or best2 < 0 or dist(best1, best2) > dist(key, p2):
                            best1, best2 = key, p2
                it = it - 1 if it > 0 else None
        out1.append(best1); out2.append(best2)
    return out1, out2
