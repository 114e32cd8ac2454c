"""Plain transcription of fill_gaps_in_fusion_transcript_sequence (output_fusions.cpp:820-1041) for the tests of -I.

A transcript is a dict: first (exon id), last (exon id), contig; exons are dicts start, end, next, prev (exon ids, None: none). `assembly` maps a contig to
its sequence (a contig missing from it has no sequence). fill() returns the filled sequence and positions and records which branch each side took."""

COMP = {"a": "t", "t": "a", "c": "g", "g": "c", "A": "T", "T": "A", "C": "G", "G": "C", "[": "]", "]": "["}


def comp(c):
    return COMP.get(c, c)


def _five(seq, pos, tr, exons, strand_fwd, itd, contig_seq, log):
    first, last = exons[tr["first"]], exons[tr["last"]]
    bp = seq.find("|")
    bp = len(seq) if bp < 0 else bp  # rows with transcripts always have one
    gap = seq.rfind(".", 0, bp + 1)  # find_last_of("...", breakpoint): the character '.'
    found = gap >= 0
    imprecise = False
    if found and gap + 1 == bp and gap >= 3:
        imprecise = True; gap -= 3
    elif found and first["start"] < pos[gap + 1] < last["end"]:
        gap += 1
    elif not found and first["start"] < pos[0] < last["end"]:
        gap = 0
    else:
        i0 = 0
        for i in range(bp):
            if first["start"] <= pos[i] <= last["end"]:
                i0 = i; break
        seq, pos = seq[i0:], pos[i0:]
        if (strand_fwd and pos[0] == first["start"]) or (not strand_fwd and pos[0] == last["end"]):
            seq, pos = "^" + seq, [-1] + pos
            log.append("5:trim^")
        else:
            log.append("5:trim")
        return seq, pos
    ov = None
    while gap != bp:
        x = tr["first"]
        while x is not None:
            if exons[x]["start"] <= pos[gap] <= exons[x]["end"]:
                ov = x; break
            x = exons[x]["next"]
        if ov is not None:
            break
        gap += 1
    ok = ov is not None
    if imprecise and ((strand_fwd and ov == tr["last"]) or (not strand_fwd and ov == tr["first"]) or itd):
        ok = False
    if not ok:
        log.append("5:imprecise-not-snapped" if imprecise else "5:no-overlap")
        return seq, pos
    seq, pos = list(seq), list(pos)
    if imprecise:
        gap = bp - 1
        pos[gap] = exons[ov]["end"] if strand_fwd else exons[ov]["start"]
        seq[gap] = contig_seq[pos[gap]] if strand_fwd else comp(contig_seq[pos[gap]])
    s, p = ["("], [-1]
    x = tr["first"] if strand_fwd else tr["last"]
    while x is not None:
        e = exons[x]
        q = e["start"] if strand_fwd else e["end"]
        while q != pos[gap] and e["start"] <= q <= e["end"]:
            s.append(contig_seq[q] if strand_fwd else comp(contig_seq[q])); p.append(q)
            q += 1 if strand_fwd else -1
        if q == pos[gap]:
            break
        s += ["_"] * 3; p += [-1] * 3
        x = e["next"] if strand_fwd else e["prev"]
    if imprecise:
        s.append(seq[gap]); p.append(pos[gap]); gap += 1
    s.append(")"); p.append(-1)
    s += seq[gap:]; p += pos[gap:]
    if (strand_fwd and p[1] == first["start"]) or (not strand_fwd and p[1] == last["end"]):
        s, p = ["^"] + s, [-1] + p
        log.append("5:imprecise-snapped^" if imprecise else "5:filled^")
    else:
        log.append("5:imprecise-snapped" if imprecise else "5:filled")
    return "".join(s), p


def _three(seq, pos, tr, exons, strand_fwd, itd, contig_seq, log):
    first, last = exons[tr["first"]], exons[tr["last"]]
    bp = seq.rfind("|")
    gap = seq.find("...", bp)
    found = gap >= 0
    n = len(seq)
    imprecise = False
    if found and gap - 1 == bp and gap + 3 < n:
        imprecise = True; gap += 3
    elif found and first["start"] < pos[gap - 1] < last["end"]:
        gap -= 1
    elif not found and first["start"] < pos[n - 1] < last["end"]:
        gap = n - 1
    else:
        i1 = n - 1
        for i in range(n - 1, bp, -1):
            if first["start"] <= pos[i] <= last["end"]:
                i1 = i; break
        if i1 < n - 1:
            seq, pos = seq[:i1 + 1], pos[:i1 + 1]
        if (strand_fwd and pos[-1] == last["end"]) or (not strand_fwd and pos[-1] == first["start"]):
            log.append("3:trim$")
            return seq + "$", pos + [-1]
        log.append("3:trim")
        return seq, pos
    ov = None
    while gap != bp:
        x = tr["first"]
        while x is not None:
            if exons[x]["start"] <= pos[gap] <= exons[x]["end"]:
                ov = x; break
            x = exons[x]["next"]
        if ov is not None:
            break
        gap -= 1
    ok = ov is not None
    if imprecise and ((strand_fwd and ov == tr["last"]) or (not strand_fwd and ov == tr["first"]) or itd):
        ok = False
    if not ok:
        log.append("3:imprecise-not-snapped" if imprecise else "3:no-overlap")
        return seq, pos
    seq, pos = list(seq), list(pos)
    if imprecise:
        gap = bp + 1
        pos[gap] = exons[ov]["start"] if strand_fwd else exons[ov]["end"]
        seq[gap] = contig_seq[pos[gap]] if strand_fwd else comp(contig_seq[pos[gap]])
    s, p = [], []
    x = ov
    while x is not None:
        e = exons[x]
        q = max(e["start"], pos[gap] + 1) if strand_fwd else min(e["end"], pos[gap] - 1)
        while e["start"] <= q <= e["end"]:
            s.append(contig_seq[q] if strand_fwd else comp(contig_seq[q])); p.append(q)
            q += 1 if strand_fwd else -1
        if (strand_fwd and e["next"] is not None) or (not strand_fwd and e["prev"] is not None):
            s += ["_"] * 3; p += [-1] * 3
        x = e["next"] if strand_fwd else e["prev"]
    seq, pos = seq[:gap + 1] + ["("] + s + [")"], pos[:gap + 1] + [-1] + p + [-1]
    if imprecise:
        seq[bp + 1], seq[bp + 2] = seq[bp + 2], seq[bp + 1]
        pos[bp + 1], pos[bp + 2] = pos[bp + 2], pos[bp + 1]
    if (strand_fwd and pos[-2] == last["end"]) or (not strand_fwd and pos[-2] == first["start"]):
        seq, pos = seq + ["$"], pos + [-1]
        log.append("3:imprecise-snapped$" if imprecise else "3:filled$")
    else:
        log.append("3:imprecise-snapped" if imprecise else "3:filled")
    return "".join(seq), pos


def fill(seq, pos, t5, t3, strand5_fwd, strand3_fwd, itd, transcripts, exons, assembly, log=None):
    """The sequence and positions after filling with transcripts t5 / t3 (None: that side is left alone)."""
    log = [] if log is None else log
    pos = list(pos)
    if t5 is not None:
        tr = transcripts[t5]
        if tr["contig"] in assembly:
            seq, pos = _five(seq, pos, tr, exons, strand5_fwd, itd, assembly[tr["contig"]], log)
        else:
            log.append("5:no-sequence")
    if t3 is not None:
        tr = transcripts[t3]
        if tr["contig"] in assembly:
            seq, pos = _three(seq, pos, tr, exons, strand3_fwd, itd, assembly[tr["contig"]], log)
        else:
            log.append("3:no-sequence")
    return seq, pos
