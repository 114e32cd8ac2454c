"""Test infrastructure: BAM records rendered as SAM text (SAMv1 section 1.4), in plain Python that shares no code with the product's parser. The rendering
keeps what the reference reads (FLAG, RNAME, POS, CIGAR, SEQ, QNAME, HI, SA) and writes every other field in whatever form the caller picks, so that
a SAM file S can be checked against a BAM file B that must mean the same."""
import struct
import bamtools

CIGAR_OPS = "MIDNSHP=X"
NT16 = "=ACMGRSVTWYHKDBN"


def aux_text(tag, t, v):
    """one BAM aux field as SAM text"""
    tag = tag.decode()
    if t == b"A":
        return "%s:A:%s" % (tag, chr(v[0]))
    if t in (b"c", b"C", b"s", b"S", b"i", b"I"):
        return "%s:i:%d" % (tag, bamtools.aux_int_value(t, v))
    if t == b"f":
        return "%s:f:%g" % (tag, struct.unpack("<f", v)[0])
    if t in (b"Z", b"H"):
        return "%s:%s:%s" % (tag, t.decode(), v[:-1].decode("latin-1"))
    if t == b"B":
        sub = v[:1]; cnt = struct.unpack_from("<I", v, 1)[0]
        fmt = {b"c": "b", b"C": "B", b"s": "h", b"S": "H", b"i": "i", b"I": "I", b"f": "f"}[sub]
        vals = struct.unpack_from("<%d%s" % (cnt, fmt), v, 5)
        return "%s:B:%s" % (tag, ",".join([sub.decode()] + ["%g" % x if fmt == "f" else str(x) for x in vals]))
    raise ValueError(t)


def record_fields(body, refs):
    """the SAM fields of one BAM record body (a list of strings: the 11 mandatory fields, then the tags)"""
    r = bamtools.split_record(body)
    ops = struct.unpack("<%dI" % (len(r["cigar"]) // 4), r["cigar"])
    cigar = "".join("%d%s" % (o >> 4, CIGAR_OPS[o & 15]) for o in ops) or "*"
    seq = "".join(NT16[(r["seq"][i >> 1] >> (4 * (1 - (i & 1)))) & 15] for i in range(r["l_seq"])) or "*"
    qual = "*" if not r["l_seq"] or r["qual"][0] == 0xFF else "".join(chr(q + 33) for q in r["qual"])
    rname = refs[r["tid"]][0] if r["tid"] >= 0 else "*"
    rnext = "*" if r["mtid"] < 0 else "=" if r["mtid"] == r["tid"] else refs[r["mtid"]][0]
    f = [r["qname"].rstrip(b"\0").decode(), str(r["flag"]), rname, str(r["pos"] + 1), str(r["mapq"]), cigar, rnext, str(r["mpos"] + 1), str(r["tlen"]), seq, qual]
    return f + [aux_text(*a) for a in r["aux"]]


def header_text(text, refs):
    """the @ lines: the BAM's own header text where it has @SQ lines, else @SQ lines from the reference list"""
    lines = [l for l in text.rstrip(b"\0").decode().split("\n") if l]
    if not any(l.startswith("@SQ\t") for l in lines):
        lines = [l for l in lines if l.startswith("@HD")] + ["@SQ\tSN:%s\tLN:%d" % (n, ln) for n, ln in refs] + [l for l in lines if not l.startswith("@HD")]
    return lines


def render(lines, newline="\n", final_newline=True):
    return (newline.join(lines) + (newline if final_newline else "")).encode("latin-1")


def bam_to_sam_lines(bam_path):
    """-> (header lines, record lines, refs, bodies)"""
    text, refs, bodies = bamtools.read_bam(bam_path)
    return header_text(text, refs), ["\t".join(record_fields(b, refs)) for b in bodies], refs, bodies


def write_bgzf(path, data, member=60000, level=6):
    with open(path, "wb") as f:
        for at in range(0, len(data), member):
            f.write(bamtools.bgzf_member(data[at: at + member], level))
        f.write(bamtools.EOF_BLOCK)
