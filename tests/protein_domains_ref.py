"""Plain reference of protein domains (-p): a literal Python transcription of load_protein_domains and annotate_retained_protein_domains
(annotate_protein_domains.cpp:14-161) and of make_annotation_index (annotation.t.hpp:25-45), with the index as dicts of key -> set built in insertion order.
It walks the index key by key like the reference does (no multiplicities), and shares no code with the product."""
import gzip
from blacklist_ref import _str_to_int, _remove_chr, _tsv

M32 = 0xFFFFFFFF
UPSTREAM, DOWNSTREAM = 1, 0
CB_PSTRAND1, CB_PSTRAND2, CB_PSTRANDS_AMBIGUOUS, CB_TSTART_GENE1 = 16, 32, 64, 128
GF_DUMMY, GF_CODING = 1, 2


def _i32(v):
    v &= M32
    return v - (1 << 32) if v >= 1 << 31 else v


def strip_ensembl_version_number(s):  # annotation.hpp:27-33
    if s[:3] == "ENS" and "." in s:
        return s[:s.rfind(".")]
    return s


def get_gff3_attribute(attributes, name, warnings):  # :14-31
    start = attributes.find(name + "=")
    if start < 0:
        warnings.append("WARNING: failed to extract %s from line in GFF3 file: %s" % (name, attributes))
        return None
    start += len(name) + 1
    end = attributes.find(";", start)
    if end < 0:
        end = len(attributes)
    return attributes[start:end]


def _hex(c):
    return c in "0123456789abcdefABCDEF"


def decode_name(name):  # :71-89
    pos = name.find("%")
    while 0 <= pos < len(name):
        if pos + 2 < len(name) and _hex(name[pos + 1]) and _hex(name[pos + 2]):
            name = name[:pos] + chr(int(name[pos + 1:pos + 3], 16)) + name[pos + 3:]
        pos = name.find("%", pos + 1)
    return "".join("_" if ord(ch) < 0x21 or ord(ch) > 0x7E or ch in ",|" else ch for ch in name)


def load_protein_domains(path, contigs, gene_ids, gene_by_name):
    """contigs: name without chr -> id; gene_ids: gene_id of every gene in annotation order ("" for dummy genes); gene_by_name: the GTF's name map.
    Returns (records as dicts with contig, start, end, gene, name; warning lines) or raises ValueError("failed to parse GFF3 file")."""
    by_id = {}
    for g, i in enumerate(gene_ids):
        by_id[strip_ensembl_version_number(i)] = g  # the last gene wins
    raw = gzip.open(path, "rb").read() if path.endswith(".gz") else open(path, "rb").read()
    lines = raw.decode("latin-1").split("\n")
    if lines and lines[-1] == "":
        lines.pop()
    records, warnings, unknown = [], [], set()
    for line in lines:
        if line.endswith("\r"):
            line = line[:-1]
        if not line or line[0] == "#":
            continue
        f = _tsv(line)
        ok = len(f) >= 9
        start = _str_to_int(f[3]) if len(f) > 3 else None
        end = _str_to_int(f[4]) if len(f) > 4 else None
        if not ok or start is None or end is None or f[0] == "" or f[6] == "" or f[8] == "":
            warnings.append("WARNING: failed to parse line in GFF3 file: " + line)
            continue
        contig, attributes = f[0], f[8]
        gene_name = get_gff3_attribute(attributes, "gene_name", warnings)
        if gene_name is None:
            continue
        gene_id = get_gff3_attribute(attributes, "gene_id", warnings)
        if gene_id is None:
            continue
        name = get_gff3_attribute(attributes, "Name", warnings)
        if name is None:
            continue
        c = contigs.get(_remove_chr(contig))
        if c is None:
            warnings.append("WARNING: unknown contig: " + contig)
            continue
        name = decode_name(name)
        gene = by_id.get(strip_ensembl_version_number(gene_id))
        if gene is None:
            gene = gene_by_name.get(gene_name)
            if gene is None:
                if gene_name + " " + gene_id not in unknown:
                    warnings.append("WARNING: unknown gene: %s %s" % (gene_name, gene_id))
                    unknown.add(gene_name + " " + gene_id)
                continue
        records.append({"contig": c, "start": _i32(start - 1), "end": _i32(end - 1), "gene": gene, "name": name})
    if not records:
        raise ValueError("failed to parse GFF3 file")
    return records, warnings


def make_annotation_index(records):
    """annotation.t.hpp:25-45: one dict per RECORD (the vector is resized to the number of records), key -> set of record indices."""
    index = [dict() for _ in records]

    def lower_bound(ix, k):
        keys = sorted(ix)
        for x in keys:
            if x >= k:
                return x
        return None

    for i, d in enumerate(records):
        ix = index[d["contig"]]
        for k in (d["end"], d["start"] - 1):
            lb = lower_bound(ix, k)
            if lb is None:
                ix.setdefault(k, set())
            else:
                ix[k] = set(ix[lb])
        keys = sorted(ix)
        j = keys.index(lower_bound(ix, d["end"]))
        while keys[j] >= d["start"]:
            ix[keys[j]].add(i)
            j -= 1
    return index


def annotate_retained_protein_domains(contig, breakpoint, predicted_strand, ambiguous, gene, direction, index, records, genes):
    """:123-161; genes: Pipeline.genes() (gene_start, gene_end, gene_strand, gene_flags)."""
    if not genes["gene_flags"][gene] & GF_CODING:
        return ""
    if ambiguous or predicted_strand != bool(genes["gene_strand"][gene]):
        return ""
    if contig >= len(index):
        return ""
    gs, ge = int(genes["gene_start"][gene]), int(genes["gene_end"][gene])
    acc = {}
    for k in sorted(index[contig]):
        if k < gs or k > ge:
            continue
        for i in index[contig][k]:
            d = records[i]
            if d["gene"] != gene:
                continue
            length = (d["end"] - d["start"] + 1) & M32
            retained = 0
            if direction == UPSTREAM and d["end"] >= breakpoint:
                retained = (d["end"] - max(d["start"], breakpoint) + 1) & M32
            elif direction == DOWNSTREAM and d["start"] <= breakpoint:
                retained = (min(d["end"], breakpoint) - d["start"] + 1) & M32
            a = acc.setdefault(d["name"], [0, 0])
            a[0] = (a[0] + length) & M32
            a[1] = (a[1] + retained) & M32
    parts = []
    for name in sorted(acc):  # code points of latin-1 text: bytewise order
        length, retained = acc[name]
        if retained:
            parts.append("%s(%d%%)" % (name, ((retained * 100) & M32) // length))
    return ",".join(parts)


def column(cand, k, index, records, genes):
    """The retained_protein_domains column of candidate k (output_fusions.cpp:1183-1190), after the 5'/3' swap of the other columns."""
    bits = int(cand["bits"][k])
    s = (1, 2) if bits & CB_TSTART_GENE1 else (2, 1)
    ambiguous = bool(bits & CB_PSTRANDS_AMBIGUOUS)
    out = []
    for w in s:
        strand = bool(bits & (CB_PSTRAND1 if w == 1 else CB_PSTRAND2))
        out.append(annotate_retained_protein_domains(int(cand["contig%d" % w][k]), int(cand["breakpoint%d" % w][k]), strand, ambiguous, int(cand["gene%d" % w][k]),
                                                     int(cand["direction%d" % w][k]), index, records, genes))
    return out[0] + "|" + out[1] if out[0] or out[1] else "."
