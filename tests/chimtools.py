"""Test infrastructure: turns a world's BAM (STAR --chimOutType WithinBAM) into the pair STAR writes with --chimOutType SeparateSAMold -- the chimeric
alignments in a file of their own (Chimeric.out.sam, given with -c) and everything else in the main file (-x) -- in plain Python on top of bamtools.py.

A read's records (one key: name and HI) are chimeric when one of them is supplementary (0x800), a discordant mate or carries an SA tag. They go to the
-c file with 0x800 turned into 0x100 (Chimeric.out.sam marks the supplementary segment as secondary) and without SA and HI tags. Variants (`kinds`) bend
this to reach the reference's two-file rules (DESIGN.md section 5):
  hi          : the -c records keep an HI tag, with values other than 1 (the -c file's loop never reads it)
  both        : proper pairs that the main file turns into read-through fragments (`read_through`: their keys) are also copied into the -c file: the
                key is then in the map before the main file's read-through test, which cannot insert its fragment
  erased      : half of such copies made malformed, so that the first pass erases them again and the read-through fragment is inserted after all: a
                hard-clipped anchor, the pair twice (four alignments), or an unclipped secondary copy of a mate (a supplementary that overlaps its split read)
  single_end  : split reads rendered single-end (the mate dropped, pairing flags cleared), which the second pass rejects
  damage      : orphans (a mate dropped), 0x800 left as it is, mate-unmapped flags, and multimapping chimeric reads moved too (their keys collapse to ",1")
"""
import random, struct, zlib
import bamtools

BF_PAIRED, BF_PROPER, BF_MUNMAP, BF_READ1, BF_READ2, BF_MREVERSE, BF_SECONDARY, BF_SUPPLEMENTARY = 1, 2, 8, 64, 128, 32, 256, 2048
C_H = 5


def _hit(r):
    for tag, t, v in r["aux"]:
        if tag == b"HI" and t in (b"c", b"C", b"s", b"S", b"i", b"I"):
            return bamtools.aux_int_value(t, v)
    return 1


def _chimeric(recs):
    return any(r["flag"] & BF_SUPPLEMENTARY or (r["flag"] & BF_PAIRED and not r["flag"] & BF_PROPER) or any(a[0] == b"SA" for a in r["aux"]) for r in recs)


def _drop(r, *tags):
    r["aux"] = [a for a in r["aux"] if a[0] not in tags]


def split(src, kinds=(), seed=5, read_through=()):
    """-> (header text, refs, -c bodies, -x bodies, number of chimeric keys moved, names of the copied keys, names of the copies made malformed)"""
    rng = random.Random(seed)
    text, refs, bodies = bamtools.read_bam(src)
    keys = {}
    for i, b in enumerate(bodies):
        r = bamtools.split_record(b)
        keys.setdefault((r["qname"], _hit(r)), []).append(i)
    to_c, c_extra, moved, copied, erased = set(), [], 0, [], []
    for (name, hit), idx in keys.items():
        recs = [bamtools.split_record(bodies[i]) for i in idx]
        if any(r["tid"] < 0 for r in recs):
            continue
        if _chimeric(recs) and (hit == 1 or "damage" in kinds):
            to_c.update(idx); moved += 1
        elif "both" in kinds or "erased" in kinds:
            key = name.rstrip(b"\0").decode() + ",1"
            if len(idx) == 2 and all(r["flag"] & BF_PROPER and not r["flag"] & (BF_SECONDARY | BF_SUPPLEMENTARY) for r in recs) and hit == 1 and key in read_through:
                copies = [dict(r) for r in recs]
                copied.append(key)
                if "erased" in kinds and rng.random() < 0.5:
                    form = rng.randrange(3)
                    if form == 0:
                        c = copies[0]; c["cigar"] = struct.pack("<I", 5 << 4 | C_H) + c["cigar"]
                    elif form == 1:
                        copies += [dict(r) for r in recs]
                    else:
                        sec = dict(copies[rng.randrange(2)]); sec["flag"] |= BF_SECONDARY; copies.append(sec)
                    erased.append(key)
                for c in copies:
                    _drop(c, b"HI", b"SA")
                c_extra.append((idx[0], copies))
    c_bodies, x_bodies = [], []
    extra = dict(c_extra)
    for i, b in enumerate(bodies):
        if i in extra:
            c_bodies += [bamtools.join_record(c) for c in extra[i]]
        if i not in to_c:
            x_bodies.append(b); continue
        r = bamtools.split_record(b)
        if r["flag"] & BF_SUPPLEMENTARY and not ("damage" in kinds and rng.random() < 0.2):
            r["flag"] = (r["flag"] & ~BF_SUPPLEMENTARY) | BF_SECONDARY
        _drop(r, b"SA", b"HI")
        if "hi" in kinds:
            r["aux"].append((b"HI", b"i", struct.pack("<i", rng.choice([2, 3, 7]))))
        if "damage" in kinds:
            if r["flag"] & BF_PAIRED and rng.random() < 0.05:
                r["flag"] |= BF_MUNMAP
            if not r["flag"] & BF_SECONDARY and r["flag"] & BF_PAIRED and rng.random() < 0.04:
                continue  # an orphan: its mate waits until the end of the file and is dropped
        if "single_end" in kinds and r["flag"] & BF_PAIRED and zlib.crc32(r["qname"]) % 4 == 0:
            if r["flag"] & BF_READ2 and not r["flag"] & BF_SECONDARY:
                continue  # the mate is dropped, the rest becomes a single-end split read
            r["flag"] &= ~(BF_PAIRED | BF_PROPER | BF_MUNMAP | BF_MREVERSE | BF_READ1 | BF_READ2)
        c_bodies.append(bamtools.join_record(r))
    return text, refs, c_bodies, x_bodies, moved, copied, erased


def write_pair(src, c_path, x_path, kinds=(), seed=5, read_through=()):
    """writes the -c file (BAM) and the main file (BAM); returns the names of the copied keys and of the copies made malformed"""
    text, refs, c_bodies, x_bodies, _, copied, erased = split(src, kinds, seed, read_through)
    bamtools.write_bam(c_path, text, refs, c_bodies, random.Random(seed + 1))
    bamtools.write_bam(x_path, text, refs, x_bodies, random.Random(seed + 2))
    return copied, erased
