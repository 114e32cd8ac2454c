"""SAM text input (-x FILE.sam, plain or BGZF): a SAM file S that means BAM file B under the rules of DESIGN.md section 5 must give what the oracle gives on B
-- the fragment table, the coverage windows and the later front-end stages (against the oracle's stage dumps of B), both output files, the WARNING lines
and the progress lines, and the same error texts. The SAM files are rendered from the BAM files by tests/samtext.py."""
import os, gzip, random, struct, subprocess, sys
import numpy as np
import pytest
import bamtools, samtext, worldutil
from arriba_b200 import lib as L, _build
from test_ingest import frag_tables_equal
from test_genomic_support import ZCHR, L151, sv_file
from test_blacklist import blacklist_file
from test_known_fusions import rules_file
from test_protein_domains import domains_file
from test_events import CFG5

WORLDS = {"small": {}, "l151": L151, "zchr": ZCHR, "cfg5": CFG5}
BF_UNMAP, BF_SECONDARY, BF_SUPPLEMENTARY = 4, 256, 2048
_SAM = {}


def world(worlds, name):
    return worlds.get(name, **WORLDS[name])


def sam_of(w, variant="plain"):
    """the SAM rendering of the world's BAM: plain or "bgzf", "crlf", "nolf" (no LF after the last line), "longheader" (@HD/@RG/@PG/@CO lines and
    @SQ lines with more fields, 20 kB of header); variants combine with "_" """
    key = (w.prefix, variant)
    if key not in _SAM:
        header, lines, _, _ = samtext.bam_to_sam_lines(w.prefix + ".bam")
        parts = variant.split("_")
        if "longheader" in parts:
            sq = [l + "\tAS:synthetic\tM5:0123456789abcdef0123456789abcdef" if l.startswith("@SQ") else l for l in header if not l.startswith("@HD")]
            header = ["@HD\tVN:1.6\tSO:unsorted"] + sq + ["@RG\tID:rg1\tSM:sample", "@PG\tID:star\tPN:STAR\tCL:STAR --chimOutType WithinBAM"] + ["@CO\tcomment %d HI:i:7 SA:Z:x" % k + "x" * 150 for k in range(120)]
        data = samtext.render(header + lines, "\r\n" if "crlf" in parts else "\n", "nolf" not in parts)
        path = w.prefix + "_" + variant + ".sam"
        if "bgzf" in parts:
            samtext.write_bgzf(path, data)
        else:
            open(path, "wb").write(data)
        _SAM[key] = path
    return _SAM[key]


def check_front_end_sam(w, path, lib_path, threads):
    """check_front_end of test_ingest.py with the input file given: table, coverage windows, strandedness, labels and candidates"""
    p = L.Pipeline(path, w.prefix + ".gtf", w.prefix + ".fa", threads=threads, lib_path=lib_path)
    p.step(L.STEP_LOAD_REFERENCE)
    p.step(L.STEP_INGEST)
    st = p.stats()
    rca = w.stage("read_chimeric_alignments")
    assert st.mapped_reads == int(rca["mapped_reads"][0])
    assert st.n_fragments == int(rca["total"][0])
    frag_tables_equal(p.fragments(), w.stage("ingest"), check_genes=False, check_pred=False)
    off = rca["coverage_off"]
    for c in range(len(off) - 1):
        cov, starts, ends = p.coverage(c)
        assert np.array_equal(cov, rca["coverage"][off[c]:off[c + 1]]), ("coverage", c)
        assert np.array_equal(starts, rca["fragment_starts"][off[c]:off[c + 1]]), ("starts", c)
        assert np.array_equal(ends, rca["fragment_ends"][off[c]:off[c + 1]]), ("ends", c)
    p.step(L.STEP_ANNOTATE)
    assert p.stats().strandedness == int(w.stage("strandedness")["strandedness"][0])
    frag_tables_equal(p.fragments(), w.stage("annotated"), check_genes=True, check_pred=True)
    p.step(L.STEP_UPLOAD); p.step(L.STEP_READ_FILTERS); p.step(L.STEP_FRAGMENT_LENGTH)
    labels, _ = p.context().fragment_filters()
    assert np.array_equal(labels, w.stage("rf_low_entropy")["frag_filter"])
    ff = w.stage("find_fusions")
    assert p.stats().max_mate_gap == int(ff["max_mate_gap"][0])
    p.step(L.STEP_FIND_FUSIONS)
    cand = p.context().candidates()
    assert cand["n"] == len(ff["gene1"])
    assert int((cand["filter"] == 0).sum()) == int(ff["remaining"][0])
    p.close()


FRONT_END = [  # world, rendering, threads, test hooks
    ("small", "plain", 1, {}), ("small", "bgzf", 1, {}), ("small", "crlf", 3, {}), ("small", "nolf", 1, {"ARB_CHUNK_BYTES": "1"}),
    ("small", "longheader_crlf_nolf", 2, {"ARB_CHUNK_BYTES": "300"}), ("small", "longheader_bgzf", 4, {"ARB_CHUNK_BYTES": "300"}),
    ("small", "plain", 2, {"ARB_KEY_HASH_BITS": "4"}), ("l151", "plain", 5, {}), ("l151", "crlf_bgzf_nolf", 5, {"ARB_CHUNK_BYTES": "70000"}),
    ("zchr", "plain", 3, {"ARB_KEY_HASH_BITS": "4"}), ("zchr", "bgzf", 1, {}),
]


@pytest.mark.parametrize("name,variant,threads,hooks", FRONT_END, ids=lambda x: x if isinstance(x, str) else str(x) if isinstance(x, int) else "-".join("%s=%s" % kv for kv in x.items()) or "default")
def test_front_end_sam_hostsim(worlds, hostsim_lib, monkeypatch, name, variant, threads, hooks):
    for k, v in hooks.items():
        monkeypatch.setenv(k, v)
    w = world(worlds, name)
    check_front_end_sam(w, sam_of(w, variant), hostsim_lib, threads)


# ---- single-record rules: a SAM file with one line changed against the BAM it means
def fragment_records(bodies):
    """indices of the records of a paired read with a proper primary pair, no secondaries, mapped, with HI"""
    by_name = {}
    for i, b in enumerate(bodies):
        by_name.setdefault(bamtools.split_record(b)["qname"], []).append(i)
    for idx in by_name.values():
        recs = [bamtools.split_record(bodies[i]) for i in idx]
        if len(idx) >= 2 and all(r["tid"] >= 0 and not r["flag"] & (BF_UNMAP | BF_SECONDARY) for r in recs) and any(t == b"HI" for t, _, _ in recs[0]["aux"]):
            yield idx


def retag(r, tag, t=None, v=None):
    """drops every `tag` and, with a type, adds it again as the first field"""
    r["aux"] = ([(tag, t, v)] if t else []) + [a for a in r["aux"] if a[0] != tag]


def sam_line_with(line, field, value):
    f = line.split("\t"); f[field] = value
    return "\t".join(f)


# name: (what the line becomes (fields -> fields), what the BAM record becomes (split record, modified in place) or None for an error, the error text)
def _rules():
    def unmapped_pos0(r): r["flag"] |= BF_UNMAP; r["pos"] = -1
    def unmapped_no_cigar(r): r["flag"] |= BF_UNMAP; r["cigar"] = b""
    def unknown_rname(r): r["flag"] |= BF_UNMAP; r["tid"] = -1
    def hi_z(r): retag(r, b"HI", b"Z", b"x\0")
    def hi_f(r): retag(r, b"HI", b"f", struct.pack("<f", 2.0))
    def secondary_no_hi(r): r["flag"] |= BF_SECONDARY; retag(r, b"HI")
    def odd_base(r): s = bytearray(r["seq"]); s[0] = (s[0] & 0x0F) | 0xF0; r["seq"] = bytes(s)
    return {
        "unknown_rname": (lambda f: sam_line_with(f, 2, "no_such_contig"), unknown_rname, None),
        "mapped_pos0": (lambda f: sam_line_with(f, 3, "0"), unmapped_pos0, None),
        "mapped_cigar_star": (lambda f: sam_line_with(f, 5, "*"), unmapped_no_cigar, None),
        "hi_z": (lambda f: "\t".join([x for x in f.split("\t") if not x.startswith("HI:")] + ["HI:Z:x"]), hi_z, None),
        "hi_f": (lambda f: "\t".join(f.split("\t")[:11] + ["HI:f:2"] + [x for x in f.split("\t")[11:] if not x.startswith("HI:")]), hi_f, None),
        "secondary_without_hi": (lambda f: "\t".join(sam_line_with(f, 1, str(int(f.split("\t")[1]) | BF_SECONDARY)).split("\t")[:11] + [x for x in f.split("\t")[11:] if not x.startswith("HI:")]), secondary_no_hi, None),
        "odd_base": (lambda f: sam_line_with(f, 9, "." + f.split("\t")[9][1:]), odd_base, None),
        "qual_length": (lambda f: sam_line_with(f, 10, f.split("\t")[10] + "I" if f.split("\t")[10] != "*" else "II"), None, "failed to load alignments"),
        "short_line": (lambda f: "\t".join(f.split("\t")[:10]), None, "failed to load alignments"),
        "empty_line": (lambda f: "", None, "failed to load alignments"),
        "bad_flag": (lambda f: sam_line_with(f, 1, "70000"), None, "failed to load alignments"),
        "bad_flag_text": (lambda f: sam_line_with(f, 1, "0x41"), None, "failed to load alignments"),
        "bad_cigar": (lambda f: sam_line_with(f, 5, f.split("\t")[5] + "5"), None, "failed to load alignments"),
        "bad_cigar_op": (lambda f: sam_line_with(f, 5, "10Q" + f.split("\t")[5]), None, "failed to load alignments"),
        "zero_length_op": (lambda f: sam_line_with(f, 5, "0S" + f.split("\t")[5]), None, "failed to load alignments"),
        "long_name": (lambda f: sam_line_with(f, 0, "n" * 255), None, "failed to load alignments"),
        "bad_tag": (lambda f: f + "\tX:i:1", None, "failed to load alignments"),
        "bad_tag_type": (lambda f: f + "\tXX:q:1", None, "failed to load alignments"),
        "bad_hi_value": (lambda f: "\t".join(f.split("\t")[:11] + ["HI:i:3000000000"] + f.split("\t")[11:]), None, "failed to load alignments"),
    }


RULES = _rules()


@pytest.fixture(scope="module")
def rule_base(worlds):
    w = world(worlds, "small")
    header, lines, refs, bodies = samtext.bam_to_sam_lines(w.prefix + ".bam")
    text = bamtools.read_bam(w.prefix + ".bam")[0]
    idx = list(fragment_records(bodies))
    return w, header, lines, refs, bodies, text, idx


def rule_case(base, root, name, k=0):
    """the SAM file and (for a meaning) the world of the BAM it means, with the rule applied to a record of the k-th suitable read"""
    w, header, lines, refs, bodies, text, idx = base
    i = idx[len(idx) // 3 + k][0]
    line_of, bam_of, _ = RULES[name]
    lines = list(lines); lines[i] = line_of(lines[i])
    d = os.path.join(root, name); os.makedirs(d, exist_ok=True)
    sam = os.path.join(d, "w.sam"); open(sam, "wb").write(samtext.render(header + lines))
    if bam_of is None:
        return sam, None
    r = bamtools.split_record(bodies[i]); bam_of(r)
    prefix = os.path.join(d, "w")
    for ext in (".fa", ".gtf"):
        os.symlink(os.path.realpath(w.prefix + ext), prefix + ext)
    bamtools.write_bam(prefix + ".bam", text, refs, bodies[:i] + [bamtools.join_record(r)] + bodies[i + 1:], random.Random(3))
    worldutil.run_oracle(prefix, os.path.join(d, "oracle"), dump=False)
    return sam, worldutil.World(prefix, os.path.join(d, "oracle"))


def run_outputs(path, w, lib_path, tmp, threads=2):
    out, disc = os.path.join(tmp, "fusions.tsv"), os.path.join(tmp, "fusions.discarded.tsv")
    p = L.Pipeline(path, w.prefix + ".gtf", w.prefix + ".fa", threads=threads, lib_path=lib_path, output=out, discarded=disc)
    try:
        p.run_all()
    finally:
        p.close()
    return open(out, "rb").read(), open(disc, "rb").read()


def ingest_error(path, w, lib_path, threads=2):
    p = L.Pipeline(path, w.prefix + ".gtf", w.prefix + ".fa", threads=threads, lib_path=lib_path)
    p.step(L.STEP_LOAD_REFERENCE)
    with pytest.raises(L.ArbError) as err:
        p.step(L.STEP_INGEST)
    p.close()
    return str(err.value)


def check_rule(base, root, name, lib_path, tmp):
    sam, meaning = rule_case(base, root, name)
    if meaning is None:
        assert RULES[name][2] in ingest_error(sam, base[0], lib_path), name
        return
    fus, disc = run_outputs(sam, meaning, lib_path, tmp)
    assert fus == open(os.path.join(meaning.outdir, "fusions.tsv"), "rb").read(), name
    assert disc == open(os.path.join(meaning.outdir, "fusions.discarded.tsv"), "rb").read(), name


@pytest.mark.parametrize("name", sorted(RULES))
def test_rule_hostsim(rule_base, hostsim_lib, tmp_path_factory, tmp_path, name):
    check_rule(rule_base, str(tmp_path_factory.mktemp("rule")), name, hostsim_lib, str(tmp_path))


def test_sq_without_length_hostsim(rule_base, hostsim_lib, tmp_path):
    w, header, lines = rule_base[:3]
    for bad in ("@SQ\tSN:extra", "@SQ\tLN:100", "@SQ\tSN:extra\tLN:0", "@SQ\tSN:extra\tLN:12x"):
        path = str(tmp_path / "h.sam"); open(path, "wb").write(samtext.render(header + [bad] + lines))
        assert ingest_error(path, w, hostsim_lib) == "failed to read SAM header", bad


def test_damage_that_bam_can_hold_hostsim(rule_base, hostsim_lib, tmp_path):
    """A CIGAR that consumes more bases than SEQ holds, and an alignment past its contig's end, give the texts the BAM path gives on the same damage;
    of two such lines the earlier one is reported, also when the later one sits in an earlier chunk's neighbourhood (small chunks)."""
    w, header, lines, refs, bodies, text, idx = rule_base
    a, b = idx[len(idx) // 4][0], idx[len(idx) // 2][0]
    def damage(i, kind):
        r = bamtools.split_record(bodies[i])
        if kind == "cigar":
            r["cigar"] = struct.pack("<I", (r["l_seq"] + 5) << 4)
        else:
            r["pos"] = refs[r["tid"]][1] - 3
        return r
    for first, second in (("cigar", "beyond"), ("beyond", "cigar")):
        ra, rb = damage(a, first), damage(b, second)
        new_bodies = list(bodies); new_bodies[a] = bamtools.join_record(ra); new_bodies[b] = bamtools.join_record(rb)
        prefix = str(tmp_path / ("d_" + first))
        bamtools.write_bam(prefix + ".bam", text, refs, new_bodies, random.Random(5))
        new_lines = list(lines); new_lines[a] = "\t".join(samtext.record_fields(new_bodies[a], refs)); new_lines[b] = "\t".join(samtext.record_fields(new_bodies[b], refs))
        open(prefix + ".sam", "wb").write(samtext.render(header + new_lines))
        want = ingest_error(prefix + ".bam", w, hostsim_lib)
        assert ra["qname"].rstrip(b"\0").decode() in want
        for hooks in ({}, {"ARB_CHUNK_BYTES": "300"}):
            os.environ.update(hooks)
            try:
                assert ingest_error(prefix + ".sam", w, hostsim_lib) == want, (first, hooks)
            finally:
                for k in hooks:
                    del os.environ[k]


def test_unreadable_line_before_a_bad_cigar_hostsim(rule_base, hostsim_lib, tmp_path):
    """an unreadable line is an error at its own position: before a later CIGAR error it wins, after it it does not"""
    w, header, lines, refs, bodies, text, idx = rule_base
    a, b = idx[len(idx) // 4][0], idx[len(idx) // 2][0]
    r = bamtools.split_record(bodies[b]); r["cigar"] = struct.pack("<I", (r["l_seq"] + 5) << 4)
    cigar_line = "\t".join(samtext.record_fields(bamtools.join_record(r), refs))
    unreadable = "\t".join(lines[a].split("\t")[:10])
    for unreadable_first in (True, False):
        new = list(lines)
        new[a], new[b] = (unreadable, cigar_line) if unreadable_first else (cigar_line, unreadable)
        path = str(tmp_path / "u.sam"); open(path, "wb").write(samtext.render(header + new))
        msg = ingest_error(path, w, hostsim_lib)
        assert msg == "failed to load alignments" if unreadable_first else msg.startswith("CIGAR string of read"), msg


def test_renderings_that_must_not_matter_hostsim(worlds, hostsim_lib, tmp_path):
    """tags in every order and type (HI retyped, before or after decoys such as XH:Z:HI:i:5, SA inside strings), lowercase SEQ, '=' bases, '*' QUAL,
    extra header lines: the product on the SAM equals the oracle on the BAM that holds the same records (with the '=' bases)"""
    w = world(worlds, "small")
    text, refs, bodies = bamtools.read_bam(w.prefix + ".bam")
    rng = random.Random(17)
    new_bodies, new_lines = [], []
    for b in bodies:
        r = bamtools.split_record(bamtools.transcode_record(b, rng))
        if rng.random() < 0.05 and r["l_seq"] > 4:
            s = bytearray(r["seq"]); s[1] &= 0x0F; r["seq"] = bytes(s)   # base 2 becomes '=' (nt16 code 0)
        if rng.random() < 0.3:
            r["aux"] = [(b"XH", b"Z", b"HI:i:5\0"), (b"XS", b"Z", b"SA:Z:1,2,+,5M,1,1;\0")] + r["aux"]
        body = bamtools.join_record(r); new_bodies.append(body)
        f = samtext.record_fields(body, refs)
        if rng.random() < 0.3:
            f[9] = f[9].lower()
        if rng.random() < 0.3:
            f[10] = "*"
        new_lines.append("\t".join(f))
    d = str(tmp_path); prefix = os.path.join(d, "w")
    for ext in (".fa", ".gtf"):
        os.symlink(os.path.realpath(w.prefix + ext), prefix + ext)
    bamtools.write_bam(prefix + ".bam", text, refs, new_bodies, random.Random(2))
    worldutil.run_oracle(prefix, os.path.join(d, "oracle"))
    meaning = worldutil.World(prefix, os.path.join(d, "oracle"))
    header = ["@HD\tVN:1.6"] + ["@SQ\tSN:%s\tLN:%d\tUR:file:x.fa" % r for r in refs] + ["@RG\tID:a", "@PG\tID:p\tPN:x", "@CO\tHI:i:1"]
    open(prefix + ".sam", "wb").write(samtext.render(header + new_lines))
    check_front_end_sam(meaning, prefix + ".sam", hostsim_lib, 3)
    fus, disc = run_outputs(prefix + ".sam", meaning, hostsim_lib, d)
    assert fus == open(os.path.join(meaning.outdir, "fusions.tsv"), "rb").read()
    assert disc == open(os.path.join(meaning.outdir, "fusions.discarded.tsv"), "rb").read()


# ---- format detection
def test_formats_refused_with_their_errors_hostsim(worlds, hostsim_lib, tmp_path):
    w = world(worlds, "small")
    sam = open(sam_of(w), "rb").read()
    cases = {"gzip": (gzip.compress(sam[:200000]), "gzip-compressed SAM must be BGZF (bgzip) or uncompressed"),
             "cram": (b"CRAM\x03\x00" + bytes(range(256)) * 4, "CRAM input is not supported"),
             "binary": (bytes(range(256)) * 16, "failed to read SAM header")}
    for name, (data, text) in cases.items():
        path = str(tmp_path / (name + ".x")); open(path, "wb").write(data)
        assert text in ingest_error(path, w, hostsim_lib), name


# ---- the command line
def warnings_of(text):
    """the warnings the product prints as the reference does: those of the input files (as the other CLI parity tests compare them) and of the ingest"""
    return [l for l in text.splitlines() if l.startswith(("WARNING: failed to", "WARNING: unknown contig", "WARNING: unknown gene", "WARNING: encountered"))
            or (l.startswith("WARNING: ") and ("SAM records were malformed" in l or "secondary alignments lack" in l))]


def progress_of(text):
    """the progress lines without the input paths and the closing line's clocks"""
    return [l.split("] ", 1)[1].split(" '")[0].strip() for l in text.splitlines() if "] " in l and l.startswith("[") and "] Done (elapsed" not in l]


def cli_parity(cli, w, sam, args, tmp):
    """both files and the warnings equal the oracle's on the BAM; the progress lines equal the product's own on the BAM (input path aside)"""
    ref = os.path.join(tmp, "oracle"); worldutil.run_oracle(w.prefix, ref, dump=False, args=args)
    runs = {}
    for kind, path in (("sam", sam), ("bam", w.prefix + ".bam")):
        d = os.path.join(tmp, kind); os.makedirs(d)
        r = subprocess.run([cli, "-x", path, "-g", w.prefix + ".gtf", "-a", w.prefix + ".fa", "-o", os.path.join(d, "fusions.tsv"), "-O", os.path.join(d, "fusions.discarded.tsv"),
                            "-@", "3"] + list(args), capture_output=True, text=True, timeout=900, encoding="latin-1")
        assert r.returncode == 0, r.stderr[-2000:]
        runs[kind] = r
    for f in ("fusions.tsv", "fusions.discarded.tsv"):
        assert open(os.path.join(tmp, "sam", f), "rb").read() == open(os.path.join(ref, f), "rb").read(), (f, args)
    assert warnings_of(runs["sam"].stderr) == warnings_of(open(os.path.join(ref, "stderr.txt"), encoding="latin-1").read())
    assert progress_of(runs["sam"].stdout) == progress_of(runs["bam"].stdout)


@pytest.fixture(scope="module")
def cli():
    return _build.build_cli_hostsim()


@pytest.mark.parametrize("name,variant,args", [("small", "plain", ("-f", "blacklist")), ("small", "bgzf", ("-f", "blacklist", "-X")), ("cfg5", "plain", ("-f", "blacklist"))])
def test_cli_parity_hostsim(worlds, cli, tmp_path, name, variant, args):
    w = world(worlds, name)
    cli_parity(cli, w, sam_of(w, variant), args, str(tmp_path))


def test_cli_parity_with_every_input_file_hostsim(worlds, cli, hostsim_lib, tmp_path_factory, tmp_path):
    w = world(worlds, "small")
    root = str(tmp_path_factory.mktemp("files"))
    args = ("-b", blacklist_file(w, hostsim_lib, root), "-k", rules_file(w, hostsim_lib, root, False), "-t", rules_file(w, hostsim_lib, root, True),
            "-p", domains_file(w, hostsim_lib, root), "-d", sv_file(w, hostsim_lib, root))
    cli_parity(cli, w, sam_of(w, "crlf"), args, str(tmp_path))


WORKER = r"""
import os, sys
sys.path.insert(0, {root!r})
import torch.distributed as dist
from arriba_b200 import lib as L, sharded
rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"])
dist.init_process_group("gloo")
out = os.path.join({outdir!r}, "rank%d" % rank); os.makedirs(out, exist_ok=True)
p = L.Pipeline({sam!r}, {prefix!r} + ".gtf", {prefix!r} + ".fa", threads=2, lib_path={lib!r},
               output=os.path.join(out, "fusions.tsv"), discarded=os.path.join(out, "fusions.discarded.tsv"))
sharded.run_sharded(p, rank, world)
p.close()
dist.destroy_process_group()
"""


def test_sharded_two_ranks_hostsim(worlds, hostsim_lib, tmp_path):
    w = world(worlds, "small")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = str(tmp_path / "worker.py")
    open(script, "w").write(WORKER.format(root=root, outdir=str(tmp_path), sam=sam_of(w, "bgzf"), prefix=w.prefix, lib=hostsim_lib))
    env = dict(os.environ, PYTHONPATH=root + os.pathsep + os.path.join(root, "tests"))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port", str(29700 + os.getpid() % 200), script]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    for f in ("fusions.tsv", "fusions.discarded.tsv"):
        assert open(os.path.join(tmp_path, "rank0", f), "rb").read() == open(os.path.join(w.outdir, f), "rb").read(), f


# ---- on the H100
GPU_FRONT_END = [("small", "plain", {}), ("small", "bgzf", {}), ("small", "plain", {"ARB_CHUNK_BYTES": "300"}), ("small", "bgzf", {"ARB_CHUNK_BYTES": "1"}),
                 ("l151", "plain", {}), ("l151", "crlf_bgzf", {}), ("l151", "nolf", {"ARB_CHUNK_BYTES": "70000"})]


@pytest.mark.gpu
@pytest.mark.parametrize("name,variant,hooks", GPU_FRONT_END, ids=lambda x: x if isinstance(x, str) else "-".join("%s=%s" % kv for kv in x.items()) or "default")
def test_front_end_sam_cuda(worlds, cuda_lib, monkeypatch, name, variant, hooks):
    for k, v in hooks.items():
        monkeypatch.setenv(k, v)
    w = world(worlds, name)
    check_front_end_sam(w, sam_of(w, variant), cuda_lib, 8)


@pytest.mark.gpu
@pytest.mark.parametrize("name,variant", [("small", "plain"), ("l151", "bgzf")])
def test_outputs_sam_cuda(worlds, cuda_lib, tmp_path, name, variant):
    w = world(worlds, name)
    fus, disc = run_outputs(sam_of(w, variant), w, cuda_lib, str(tmp_path), threads=8)
    assert fus == open(os.path.join(w.outdir, "fusions.tsv"), "rb").read()
    assert disc == open(os.path.join(w.outdir, "fusions.discarded.tsv"), "rb").read()


@pytest.mark.gpu
def test_rules_cuda(rule_base, cuda_lib, tmp_path_factory, tmp_path):
    root = str(tmp_path_factory.mktemp("rule"))
    for name in sorted(RULES):
        d = os.path.join(str(tmp_path), name); os.makedirs(d)
        check_rule(rule_base, root, name, cuda_lib, d)
