"""A separate chimeric alignment file (-c Chimeric.out.sam, STAR --chimOutType SeparateSAMold): the pair that tests/chimtools.py splits from a world's
WithinBAM file must give what the oracle gives on the same pair -- the fragment table, the coverage windows and the later front-end stages (the oracle dumps
read_chimeric_alignments once per file: occurrence 0 is the -c file's call, 1 the final state), both output files, both WARNING lines and both progress
lines, and the errors in the reference's order."""
import os, random, re, shutil, struct, subprocess, sys
import numpy as np
import pytest
import bamtools, chimtools, samtext, worldutil
from arriba_b200 import lib as L, _build
from test_ingest import frag_tables_equal
from test_genomic_support import L151
from test_sam_input import warnings_of

WORLDS = {"small": {}, "l151": L151}
_PAIRS = {}
_COPIES = {}


def table(stage):
    """name -> number of alignments of the fragments of an oracle table dump"""
    names, off = bytes(stage["names"]), stage["name_off"]
    return {names[off[i]:off[i + 1]].decode(): int(stage["n_aln"][i]) for i in range(len(off) - 1)}


def pair(worlds, name, kinds=(), form="bam"):
    """(world of the -x file with the oracle run on the pair, path of the -c file in the given form: bam, sam or bgzf)"""
    w = worlds.get(name, **WORLDS[name])
    key = (w.prefix, tuple(kinds))
    if key not in _PAIRS:
        d = os.path.join(os.path.dirname(w.prefix), "chim_" + ("_".join(kinds) or "plain")); os.makedirs(d, exist_ok=True)
        prefix = os.path.join(d, "w")
        for ext in (".fa", ".gtf"):
            if not os.path.exists(prefix + ext):
                os.symlink(os.path.realpath(w.prefix + ext), prefix + ext)
        read_through = [k for k in table(w.stage("ingest")) if k.endswith(",1")]  # the WithinBAM run's fragments: read-through where the pair is not chimeric
        _COPIES[key] = chimtools.write_pair(w.prefix + ".bam", prefix + "_chimeric.bam", prefix + ".bam", kinds, read_through=set(read_through))
        worldutil.run_oracle(prefix, os.path.join(d, "oracle"), args=("-c", prefix + "_chimeric.bam", "-f", "blacklist"))
        _PAIRS[key] = worldutil.World(prefix, os.path.join(d, "oracle"))
    cw = _PAIRS[key]
    c = cw.prefix + "_chimeric.bam"
    if form != "bam":
        path = cw.prefix + "_chimeric_" + form + ".sam"
        if not os.path.exists(path):
            header, lines, _, _ = samtext.bam_to_sam_lines(c)
            data = samtext.render(header + lines)
            if form == "bgzf":
                samtext.write_bgzf(path, data, member=7000)
            else:
                open(path, "wb").write(data)
        c = path
    return cw, c


def check_front_end(w, c, lib_path, threads):
    p = L.Pipeline(w.prefix + ".bam", w.prefix + ".gtf", w.prefix + ".fa", threads=threads, lib_path=lib_path, chimeric=c)
    p.step(L.STEP_LOAD_REFERENCE)
    p.step(L.STEP_INGEST)
    st = p.stats()
    first, rca = w.stage("read_chimeric_alignments", 0), w.stage("read_chimeric_alignments", 1)
    assert st.chimeric_total == int(first["total"][0])
    assert st.mapped_reads == int(rca["mapped_reads"][0])
    assert st.n_fragments == int(rca["total"][0])
    frag_tables_equal(p.fragments(), w.stage("ingest"), check_genes=False, check_pred=False)
    off = rca["coverage_off"]
    for k in range(len(off) - 1):
        cov, starts, ends = p.coverage(k)
        assert np.array_equal(cov, rca["coverage"][off[k]:off[k + 1]]), ("coverage", k)
        assert np.array_equal(starts, rca["fragment_starts"][off[k]:off[k + 1]]), ("starts", k)
        assert np.array_equal(ends, rca["fragment_ends"][off[k]:off[k + 1]]), ("ends", k)
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
    return st


def totals(stdout):
    """the totals of the "Reading chimeric alignments" progress lines, in order"""
    return [int(m.group(1)) for m in re.finditer(r"Reading chimeric alignments from '[^']*' \(total=(\d+)\)", stdout)]


def cli_parity(cli, w, c, tmp, args=("-f", "blacklist")):
    r = subprocess.run([cli, "-c", c, "-x", w.prefix + ".bam", "-g", w.prefix + ".gtf", "-a", w.prefix + ".fa", "-o", os.path.join(tmp, "fusions.tsv"),
                        "-O", os.path.join(tmp, "fusions.discarded.tsv"), "-@", "3"] + list(args), capture_output=True, text=True, timeout=900, encoding="latin-1")
    assert r.returncode == 0, r.stderr[-2000:]
    for f in ("fusions.tsv", "fusions.discarded.tsv"):
        assert open(os.path.join(tmp, f), "rb").read() == open(os.path.join(w.outdir, f), "rb").read(), f
    ref_err = open(os.path.join(w.outdir, "stderr.txt"), encoding="latin-1").read()
    assert warnings_of(r.stderr) == warnings_of(ref_err)
    ref_out = open(os.path.join(w.outdir, "stdout.txt"), encoding="latin-1").read()
    assert len(totals(ref_out)) == 2 and totals(r.stdout) == totals(ref_out)
    return r


@pytest.fixture(scope="module")
def cli():
    return _build.build_cli_hostsim()


# world, variant, -c form, threads, test hooks
FRONT_END = [("small", (), "bam", 2, {}), ("small", ("hi",), "sam", 1, {}), ("small", ("both",), "bam", 3, {}), ("small", ("erased",), "bgzf", 2, {}),
             ("small", ("single_end",), "bam", 2, {}), ("small", ("damage",), "sam", 2, {}),
             ("small", ("erased", "single_end", "damage"), "bgzf", 3, {"ARB_CHUNK_BYTES": "3000"}),
             ("small", ("both", "erased"), "sam", 2, {"ARB_KEY_HASH_BITS": "4", "ARB_CHUNK_BYTES": "20000"}), ("l151", ("erased", "single_end"), "bam", 4, {})]


def _id(x):
    return "-".join(x) or "plain" if isinstance(x, tuple) else x if isinstance(x, str) else str(x) if isinstance(x, int) else "-".join("%s=%s" % kv for kv in x.items()) or "default"


@pytest.mark.parametrize("name,kinds,form,threads,hooks", FRONT_END, ids=_id)
def test_front_end_hostsim(worlds, hostsim_lib, monkeypatch, name, kinds, form, threads, hooks):
    for k, v in hooks.items():
        monkeypatch.setenv(k, v)
    w, c = pair(worlds, name, kinds, form)
    check_front_end(w, c, hostsim_lib, threads)


@pytest.mark.parametrize("name,kinds,form", [("small", (), "bam"), ("small", ("hi", "both"), "sam"), ("small", ("erased", "single_end", "damage"), "bgzf"),
                                             ("l151", ("single_end", "both"), "bam")], ids=_id)
def test_cli_parity_hostsim(worlds, cli, tmp_path, name, kinds, form):
    w, c = pair(worlds, name, kinds, form)
    cli_parity(cli, w, c, str(tmp_path))


def test_single_end_quirk_hostsim(worlds, hostsim_lib):
    """single-end -c fragments that the first pass kept are rejected by the second one, and counted in the second warning (DESIGN.md section 5)"""
    w, c = pair(worlds, "small", ("single_end",))
    warn = [l for l in open(os.path.join(w.outdir, "stderr.txt")).read().splitlines() if "SAM records were malformed" in l]
    assert len(warn) == 2
    st = check_front_end(w, c, hostsim_lib, 2)
    assert st.chimeric_malformed == int(warn[0].split()[1]) and st.malformed == int(warn[1].split()[1])
    assert st.chimeric_total > 0


def test_synth_separate_chimeric_hostsim(cli, tmp_path):
    """tools/synth.cpp --separate-chimeric writes the world as STAR's SeparateSAMold pair (the -c file as SAM text); the pair gives the oracle's outputs"""
    prefix = str(tmp_path / "w")
    worldutil.run_synth(prefix, extra=("--separate-chimeric",))
    _, refs, bodies = bamtools.read_bam(prefix + ".bam")
    _, _, x_bodies = bamtools.read_bam(prefix + ".Aligned.out.bam")
    c_lines = [l for l in open(prefix + ".Chimeric.out.sam") if not l.startswith("@")]
    assert len(c_lines) > 0 and len(x_bodies) > 0 and len(c_lines) + len(x_bodies) == len(bodies)
    assert all("\tSA:" not in l and "\tHI:" not in l and not int(l.split("\t")[1]) & 2048 for l in c_lines)
    d = str(tmp_path / "pair"); os.makedirs(d)
    pp = os.path.join(d, "w")
    for ext in (".fa", ".gtf"):
        os.symlink(prefix + ext, pp + ext)
    os.symlink(prefix + ".Aligned.out.bam", pp + ".bam")
    bamtools.write_bam(pp + "_chimeric.bam", b"", refs, [bamtools.join_record(samtext_record(l, refs)) for l in c_lines], random.Random(2))
    worldutil.run_oracle(pp, os.path.join(d, "oracle"), dump=False, args=("-c", pp + "_chimeric.bam", "-f", "blacklist"))
    cli_parity(cli, worldutil.World(pp, os.path.join(d, "oracle")), prefix + ".Chimeric.out.sam", str(tmp_path))


def samtext_record(line, refs):
    """a SAM line of synth's (integer and string tags only) as a split BAM record, for the oracle (which reads the -c file as BAM)"""
    f = line.rstrip("\n").split("\t")
    names = [n for n, _ in refs]
    ops = "MIDNSHP=X"
    cig = re.findall(r"(\d+)([MIDNSHP=X])", f[5]) if f[5] != "*" else []
    seq = f[9] if f[9] != "*" else ""
    nt = "=ACMGRSVTWYHKDBN"
    packed = bytearray((len(seq) + 1) // 2)
    for i, ch in enumerate(seq):
        packed[i // 2] |= nt.index(ch) << (0 if i & 1 else 4)
    aux = []
    for t in f[11:]:
        tag, typ, val = t.split(":", 2)
        aux.append((tag.encode(), b"C", struct.pack("<B", int(val))) if typ == "i" else (tag.encode(), b"Z", val.encode() + b"\0"))
    tid = names.index(f[2]) if f[2] != "*" else -1
    mtid = tid if f[6] == "=" else (names.index(f[6]) if f[6] != "*" else -1)
    return dict(tid=tid, pos=int(f[3]) - 1, mapq=int(f[4]), bin=0, flag=int(f[1]), l_seq=len(seq), mtid=mtid, mpos=int(f[7]) - 1, tlen=int(f[8]),
                qname=f[0].encode() + b"\0", cigar=b"".join(struct.pack("<I", int(n) << 4 | ops.index(o)) for n, o in cig), seq=bytes(packed),
                qual=bytes(ord(q) - 33 for q in f[10]) if f[10] != "*" else b"\xff" * len(seq), aux=aux)


def test_copied_keys_block_and_erased_keys_reinsert_hostsim(worlds, hostsim_lib):
    """The "both" and "erased" variants reach the rule they are for. A copied read-through pair that the first pass keeps blocks the main file's insert:
    where the WithinBAM run split the pair at an intron (3 alignments), the table now holds the unsplit copy (2). A copy the first pass erases leaves the
    name free, and the main file's read-through fragment takes it again (as in the WithinBAM run)."""
    base = worlds.get("small")
    within = table(base.stage("ingest"))
    for kinds in (("both",), ("erased",)):
        w, c = pair(worlds, "small", kinds)
        copied, erased = _COPIES[(base.prefix, kinds)]
        final = table(w.stage("ingest"))
        kept = [k for k in copied if k not in erased]
        blocked = [k for k in kept if within.get(k) == 3 and final.get(k) == 2]
        assert kept and blocked, kinds
        if erased:
            reinserted = [k for k in erased if k in final and final[k] == within[k]]
            assert reinserted, kinds
        check_front_end(w, c, hostsim_lib, 2)


# ---- errors, in the reference's order
def run_error(w, c, lib_path, x=None):
    p = L.Pipeline(x or w.prefix + ".bam", w.prefix + ".gtf", w.prefix + ".fa", threads=2, lib_path=lib_path, chimeric=c)
    p.step(L.STEP_LOAD_REFERENCE)
    with pytest.raises(L.ArbError) as err:
        p.step(L.STEP_INGEST)
    p.close()
    return str(err.value)


def oracle_error(w, c, tmp):
    with pytest.raises(RuntimeError) as err:
        worldutil.run_oracle(w.prefix, tmp, dump=False, args=("-c", c, "-f", "blacklist"))
    return str(err.value)


NO_CHIMERIC = "no split reads or discordant mates found"


def test_errors_hostsim(worlds, hostsim_lib, tmp_path):
    w, c = pair(worlds, "small")
    text, refs, c_bodies = bamtools.read_bam(c)
    rng = random.Random(1)
    # a -c file with a header only
    empty = str(tmp_path / "empty.bam"); bamtools.write_bam(empty, text, refs, [], rng)
    assert NO_CHIMERIC in run_error(w, empty, hostsim_lib)
    assert NO_CHIMERIC in oracle_error(w, empty, str(tmp_path / "o1"))
    # a -c record without a reference: undefined in the reference, an error that names the read here
    r = bamtools.split_record(c_bodies[len(c_bodies) // 2]); r["tid"] = -1
    bad = str(tmp_path / "unmapped.bam"); bamtools.write_bam(bad, text, refs, c_bodies[:5] + [bamtools.join_record(r)] + c_bodies[5:], rng)
    e = run_error(w, bad, hostsim_lib)
    assert "in the chimeric alignment file has no reference sequence" in e and r["qname"].rstrip(b"\0").decode() in e
    # a -c file without chimeric reads (one orphan mate) and a CIGAR that does not fit its sequence in the main file: the -c file's error comes first
    orphan = next(b for b in c_bodies if bamtools.split_record(b)["flag"] & 1 and not bamtools.split_record(b)["flag"] & 256)
    lone = str(tmp_path / "orphan.bam"); bamtools.write_bam(lone, text, refs, [orphan], rng)
    _, xrefs, x_bodies = bamtools.read_bam(w.prefix + ".bam")
    xr = bamtools.split_record(x_bodies[10]); xr["cigar"] = struct.pack("<I", (xr["l_seq"] + 5) << 4)
    xbad = str(tmp_path / "x_bad_cigar.bam"); bamtools.write_bam(xbad, text, xrefs, x_bodies[:10] + [bamtools.join_record(xr)] + x_bodies[11:], rng)
    assert NO_CHIMERIC in run_error(w, lone, hostsim_lib, x=xbad)
    assert "does not fit its sequence" in run_error(w, c, hostsim_lib, x=xbad)  # with chimeric reads in -c, the main file's error stands


def test_chimeric_call_ends_before_a_main_file_error_hostsim(worlds, cli, tmp_path):
    """a record error in the main file comes after the -c call's first warning and progress line, as the reference prints them before reading -x"""
    w, c = pair(worlds, "small", ("erased",))
    text, xrefs, x_bodies = bamtools.read_bam(w.prefix + ".bam")
    xr = bamtools.split_record(x_bodies[-10]); xr["cigar"] = struct.pack("<I", (xr["l_seq"] + 5) << 4)
    xbad = str(tmp_path / "x_bad_cigar.bam"); bamtools.write_bam(xbad, text, xrefs, x_bodies[:-10] + [bamtools.join_record(xr)] + x_bodies[-9:], random.Random(4))
    r = subprocess.run([cli, "-c", c, "-x", xbad, "-g", w.prefix + ".gtf", "-a", w.prefix + ".fa", "-o", str(tmp_path / "f.tsv"), "-f", "blacklist"],
                       capture_output=True, text=True, timeout=900, encoding="latin-1")
    assert r.returncode != 0
    ref_err = open(os.path.join(w.outdir, "stderr.txt"), encoding="latin-1").read()
    first_warning = [l for l in ref_err.splitlines() if "SAM records were malformed" in l][0]
    lines = [l for l in r.stderr.splitlines() if l.startswith(("WARNING", "ERROR"))]
    assert lines[0] == first_warning and lines[-1].startswith("ERROR: CIGAR string of read") and len(lines) == 2
    assert totals(r.stdout) == totals(open(os.path.join(w.outdir, "stdout.txt"), encoding="latin-1").read())[:1]


def test_cli_options_hostsim(worlds, cli, tmp_path):
    w, c = pair(worlds, "small")
    base = [cli, "-x", w.prefix + ".bam", "-g", w.prefix + ".gtf", "-a", w.prefix + ".fa", "-o", str(tmp_path / "f.tsv"), "-f", "blacklist"]
    r = subprocess.run(base + ["-c", str(tmp_path / "missing.sam")], capture_output=True, text=True)
    assert r.returncode != 0 and "ERROR: file not found/readable: " + str(tmp_path / "missing.sam") in r.stderr
    junction = str(tmp_path / "Chimeric.out.junction"); shutil.copy(c, junction)
    r = subprocess.run(base + ["-c", junction], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "WARNING: it seems you passed the chimeric junction file ('Chimeric.out.junction') to the parameter -c, but this parameter takes the chimeric alignments file ('Chimeric.out.sam') as input" in r.stderr
    assert open(tmp_path / "f.tsv", "rb").read() == open(os.path.join(w.outdir, "fusions.tsv"), "rb").read()
    u = subprocess.run([cli, "-h"], capture_output=True, text=True)
    assert "[-c Chimeric.out.sam]" in u.stdout


def test_runs_without_c_unchanged_hostsim(worlds, hostsim_lib, tmp_path):
    """no -c: the stats of the -c file stay zero (the outputs are checked by every other test of the suite)"""
    w = worlds.get("small")
    p = L.Pipeline(w.prefix + ".bam", w.prefix + ".gtf", w.prefix + ".fa", threads=2, lib_path=hostsim_lib)
    p.step(L.STEP_LOAD_REFERENCE); p.step(L.STEP_INGEST)
    st = p.stats()
    assert (st.chimeric_records, st.chimeric_malformed, st.chimeric_total) == (0, 0, 0)
    assert st.n_fragments == int(w.stage("read_chimeric_alignments")["total"][0])
    p.close()


WORKER = r"""
import os, sys
sys.path.insert(0, {root!r})
import torch.distributed as dist
from arriba_b200 import lib as L, sharded
rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"])
dist.init_process_group("gloo")
out = os.path.join({outdir!r}, "rank%d" % rank); os.makedirs(out, exist_ok=True)
p = L.Pipeline({prefix!r} + ".bam", {prefix!r} + ".gtf", {prefix!r} + ".fa", threads=2, lib_path={lib!r}, chimeric={chim!r},
               output=os.path.join(out, "fusions.tsv"), discarded=os.path.join(out, "fusions.discarded.tsv"))
sharded.run_sharded(p, rank, world)
p.close()
dist.destroy_process_group()
"""


def test_sharded_two_ranks_hostsim(worlds, hostsim_lib, tmp_path):
    w, c = pair(worlds, "small", ("both", "single_end"), "sam")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = str(tmp_path / "worker.py")
    open(script, "w").write(WORKER.format(root=root, outdir=str(tmp_path), prefix=w.prefix, chim=c, lib=hostsim_lib))
    env = dict(os.environ, PYTHONPATH=root + os.pathsep + os.path.join(root, "tests"))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port", str(29500 + os.getpid() % 200), script]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    for f in ("fusions.tsv", "fusions.discarded.tsv"):
        assert open(os.path.join(tmp_path, "rank0", f), "rb").read() == open(os.path.join(w.outdir, f), "rb").read(), f


# ---- on the H100
GPU_FRONT_END = [("small", ("erased", "single_end", "damage"), "bam", {}), ("small", ("both", "hi"), "sam", {"ARB_CHUNK_BYTES": "3000"}),
                 ("l151", ("erased", "single_end"), "bam", {}), ("l151", ("both",), "bgzf", {"ARB_KEY_HASH_BITS": "4"})]


@pytest.mark.gpu
@pytest.mark.parametrize("name,kinds,form,hooks", GPU_FRONT_END, ids=_id)
def test_front_end_cuda(worlds, cuda_lib, monkeypatch, name, kinds, form, hooks):
    for k, v in hooks.items():
        monkeypatch.setenv(k, v)
    w, c = pair(worlds, name, kinds, form)
    check_front_end(w, c, cuda_lib, 8)


@pytest.mark.gpu
@pytest.mark.parametrize("name,kinds,form", [("small", ("erased", "single_end", "damage"), "bam"), ("l151", ("both", "single_end"), "sam")], ids=_id)
def test_outputs_cuda(worlds, cuda_lib, tmp_path, name, kinds, form):
    w, c = pair(worlds, name, kinds, form)
    out, disc = str(tmp_path / "fusions.tsv"), str(tmp_path / "fusions.discarded.tsv")
    p = L.Pipeline(w.prefix + ".bam", w.prefix + ".gtf", w.prefix + ".fa", threads=8, lib_path=cuda_lib, chimeric=c, output=out, discarded=disc)
    p.run_all(); p.close()
    for got, f in ((out, "fusions.tsv"), (disc, "fusions.discarded.tsv")):
        assert open(got, "rb").read() == open(os.path.join(w.outdir, f), "rb").read(), f


@pytest.mark.gpu
def test_errors_cuda(worlds, cuda_lib, tmp_path):
    w, c = pair(worlds, "small")
    text, refs, c_bodies = bamtools.read_bam(c)
    empty = str(tmp_path / "empty.bam"); bamtools.write_bam(empty, text, refs, [], random.Random(1))
    assert NO_CHIMERIC in run_error(w, empty, cuda_lib)
