"""Genomic breakpoints from whole-genome sequencing (-d, -D): the SV file is read like the reference reads it, every candidate is matched to its closest
genomic breakpoint pair on the device (csrc/genomic_hd.h), and the genomic_support / no_genomic_support filters and the confidence raise follow.
Both output files and the WARNING lines must equal the reference's; closest_genomic_breakpoint1/2 of every candidate must equal tests/genomic_ref.py."""
import os
import random
import subprocess
import numpy as np
import pytest
import genomic_ref
import svtools
import worldutil
from arriba_b200 import lib as L, _build

CLI_BASE = ("-f", "blacklist")
ZCHR = dict(seed=11, extra=("--compress", "6", "--chr", "--normal-frac", "0.5"))
L151 = dict(read_length=151, seed=7, extra=("--shuffle", "--varnames"))


def contig_names(world):
    d = world.stage("read_chimeric_alignments")
    blob = bytes(d["contig_names"]).decode(); off = d["contig_name_off"]
    return [blob[off[k]:off[k + 1]] for k in range(len(off) - 1)]


def contig_ids(world):
    return {genomic_ref._remove_chr(n): k for k, n in enumerate(contig_names(world))}


def world_tables(world, lib_path):
    """The candidates find_fusions made and the gene table (dummy genes included), from the product run without -d."""
    p = L.Pipeline(world.prefix + ".bam", world.prefix + ".gtf", world.prefix + ".fa", threads=2, lib_path=lib_path)
    p.run(); p.events(0)
    cand = p.candidates(); genes = p.genes(); p.close()
    return cand, genes["gene_start"], genes["gene_end"], (genes["gene_flags"] & 1).astype(bool)


_FILES = {}


def sv_file(world, lib_path, tmp_root, variant="plain", seed=5):
    key = (world.prefix, variant, seed)
    if key not in _FILES:
        cand, gs, ge, gd = world_tables(world, lib_path)
        lines = svtools.sv_lines(cand, gs, ge, gd, contig_names(world), random.Random(seed))
        path = os.path.join(tmp_root, "sv_%d_%s_%d%s" % (len(_FILES), variant, seed, ".vcf.gz" if variant == "gz" else ".txt"))
        svtools.write(path, lines, crlf=variant == "crlf")
        _FILES[key] = path
    return _FILES[key]


def oracle_run(world, args, outdir):
    worldutil.run_oracle(world.prefix, outdir, args=args)
    return worldutil.World(world.prefix, outdir)


def warnings_of(text):
    return [l for l in text.splitlines() if l.startswith("WARNING: failed to parse line")]


def cli_parity(cli, world, args, tmp, env=None):
    ref = oracle_run(world, args, os.path.join(tmp, "oracle"))
    out = os.path.join(tmp, "fusions.tsv"); disc = os.path.join(tmp, "fusions.discarded.tsv")
    r = subprocess.run([cli, "-x", world.prefix + ".bam", "-g", world.prefix + ".gtf", "-a", world.prefix + ".fa", "-o", out, "-O", disc, "-@", "3"] + list(args),
                       capture_output=True, text=True, timeout=900, env=dict(os.environ, **(env or {})))
    assert r.returncode == 0, r.stderr[-2000:]
    assert open(out, "rb").read() == open(os.path.join(ref.outdir, "fusions.tsv"), "rb").read(), "fusions.tsv differs with %s" % (args,)
    assert open(disc, "rb").read() == open(os.path.join(ref.outdir, "fusions.discarded.tsv"), "rb").read(), "fusions.discarded.tsv differs with %s" % (args,)
    assert warnings_of(r.stderr) == warnings_of(open(os.path.join(ref.outdir, "stderr.txt")).read())
    marked = [l for l in r.stdout.splitlines() if "Marking fusions with support from whole-genome sequencing" in l]
    assert len(marked) == 1 and marked[0].split("] ", 1)[1] in open(os.path.join(ref.outdir, "stdout.txt")).read(), marked
    return ref


@pytest.fixture(scope="module")
def cli():
    return _build.build_cli_hostsim()


@pytest.fixture(scope="module")
def sv_root(tmp_path_factory):
    return str(tmp_path_factory.mktemp("sv"))


CASES = [
    ("small", {}, "plain", ()), ("small", {}, "crlf", ("-D", "0")), ("small", {}, "gz", ("-D", "1000")),
    ("small", {}, "plain", ("-f", "blacklist,genomic_support")), ("small", {}, "plain", ("-f", "blacklist,no_genomic_support")),
    ("small", {}, "plain", ("-f", "blacklist,many_spliced,select_best")), ("small", {}, "plain", ("-f", "blacklist,genomic_support,no_genomic_support")),
    ("small", {}, "plain", ("-v", "1,2,3,4,5,6,7,8")), ("small", {}, "plain", ("-X",)),
    ("l151", L151, "plain", ()), ("zchr", ZCHR, "plain", ()), ("cfg5", None, "plain", ()),
]


@pytest.mark.parametrize("name,kw,variant,extra", CASES, ids=lambda x: x if isinstance(x, str) else " ".join(x) if isinstance(x, tuple) else None)
def test_genomic_cli_parity(worlds, cli, hostsim_lib, sv_root, tmp_path, name, kw, variant, extra):
    if kw is None:
        from test_events import CFG5
        kw = CFG5
    w = worlds.get(name, **kw)
    path = sv_file(w, hostsim_lib, sv_root, variant)
    args = tuple(extra) + ("-d", path) if "-f" in extra else CLI_BASE + tuple(extra) + ("-d", path)
    cli_parity(cli, w, args, str(tmp_path))


def test_genomic_cli_parity_scattered_and_poisoned(worlds, cli, hostsim_lib, sv_root, tmp_path):
    w = worlds.get("small")
    cli_parity(cli, w, CLI_BASE + ("-d", sv_file(w, hostsim_lib, sv_root)), str(tmp_path), env={"ARB_HOSTSIM_ORDER": "2", "ARB_HOSTSIM_POISON": "1", "ARB_GENOMIC_SHORT_RANGE": "2"})


def check_every_candidate(w, lib_path, path, max_distance=100000, oracle=None, short_range=None):
    if short_range is not None:
        os.environ["ARB_GENOMIC_SHORT_RANGE"] = str(short_range)
    try:
        p = L.Pipeline(w.prefix + ".bam", w.prefix + ".gtf", w.prefix + ".fa", threads=2, lib_path=lib_path, genomic_breakpoints=path, max_genomic_breakpoint_distance=max_distance)
        p.run(); p.events(0)
        cand = p.candidates(); genes = p.genes()
        timings = p.context().timings()
        recs, _ = genomic_ref.read_records(path, contig_ids(w))
        want1, want2 = genomic_ref.mark(recs, cand, genes["gene_start"], genes["gene_end"], (genes["gene_flags"] & 1).astype(bool), max_distance)
        assert np.array_equal(cand["closest_genomic_breakpoint1"], np.array(want1, np.int32))
        assert np.array_equal(cand["closest_genomic_breakpoint2"], np.array(want2, np.int32))
        if oracle is not None:  # the reference's own marks (stage dump after merge_adjacent, in its iteration order) and its final confidence
            d = oracle.stage("ev_merge_adjacent")
            assert np.array_equal(cand["closest_genomic_breakpoint1"][cand["order"]], d["closest_genomic_breakpoint1"])
            assert np.array_equal(cand["closest_genomic_breakpoint2"][cand["order"]], d["closest_genomic_breakpoint2"])
            p.events(L.EV_NAMES.index("confidence"))
            conf = p.candidates()["confidence"]
            assert np.array_equal(conf[cand["order"]], oracle.stage("ev_confidence", 1)["confidence"])
        p.close()
        return int((cand["closest_genomic_breakpoint1"] >= 0).sum()), timings
    finally:
        os.environ.pop("ARB_GENOMIC_SHORT_RANGE", None)


@pytest.mark.parametrize("short_range", [None, 0])
def test_closest_of_every_candidate(worlds, hostsim_lib, sv_root, tmp_path, short_range):
    w = worlds.get("small")
    path = sv_file(w, hostsim_lib, sv_root)
    ref = oracle_run(w, CLI_BASE + ("-d", path), str(tmp_path / "oracle"))
    marked, _ = check_every_candidate(w, hostsim_lib, path, oracle=ref, short_range=short_range)
    assert marked > 50


def dense_file(w, lib_path, root, n=100000):
    path = os.path.join(root, "dense_%s.txt" % os.path.basename(os.path.dirname(w.prefix)))
    if not os.path.exists(path):
        cand, gs, ge, _ = world_tables(w, lib_path)
        svtools.write(path, svtools.dense_lines(cand, gs, ge, contig_names(w), random.Random(9), n))
    return path


def test_dense_file_hostsim(worlds, hostsim_lib, sv_root):
    w = worlds.get("small")
    marked, t = check_every_candidate(w, hostsim_lib, dense_file(w, hostsim_lib, sv_root))
    assert marked > 0


def test_cli_genomic_errors(worlds, cli, tmp_path):
    """A missing -d file and a bad -D stop both programs with the same exit code; the missing file with the same ERROR line."""
    w = worlds.get("small")
    oracle = _build.build_oracle()
    base = ["-x", w.prefix + ".bam", "-g", w.prefix + ".gtf", "-a", w.prefix + ".fa", "-o", str(tmp_path / "o.tsv"), "-f", "blacklist"]
    for extra, same_text in ((["-d", str(tmp_path / "missing.vcf")], True), (["-D", "-1"], False), (["-D", "abc"], False), (["-D", "12x"], False)):
        seen = []
        for exe in (oracle, cli):
            r = subprocess.run([exe] + base + extra, capture_output=True, text=True, timeout=300)
            seen.append((r.returncode, [l for l in r.stderr.splitlines() if l.startswith("ERROR")]))
        assert seen[0][0] == seen[1][0] == 1, (extra, seen)
        if same_text:
            assert seen[0][1] == seen[1][1], (extra, seen)
        else:
            assert seen[1][1] == ["ERROR: invalid argument to -D"], seen
    r = subprocess.run([cli] + base + ["-D", "500"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "Marking fusions" not in r.stdout, r.stderr[-2000:]  # -D without -d is accepted and changes nothing


WORKER = r"""
import os, sys
sys.path.insert(0, {root!r})
import torch.distributed as dist
from arriba_b200 import lib as L, sharded
rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"])
dist.init_process_group("gloo")
out = os.path.join({outdir!r}, "rank%d" % rank); os.makedirs(out, exist_ok=True)
p = L.Pipeline({prefix!r} + ".bam", {prefix!r} + ".gtf", {prefix!r} + ".fa", threads=2, lib_path={lib!r}, genomic_breakpoints={sv!r},
               output=os.path.join(out, "fusions.tsv"), discarded=os.path.join(out, "fusions.discarded.tsv"))
sharded.run_sharded(p, rank, world)
p.close()
dist.destroy_process_group()
"""


def test_sharded_two_ranks_with_genomic_support(worlds, hostsim_lib, sv_root, tmp_path):
    import sys
    w = worlds.get("small")
    path = sv_file(w, hostsim_lib, sv_root)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = str(tmp_path / "worker.py")
    open(script, "w").write(WORKER.format(root=root, outdir=str(tmp_path), prefix=w.prefix, lib=hostsim_lib, sv=path))
    env = dict(os.environ, PYTHONPATH=root + os.pathsep + os.path.join(root, "tests"))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port", str(29700 + os.getpid() % 200), script]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    single = str(tmp_path / "single"); os.makedirs(single)
    p = L.Pipeline(w.prefix + ".bam", w.prefix + ".gtf", w.prefix + ".fa", threads=2, lib_path=hostsim_lib, genomic_breakpoints=path,
                   output=os.path.join(single, "fusions.tsv"), discarded=os.path.join(single, "fusions.discarded.tsv"))
    p.run_all(); p.close()
    for f in ("fusions.tsv", "fusions.discarded.tsv"):
        assert open(os.path.join(tmp_path, "rank0", f), "rb").read() == open(os.path.join(single, f), "rb").read(), f


# ---- on the H100
def pipeline_parity(world, lib_path, args, path, tmp):
    ref = oracle_run(world, args + ("-d", path), os.path.join(tmp, "oracle"))
    out = os.path.join(tmp, "fusions.tsv"); disc = os.path.join(tmp, "fusions.discarded.tsv")
    p = L.Pipeline(world.prefix + ".bam", world.prefix + ".gtf", world.prefix + ".fa", threads=8, lib_path=lib_path, genomic_breakpoints=path, output=out, discarded=disc)
    p.run_all(); p.close()
    for f in ("fusions.tsv", "fusions.discarded.tsv"):
        assert open(os.path.join(tmp, f), "rb").read() == open(os.path.join(ref.outdir, f), "rb").read(), f
    return ref


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small", "cfg5"])
def test_genomic_parity_cuda(worlds, cuda_lib, hostsim_lib, sv_root, tmp_path, name):
    from test_events import CFG5
    w = worlds.get(name, **(CFG5 if name == "cfg5" else {}))
    path = sv_file(w, hostsim_lib, sv_root)
    pipeline_parity(w, cuda_lib, CLI_BASE, path, str(tmp_path / "lib"))
    cli_parity(_build.build_cli(), w, CLI_BASE + ("-X", "-d", path), str(tmp_path / "cli"))


@pytest.mark.gpu
def test_dense_file_cuda(worlds, cuda_lib, hostsim_lib, sv_root):
    w = worlds.get("small")
    path = dense_file(w, hostsim_lib, sv_root)
    marked, t = check_every_candidate(w, cuda_lib, path)
    assert marked > 0 and t.genomic_support_ms > 0
    check_every_candidate(w, cuda_lib, path, short_range=0)  # every range through the lane groups
