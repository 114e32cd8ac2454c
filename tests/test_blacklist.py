"""Blacklist (-b): the file is read like the reference reads it, the rules are matched to the eligible candidates on the device (csrc/blacklist_hd.h) and the
blacklist filter is applied just before short_anchor. Both output files, the WARNING lines and the progress line must equal the reference's; the verdict of
every candidate must equal tests/blacklist_ref.py, a plain transcription of the reference loop."""
import os
import random
import subprocess
import sys
import numpy as np
import pytest
import blacklist_ref
import blacklisttools
import worldutil
from arriba_b200 import lib as L, _build
from test_genomic_support import contig_names, contig_ids, oracle_run, sv_file, ZCHR, L151

F_BLACKLIST, F_NO_GENOMIC_SUPPORT = 20, 29
MANY_SPLICED, SHORT_ANCHOR = L.EV_NAMES.index("many_spliced"), L.EV_NAMES.index("short_anchor")


def world_state(world, lib_path, sv=None):
    """The candidates as the blacklist stage sees them (after many_spliced, and no_genomic_support with -d), the genes, their names and max_mate_gap."""
    p = L.Pipeline(world.prefix + ".bam", world.prefix + ".gtf", world.prefix + ".fa", threads=2, lib_path=lib_path, genomic_breakpoints=sv)
    p.run(); p.events(MANY_SPLICED)
    cand = p.candidates(); genes = p.genes(); mmg = int(p.stats().max_mate_gap); p.close()
    names = blacklisttools.gene_names(world.prefix + ".gtf", genes, contig_ids(world))
    return cand, genes, names, mmg


_FILES = {}


def blacklist_file(world, lib_path, root, variant="plain", seed=3, sv=None):
    key = (world.prefix, variant, seed, sv)
    if key not in _FILES:
        cand, genes, names, mmg = world_state(world, lib_path, sv)
        lines = blacklisttools.rule_lines(cand, genes, names, contig_names(world), random.Random(seed), mmg)
        path = os.path.join(root, "bl_%d_%s%s" % (len(_FILES), variant, ".tsv.gz" if variant == "gz" else ".tsv"))
        blacklisttools.write(path, lines, crlf=variant == "crlf")
        _FILES[key] = path
    return _FILES[key]


def warnings_of(text):
    return [l for l in text.splitlines() if l.startswith("WARNING: unknown gene") or l.startswith("WARNING: encountered a line")]


def cli_run(cli, world, args, tmp, env=None):
    out = os.path.join(tmp, "fusions.tsv"); disc = os.path.join(tmp, "fusions.discarded.tsv")
    r = subprocess.run([cli, "-x", world.prefix + ".bam", "-g", world.prefix + ".gtf", "-a", world.prefix + ".fa", "-o", out, "-O", disc, "-@", "3"] + list(args),
                       capture_output=True, text=True, timeout=900, env=dict(os.environ, **(env or {})))
    assert r.returncode == 0, r.stderr[-2000:]
    return r, open(out, "rb").read(), open(disc, "rb").read()


def cli_parity(cli, world, args, tmp, env=None):
    ref = oracle_run(world, args, os.path.join(tmp, "oracle"))
    r, fus, disc = cli_run(cli, world, args, tmp, env)
    assert fus == open(os.path.join(ref.outdir, "fusions.tsv"), "rb").read(), "fusions.tsv differs with %s" % (args,)
    assert disc == open(os.path.join(ref.outdir, "fusions.discarded.tsv"), "rb").read(), "fusions.discarded.tsv differs with %s" % (args,)
    assert warnings_of(r.stderr) == warnings_of(open(os.path.join(ref.outdir, "stderr.txt")).read())
    ref_out = open(os.path.join(ref.outdir, "stdout.txt")).read()
    mine = [l.split("] ", 1)[1].strip() for l in r.stdout.splitlines() if "Filtering blacklisted fusions" in l]
    theirs = [l.split("] ", 1)[1].strip() for l in ref_out.splitlines() if "Filtering blacklisted fusions" in l]
    assert len(mine) == 1 and mine == theirs, (mine, theirs)
    return ref


@pytest.fixture(scope="module")
def cli():
    return _build.build_cli_hostsim()


@pytest.fixture(scope="module")
def bl_root(tmp_path_factory):
    return str(tmp_path_factory.mktemp("bl"))


def _world(worlds, name):
    if name == "cfg5":
        from test_events import CFG5
        return worlds.get(name, **CFG5)
    return worlds.get(name, **{"small": {}, "l151": L151, "zchr": ZCHR}[name])


CASES = [
    ("small", "plain", ()), ("small", "crlf", ("-E", "0.3")), ("small", "gz", ("-E", "1000")), ("small", "plain", ("-X",)),
    ("small", "plain", ("-v", "1,2,3,4,5,6,7,8")), ("l151", "plain", ()), ("zchr", "plain", ()), ("cfg5", "plain", ()),
]


@pytest.mark.parametrize("name,variant,extra", CASES, ids=lambda x: x if isinstance(x, str) else " ".join(x) if isinstance(x, tuple) else None)
def test_blacklist_cli_parity(worlds, cli, hostsim_lib, bl_root, tmp_path, name, variant, extra):
    w = _world(worlds, name)
    cli_parity(cli, w, tuple(extra) + ("-b", blacklist_file(w, hostsim_lib, bl_root, variant)), str(tmp_path))


def test_blacklist_cli_parity_with_genomic_support(worlds, cli, hostsim_lib, bl_root, tmp_path):
    """-d and -b: candidates filtered earlier but with genomic support are eligible, and the blacklist label overwrites their filter."""
    w = worlds.get("small")
    sv = sv_file(w, hostsim_lib, bl_root)
    cand, genes, names, mmg = world_state(w, hostsim_lib, sv)
    supported = [k for k in range(int(cand["n"])) if cand["closest_genomic_breakpoint1"][k] >= 0 and cand["filter"][k] != 0]
    assert supported
    nm = contig_names(w)
    lines = blacklisttools.rule_lines(cand, genes, names, nm, random.Random(4), mmg)
    lines += ["%s:%d\tany" % (nm[cand["contig1"][k]], cand["breakpoint1"][k] + 1) for k in supported]
    path = os.path.join(bl_root, "bl_genomic.tsv"); blacklisttools.write(path, lines)
    ref = cli_parity(cli, w, ("-d", sv, "-b", path), str(tmp_path))
    verdicts_against_reference(w, hostsim_lib, path, sv=sv, oracle=ref)


def test_blacklist_cli_disabled_filter(worlds, cli, hostsim_lib, bl_root, tmp_path):
    """-f blacklist -b FILE: the file is not read, and the output equals the run without -b."""
    w = worlds.get("small")
    path = blacklist_file(w, hostsim_lib, bl_root)
    r1, f1, d1 = cli_run(cli, w, ("-f", "blacklist"), str(tmp_path))
    r2, f2, d2 = cli_run(cli, w, ("-f", "blacklist", "-b", path), str(tmp_path))
    assert f1 == f2 and d1 == d2 and warnings_of(r2.stderr) == [] and "Filtering blacklisted" not in r2.stdout
    ref = oracle_run(w, ("-f", "blacklist", "-b", path), str(tmp_path / "oracle"))
    assert f2 == open(os.path.join(ref.outdir, "fusions.tsv"), "rb").read()


def test_blacklist_cli_parity_scattered_and_poisoned(worlds, cli, hostsim_lib, bl_root, tmp_path):
    w = worlds.get("small")
    cli_parity(cli, w, ("-b", blacklist_file(w, hostsim_lib, bl_root)), str(tmp_path), env={"ARB_HOSTSIM_ORDER": "2", "ARB_HOSTSIM_POISON": "1", "ARB_BLACKLIST_SHORT_LIST": "0"})


def verdicts_against_reference(w, lib_path, path, sv=None, oracle=None, short_list=None, evalue_cutoff=3.0):
    """Every candidate's verdict: the product's blacklist labels after the stage against blacklist_ref.py (and the reference's own stage dump)."""
    if short_list is not None:
        os.environ["ARB_BLACKLIST_SHORT_LIST"] = str(short_list)
    try:
        p = L.Pipeline(w.prefix + ".bam", w.prefix + ".gtf", w.prefix + ".fa", threads=2, lib_path=lib_path, genomic_breakpoints=sv, blacklist=path)
        p.run(); p.events(MANY_SPLICED)
        before = p.candidates(); genes = p.genes(); mmg = int(p.stats().max_mate_gap)
        p.events(SHORT_ANCHOR)
        after = p.candidates(); timings = p.context().timings(); p.close()
        names = blacklisttools.gene_names(w.prefix + ".gtf", genes, contig_ids(w))
        rules, _ = blacklist_ref.read_rules(path, contig_ids(w), blacklisttools.gene_by_name(names), genes["gene_contig"], genes["gene_start"], genes["gene_end"])
        closest = before["closest_genomic_breakpoint1"] if sv else None
        if sv:  # no_genomic_support runs at the head of the same stage, before the blacklist (arriba.cpp:516-530)
            before["filter"] = np.where(after["filter"] == F_NO_GENOMIC_SUPPORT, F_NO_GENOMIC_SUPPORT, before["filter"]).astype(np.uint8)
        want = blacklist_ref.blacklisted(rules, before, genes["gene_start"], genes["gene_end"], float(np.float32(evalue_cutoff)), mmg, closest)
        got = set(np.flatnonzero(after["filter"] == F_BLACKLIST).tolist())
        assert got == want, (sorted(got - want)[:10], sorted(want - got)[:10])
        if oracle is not None:  # blacklist runs just before short_anchor: the reference's dump of that stage, in its iteration order
            d = oracle.stage("ev_short_anchor")
            assert np.array_equal(after["filter"][after["order"]] == F_BLACKLIST, d["filter"] == F_BLACKLIST)
        return len(got), timings
    finally:
        os.environ.pop("ARB_BLACKLIST_SHORT_LIST", None)


@pytest.mark.parametrize("short_list", [None, 0])
def test_verdict_of_every_candidate(worlds, hostsim_lib, bl_root, tmp_path, short_list):
    w = worlds.get("small")
    path = blacklist_file(w, hostsim_lib, bl_root)
    ref = oracle_run(w, ("-b", path), str(tmp_path / "oracle"))
    n, _ = verdicts_against_reference(w, hostsim_lib, path, oracle=ref, short_list=short_list)
    assert n > 20


def dense_file(w, lib_path, root, n=100000):
    path = os.path.join(root, "dense_%s.tsv" % os.path.basename(os.path.dirname(w.prefix)))
    if not os.path.exists(path):
        cand, genes, names, mmg = world_state(w, lib_path)
        blacklisttools.write(path, blacklisttools.dense_lines(cand, genes, contig_names(w), random.Random(9), n, mmg))
    return path


def test_dense_file_hostsim(worlds, hostsim_lib, bl_root):
    w = worlds.get("small")
    n, _ = verdicts_against_reference(w, hostsim_lib, dense_file(w, hostsim_lib, bl_root))
    assert n > 0


def test_cli_blacklist_errors(worlds, cli, tmp_path):
    """A missing -b file stops both programs with the same ERROR line; the two inputs the reference has no defined behaviour for stop the product with an error."""
    w = worlds.get("small")
    oracle = _build.build_oracle()
    base = ["-x", w.prefix + ".bam", "-g", w.prefix + ".gtf", "-a", w.prefix + ".fa", "-o", str(tmp_path / "o.tsv")]
    seen = []
    for exe in (oracle, cli):
        r = subprocess.run([exe] + base + ["-b", str(tmp_path / "missing.tsv")], capture_output=True, text=True, timeout=300)
        seen.append((r.returncode, [l for l in r.stderr.splitlines() if l.startswith("ERROR")]))
    assert seen[0] == seen[1] and seen[0][0] == 1, seen
    r = subprocess.run([cli] + base, capture_output=True, text=True, timeout=300)
    assert r.returncode == 1 and "missing option -b" in r.stderr
    nm = contig_names(w)[0]
    for line, why in (("~~~*:100\tany", "sorts after every contig name"), ("%s:2147483000\tany" % nm, "overflow int"), ("%s:1-2147483000\tany" % nm, "overflow int")):
        path = str(tmp_path / "ub.tsv"); blacklisttools.write(path, ["%s:100\tany" % nm, line])
        r = subprocess.run([cli] + base + ["-b", path], capture_output=True, text=True, timeout=300)
        assert r.returncode == 1 and why in r.stderr and "line 2" in r.stderr, r.stderr[-2000:]


def test_no_blacklist_changes_nothing(worlds, hostsim_lib, bl_root, tmp_path):
    """Without -b, or with -b while the filter is off, the files and the number of kernel launches equal those of a run that never heard of -b."""
    w = worlds.get("small")
    path = blacklist_file(w, hostsim_lib, bl_root)
    lib = L.load(hostsim_lib)
    res = []
    for bl, on in ((None, True), (path, False), (None, False)):
        d = str(tmp_path / ("run%d" % len(res))); os.makedirs(d)
        prm = L.Params(); lib.arb_default_params(C_byref(prm))
        if not on:
            prm.filter_mask &= ~(1 << F_BLACKLIST)
        p = L.Pipeline(w.prefix + ".bam", w.prefix + ".gtf", w.prefix + ".fa", threads=2, lib_path=hostsim_lib, params=prm, blacklist=bl,
                       output=os.path.join(d, "fusions.tsv"), discarded=os.path.join(d, "fusions.discarded.tsv"))
        k0 = lib.arb_kernel_launches(); p.run_all(); k1 = lib.arb_kernel_launches(); p.close()
        res.append((k1 - k0, open(os.path.join(d, "fusions.tsv"), "rb").read(), open(os.path.join(d, "fusions.discarded.tsv"), "rb").read()))
    assert res[0] == res[1] == res[2]


def C_byref(x):
    import ctypes
    return ctypes.byref(x)


WORKER = r"""
import os, sys
sys.path.insert(0, {root!r})
import torch.distributed as dist
from arriba_b200 import lib as L, sharded
rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"])
dist.init_process_group("gloo")
out = os.path.join({outdir!r}, "rank%d" % rank); os.makedirs(out, exist_ok=True)
p = L.Pipeline({prefix!r} + ".bam", {prefix!r} + ".gtf", {prefix!r} + ".fa", threads=2, lib_path={lib!r}, blacklist={bl!r},
               output=os.path.join(out, "fusions.tsv"), discarded=os.path.join(out, "fusions.discarded.tsv"))
sharded.run_sharded(p, rank, world)
p.close()
dist.destroy_process_group()
"""


def test_sharded_two_ranks_with_blacklist(worlds, hostsim_lib, bl_root, tmp_path):
    w = worlds.get("small")
    path = blacklist_file(w, hostsim_lib, bl_root)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = str(tmp_path / "worker.py")
    open(script, "w").write(WORKER.format(root=root, outdir=str(tmp_path), prefix=w.prefix, lib=hostsim_lib, bl=path))
    env = dict(os.environ, PYTHONPATH=root + os.pathsep + os.path.join(root, "tests"))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port", str(29500 + os.getpid() % 200), script]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    single = str(tmp_path / "single"); os.makedirs(single)
    p = L.Pipeline(w.prefix + ".bam", w.prefix + ".gtf", w.prefix + ".fa", threads=2, lib_path=hostsim_lib, blacklist=path,
                   output=os.path.join(single, "fusions.tsv"), discarded=os.path.join(single, "fusions.discarded.tsv"))
    p.run_all(); p.close()
    for f in ("fusions.tsv", "fusions.discarded.tsv"):
        assert open(os.path.join(tmp_path, "rank0", f), "rb").read() == open(os.path.join(single, f), "rb").read(), f
    assert b"\tblacklist" in open(os.path.join(single, "fusions.discarded.tsv"), "rb").read()


# ---- on the H100
def pipeline_parity(world, lib_path, args, path, tmp):
    ref = oracle_run(world, args + ("-b", path), os.path.join(tmp, "oracle"))
    out = os.path.join(tmp, "fusions.tsv"); disc = os.path.join(tmp, "fusions.discarded.tsv")
    p = L.Pipeline(world.prefix + ".bam", world.prefix + ".gtf", world.prefix + ".fa", threads=8, lib_path=lib_path, blacklist=path, output=out, discarded=disc)
    p.run_all(); p.close()
    for f in ("fusions.tsv", "fusions.discarded.tsv"):
        assert open(os.path.join(tmp, f), "rb").read() == open(os.path.join(ref.outdir, f), "rb").read(), f


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small", "cfg5"])
def test_blacklist_parity_cuda(worlds, cuda_lib, hostsim_lib, bl_root, tmp_path, name):
    w = _world(worlds, name)
    path = blacklist_file(w, hostsim_lib, bl_root)
    pipeline_parity(w, cuda_lib, (), path, str(tmp_path / "lib"))
    cli = _build.build_cli()
    cli_parity(cli, w, ("-b", path), str(tmp_path / "cli"))
    cli_parity(cli, w, ("-X", "-b", path), str(tmp_path / "cli_x"))


@pytest.mark.gpu
def test_dense_file_cuda(worlds, cuda_lib, hostsim_lib, bl_root):
    w = worlds.get("small")
    path = dense_file(w, hostsim_lib, bl_root)
    n, t = verdicts_against_reference(w, cuda_lib, path)
    assert n > 0 and t.blacklist_ms > 0
    verdicts_against_reference(w, cuda_lib, path, short_list=0)  # every list through the lane groups
