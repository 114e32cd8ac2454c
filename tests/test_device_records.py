"""The record loop of the ingest runs on the device (csrc/records.cu): records are kept in a store across chunks, grouped by "<qname>,<HI>" and
replayed in file order. Files whose record order the aligner would not write -- every record backwards (supplementaries before their primaries, second
mates first), first mates that never meet a second one, three primaries of one key -- go through the oracle and through the product's front end, read in
small chunks so that keys are split over chunks; runs of one key hash that hold many keys (ARB_KEY_HASH_BITS, a test hook) must read the same; of two
record errors the one earlier in the file is reported."""
import os, random
import pytest
import bamtools, worldutil
from arriba_b200 import lib as L
from test_ingest import check_front_end

BF_PAIRED, BF_PROPER, BF_SECONDARY, BF_SUPPLEMENTARY = 1, 2, 256, 2048


def _proper_first_mates(bodies):
    """indices of the first record of every proper pair (by name, primary alignments)"""
    seen, firsts = set(), []
    for i, b in enumerate(bodies):
        r = bamtools.split_record(b)
        if r["flag"] & (BF_SECONDARY | BF_SUPPLEMENTARY) or not (r["flag"] & BF_PAIRED and r["flag"] & BF_PROPER):
            continue
        if r["qname"] not in seen:
            seen.add(r["qname"]); firsts.append(i)
    return firsts


def reorder(bodies, kind):
    if kind == "reversed":
        return bodies[::-1]
    firsts = _proper_first_mates(bodies)
    if kind == "orphans":  # the second mate never arrives
        drop = set(firsts[::7])
        return [b for i, b in enumerate(bodies) if i not in drop]
    if kind == "triplets":  # one mate twice: three primaries of one key
        again = set(firsts[::11])
        out = []
        for i, b in enumerate(bodies):
            out.append(b)
            if i in again:
                out.append(b)
        return out
    raise ValueError(kind)


def reordered_world(worlds, root, kind):
    base = worlds.get("l151", read_length=151, seed=7, extra=("--shuffle", "--varnames"))
    d = os.path.join(str(root), kind); os.makedirs(d, exist_ok=True)
    prefix = os.path.join(d, "w")
    for ext in (".fa", ".gtf"):
        if not os.path.exists(prefix + ext):
            os.symlink(base.prefix + ext, prefix + ext)
    if not os.path.exists(prefix + ".bam"):
        text, refs, bodies = bamtools.read_bam(base.prefix + ".bam")
        bamtools.write_bam(prefix + ".bam", text, refs, reorder(bodies, kind), random.Random(3))
        worldutil.run_oracle(prefix, os.path.join(d, "oracle"))
    return worldutil.World(prefix, os.path.join(d, "oracle"))


KINDS = ["reversed", "orphans", "triplets"]


@pytest.fixture(scope="module")
def reordered(worlds, tmp_path_factory):
    root = tmp_path_factory.mktemp("reordered")
    return {k: reordered_world(worlds, root, k) for k in KINDS}


@pytest.mark.parametrize("kind", KINDS)
def test_front_end_hostsim_reordered(reordered, hostsim_lib, monkeypatch, kind):
    monkeypatch.setenv("ARB_CHUNK_BYTES", "30000")
    check_front_end(reordered[kind], hostsim_lib, threads=2)


@pytest.mark.parametrize("kind", ["reversed", "triplets"])
def test_front_end_hostsim_colliding_key_hashes(reordered, hostsim_lib, monkeypatch, kind):
    """keys that share a hash are told apart by their names: 16 hashes for the whole file"""
    monkeypatch.setenv("ARB_KEY_HASH_BITS", "4")
    check_front_end(reordered[kind], hostsim_lib, threads=1)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_front_end_cuda_reordered(reordered, cuda_lib, monkeypatch, kind):
    monkeypatch.setenv("ARB_CHUNK_BYTES", "30000")
    check_front_end(reordered[kind], cuda_lib, threads=2)


@pytest.mark.gpu
def test_front_end_cuda_colliding_key_hashes(reordered, cuda_lib, monkeypatch):
    monkeypatch.setenv("ARB_KEY_HASH_BITS", "4")
    check_front_end(reordered["reversed"], cuda_lib, threads=1)


def _two_errors(worlds, tmp_path):
    """two alignments past the end of their contigs; returns (path, name of the earlier record)"""
    base = worlds.get("small")
    text, refs, bodies = bamtools.read_bam(base.prefix + ".bam")
    picked = []
    for i, b in enumerate(bodies):
        r = bamtools.split_record(b)
        if r["tid"] >= 0 and not r["flag"] & 4:
            picked.append(i)
    first, second = picked[len(picked) // 3], picked[2 * len(picked) // 3]
    for i in (second, first):
        r = bamtools.split_record(bodies[i])
        r["pos"] = refs[r["tid"]][1] - 5
        bodies[i] = bamtools.join_record(r)
    path = os.path.join(str(tmp_path), "w.bam")
    bamtools.write_bam(path, text, refs, bodies, random.Random(4))
    return base, path, bamtools.split_record(bodies[first])["qname"].rstrip(b"\0").decode()


def _expect_error(base, path, lib_path, name):
    p = L.Pipeline(path, base.prefix + ".gtf", base.prefix + ".fa", threads=2, lib_path=lib_path)
    p.step(L.STEP_LOAD_REFERENCE)
    with pytest.raises(Exception) as e:
        p.step(L.STEP_INGEST)
    assert ("alignment of read '%s' extends beyond the end of contig" % name) in str(e.value), str(e.value)


def test_earlier_record_error_wins_hostsim(worlds, hostsim_lib, monkeypatch, tmp_path):
    base, path, name = _two_errors(worlds, tmp_path)
    for chunk in (None, "200000"):
        if chunk:
            monkeypatch.setenv("ARB_CHUNK_BYTES", chunk)
        _expect_error(base, path, hostsim_lib, name)


@pytest.mark.gpu
def test_earlier_record_error_wins_cuda(worlds, cuda_lib, tmp_path):
    base, path, name = _two_errors(worlds, tmp_path)
    _expect_error(base, path, cuda_lib, name)


# ---- the ingest alone against the oracle: fragment table, mapped reads, coverage windows
def check_ingest(world, lib_path, threads=2, params=None):
    import numpy as np
    from test_ingest import frag_tables_equal
    p = L.Pipeline(world.prefix + ".bam", world.prefix + ".gtf", world.prefix + ".fa", threads=threads, lib_path=lib_path, params=params)
    p.step(L.STEP_LOAD_REFERENCE)
    p.step(L.STEP_INGEST)
    rca = world.stage("read_chimeric_alignments")
    st = p.stats()
    assert st.mapped_reads == int(rca["mapped_reads"][0])
    assert st.n_fragments == int(rca["total"][0])
    frag_tables_equal(p.fragments(), world.stage("ingest"), check_genes=False, check_pred=False)
    off = rca["coverage_off"]
    for c in range(len(off) - 1):
        cov, starts, ends = p.coverage(c)
        assert np.array_equal(cov, rca["coverage"][off[c]:off[c + 1]]), ("coverage", c)
        assert np.array_equal(starts, rca["fragment_starts"][off[c]:off[c + 1]]), ("starts", c)
        assert np.array_equal(ends, rca["fragment_ends"][off[c]:off[c + 1]]), ("ends", c)
    p.close()


def stacked_world(worlds, root, per_gene, n_genes=40):
    """the small world with `per_gene` extra genes stacked over each of its first `n_genes` genes: the read-through test's gene sets get that large"""
    base = worlds.get("small")
    d = os.path.join(str(root), "stacked_%d" % per_gene); os.makedirs(d, exist_ok=True)
    prefix = os.path.join(d, "w")
    for ext in (".fa", ".bam"):
        if not os.path.exists(prefix + ext):
            os.symlink(base.prefix + ext, prefix + ext)
    if not os.path.exists(prefix + ".gtf"):
        lines = open(base.prefix + ".gtf").read().splitlines()
        genes = [l.split("\t") for l in lines if not l.startswith("#") and l.split("\t")[2] == "gene"][:n_genes]
        extra = []
        for g, f in enumerate(genes):
            for k in range(per_gene):
                gid, tid = "ENSGSTACK%03d%04d" % (g, k), "ENSTSTACK%03d%04d" % (g, k)
                extra.append("\t".join(f[:2] + ["gene"] + f[3:8] + ['gene_id "%s"; gene_name "STACK%d_%d";' % (gid, g, k)]))
                extra.append("\t".join(f[:2] + ["exon"] + f[3:8] + ['gene_id "%s"; transcript_id "%s"; gene_name "STACK%d_%d"; exon_number "1";' % (gid, tid, g, k)]))
        open(prefix + ".gtf", "w").write("\n".join(lines + extra) + "\n")
    return base, prefix, d


@pytest.fixture(scope="module")
def stacked(worlds, tmp_path_factory):
    """40 genes at a locus: more than the 32 the first replay launch holds, so those keys go to the second launch"""
    base, prefix, d = stacked_world(worlds, tmp_path_factory.mktemp("stacked"), 40)
    if not os.path.exists(os.path.join(d, "oracle", "dump")):
        worldutil.run_oracle(prefix, os.path.join(d, "oracle"))
    return worldutil.World(prefix, os.path.join(d, "oracle"))


def test_ingest_hostsim_large_gene_sets(stacked, hostsim_lib):
    check_ingest(stacked, hostsim_lib)


@pytest.mark.gpu
def test_ingest_cuda_large_gene_sets(stacked, cuda_lib):
    check_ingest(stacked, cuda_lib)


def _too_many_genes(worlds, tmp_path, lib_path):
    base, prefix, _ = stacked_world(worlds, tmp_path, 1100)
    p = L.Pipeline(prefix + ".bam", prefix + ".gtf", prefix + ".fa", threads=2, lib_path=lib_path)
    p.step(L.STEP_LOAD_REFERENCE)
    with pytest.raises(Exception) as e:
        p.step(L.STEP_INGEST)
    assert "too many overlapping annotation records at one locus" in str(e.value), str(e.value)


def test_too_many_genes_at_one_locus_hostsim(worlds, hostsim_lib, tmp_path):
    _too_many_genes(worlds, tmp_path, hostsim_lib)


@pytest.mark.gpu
def test_too_many_genes_at_one_locus_cuda(worlds, cuda_lib, tmp_path):
    _too_many_genes(worlds, tmp_path, cuda_lib)


# ---- the tandem-duplication search at other maximum lengths: 5000 puts the search window of many reads across a contig's start or end
@pytest.mark.parametrize("max_itd", [13, 5000])
def test_ingest_hostsim_max_itd_length(worlds, hostsim_lib, max_itd):
    w = worlds.get("small", oracle_args=("-f", "blacklist", "-l", str(max_itd)))
    import ctypes
    params = L.Params(); L.load(hostsim_lib).arb_default_params(ctypes.byref(params))
    params.max_itd_length = max_itd
    check_ingest(w, hostsim_lib, params=params)


# ---- sizes the fragment table cannot address stop the run with the sizes, before the pools are written
def _pool_limit(worlds, lib_path, monkeypatch):
    monkeypatch.setenv("ARB_REPLAY_POOL_LIMIT", "1000")
    w = worlds.get("small")
    p = L.Pipeline(w.prefix + ".bam", w.prefix + ".gtf", w.prefix + ".fa", threads=2, lib_path=lib_path)
    p.step(L.STEP_LOAD_REFERENCE)
    with pytest.raises(Exception) as e:
        p.step(L.STEP_INGEST)
    assert "the sample is too large for one fragment table" in str(e.value) and "(limit 1000)" in str(e.value), str(e.value)


def test_pool_limits_hostsim(worlds, hostsim_lib, monkeypatch):
    _pool_limit(worlds, hostsim_lib, monkeypatch)


@pytest.mark.gpu
def test_pool_limits_cuda(worlds, cuda_lib, monkeypatch):
    _pool_limit(worlds, cuda_lib, monkeypatch)
