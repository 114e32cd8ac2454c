"""The replay of the BAM record loop (csrc/records.cu) against the oracle where its coverage counters saturate: the small world with one proper pair
copied 70,000 times under new names, so that the windows it covers are counted past 65,535 -- the reference's 16-bit counters stop there, and a pack that
wrapped instead would read 70,000 - 65,536. The coverage windows, the fragment table and both output files must equal the oracle's, also with 256 key
hashes for the whole file (long runs of one hash) and in chunks of 200 kB. In a second world the pair lies inside a gene that 40 others overlap, so that
its keys take the replay launch with the large gene sets (the ingest only: the annotation stage takes at most 32 genes under one alignment)."""
import os, random
import numpy as np
import pytest
import bamtools, worldutil
from arriba_b200 import lib as L
from test_device_records import check_ingest, stacked_world

BF_PAIRED, BF_PROPER, BF_SECONDARY, BF_SUPPLEMENTARY = 1, 2, 256, 2048
COPIES = 70000


def _stacked_genes(gtf, n_genes=40):
    """(contig, start, end) of the genes that stacked_world piles 40 more onto (its first 40 gene lines), 0-based half-open"""
    genes = [l.split("\t") for l in open(gtf).read().splitlines() if not l.startswith("#") and l.split("\t")[2] == "gene"][:n_genes]
    return [(f[0], int(f[3]) - 1, int(f[4])) for f in genes]


def _plain_pair(bodies, refs, genes):
    """indices of the two records of a proper pair without SA tag or clipping, both inside one of `genes`"""
    by_name = {}
    for i, b in enumerate(bodies):
        r = bamtools.split_record(b)
        if r["flag"] & (BF_SECONDARY | BF_SUPPLEMENTARY) or (r["flag"] & (BF_PAIRED | BF_PROPER)) != (BF_PAIRED | BF_PROPER) or r["tid"] < 0:
            continue
        if any(tag == b"SA" for tag, _, _ in r["aux"]) or any(op & 15 not in (0, 7, 8) for op in np.frombuffer(r["cigar"], dtype="<u4")):
            continue
        by_name.setdefault(r["qname"], []).append((i, r))
    for pair in by_name.values():
        if len(pair) != 2:
            continue
        (i, a), (j, b) = pair
        contig = refs[a["tid"]][0]
        for c, s, e in genes:
            if c.lstrip("chr") == contig.lstrip("chr") and s <= min(a["pos"], b["pos"]) and max(a["pos"], b["pos"]) + len(a["seq"]) * 2 <= e:
                return i, j
    raise AssertionError("no plain proper pair inside a stacked gene")


def deep_world(worlds, root, stacked):
    """the small world (with stacked genes: stacked_world's GTF) and the pileup; `stacked`: the pair lies inside one of the stacked genes"""
    base, stacked_prefix, d = stacked_world(worlds, root, 40)
    prefix = os.path.join(d, "deep")
    os.symlink(os.path.realpath(base.prefix + ".fa"), prefix + ".fa")
    os.symlink(os.path.realpath((stacked_prefix if stacked else base.prefix) + ".gtf"), prefix + ".gtf")
    text, refs, bodies = bamtools.read_bam(base.prefix + ".bam")
    i, j = _plain_pair(bodies, refs, _stacked_genes(stacked_prefix + ".gtf") if stacked else [(refs[k][0], 0, refs[k][1]) for k in range(len(refs))])
    copies = []
    for k in range(COPIES):
        for x in (i, j):
            r = bamtools.split_record(bodies[x])
            r["qname"] = r["qname"].rstrip(b"\0") + b"_deep%d\0" % k
            copies.append(bamtools.join_record(r))
    bamtools.write_bam(prefix + ".bam", text, refs, bodies[:j + 1] + copies + bodies[j + 1:], random.Random(11))
    outdir = os.path.join(d, "oracle_deep")
    worldutil.run_oracle(prefix, outdir)
    w = worldutil.World(prefix, outdir)
    cov = w.stage("read_chimeric_alignments")["coverage"]
    assert int(cov.max()) == 65535, int(cov.max())   # the world reaches saturation
    return w


@pytest.fixture(scope="module")
def deep(worlds, tmp_path_factory):
    return deep_world(worlds, tmp_path_factory.mktemp("deep"), False)


@pytest.fixture(scope="module")
def deep_stacked(worlds, tmp_path_factory):
    return deep_world(worlds, tmp_path_factory.mktemp("deep_stacked"), True)


def check_outputs(world, lib_path, tmp_path):
    out, disc = os.path.join(str(tmp_path), "fusions.tsv"), os.path.join(str(tmp_path), "fusions.discarded.tsv")
    p = L.Pipeline(world.prefix + ".bam", world.prefix + ".gtf", world.prefix + ".fa", threads=2, lib_path=lib_path, output=out, discarded=disc)
    p.run_all(); p.close()
    for name, path in (("fusions.tsv", out), ("fusions.discarded.tsv", disc)):
        assert open(path, "rb").read() == open(os.path.join(world.outdir, name), "rb").read(), name


HOOKS = {"plain": {}, "few_hashes": {"ARB_KEY_HASH_BITS": "8"}, "small_chunks": {"ARB_CHUNK_BYTES": "200000"}}


@pytest.mark.parametrize("hooks", sorted(HOOKS))
def test_saturated_coverage_hostsim(deep, hostsim_lib, monkeypatch, tmp_path, hooks):
    for k, v in HOOKS[hooks].items():
        monkeypatch.setenv(k, v)
    check_ingest(deep, hostsim_lib)
    check_outputs(deep, hostsim_lib, tmp_path)


def test_saturated_coverage_large_gene_sets_hostsim(deep_stacked, hostsim_lib, monkeypatch):
    monkeypatch.setenv("ARB_KEY_HASH_BITS", "8")
    check_ingest(deep_stacked, hostsim_lib)


@pytest.mark.gpu
@pytest.mark.parametrize("hooks", sorted(HOOKS))
def test_saturated_coverage_cuda(deep, cuda_lib, monkeypatch, tmp_path, hooks):
    for k, v in HOOKS[hooks].items():
        monkeypatch.setenv(k, v)
    check_ingest(deep, cuda_lib)
    check_outputs(deep, cuda_lib, tmp_path)


@pytest.mark.gpu
def test_saturated_coverage_large_gene_sets_cuda(deep_stacked, cuda_lib, monkeypatch):
    monkeypatch.setenv("ARB_KEY_HASH_BITS", "8")
    check_ingest(deep_stacked, cuda_lib)
