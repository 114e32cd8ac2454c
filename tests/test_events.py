"""Event-level chain: after every stage the candidate table (filter, read counts, e-value) must equal the oracle's."""
import numpy as np
import pytest
import worldutil
from arriba_b200 import lib as L
from test_find_fusions import key_of


def compare_stage(got, want, stage, check_evalue):
    index = {key_of(want, i): i for i in range(len(want["gene1"]))}
    perm = np.array([index[key_of(got, i)] for i in range(got["n"])])
    for name in ("filter", "split_reads1", "split_reads2", "discordant_mates"):
        w = want[name][perm]
        bad = np.nonzero(got[name] != w)[0]
        assert len(bad) == 0, (stage, name, len(bad), [key_of(got, i) for i in bad[:5]], got[name][bad[:5]], w[bad[:5]])
    if check_evalue:
        w = want["evalue"][perm]
        bad = np.nonzero(got["evalue"].view(np.uint32) != w.view(np.uint32))[0]
        assert len(bad) == 0, (stage, "evalue", len(bad), got["evalue"][bad[:5]], w[bad[:5]], [key_of(got, i) for i in bad[:5]])
    for lname, oname in (("list1", "list1_off"), ("list2", "list2_off")):
        gs = np.diff(got[oname].astype(np.int64)); ws = np.diff(want[oname].astype(np.int64))[perm]
        assert np.array_equal(gs, ws), (stage, lname + " sizes")
    return perm


def check_events(world, lib_path, threads=4, keep=False):
    p = L.Pipeline(world.prefix + ".bam", world.prefix + ".gtf", world.prefix + ".fa", threads=threads, lib_path=lib_path)
    p.run(L.STEP_FIND_FUSIONS)
    p.events(0)
    got = p.candidates()
    ff = world.stage("find_fusions")
    # the replayed unordered_map iteration order must be the reference's
    want_keys = [key_of(ff, i) for i in range(len(ff["gene1"]))]
    got_keys = [key_of(got, int(i)) for i in got["order"]]
    assert got_keys == want_keys, "iteration order of the candidate table differs from the reference's unordered_map"
    stages = ["merge_adjacent", "multimappers", "evalue", "non_coding_neighbors", "intragenic_exonic", "min_support", "relative_support", "internal_tandem_duplication",
              "intronic", "in_vitro", "spliced", "select_best", "marginal_read_through", "many_spliced", "short_anchor", "end_to_end", "no_coverage",
              "kmer_index", "homologs", "mismappers", "select_best", "isoforms", "confidence"]
    occurrence = {}
    seen_evalue = False
    for s, name in enumerate(stages, start=1):
        p.events(s)
        got = p.candidates()
        if name == "kmer_index":
            continue
        occ = occurrence.get(name, 0); occurrence[name] = occ + 1
        want = world.stage("ev_" + name, occ)
        seen_evalue = seen_evalue or name == "evalue"
        compare_stage(got, want, name, seen_evalue)
        if "frag_filter" in want:
            assert np.array_equal(got["labels"], want["frag_filter"]), (name, "fragment labels")
        assert int((got["filter"] == 0).sum()) == int(want["remaining"][0]) or name in ("evalue", "confidence"), name
        if name == "confidence":
            assert np.array_equal(got["confidence"], want["confidence"][compare_stage(got, want, name, True)])
    if keep:
        return p
    p.close()


def test_events_hostsim(worlds, hostsim_lib):
    check_events(worlds.get("small"), hostsim_lib)


def test_events_hostsim_l151(worlds, hostsim_lib):
    check_events(worlds.get("l151", read_length=151, seed=7, extra=("--shuffle", "--varnames")), hostsim_lib)


CFG5 = dict(scale=0.002, genes=800, breakpoints=400, fragments=40000, extra=("--mismapper-frac", "0.3", "--paralog-frac", "0.15"))


def test_events_hostsim_mismapper_heavy(worlds, hostsim_lib):
    """BASELINE.json configs[4] in miniature: homologous partners, clipped segments alignable in the donor, adjacent breakpoints, ITD merges."""
    w = worlds.get("cfg5", **CFG5)
    mm = w.stage("ev_mismappers")
    assert (mm["frag_filter"] == 11).sum() > 1000 and (mm["filter"] == 11).sum() > 20 and (w.stage("ev_homologs")["filter"] == 37).sum() > 5
    assert (w.stage("ev_merge_adjacent")["filter"] == 23).sum() > 20
    check_events(w, hostsim_lib)


def test_events_hostsim_cooperative_realignment(worlds, hostsim_lib, monkeypatch):
    """A tiny step budget pushes almost every (candidate, read) pair through the cooperative second pass; labels must not change."""
    monkeypatch.setenv("ARB_MISMAP_BUDGET", "24"); monkeypatch.setenv("ARB_MISMAP_LANES", "7"); monkeypatch.setenv("ARB_MISMAP_TASK_LANES", "3")
    p = check_events(worlds.get("cfg5", **CFG5), hostsim_lib, keep=True)
    tm = p.context().timings(); p.close()
    assert tm.mismapper_heavy_items > 0.2 * tm.mismapper_items
    assert tm.mismapper_tasks > 1000 and tm.mismapper_rounds >= 2   # continuations of continuations were registered as well


@pytest.mark.parametrize("table", ["1048576", "64", "1"])
def test_events_hostsim_continuation_registry(worlds, hostsim_lib, monkeypatch, table):
    """A registry large enough for every continuation, and first registries so small that registrations fail: the items they belong to are re-aligned again
    with a larger one."""
    monkeypatch.setenv("ARB_MISMAP_BUDGET", "24"); monkeypatch.setenv("ARB_MISMAP_LANES", "5")
    monkeypatch.setenv("ARB_MISMAP_TASK_LANES", "4"); monkeypatch.setenv("ARB_MISMAP_TABLE_TOTAL", table)
    p = check_events(worlds.get("cfg5", **CFG5), hostsim_lib, keep=True)
    tm = p.context().timings(); p.close()
    if int(table) <= 64:
        assert tm.mismapper_overflow > 0


@pytest.mark.parametrize("lanes", ["1", "7"])
def test_events_hostsim_homolog_lanes(worlds, hostsim_lib, monkeypatch, lanes):
    """filter_homologs' identity test with one thread per gene pair and with lanes that split the positions: same verdicts."""
    monkeypatch.setenv("ARB_HOMOLOG_LANES", lanes)
    check_events(worlds.get("cfg5", **CFG5), hostsim_lib)


@pytest.mark.gpu
@pytest.mark.parametrize("lanes", ["1", "32"])
def test_events_cuda_homolog_lanes(worlds, cuda_lib, monkeypatch, lanes):
    monkeypatch.setenv("ARB_HOMOLOG_LANES", lanes)
    check_events(worlds.get("cfg5", **CFG5), cuda_lib)


@pytest.mark.gpu
def test_events_cuda_mismapper_heavy(worlds, cuda_lib):
    check_events(worlds.get("cfg5", **CFG5), cuda_lib)


@pytest.mark.gpu
@pytest.mark.parametrize("budget,lanes,task_lanes", [("16", "32", "32"), ("200", "256", "32"), ("0", "1", "1"), ("64", "8", "5")])
def test_events_cuda_cooperative_realignment(worlds, cuda_lib, monkeypatch, budget, lanes, task_lanes):
    monkeypatch.setenv("ARB_MISMAP_BUDGET", budget); monkeypatch.setenv("ARB_MISMAP_LANES", lanes); monkeypatch.setenv("ARB_MISMAP_TASK_LANES", task_lanes)
    check_events(worlds.get("cfg5", **CFG5), cuda_lib)


@pytest.mark.gpu
def test_events_cuda(worlds, cuda_lib):
    check_events(worlds.get("small"), cuda_lib)
