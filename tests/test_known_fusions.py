"""Known fusions (-k) and tags (-t): both files are read like the reference reads them and matched to the candidates on the device (csrc/blacklist_hd.h).
Known fusions put candidates that min_support or relative_support removed back, right after the intronic filter; tags fill the tags column of every written
row. Both output files, the WARNING lines and the progress lines must equal the reference's; every rescue verdict and every row's tags must equal
tests/known_fusions_ref.py, a plain transcription of the reference loops."""
import gzip
import os
import random
import subprocess
import sys
import numpy as np
import pytest
import blacklisttools
import known_fusions_ref as kref
from arriba_b200 import lib as L, _build
from test_genomic_support import contig_names, contig_ids, oracle_run, sv_file, ZCHR, L151

F_NONE, F_KNOWN_FUSIONS, F_RELATIVE_SUPPORT, F_MIN_SUPPORT = 0, 18, 12, 17
CB_TSTART_GENE1 = 128
INTRONIC = L.EV_NAMES.index("intronic")
NO_BL = ("-f", "blacklist")


def _world(worlds, name):
    if name == "cfg5":
        from test_events import CFG5
        return worlds.get(name, **CFG5)
    return worlds.get(name, **{"small": {}, "l151": L151, "zchr": ZCHR}[name])


def stage_state(w, lib_path, known_fusions=None):
    """The candidates after the intronic stage (with known_fusions: after the rescue), the genes, the gene names, max_mate_gap and the coverage windows."""
    p = L.Pipeline(w.prefix + ".bam", w.prefix + ".gtf", w.prefix + ".fa", threads=2, lib_path=lib_path, known_fusions=known_fusions)
    p.run(); p.events(INTRONIC)
    cand = p.candidates(); genes = p.genes(); mmg = int(p.stats().max_mate_gap)
    windows = [p.coverage(c)[0] for c in range(int(genes["n_contigs"]))]
    p.close()
    names = blacklisttools.gene_names(w.prefix + ".gtf", genes, contig_ids(w))
    return cand, genes, names, mmg, windows


def _name(nm, c, rng):
    n = nm[c]
    bare = n[3:] if n.startswith("chr") else n
    return rng.choice([bare, "chr" + bare])


TAGS = ["driver", "COSMIC", "a,b", "a b", "a_b", "two words", "\xe9t\xe9", "tab\x7fdel", "x", "driver"]


def rule_lines(cand, genes, names, nm, rng, mmg, tags=False, n_candidates=300):
    """Rules written from the world's candidates: 5'->3' and swapped, positions, genes, ranges at the 0.5 overlap, strands, wildcards, keywords (warnings),
    and with tags, the third column (several per candidate, some empty, some that sanitise to one string)."""
    n = len(cand["breakpoint1"])
    gs, ge = genes["gene_start"], genes["gene_end"]
    eligible = [k for k in range(n) if cand["filter"][k] in (F_RELATIVE_SUPPORT, F_MIN_SUPPORT) and cand["gene1"][k] != cand["gene2"][k]]
    others = [k for k in range(n) if k not in set(eligible)]
    pick = rng.sample(eligible, min(len(eligible), n_candidates)) + rng.sample(others, min(len(others), n_candidates // 3 if tags else 20))
    out = ["# written from the world's candidates", ""]

    def side(k, w):
        return int(cand["contig%d" % w][k]), int(cand["breakpoint%d" % w][k]), int(cand["gene%d" % w][k])

    def item(k, w, kind=None):
        c, b, g = side(k, w)
        kind = kind or rng.choice(["pos", "pos", "gene", "range", "strand", "wild"])
        if kind == "gene" and names[g] is not None:
            return names[g]
        if kind == "range":
            s, e = int(gs[g]), int(ge[g]); h = (e - s + 1) // 2
            return rng.choice(["%s:%d-%d" % (_name(nm, c, rng), s - 2, e + 4), "%s:%d-%d" % (_name(nm, c, rng), s + 1, s + 1 + h + rng.choice((-1, 0, 1))),
                               "%s:%d-%d" % (_name(nm, c, rng), s - 10, s + h + rng.choice((-1, 0, 1)))])
        if kind == "strand":
            return "%s%s:%d" % (rng.choice("+-"), _name(nm, c, rng), b + 1)
        if kind == "wild":
            bare = nm[c][3:] if nm[c].startswith("chr") else nm[c]
            return "%s*:%d" % (bare, b + 1)
        return "%s:%d" % (_name(nm, c, rng), b + 1 + (rng.choice((0, 0, 0, 1, -1, mmg, -mmg)) if int(cand["split_reads1"][k]) + int(cand["split_reads2"][k]) == 0 else 0))

    def tag():
        return rng.choice(TAGS)

    for k in pick:
        g5 = 1 if int(cand["bits"][k]) & CB_TSTART_GENE1 else 2
        g3 = 3 - g5
        rows = [(item(k, g5), item(k, g3)), (item(k, g5, "pos"), item(k, g3, "pos")), (item(k, g3), item(k, g5))]  # 5'->3', positions, swapped
        if rng.random() < 0.3:
            rows.append((item(k, g5, "gene"), item(k, g3, "range")))
        for a, b in rows:
            out.append("%s\t%s\t%s" % (a, b, tag()) if tags else "%s\t%s" % (a, b))
        if tags and rng.random() < 0.5:
            out.append("%s\t%s\t%s" % (item(k, g5, "pos"), item(k, g3, "pos"), tag()))  # a second tag on the same row
    nm0 = nm[int(cand["contig1"][pick[0]])] if pick else nm[0]
    junk = ["any\t%s:100" % nm0, "%s:100\tany" % nm0, "%s:100\tsplit_read_any" % nm0, "\t%s:100" % nm0, "%s:100\t" % nm0, "nocolon\t%s:5" % nm0, "unknown_contig:100\t%s:5" % nm0,
            "no_such_gene\t%s:7" % nm0, "# comment"]
    if tags:
        junk = ["%s\tT%d" % (l, x) for x, l in enumerate(junk)] + ["%s:100\t%s:200" % (nm0, nm0), "%s:100\t%s:200\t" % (nm0, nm0), "%s:100\t%s:200\t\tlate" % (nm0, nm0)]
    out += junk
    rng.shuffle(out)
    return out


def write(path, lines, crlf=False):
    data = (("\r\n" if crlf else "\n").join(lines) + "\n").encode("latin-1")
    if path.endswith(".gz"):
        with gzip.open(path, "wb") as f:
            f.write(data)
    else:
        open(path, "wb").write(data)


_FILES = {}


def rules_file(w, lib_path, root, tags, variant="plain", seed=5):
    key = (w.prefix, tags, variant, seed)
    if key not in _FILES:
        cand, genes, names, mmg, _ = stage_state(w, lib_path)
        lines = rule_lines(cand, genes, names, contig_names(w), random.Random(seed), mmg, tags)
        path = os.path.join(root, "%s_%d_%s%s" % ("tags" if tags else "kf", len(_FILES), variant, ".tsv.gz" if variant == "gz" else ".tsv"))
        write(path, lines, crlf=variant == "crlf")
        _FILES[key] = path
    return _FILES[key]


@pytest.fixture(scope="module")
def cli():
    return _build.build_cli_hostsim()


@pytest.fixture(scope="module")
def kf_root(tmp_path_factory):
    return str(tmp_path_factory.mktemp("kf"))


def warnings_of(text):
    return [l for l in text.splitlines() if l.startswith("WARNING: unknown gene") or l.startswith("WARNING: encountered a line")]


def progress_of(text):
    return [l.split("] ", 1)[1].strip() for l in text.splitlines() if "Searching for known fusions" in l or "Loading tags" in l]


def cli_run(cli, w, args, tmp, env=None, discarded=True):
    out = os.path.join(tmp, "fusions.tsv"); disc = os.path.join(tmp, "fusions.discarded.tsv")
    cmd = [cli, "-x", w.prefix + ".bam", "-g", w.prefix + ".gtf", "-a", w.prefix + ".fa", "-o", out, "-@", "3"] + (["-O", disc] if discarded else []) + list(args)
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=dict(os.environ, **(env or {})))
    assert r.returncode == 0, r.stderr[-2000:]
    return r, open(out, "rb").read(), open(disc, "rb").read() if discarded else None


def cli_parity(cli, w, args, tmp, env=None, discarded=True):
    ref = oracle_run(w, args, os.path.join(tmp, "oracle"))
    r, fus, disc = cli_run(cli, w, args, tmp, env, discarded)
    assert fus == open(os.path.join(ref.outdir, "fusions.tsv"), "rb").read(), "fusions.tsv differs with %s" % (args,)
    if discarded:
        assert disc == open(os.path.join(ref.outdir, "fusions.discarded.tsv"), "rb").read(), "fusions.discarded.tsv differs with %s" % (args,)
    assert warnings_of(r.stderr) == warnings_of(open(os.path.join(ref.outdir, "stderr.txt"), encoding="latin-1").read())
    assert progress_of(r.stdout) == progress_of(open(os.path.join(ref.outdir, "stdout.txt")).read())
    return ref, fus, disc


def tagged_rows(blob):
    return [l.split(b"\t")[16] for l in blob.splitlines()[1:] if l.split(b"\t")[16] != b"."]


CASES = [
    ("small", "plain", "k", ()), ("small", "plain", "t", ()), ("small", "plain", "kt", ()), ("small", "crlf", "kt", ("-E", "0.3")), ("small", "gz", "kt", ("-E", "1000")),
    ("small", "plain", "kt", ("-X",)), ("l151", "plain", "kt", ()), ("zchr", "plain", "kt", ()), ("cfg5", "plain", "kt", ()),
]


@pytest.mark.parametrize("name,variant,which,extra", CASES, ids=lambda x: x if isinstance(x, str) else " ".join(x) if isinstance(x, tuple) else None)
def test_cli_parity(worlds, cli, hostsim_lib, kf_root, tmp_path, name, variant, which, extra):
    w = _world(worlds, name)
    args = tuple(extra) + NO_BL
    if "k" in which:
        args += ("-k", rules_file(w, hostsim_lib, kf_root, False, variant))
    if "t" in which:
        args += ("-t", rules_file(w, hostsim_lib, kf_root, True, variant))
    ref, fus, disc = cli_parity(cli, w, args, str(tmp_path))
    if "t" in which:
        rows = tagged_rows(fus) + tagged_rows(disc)
        assert tagged_rows(disc) and any(b"," in t for t in rows), "no discarded row carries a tag, or no row carries two"
        if name == "small":
            assert tagged_rows(fus)


def test_cli_parity_with_blacklist_and_genomic(worlds, cli, hostsim_lib, kf_root, tmp_path):
    w = worlds.get("small")
    k, t = rules_file(w, hostsim_lib, kf_root, False), rules_file(w, hostsim_lib, kf_root, True)
    cand, genes, names, mmg, _ = stage_state(w, hostsim_lib)
    bl = os.path.join(kf_root, "bl.tsv")
    blacklisttools.write(bl, blacklisttools.rule_lines(cand, genes, names, contig_names(w), random.Random(3), mmg, n_candidates=40))
    cli_parity(cli, w, ("-b", bl, "-k", k, "-t", t), str(tmp_path / "b"))
    sv = sv_file(w, hostsim_lib, kf_root)
    cli_parity(cli, w, NO_BL + ("-d", sv, "-k", k, "-t", t), str(tmp_path / "d"))


def test_cli_parity_filter_off_and_no_discarded_file(worlds, cli, hostsim_lib, kf_root, tmp_path):
    """-f known_fusions: the file is never read (no warnings, no progress line), the output equals the run without -k; without -O only fusions.tsv is tagged."""
    w = worlds.get("small")
    k, t = rules_file(w, hostsim_lib, kf_root, False), rules_file(w, hostsim_lib, kf_root, True)
    r1, f1, d1 = cli_run(cli, w, ("-f", "blacklist,known_fusions"), str(tmp_path))
    r2, f2, d2 = cli_run(cli, w, ("-f", "blacklist,known_fusions", "-k", k), str(tmp_path))
    assert f1 == f2 and d1 == d2 and warnings_of(r2.stderr) == [] and "known fusions" not in r2.stdout
    cli_parity(cli, w, ("-f", "blacklist,known_fusions", "-k", k, "-t", t), str(tmp_path / "off"))
    cli_parity(cli, w, NO_BL + ("-k", k, "-t", t), str(tmp_path / "noO"), discarded=False)


def test_cli_parity_scattered_and_poisoned(worlds, cli, hostsim_lib, kf_root, tmp_path):
    w = worlds.get("small")
    cli_parity(cli, w, NO_BL + ("-k", rules_file(w, hostsim_lib, kf_root, False), "-t", rules_file(w, hostsim_lib, kf_root, True)), str(tmp_path),
               env={"ARB_HOSTSIM_ORDER": "2", "ARB_HOSTSIM_POISON": "1", "ARB_BLACKLIST_SHORT_LIST": "0"})


# ---- per candidate, through the C ABI
def _parse(w, path, genes, names, tags):
    return kref.read_rules(path, contig_ids(w), blacklisttools.gene_by_name(names), genes["gene_contig"], genes["gene_start"], genes["gene_end"], tags=tags)


def rescue_against_reference(w, lib_path, path, short_list=None):
    """The rescued candidates of the product (after intronic, with -k, against the same stage without it) against known_fusions_ref.py."""
    if short_list is not None:
        os.environ["ARB_BLACKLIST_SHORT_LIST"] = str(short_list)
    try:
        before, genes, names, mmg, windows = stage_state(w, lib_path)
        p = L.Pipeline(w.prefix + ".bam", w.prefix + ".gtf", w.prefix + ".fa", threads=2, lib_path=lib_path, known_fusions=path)
        p.run(); p.events(INTRONIC)
        after = p.candidates(); timings = p.context().timings(); p.close()
        rules, _ = _parse(w, path, genes, names, False)
        want = kref.rescued(rules, before, genes, mmg, windows)
        got = set(np.flatnonzero((after["filter"] == F_NONE) & (before["filter"] != F_NONE)).tolist())
        assert got == set(want), (sorted(got - set(want))[:10], sorted(set(want) - got)[:10])
        return want, before, timings
    finally:
        os.environ.pop("ARB_BLACKLIST_SHORT_LIST", None)


def tags_against_reference(w, lib_path, path, short_list=None, sample=None):
    """The tags arb_annotate_tags finds for the rows against known_fusions_ref.py, on the candidates after all stages: every candidate, or with `sample`, the
    unfiltered ones and `sample` others (the transcription is slow on dense files); the rows not asked for must have none."""
    if short_list is not None:
        os.environ["ARB_BLACKLIST_SHORT_LIST"] = str(short_list)
    try:
        p = L.Pipeline(w.prefix + ".bam", w.prefix + ".gtf", w.prefix + ".fa", threads=2, lib_path=lib_path)
        p.run(); p.events(len(L.EV_NAMES) - 1)
        cand = p.candidates(); genes = p.genes(); mmg = int(p.stats().max_mate_gap)
        names = blacklisttools.gene_names(w.prefix + ".gtf", genes, contig_ids(w))
        rules, _ = _parse(w, path, genes, names, True)
        ctx = p.context()
        ctx.set_candidate_state(cand["filter"], cand["split_reads1"], cand["split_reads2"], cand["discordant_mates"], cand["evalue"])
        ctx.set_tags(kref.rule_columns(rules), [r[2] for r in rules])
        ids = np.arange(int(cand["n"]), dtype=np.uint32)
        if sample is not None:
            rest = [k for k in ids.tolist() if cand["filter"][k] != F_NONE]
            ids = np.array(sorted(set(np.flatnonzero(cand["filter"] == F_NONE).tolist()) | set(random.Random(2).sample(rest, min(sample, len(rest))))), np.uint32)
        got = ctx.annotate_tags(ids, mmg)
        timings = ctx.timings(); p.close()
        want = {k: [] for k in range(int(cand["n"]))}
        want.update(kref.tags_of(rules, cand, genes, mmg, ids.tolist()))
        bad = [k for k in range(int(cand["n"])) if [t.decode("latin-1") for t in got[k]] != want[k]]
        assert not bad, [(k, got[k], want[k]) for k in bad[:5]]
        return want, timings
    finally:
        os.environ.pop("ARB_BLACKLIST_SHORT_LIST", None)


@pytest.mark.parametrize("short_list", [None, 0])
def test_rescue_of_every_candidate(worlds, hostsim_lib, kf_root, short_list):
    w = worlds.get("small")
    want, _, _ = rescue_against_reference(w, hostsim_lib, rules_file(w, hostsim_lib, kf_root, False), short_list)
    assert len(want) > 5


@pytest.mark.parametrize("short_list", [None, 0])
def test_tags_of_every_candidate(worlds, hostsim_lib, kf_root, short_list):
    w = worlds.get("small")
    want, _ = tags_against_reference(w, hostsim_lib, rules_file(w, hostsim_lib, kf_root, True), short_list)
    assert sum(1 for v in want.values() if len(v) >= 2) > 0 and sum(1 for v in want.values() if v) > 20


IN_VITRO = L.EV_NAMES.index("in_vitro")


def _eligible(c, k):
    return int(c["filter"][k]) in (F_RELATIVE_SUPPORT, F_MIN_SUPPORT) and int(c["gene1"][k]) != int(c["gene2"][k])


def _far(c, k, distance=1000000):
    return int(c["contig1"][k]) != int(c["contig2"][k]) or abs(int(c["breakpoint2"][k]) - int(c["breakpoint1"][k])) > distance


def test_swapped_order_probes(worlds, hostsim_lib, kf_root):
    """One swapped-only rule (3' position, then 5' position) per target candidate and nothing else for it: it rescues a candidate with an ambiguous transcript
    start whose breakpoints are more than 1 Mb apart, and neither one within 1 Mb nor one whose transcript start is certain."""
    w = worlds.get("small")
    cand, genes, names, mmg, _ = stage_state(w, hostsim_lib)
    nm = contig_names(w)
    pos = lambda k, s: (int(cand["contig%d" % s][k]), int(cand["breakpoint%d" % s][k]))
    n = int(cand["n"])
    # a target's rule must not match another candidate with the same breakpoints
    seen = {}
    for k in range(n):
        key = frozenset((pos(k, 1), pos(k, 2))); seen[key] = seen.get(key, 0) + 1
    unique = lambda k: seen[frozenset((pos(k, 1), pos(k, 2)))] == 1
    far_ambiguous, close_ambiguous, certain = [], [], []
    for k in range(n):
        if not _eligible(cand, k) or not unique(k):
            continue
        if int(cand["bits2"][k]) and _far(cand, k):
            far_ambiguous.append(k)
        elif int(cand["bits2"][k]) and not _far(cand, k, 999999) and abs(int(cand["breakpoint2"][k]) - int(cand["breakpoint1"][k])) > 2 * mmg + 2:
            close_ambiguous.append(k)
        elif not int(cand["bits2"][k]) and _far(cand, k):
            certain.append(k)
    assert far_ambiguous and close_ambiguous and certain, (len(far_ambiguous), len(close_ambiguous), len(certain))
    lines = []
    for k in far_ambiguous + close_ambiguous + certain:
        g5 = 1 if int(cand["bits"][k]) & CB_TSTART_GENE1 else 2
        (c3, b3), (c5, b5) = pos(k, 3 - g5), pos(k, g5)
        lines.append("%s:%d\t%s:%d" % (nm[c3], b3 + 1, nm[c5], b5 + 1))
    path = os.path.join(kf_root, "swapped.tsv"); write(path, lines)
    # a control that some line matches in the 5'->3' order (another candidate's rule at the same positions, or within max_mate_gap) proves nothing
    rules, _ = _parse(w, path, genes, names, False)
    unambiguous = dict(cand); unambiguous["bits2"] = np.zeros_like(cand["bits2"])
    direct = set(kref.rescued(rules, unambiguous, genes, mmg, [p.tolist() for p in stage_state(w, hostsim_lib)[4]]))
    controls = (set(close_ambiguous) | set(certain)) - direct
    assert len(controls & set(close_ambiguous)) >= 5 and len(controls & set(certain)) >= 5
    for short_list in (None, 0):
        want, _, _ = rescue_against_reference(w, hostsim_lib, path, short_list)
        assert set(far_ambiguous) <= set(want), sorted(set(far_ambiguous) - set(want))[:5]
        assert not controls & set(want), sorted(controls & set(want))[:5]


def abi_probes(w, lib_path, short_list=None):
    """Through the C ABI on a world's candidates after in_vitro (coverage resident), with candidate states set by the test:
    - spliced: both breakpoints spliced, coverage < 200, > 1 Mb apart, given one read and a low-support filter, and one rule of the two gene ranges each:
      every one is rescued, and only by the spliced way;
    - bins: the same candidates made discordant-only, with a rule of two positions in the direction the mates point, within max_mate_gap (set to 3 Mb here)
      but in 100 kb bins that none of the candidate's four ranges touch: the rule's bins are not widened, so none is found; the same rule moved into the
      breakpoints' own bins is found."""
    if short_list is not None:
        os.environ["ARB_BLACKLIST_SHORT_LIST"] = str(short_list)
    try:
        p = L.Pipeline(w.prefix + ".bam", w.prefix + ".gtf", w.prefix + ".fa", threads=2, lib_path=lib_path)
        p.run(); p.events(IN_VITRO)
        cand = p.candidates(); genes = p.genes()
        windows = [p.coverage(c)[0] for c in range(int(genes["n_contigs"]))]
        names = blacklisttools.gene_names(w.prefix + ".gtf", genes, contig_ids(w))
        nm = contig_names(w)
        ctx = p.context()
        gs, ge = genes["gene_start"], genes["gene_end"]
        cov = lambda k: (kref.coverage_get(windows, int(cand["contig1"][k]), int(cand["breakpoint1"][k]), 1 - int(cand["direction1"][k]))
                         + kref.coverage_get(windows, int(cand["contig2"][k]), int(cand["breakpoint2"][k]), 1 - int(cand["direction2"][k])))
        targets = [k for k in range(int(cand["n"])) if int(cand["gene1"][k]) != int(cand["gene2"][k]) and kref._both_spliced(cand, k, genes["gene_strand"])
                   and cov(k) < 200 and _far(cand, k)]
        assert len(targets) >= 5, len(targets)
        tmp = os.path.join(os.path.dirname(w.prefix), "abi_probe.tsv")

        def run(state, lines, mmg):
            write(tmp, lines)
            rules, _ = kref.read_rules(tmp, contig_ids(w), blacklisttools.gene_by_name(names), genes["gene_contig"], gs, ge)
            ctx.set_candidate_state(state["filter"], state["split_reads1"], state["split_reads2"], state["discordant_mates"], state["evalue"])
            ctx.set_known_fusions(kref.rule_columns(rules))
            ids = np.array([k for k in range(int(state["n"])) if _eligible(state, k)], np.uint32)
            got = set(ids[ctx.recover_known_fusions(ids, mmg) != 0].tolist())
            want = kref.rescued(rules, state, genes, mmg, windows)
            assert got == set(want), (sorted(got - set(want))[:5], sorted(set(want) - got)[:5])
            return want

        def state_with(sr1, sr2, dm):
            st = dict(cand)
            for col in ("filter", "split_reads1", "split_reads2", "discordant_mates"):
                st[col] = st[col].copy()
            st["filter"][targets] = F_MIN_SUPPORT; st["split_reads1"][targets] = sr1; st["split_reads2"][targets] = sr2; st["discordant_mates"][targets] = dm
            return st

        def side(k, s):
            return int(cand["contig%d" % s][k]), int(cand["breakpoint%d" % s][k]), int(cand["direction%d" % s][k]), int(cand["gene%d" % s][k])

        # spliced
        lines = []
        for k in targets:
            g5 = 1 if int(cand["bits"][k]) & CB_TSTART_GENE1 else 2
            rng = lambda s: "%s:%d-%d" % (nm[side(k, s)[0]], int(gs[side(k, s)[3]]) + 1, int(ge[side(k, s)[3]]) + 1)
            lines.append("%s\t%s" % (rng(g5), rng(3 - g5)))
        want = run(state_with(1, 0, 0), lines, 120)
        assert all(want.get(k) == "spliced" for k in targets), [(k, want.get(k)) for k in targets if want.get(k) != "spliced"][:5]

        # bins: positions 1.5-2.5 Mb away in the direction of the mates, outside every bin of the candidate's four ranges
        MMG = 3000000
        far_lines, near_lines, probed = [], [], []
        for k in targets:
            ranges = []
            for s in (1, 2):
                c, b, d, g = side(k, s)
                ranges += kref._bins(c, b, b) + kref._bins(c, int(gs[g]), int(ge[g]))
            items = []
            for s in (1, 2):
                c, b, d, g = side(k, s)
                q = b + 2000000 if d == kref.DOWNSTREAM else b - 2000000
                items.append((c, q))
            if any(q < 0 for c, q in items) or any(bn in ranges for c, q in items for bn in kref._bins(c, q, q)):
                continue
            g5 = 1 if int(cand["bits"][k]) & CB_TSTART_GENE1 else 2
            it5, it3 = items[g5 - 1], items[2 - g5]
            far_lines.append("%s:%d\t%s:%d" % (nm[it5[0]], it5[1] + 1, nm[it3[0]], it3[1] + 1))
            near_lines.append("%s:%d\t%s:%d" % (nm[side(k, g5)[0]], side(k, g5)[1] + 1, nm[side(k, 3 - g5)[0]], side(k, 3 - g5)[1] + 1))
            probed.append(k)
        assert len(probed) >= 3, len(probed)
        discordant_only = state_with(0, 0, 1)
        assert not set(probed) & set(run(discordant_only, far_lines, MMG))
        assert set(probed) <= set(run(discordant_only, near_lines, MMG))
        p.close()
        return targets, probed
    finally:
        os.environ.pop("ARB_BLACKLIST_SHORT_LIST", None)


@pytest.mark.parametrize("short_list", [None, 0])
def test_abi_probes(worlds, hostsim_lib, short_list):
    abi_probes(worlds.get("small"), hostsim_lib, short_list)


def dense_file(w, lib_path, root, tags, n=100000):
    path = os.path.join(root, "dense_%s_%d.tsv" % (os.path.basename(os.path.dirname(w.prefix)), tags))
    if not os.path.exists(path):
        cand, genes, names, mmg, _ = stage_state(w, lib_path)
        rng = random.Random(9)
        lines = blacklisttools.dense_lines(cand, genes, contig_names(w), rng, n, mmg)
        if tags:
            lines = ["%s\tt%d" % (l, rng.randint(0, 40)) for l in lines]
        write(path, lines)
    return path


def test_dense_files_hostsim(worlds, hostsim_lib, kf_root):
    w = worlds.get("small")
    rescue_against_reference(w, hostsim_lib, dense_file(w, hostsim_lib, kf_root, False))
    want, _ = tags_against_reference(w, hostsim_lib, dense_file(w, hostsim_lib, kf_root, True), sample=400)
    assert any(want.values())


def test_cli_errors(worlds, cli, tmp_path):
    """Unreadable -k / -t stop both programs with the same ERROR line; the inputs the reference has no defined behaviour for name the file's kind."""
    w = worlds.get("small")
    oracle = _build.build_oracle()
    base = ["-x", w.prefix + ".bam", "-g", w.prefix + ".gtf", "-a", w.prefix + ".fa", "-o", str(tmp_path / "o.tsv"), "-f", "blacklist"]
    for opt in ("-k", "-t"):
        seen = []
        for exe in (oracle, cli):
            r = subprocess.run([exe] + base + [opt, str(tmp_path / "missing.tsv")], capture_output=True, text=True, timeout=300)
            seen.append((r.returncode, [l for l in r.stderr.splitlines() if l.startswith("ERROR")]))
        assert seen[0] == seen[1] and seen[0][0] == 1, seen
    nm = contig_names(w)[0]
    for opt, kind, suffix in (("-k", "known fusions", ""), ("-t", "tags", "\tT")):
        for line, why in (("~~~*:100\t%s:5" % nm, "sorts after every contig name"), ("%s:1-2147483000\t%s:5" % (nm, nm), "overflow int")):
            path = str(tmp_path / "ub.tsv"); write(path, ["%s:100\t%s:5%s" % (nm, nm, suffix), line + suffix])
            r = subprocess.run([cli] + base + [opt, path], capture_output=True, text=True, timeout=300)
            assert r.returncode == 1 and why in r.stderr and "line 2" in r.stderr and "%s '" % kind in r.stderr, r.stderr[-2000:]
    path = str(tmp_path / "ok.tsv"); write(path, ["%s:2147383000\t%s:5" % (nm, nm)])  # not widened by max_mate_gap: still within int for -k
    r = subprocess.run([cli] + base + ["-k", path], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]


def C_byref(x):
    import ctypes
    return ctypes.byref(x)


def test_no_options_change_nothing(worlds, hostsim_lib, kf_root, tmp_path):
    """Without -k / -t, or with -k while the filter is off, the files and the number of kernel launches equal those of a run that never heard of them."""
    w = worlds.get("small")
    path = rules_file(w, hostsim_lib, kf_root, False)
    lib = L.load(hostsim_lib)
    res = []
    for kf, on in ((None, True), (path, False), (None, False)):
        d = str(tmp_path / ("run%d" % len(res))); os.makedirs(d)
        prm = L.Params(); lib.arb_default_params(C_byref(prm))
        if not on:
            prm.filter_mask &= ~(1 << F_KNOWN_FUSIONS)
        p = L.Pipeline(w.prefix + ".bam", w.prefix + ".gtf", w.prefix + ".fa", threads=2, lib_path=hostsim_lib, params=prm, known_fusions=kf,
                       output=os.path.join(d, "fusions.tsv"), discarded=os.path.join(d, "fusions.discarded.tsv"))
        k0 = lib.arb_kernel_launches(); p.run_all(); k1 = lib.arb_kernel_launches(); p.close()
        res.append((k1 - k0, open(os.path.join(d, "fusions.tsv"), "rb").read(), open(os.path.join(d, "fusions.discarded.tsv"), "rb").read()))
    assert res[0] == res[1] == res[2]


WORKER = r"""
import os, sys
sys.path.insert(0, {root!r})
import torch.distributed as dist
from arriba_b200 import lib as L, sharded
rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"])
dist.init_process_group("gloo")
out = os.path.join({outdir!r}, "rank%d" % rank); os.makedirs(out, exist_ok=True)
p = L.Pipeline({prefix!r} + ".bam", {prefix!r} + ".gtf", {prefix!r} + ".fa", threads=2, lib_path={lib!r}, known_fusions={kf!r}, tags={tags!r},
               output=os.path.join(out, "fusions.tsv"), discarded=os.path.join(out, "fusions.discarded.tsv"))
sharded.run_sharded(p, rank, world)
p.close()
dist.destroy_process_group()
"""


def test_sharded_two_ranks(worlds, hostsim_lib, kf_root, tmp_path):
    w = worlds.get("small")
    kf, tags = rules_file(w, hostsim_lib, kf_root, False), rules_file(w, hostsim_lib, kf_root, True)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = str(tmp_path / "worker.py")
    open(script, "w").write(WORKER.format(root=root, outdir=str(tmp_path), prefix=w.prefix, lib=hostsim_lib, kf=kf, tags=tags))
    env = dict(os.environ, PYTHONPATH=root + os.pathsep + os.path.join(root, "tests"))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port", str(29700 + os.getpid() % 200), script]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    single = str(tmp_path / "single"); os.makedirs(single)
    p = L.Pipeline(w.prefix + ".bam", w.prefix + ".gtf", w.prefix + ".fa", threads=2, lib_path=hostsim_lib, known_fusions=kf, tags=tags,
                   output=os.path.join(single, "fusions.tsv"), discarded=os.path.join(single, "fusions.discarded.tsv"))
    p.run_all(); p.close()
    for f in ("fusions.tsv", "fusions.discarded.tsv"):
        assert open(os.path.join(tmp_path, "rank0", f), "rb").read() == open(os.path.join(single, f), "rb").read(), f
    assert tagged_rows(open(os.path.join(single, "fusions.discarded.tsv"), "rb").read())


# ---- on the H100
def pipeline_parity(w, lib_path, args, kf, tags, tmp, blacklist=None):
    ref = oracle_run(w, args, os.path.join(tmp, "oracle"))
    out = os.path.join(tmp, "fusions.tsv"); disc = os.path.join(tmp, "fusions.discarded.tsv")
    p = L.Pipeline(w.prefix + ".bam", w.prefix + ".gtf", w.prefix + ".fa", threads=8, lib_path=lib_path, known_fusions=kf, tags=tags, blacklist=blacklist, output=out, discarded=disc)
    p.run_all(); p.close()
    for f in ("fusions.tsv", "fusions.discarded.tsv"):
        assert open(os.path.join(tmp, f), "rb").read() == open(os.path.join(ref.outdir, f), "rb").read(), f


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small", "cfg5"])
def test_parity_cuda(worlds, cuda_lib, hostsim_lib, kf_root, tmp_path, name):
    w = _world(worlds, name)
    kf, tags = rules_file(w, hostsim_lib, kf_root, False), rules_file(w, hostsim_lib, kf_root, True)
    pipeline_parity(w, cuda_lib, NO_BL + ("-k", kf, "-t", tags), kf, tags, str(tmp_path / "lib"))
    cli = _build.build_cli()
    cli_parity(cli, w, NO_BL + ("-k", kf, "-t", tags), str(tmp_path / "cli"))
    cand, genes, names, mmg, _ = stage_state(w, hostsim_lib)
    bl = os.path.join(kf_root, "bl_%s.tsv" % name)
    blacklisttools.write(bl, blacklisttools.rule_lines(cand, genes, names, contig_names(w), random.Random(3), mmg, n_candidates=40))
    cli_parity(cli, w, ("-X", "-k", kf, "-t", tags, "-b", bl), str(tmp_path / "cli_x"))


@pytest.mark.gpu
def test_dense_files_cuda(worlds, cuda_lib, hostsim_lib, kf_root):
    w = worlds.get("small")
    for short_list in (None, 0):
        _, _, t = rescue_against_reference(w, cuda_lib, dense_file(w, hostsim_lib, kf_root, False), short_list)
        assert t.known_fusions_ms > 0
        want, t = tags_against_reference(w, cuda_lib, dense_file(w, hostsim_lib, kf_root, True), short_list, sample=400)
        assert any(want.values()) and t.tags_ms > 0


@pytest.mark.gpu
def test_abi_probes_cuda(worlds, cuda_lib):
    for short_list in (None, 0):
        abi_probes(worlds.get("small"), cuda_lib, short_list)
