"""The re-alignment stage (`arb_filter_mismappers`), the gene homology test (`arb_homolog_pairs`) and the k-mer index under both
(`arb_build_kmer_index`, `arb_selftest_kmer_lookup`) against the plain reference in mismaprules.py, on the world of mismapworld.py.

Every check runs through the CPU stand-in (*_hostsim) and the device (*_cuda). The re-alignment reads its test hooks (ARB_MISMAP_BUDGET,
ARB_MISMAP_LANES, ARB_MISMAP_TASK_LANES, ARB_MISMAP_TABLE_TOTAL, ARB_HOMOLOG_LANES) when a context is created, so every configuration gets a
context of its own; `Timings` shows that each one sent work down the path it is meant for. On the device every distinct fragment is
repeated many times, so that pass 1's 16-lane groups sit at every position of a block."""
import contextlib
import os
import time
import zlib
import numpy as np
import pytest
import mismaprules as R
import mismapworld as MW
import seqworld as W
from arriba_b200 import lib

DEAD_GENE = 10                         # a gene on the contig beyond the index: nothing aligns there
FRACTIONS = (0.8, 0.55)                # max_mismapper_fraction: the default and a second value
COUNT_TOTALS = (1, 2, 5, 7, 10, 13, 20, 31)
WRAP_MISMAPPERS, WRAP_OTHERS = 65_538, 10   # 65,548 listed reads: the 16-bit counters of the reference wrap
ENV_KEYS = ("ARB_MISMAP_BUDGET", "ARB_MISMAP_LANES", "ARB_MISMAP_TASK_LANES", "ARB_MISMAP_TABLE_TOTAL", "ARB_HOMOLOG_LANES")


# ------------------------------------------------------------------------------------------------ the world
class World:
    def __init__(self, seed, n_attempts, copies, padding=MW.MAX_MATE_GAP + 300):
        t0 = time.time()
        rng = np.random.default_rng(seed)
        self.rng = rng
        genes, many = MW.make_genes(rng)
        contigs = MW.make_genome(rng)
        contigs, self.homolog_planted = MW.plant_homologs(rng, contigs, genes)
        self.genes, self.many = genes, many
        self.splice = MW.splice_sites_for(rng, genes)
        self.stages = {}
        self.contigs = contigs
        self.intervals = {}
        for name, pad in (("default", padding), ("small_padding", 40)):
            iv = R.index_intervals([(c, s, e) for c, s, e, _ in genes if c < MW.N_INDEX], pad, MW.LENGTHS)
            self.intervals[name] = iv
            self.stages[name] = R.Stage(contigs, genes, self.splice, R.KmerIndex(contigs, iv, MW.N_INDEX), MW.MAX_MATE_GAP)
        self.stage = self.stages["default"]
        fam = MW.Families(rng, self.stage, many, DEAD_GENE)
        self.frags, self.twins, self.family = [], [], []
        self.same = []
        for k in range(n_attempts):
            family = MW.FAMILIES[k % len(MW.FAMILIES)]
            name, same, twins, plain = fam.one(family)
            if twins:
                self.twins.append((len(self.frags), len(self.frags) + 1))
                for f in twins:
                    self.frags.append(f); self.family.append(name); self.same.append(same)
            elif plain is not None:
                self.frags.append(plain); self.family.append(name); self.same.append(same)
        b = MW.Builder(rng, contigs, genes)
        self.dead, self.preset_mismappers, self.duplicates = [], [], []
        for k in range(40):   # random segments: not mis-mapped; fragments preset to mismappers / duplicates
            for lst, fam_name in ((self.dead, "dead"), (self.preset_mismappers, "preset_mismappers"), (self.duplicates, "duplicates")):
                lst.append(len(self.frags))
                self.frags.append(b.split(b.dead(30), b.dead(50), [DEAD_GENE], [DEAD_GENE])); self.family.append(fam_name); self.same.append(False)
        self.n_unique = len(self.frags)
        self.order = np.concatenate([rng.permutation(self.n_unique) for _ in range(copies)])
        self.cache = {}
        print("world: %d fragments (%d twins), %.1f s" % (self.n_unique, len(self.twins), time.time() - t0))

    def verdict(self, stage_name, frag, uid, swapped, kind, same):
        key = (stage_name, uid, swapped, kind, same)
        if key not in self.cache:
            self.cache[key] = self.stages[stage_name].fragment_is_mismapper(frag, kind, same)
        return self.cache[key]


def chunk_of(world, layout, rng):
    ch = W.build_chunk(world.frags, world.order, layout, rng)
    n = len(world.order)
    pool, off, cnt = [], np.zeros(3 * n, np.uint32), np.zeros(3 * n, np.uint16)
    for i, u in enumerate(world.order):
        for s, a in enumerate(world.frags[u]["alignments"]):
            off[s * n + i] = len(pool); cnt[s * n + i] = len(a["genes"]); pool += a["genes"]
    ch["genes_off"], ch["genes_cnt"], ch["genes"] = off, cnt, np.array(pool or [0], np.uint32)
    return ch


def splice_columns(splice):
    off = np.zeros(len(splice) + 1, np.uint32)
    off[1:] = np.cumsum([len(s) for s in splice])
    return off, np.array([x for s in splice for x in s] or [0], np.int32)


@contextlib.contextmanager
def environment(env):
    """The test hooks in `env` set, every other one unset, for the duration."""
    old = {k: os.environ.get(k) for k in ENV_KEYS}
    try:
        for k in ENV_KEYS:
            os.environ.pop(k, None)
        os.environ.update({k: str(v) for k, v in env.items()})
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def new_context(lib_path, env, contigs):
    with environment(env):
        ctx = lib.Context(0, lib_path)
    ctx.set_contigs(np.ones(len(contigs), np.uint8), [c.encode() for c in contigs])
    return ctx


def index_context(world, lib_path, env, stage_name="default", contigs=None):
    ctx = new_context(lib_path, env, contigs or world.contigs)
    ctx.set_annotation(MW.annotation(world.genes, len(world.contigs)))
    iv = world.intervals[stage_name]
    n = ctx.build_kmer_index([c for c, _, _ in iv], [s for _, s, _ in iv], [e for _, _, e in iv], MW.N_INDEX)
    assert n == len(world.stages[stage_name].index.pos)
    return ctx


# ------------------------------------------------------------------------------------------------ the reference against itself
def test_memoized_search_matches_plain_recursion():
    """The memo only caches a pure function: verdicts with and without it agree, on reads in tandem repeats, across splice sites and
    around the score threshold."""
    w = world_for(None, False)
    n = 0
    for u in range(0, w.n_unique, 5):
        f = w.frags[u]
        if max(len(s) for s in f["sequences"]) > 110 or n >= 50:
            continue
        for same in (False, True):
            a = w.stage.fragment_is_mismapper(f, f["kind"], same, memo=True)
            b = w.stage.fragment_is_mismapper(f, f["kind"], same, memo=False)
            assert a == b, (u, w.family[u], same)
            n += 1
    assert n >= 40


def test_world_reaches_its_edges():
    """The shapes the world promises: twins whose probe slice starts at every offset modulo 32 of the sequence pool, reverse-strand twins
    decided by an IUPAC code at every position of an 8-base word, 0-8 base segments in indexed genes, two-intron placements."""
    w = world_for(None, False)
    members = [x for pair in w.twins for x in pair]
    offsets = {MW.slice_offset(w.frags[u]) % 32 for u in members if w.frags[u].get("slot") in ("seg0", "seg1")}
    assert offsets == set(range(32)), sorted(set(range(32)) - offsets)
    positions = {w.frags[u]["iupac_word_position"] for u in members if "iupac_word_position" in w.frags[u]}
    assert positions == set(range(8)), sorted(set(range(8)) - positions)
    short = {(w.frags[u]["slot"], MW.probe_length(w.frags[u])) for u in range(w.n_unique) if w.family[u] == "short"}
    assert {L for _, L in short} == set(range(9)) and {slot for slot, _ in short} == {"seg0", "seg1", "disc"}, sorted(short)


# ------------------------------------------------------------------------------------------------ index lookups
def lookup_queries(world, rng):
    ix = world.stage.index
    cs, ks, fs = [], [], []
    present = np.unique(ix.key)
    for c in range(MW.N_INDEX):
        L = MW.LENGTHS[c]
        bounds = [0, -1, -5, -(1 << 20), L - 1, L - 2] + [b * MW.BLOCK + d for b in range(1, L // MW.BLOCK + 1) for d in (-1, 0, 1)]
        keys = present[(present >> 16) == c] & 0xFFFF
        keys = list(rng.choice(keys, min(len(keys), 400), replace=False)) + list(rng.integers(0, 65536, 40))
        for k in keys:
            for bnd in bounds + [int(x) for x in rng.integers(0, L, 3)]:
                cs.append(c); ks.append(int(k)); fs.append(int(bnd))
        # every hit of a few buckets as a bound, and one past it
        for k in keys[:30]:
            lo, hi, _ = ix.lookup(c, int(k), 0)
            for p in ix.pos[lo:hi]:
                for d in (0, 1):
                    if p + d < L:
                        cs.append(c); ks.append(int(k)); fs.append(int(p) + d)
    return np.array(cs, np.uint32), np.array(ks, np.uint32), np.array(fs, np.int32)


def check_lookups(world, lib_path):
    ctx = index_context(world, lib_path, {})
    c, k, f = lookup_queries(world, np.random.default_rng(5))
    fn = ctx.lib.arb_selftest_kmer_lookup
    fn.argtypes = [lib.C.c_void_p, lib._p(lib.C.c_uint32), lib._p(lib.C.c_uint32), lib._p(lib.C.c_int32), lib.C.c_uint32, lib._p(lib.C.c_uint32)]
    out = np.zeros((len(c), 6), np.uint32)
    ctx._check(fn(ctx.h, lib.ptr(c), lib.ptr(k), lib.ptr(f), len(c), lib.ptr(out)))
    ix = world.stage.index
    want = np.zeros((len(c), 6), np.uint32)
    for j in range(len(c)):
        lo, hi, h = ix.lookup(int(c[j]), int(k[j]), int(f[j]))
        p = int(ix.pos[h]) if h < hi else 0xFFFFFFFF
        want[j] = (lo, hi, h, p, h, p)
    for col, what in ((slice(0, 2), "bucket bounds"), (slice(2, 4), "first_at_or_after"), (slice(4, 6), "env_first_hit")):
        bad = np.nonzero((out[:, col] != want[:, col]).any(1))[0]
        assert len(bad) == 0, "%s differs for %d of %d queries, first (contig, 8-mer, bound) %s: got %s want %s" % (
            what, len(bad), len(c), (c[bad[0]], k[bad[0]], f[bad[0]]), out[bad[0]], want[bad[0]])
    ctx.close()
    return len(c)


def test_kmer_lookup_hostsim(hostsim_lib):
    check_lookups(world_for(hostsim_lib, False), hostsim_lib)


@pytest.mark.gpu
def test_kmer_lookup_cuda(cuda_lib):
    check_lookups(world_for(cuda_lib, True), cuda_lib)


# ------------------------------------------------------------------------------------------------ gene homology
def identity_edge(stage, g1, g2):
    """The largest identity at which is_homolog still says yes (to 1e-12), by bisection. Only used to pick identities at the edge; the
    verdicts come from the literal is_homolog."""
    lo, hi = 0.0, 1.5
    for _ in range(40):
        mid = (lo + hi) / 2
        if R.is_homolog(stage, g1, g2, mid):
            lo = mid
        else:
            hi = mid
    return lo


def homolog_pairs_of(world):
    pairs = list(world.homolog_planted) + [(b, a) for a, b in world.homolog_planted]
    pairs += [(11, 12), (12, 11), (3, 3), (0, 1), (7, 8), (2, 36), (36, 2)]   # overlapping, the same gene, unrelated
    rng = np.random.default_rng(9)
    idx = [g for g, x in enumerate(world.genes) if x[0] < MW.N_INDEX]
    pairs += [(int(rng.choice(idx)), int(rng.choice(idx))) for _ in range(30)]
    return pairs


def identities(world):
    """0.3, and per planted pair the identities where length * identity falls on 8 * matches, one float step below and above it."""
    out = {np.float32(0.3)}
    for a, b in world.homolog_planted:
        ident = identity_edge(world.stage, a, b)
        (sc, ss, se, _), (bc, bs, be, _) = world.genes[a], world.genes[b]
        length = min(se - ss, be - bs)
        m = int(np.float32(length) * np.float32(ident) / 8 + 1e-6)
        for k in (m, m + 1):
            x = np.float32(8 * k / length)
            out.update((x, np.nextafter(x, np.float32(0)), np.nextafter(x, np.float32(2))))
    return sorted(float(x) for x in out if 0 < x < 1.5)


def check_homologs(world, lib_path, lanes):
    ctx = index_context(world, lib_path, {"ARB_HOMOLOG_LANES": lanes})
    pairs = homolog_pairs_of(world)
    a = np.array([p[0] for p in pairs], np.uint32); b = np.array([p[1] for p in pairs], np.uint32)
    idents = identities(world)
    flips = 0
    for ident in idents:
        p = ctx.default_params(); p.max_homolog_identity = ident; ctx.set_params(p)
        got = ctx.homolog_pairs(a, b)
        want = np.array([R.is_homolog(world.stage, int(x), int(y), np.float32(ident)) for x, y in pairs])
        bad = np.nonzero(got != want)[0]
        assert len(bad) == 0, "lanes %d, identity %r: pairs %s differ (got %s)" % (lanes, ident, [pairs[i] for i in bad[:5]], got[bad[:5]])
        flips += int(want.sum())
    assert 0 < flips < len(idents) * len(pairs)
    ctx.close()


@pytest.mark.parametrize("lanes", [1, 7, 32])
def test_homolog_pairs_hostsim(hostsim_lib, lanes):
    check_homologs(world_for(hostsim_lib, False), hostsim_lib, lanes)


@pytest.mark.gpu
@pytest.mark.parametrize("lanes", [1, 7, 32])
def test_homolog_pairs_cuda(cuda_lib, lanes):
    check_homologs(world_for(cuda_lib, True), cuda_lib, lanes)


# ------------------------------------------------------------------------------------------------ re-alignment
class Run:
    """One context: candidates from the device, lists and state set on them, the reference's expectations."""

    def __init__(self, world, lib_path, env, layout="canonical", stage_name="default", exotic=False, seed=0):
        self.world, self.stage_name, self.env = world, stage_name, env
        contigs = MW.with_exotic(world.contigs) if exotic else world.contigs
        ctx = new_context(lib_path, env, contigs)
        self.ctx = ctx
        ctx.set_annotation(MW.annotation(world.genes, len(world.contigs)))
        ctx.push_chunk(chunk_of(world, layout, np.random.default_rng(seed)))   # the layout depends on the configuration only
        p = ctx.default_params(); p.subsampling_threshold = 1 << 30; ctx.set_params(p)
        ctx.set_fragment_filters(np.zeros(len(world.order), np.uint8))
        ctx.find_fusions(MW.MAX_MATE_GAP)
        self.cands = ctx.candidates()
        self.swapped = ctx.slot_swaps()
        iv = world.intervals[stage_name]
        ctx.build_kmer_index([c for c, _, _ in iv], [s for _, s, _ in iv], [e for _, _, e in iv], MW.N_INDEX)
        ctx.set_splice_sites(*splice_columns(world.splice))
        self.frags = []
        for i, u in enumerate(world.order):   # the reference's copy of the fragments, in the device's canonical mate order
            f = world.frags[u]
            if self.swapped[i]:
                f = dict(f); f["alignments"] = [f["alignments"][1], f["alignments"][0]] + f["alignments"][2:]; f["sequences"] = f["sequences"][::-1]
            self.frags.append(f)
        self._plan()

    def _plan(self):
        w, c, rng = self.world, self.cands, np.random.default_rng(77)
        n = c["n"]
        same = c["contig1"] == c["contig2"]
        has_d = np.diff(c["listd_off"]) > 0
        free = [k for k in range(n) if not has_d[k]]
        rng.shuffle(free)
        assert len(free) > 4 * len(COUNT_TOTALS), "find_fusions gave too few candidates without discordant mates"
        self.count_cands = free[:2 * len(COUNT_TOTALS)]
        self.wrap_cand = free[2 * len(COUNT_TOTALS)]
        rest = free[2 * len(COUNT_TOTALS) + 1:]
        self.filtered = rest[:len(rest) // 10]
        self.filter = np.zeros(n, np.uint8); self.filter[self.filtered] = MW.F_OTHER_CANDIDATE_FILTER
        usable = [k for k in range(n) if k not in set(self.count_cands) | {self.wrap_cand} | set(self.filtered)]
        by_class = {s: [k for k in usable if bool(same[k]) == s] for s in (False, True)}
        assert by_class[False] and by_class[True], "find_fusions gave no candidate of one contig class"
        l1 = [[] for _ in range(n)]; l2 = [[] for _ in range(n)]
        uid = w.order
        for i, u in enumerate(uid):
            f = w.frags[u]
            if f["kind"] != 0 or w.family[u] in ("dead", "preset_mismappers"):
                continue
            s = w.same[u]
            targets = [int(rng.choice(by_class[s]))]
            if rng.random() < 0.2:
                targets.append(int(rng.choice(by_class[s])))
            if self.filtered and rng.random() < 0.1:
                targets.append(int(rng.choice(self.filtered)))
            if u not in self._twin_members() and rng.random() < 0.15:   # a plain shape also under the other contig class
                targets.append(int(rng.choice(by_class[not s])))
            for t in targets:
                (l1 if rng.random() < 0.6 else l2)[t].append(i)
        self.base_l1, self.base_l2 = l1, l2
        self.split_reads = [rng.choice([0, 1, int(rng.integers(2, 1 << 15))], n).astype(np.uint32) for _ in range(3)]
        self.presets = np.zeros(len(uid), np.uint8)
        for i, u in enumerate(uid):
            if w.family[u] == "preset_mismappers":
                self.presets[i] = MW.F_MISMAPPERS
            elif w.family[u] == "duplicates":
                self.presets[i] = MW.F_DUPLICATES
        self.copies_of = {}
        for i, u in enumerate(uid):
            self.copies_of.setdefault(int(u), []).append(i)

    def many_gene_items(self):
        """Work items (candidate, fragment) of the fragments whose clipped segment is searched against the 34 genes, under unfiltered candidates."""
        many = [i for i, u in enumerate(self.world.order) if self.world.family[u] == "many_genes"]
        return sum(ls.count(i) for k, ls in enumerate(self.base_l1 + self.base_l2) if self.filter[k % len(self.filter)] == 0 for i in many)

    def _twin_members(self):
        if not hasattr(self, "_tm"):
            self._tm = {x for pair in self.world.twins for x in pair}
        return self._tm

    def lists_for(self, fraction, wrap):
        """list1 / list2 of every candidate: the planned lists, count candidates with mismappers at floor(fraction * total) and one below,
        and with `wrap` the candidate whose 65,548 reads wrap the 16-bit counters."""
        w = self.world
        l1 = [list(x) for x in self.base_l1]; l2 = [list(x) for x in self.base_l2]
        pm = [i for u in w.preset_mismappers for i in self.copies_of[u]]
        dead = [i for u in w.dead for i in self.copies_of[u]]
        k = 0
        for total in COUNT_TOTALS:
            edge = int(np.floor(np.float32(fraction) * np.float32(total)))
            for m in (edge, edge - 1):
                m = min(max(m, 0), total)
                cand = self.count_cands[k]; k += 1
                l1[cand] = [pm[j % len(pm)] for j in range(m)] + [dead[j % len(dead)] for j in range(total - m)]
        if wrap:
            l1[self.wrap_cand] = [pm[j % len(pm)] for j in range(WRAP_MISMAPPERS)] + [dead[j % len(dead)] for j in range(WRAP_OTHERS)]
        return l1, l2

    def expect(self, fraction, l1, l2):
        c = self.cands
        cols = {"filter": self.filter, "split_reads1": self.split_reads[0], "split_reads2": self.split_reads[1], "discordant_mates": self.split_reads[2],
                "contig1": c["contig1"], "contig2": c["contig2"], "list1": l1, "list2": l2,
                "listd": [c["listd"][c["listd_off"][k]:c["listd_off"][k + 1]].tolist() for k in range(c["n"])]}
        uid = self.world.order
        verdict = lambda i, kind, same: self.world.verdict(self.stage_name, self.frags[i], int(uid[i]), bool(self.swapped[i]), kind, bool(same))
        return R.filter_mismappers(self.world.stage, self.frags, cols, self.presets, fraction, verdict)

    def run(self, fraction, wrap):
        ctx = self.ctx
        l1, l2 = self.lists_for(fraction, wrap)
        off = lambda ls: np.concatenate([[0], np.cumsum([len(x) for x in ls])]).astype(np.uint32)
        flat = lambda ls: np.array([i for x in ls for i in x], np.uint32)
        ctx.set_candidate_lists(off(l1), flat(l1), off(l2), flat(l2))
        n = self.cands["n"]
        ctx.set_candidate_state(self.filter, *self.split_reads, np.zeros(n, np.float32))
        p = ctx.default_params(); p.subsampling_threshold = 1 << 30; p.max_mismapper_fraction = fraction; ctx.set_params(p)
        ctx.set_fragment_filters(self.presets)
        with environment(self.env):   # the registry's first size is read when the stage runs
            ctx.filter_mismappers(MW.MAX_MATE_GAP)
        got_labels = ctx.fragment_filters()[0]
        got = ctx.candidates()
        want = self.expect(fraction, l1, l2)
        return got_labels, got, want, l1, l2


def compare_run(run, fraction, wrap, what):
    labels, got, want, l1, l2 = run.run(fraction, wrap)
    w = run.world
    bad = np.nonzero(labels != want[0])[0]
    if len(bad):
        detail = ["%d (%s, twin of a pair: %s) got %d want %d" % (i, w.family[w.order[i]], int(w.order[i]) in run._twin_members(), labels[i], want[0][i]) for i in bad[:6]]
        raise AssertionError("%s, fraction %g: %d fragment labels differ: %s" % (what, fraction, len(bad), "; ".join(detail)))
    for k, name in ((1, "filter"), (2, "split_reads1"), (3, "split_reads2"), (4, "discordant_mates")):
        g = got[name].astype(np.int64); x = np.asarray(want[k]).astype(np.int64)
        bad = np.nonzero(g != x)[0]
        assert len(bad) == 0, "%s, fraction %g: candidate %s differs at %s: got %s want %s" % (what, fraction, name, bad[:6], g[bad[:6]], x[bad[:6]])
    # each count candidate sits on its edge: mismappers at the floor discard it, one below keeps it
    edge = [want[1][cand] for cand in run.count_cands]
    floors = [int(np.floor(np.float32(fraction) * np.float32(t))) for t in COUNT_TOTALS]
    assert all(e == R.F_MISMAPPERS for e, fl in zip(edge[0::2], floors) if fl >= 1) and all(e == R.F_NONE for e in edge[1::2])
    if wrap:
        assert want[1][run.wrap_cand] == R.F_NONE, "with 16-bit counters 2 mismappers out of 12 keep the candidate"
    return want[0]


def twin_coverage(run, labels):
    w = run.world
    pairs = [(run.copies_of[a][0], run.copies_of[b][0]) for a, b in w.twins]
    listed = np.zeros(len(w.order), bool)
    for ls in (run.base_l1, run.base_l2):
        for k, x in enumerate(ls):
            if run.filter[k] == 0:
                listed[x] = True
    c = run.cands
    for k in range(c["n"]):
        if run.filter[k] == 0:
            listed[c["listd"][c["listd_off"][k]:c["listd_off"][k + 1]]] = True
    pairs = [(a, b) for a, b in pairs if listed[a] and listed[b]]
    differ = sum(1 for a, b in pairs if labels[a] != labels[b])
    return differ / max(len(pairs), 1), len(pairs)


CONFIGS = {   # name: (environment, layout, index, genome with an 'X', what Timings must show)
    "default": ({}, "canonical", "default", False, ("heavy", "tasks", "natural")),
    "budget1_lanes1": ({"ARB_MISMAP_BUDGET": 1, "ARB_MISMAP_LANES": 1, "ARB_MISMAP_TASK_LANES": 1}, "permuted", "default", False, ("heavy", "tasks")),
    "budget1_lanes7": ({"ARB_MISMAP_BUDGET": 1, "ARB_MISMAP_LANES": 7, "ARB_MISMAP_TASK_LANES": 3}, "canonical", "default", False, ("heavy", "tasks")),
    "budget1_lanes32": ({"ARB_MISMAP_BUDGET": 1, "ARB_MISMAP_LANES": 32, "ARB_MISMAP_TASK_LANES": 32}, "permuted", "default", False, ("heavy", "tasks")),
    "table1": ({"ARB_MISMAP_BUDGET": 1, "ARB_MISMAP_TABLE_TOTAL": 1}, "canonical", "default", False, ("heavy", "tasks", "overflow")),
    "table64": ({"ARB_MISMAP_BUDGET": 1, "ARB_MISMAP_TABLE_TOTAL": 64}, "permuted", "default", False, ("heavy", "tasks", "overflow")),
    "character_path": ({}, "permuted", "default", True, ("heavy", "tasks", "natural")),
    "small_padding": ({}, "canonical", "small_padding", False, ("heavy", "tasks")),
}


def check_config(world, lib_path, name, wrap):
    env, layout, index, exotic, paths = CONFIGS[name]
    run = Run(world, lib_path, env, layout, index, exotic, seed=zlib.crc32(name.encode()))
    labels = None
    for fraction in FRACTIONS:
        labels_f = compare_run(run, fraction, wrap and fraction == FRACTIONS[0], name)
        labels = labels if labels is not None else labels_f
        t = run.ctx.timings()
        if "heavy" in paths:
            assert t.mismapper_heavy_items > 0, "%s: no item reached pass 2" % name
        if "tasks" in paths:
            assert t.mismapper_tasks > 0 and t.mismapper_rounds > 0, "%s: no continuation ran as a task" % name
        if "overflow" in paths:
            assert t.mismapper_overflow > 0, "%s: the registry never overflowed" % name
        if "natural" in paths:   # under the default budget, more items reach pass 2 than the 34-gene alignment sends there straight away
            assert t.mismapper_heavy_items > run.many_gene_items(), "%s: only the 34-gene items reached pass 2 (%d)" % (name, t.mismapper_heavy_items)
    coverage, n_pairs = twin_coverage(run, labels)
    assert n_pairs > 0.8 * len(world.twins), "%s: only %d of %d twins are listed under an unfiltered candidate" % (name, n_pairs, len(world.twins))
    if index == "default":   # the twins were bisected on this index; with less padding some of them fall out of it
        assert coverage >= 0.9, "%s: the reference separates only %.3f of the twins" % (name, coverage)
    print("%s: %d twins, %.3f separated; heavy items %d, tasks %d, rounds %d, overflow %d" % (
        name, n_pairs, coverage, t.mismapper_heavy_items, t.mismapper_tasks, t.mismapper_rounds, t.mismapper_overflow))
    run.ctx.close()


_WORLDS = {}


def world_for(lib_path, gpu):
    key = "gpu" if gpu else "cpu"
    if key not in _WORLDS:
        _WORLDS[key] = World(seed=4242, n_attempts=450, copies=60 if gpu else 1)
    return _WORLDS[key]


@pytest.mark.parametrize("config", list(CONFIGS))
def test_filter_mismappers_hostsim(hostsim_lib, config):
    check_config(world_for(hostsim_lib, False), hostsim_lib, config, wrap=config == "default")


@pytest.mark.gpu
@pytest.mark.parametrize("config", list(CONFIGS))
def test_filter_mismappers_cuda(cuda_lib, config):
    check_config(world_for(cuda_lib, True), cuda_lib, config, wrap=config in ("default", "budget1_lanes7"))
