"""Gap filling of the fusion transcript (-I): every side of a row is filled on the device from the resident assembly and exons (csrc/fill_gaps_hd.h).

Per job, through the stage entry points: the filled sides must equal tests/fill_gaps_ref.py, a plain transcription of fill_gaps_in_fusion_transcript_sequence,
and for every transcript pair P5 + seq[b5 .. b3] + S3 must equal the transcription applied to the whole sequence. On the command line: both output files and
the WARNING lines must equal the reference's, with -I changing rows. `python tests/test_fill_gaps.py SEED N` runs N random worlds against the reference."""
import os
import random
import subprocess
import sys
import pytest
import fill_gaps_ref as fref
import genomic_ref
import worldutil
from arriba_b200 import lib as L, _build
from test_genomic_support import contig_names, oracle_run
from test_known_fusions import _world
from test_protein_domains import cli_parity, cli_run, rules_file, domains_file, NO_BL

SEQ_COL = 27

# ---- per job, through the C ABI


INTERESTING = [str(i) for i in range(1, 23)] + ["X", "Y"]


class UnsequencedWorld:
    """A world with one contig left out of the FASTA and of the interesting contigs (the reference requires the sequence of every interesting contig). Its
    genes stay in the GTF and its reads in the BAM, so rows and transcripts on it remain: the fill must leave their sides as they are."""

    def __init__(self, w, drop="3"):
        d = os.path.dirname(w.prefix) + "_without_" + drop
        os.makedirs(d, exist_ok=True)
        self.prefix = os.path.join(d, "w")
        for ext in (".bam", ".gtf"):
            if not os.path.exists(self.prefix + ext):
                os.symlink(w.prefix + ext, self.prefix + ext)
        if not os.path.exists(self.prefix + ".fa"):
            keep = True
            with open(w.prefix + ".fa") as src, open(self.prefix + ".fa.tmp", "w") as dst:
                for line in src:
                    if line.startswith(">"):
                        keep = genomic_ref._remove_chr(line[1:].split()[0]) != drop
                    if keep:
                        dst.write(line)
            os.replace(self.prefix + ".fa.tmp", self.prefix + ".fa")
        self.interesting = [c for c in INTERESTING if c != drop]
        self.args = ("-i", ",".join(self.interesting))
        ref = os.path.join(d, "oracle")  # the contig order of this run (the missing sequence moves the contig)
        if not os.path.exists(os.path.join(ref, "fusions.tsv")):
            worldutil.run_oracle(self.prefix, ref, args=NO_BL + self.args)
        self.names = contig_names(worldutil.World(self.prefix, ref))


def _tables(w, lib_path):
    """A pipeline over the world (the annotation and assembly resident on its context), its exons and the sequence of each device contig (None: none)."""
    p = L.Pipeline(w.prefix + ".bam", w.prefix + ".gtf", w.prefix + ".fa", threads=2, lib_path=lib_path, interesting_contigs=w.interesting)
    p.run(L.STEP_UPLOAD)
    genes = p.genes()
    names, seqs = worldutil.read_fasta(w.prefix + ".fa")
    by_name = {genomic_ref._remove_chr(n): s.decode() for n, s in zip(names, seqs)}
    contigs = [by_name.get(genomic_ref._remove_chr(n)) for n in w.names]
    return p, genes, contigs


def _transcripts(genes, contigs, rng, n=60):
    """Transcripts made of the exons of one gene (one to five, ascending), the exon chains; the genes of a contig without sequence among them."""
    by_gene = {}
    for x in range(len(genes["exon_start"])):
        by_gene.setdefault(int(genes["exon_gene"][x]), []).append(x)
    n_exons = len(genes["exon_start"])
    nxt, prv = [-1] * n_exons, [-1] * n_exons
    used, transcripts = set(), []
    unsequenced = sorted(g for g in by_gene if contigs[int(genes["gene_contig"][g])] is None)
    for g in rng.sample(sorted(by_gene), min(n, len(by_gene))) + unsequenced[:5]:
        ex = sorted((x for x in by_gene[g] if x not in used), key=lambda x: (int(genes["exon_start"][x]), x))
        # disjoint exons only: a chain walks them in order
        chain = []
        for x in ex:
            if not chain or int(genes["exon_start"][x]) > int(genes["exon_end"][chain[-1]]) + 1:
                chain.append(x)
        chain = chain[:rng.randint(1, 5)]
        if not chain:
            continue
        if rng.random() < 0.15:  # a chain against the genomic order: the walks' ends fall elsewhere (the plain "filled" / "snapped" cases without "^" / "$")
            chain.reverse()
        used.update(chain)
        for a, b in zip(chain, chain[1:]):
            nxt[a] = b; prv[b] = a
        transcripts.append({"first": chain[0], "last": chain[-1], "contig": int(genes["gene_contig"][g])})
    exons = [{"start": int(genes["exon_start"][x]), "end": int(genes["exon_end"][x]), "next": nxt[x] if nxt[x] >= 0 else None, "prev": prv[x] if prv[x] >= 0 else None}
             for x in range(n_exons)]
    return transcripts, exons, nxt, prv


def _side(tr, exons, contig, rng, five, fwd):
    """Characters and positions of one side, built around the transcript: runs of bases inside, before or after its exons, "..." and "___" gaps,
    lower-case bases without positions next to the junction, and the imprecise "...|" / "|..." forms."""
    chain = [tr["first"]]
    while exons[chain[-1]]["next"] is not None:
        chain.append(exons[chain[-1]]["next"])
    lo, hi = exons[chain[0]]["start"], exons[chain[-1]]["end"]
    s, p = [], []

    def run(a, b):  # genomic positions a..b in transcription order
        step = 1 if a <= b else -1
        for q in range(a, b + step, step):
            if 0 <= q < len(contig):
                s.append(contig[q] if fwd else fref.comp(contig[q])); p.append(q)

    def marks(t):
        s.extend(t); p.extend([-1] * len(t))

    kind = rng.random()
    e = exons[rng.choice(chain[:-1] if len(chain) > 1 and rng.random() < 0.7 else chain)]
    inner = rng.randint(e["start"], e["end"])
    introns = [(exons[x]["end"] + 1, exons[exons[x]["next"]]["start"] - 1) for x in chain[:-1] if exons[exons[x]["next"]]["start"] - exons[x]["end"] > 2]
    if kind < 0.1 and introns:  # only intronic bases: no exon overlaps the side
        a, b = rng.choice(introns)
        run(a, b) if fwd else run(b, a)
        return s, p
    if kind < 0.35:  # imprecise breakpoint: one base, then "..."
        if five:
            run(inner, inner); marks("...")
        else:
            marks("..."); run(inner, inner)
        return s, p
    # a run that reaches or passes the end of the transcript, or stops inside it, with a gap in between or not
    outer = rng.choice([lo - rng.randint(0, 30), lo, lo + rng.randint(1, 5), hi, hi + rng.randint(0, 30), hi - rng.randint(1, 5)])
    near = rng.choice([inner, inner, e["start"], e["end"], lo - 3])
    a, b = (outer, near) if five == fwd else (near, outer)
    if not fwd:
        a, b = b, a
    a, b = (min(a, b), max(a, b)) if fwd else (max(a, b), min(a, b))
    mid = (a + b) // 2
    if rng.random() < 0.4:
        run(a, mid); marks(rng.choice(["...", "___", "...___"])); run(mid + (1 if fwd else -1), b)
    else:
        run(a, b)
    if rng.random() < 0.2:  # non-template bases at the junction
        marks(rng.choice(["acg", "t"]) if five else rng.choice(["gga", "c"]))
    if not s:
        run(inner, inner)
    return s, p


def _rows(transcripts, exons, contigs, rng, n_rows=2000):
    rows, jobs, want = [], [], []
    for r in range(n_rows):
        k5 = rng.randrange(len(transcripts)); k3 = rng.randrange(len(transcripts))
        t5, t3 = transcripts[k5], transcripts[k3]
        f5, f3 = rng.random() < 0.5, rng.random() < 0.5
        c5 = contigs[t5["contig"]] or contigs[[t for t in transcripts if contigs[t["contig"]]][0]["contig"]]
        c3 = contigs[t3["contig"]] or c5
        s5, p5 = _side(t5, exons, c5, rng, True, f5)
        s3, p3 = _side(t3, exons, c3, rng, False, f3)
        mid = rng.choice(["|", "|", "|", "|tt|", "|a|"])
        seq = "".join(s5) + mid + "".join(s3)
        pos = p5 + [-1] * len(mid) + p3
        if rng.random() < 0.1:
            pos = pos + [rng.randint(0, 1000)] * rng.randint(1, 3)  # positions beyond the text (insertions that went to the clipped bases)
        itd = rng.random() < 0.15
        if rng.random() < 0.15:  # the strand against the order of the positions
            f5, f3 = (not f5, f3) if rng.random() < 0.5 else (f5, not f3)
        rows.append((seq, pos, k5, k3, f5, f3, itd))
    return rows


def _crafted(transcripts, exons, contigs):
    """Rows whose positions run against the strand, on transcripts with an intron after their first exon: the 5' side's first base in an exon is the
    transcript's first base (an empty walk: "()" without "^"), the 3' side's is its last base (an empty walk without "$")."""
    rows = []
    for k, t in enumerate(transcripts):
        a = exons[t["first"]]
        if contigs[t["contig"]] is None or a["next"] is None or exons[a["next"]]["start"] <= a["end"] + 1:
            continue
        m, z = a["end"] + 1, exons[t["last"]]  # m: intronic, inside the transcript
        seq = "a...CG" + "|" + "TC...A"
        pos = [-1, -1, -1, -1, m, a["start"], -1, z["end"], m, -1, -1, -1, -1]
        rows.append((seq, pos, k, k, True, True, False))
        if len(rows) == 3:
            break
    assert rows
    return rows


def per_job(w, lib_path, seed=7):
    rng = random.Random(seed)
    p, genes, contigs = _tables(w, lib_path)
    ctx = p.context()
    transcripts, exons, nxt, prv = _transcripts(genes, contigs, rng)
    assembly = {c: contigs[c] for c in range(len(contigs)) if contigs[c] is not None}
    ctx.set_fill_transcripts([t["first"] for t in transcripts], [t["last"] for t in transcripts], [t["contig"] for t in transcripts], nxt, prv)
    rows = _rows(transcripts, exons, contigs, rng) + _crafted(transcripts, exons, contigs)
    jobs = []
    for r, (seq, pos, k5, k3, f5, f3, itd) in enumerate(rows):
        flags = ctx.FILL_ITD if itd else 0
        jobs.append((r, k5, flags | (ctx.FILL_FORWARD if f5 else 0)))
        jobs.append((r, k3, flags | ctx.FILL_THREE | (ctx.FILL_FORWARD if f3 else 0)))
    out = ctx.fill_gaps([s.encode() for s, *_ in rows], [pos for _, pos, *_ in rows], jobs)
    branches = set()
    for r, (seq, pos, k5, k3, f5, f3, itd) in enumerate(rows):
        (c5, q5), (c3, q3) = out[2 * r], out[2 * r + 1]
        b5, b3 = seq.find("|"), seq.rfind("|")
        log5, log3 = [], []
        w5, wp5 = fref.fill(seq, pos, k5, None, f5, f3, itd, transcripts, exons, assembly, log5)
        w3, wp3 = fref.fill(seq, pos, None, k3, f5, f3, itd, transcripts, exons, assembly, log3)
        branches.update(log5 + log3)
        # P5 replaces seq[0, b5), S3 replaces seq(b3, end)
        assert c5.decode() + seq[b5:] == w5, (r, log5, seq, c5)
        assert q5 + pos[b5:len(seq)] == wp5[:len(w5)], (r, log5)
        assert seq[:b3 + 1] + c3.decode() == w3, (r, log3, seq, c3)
        assert pos[:b3 + 1] + q3 == wp3[:len(w3)], (r, log3)
        # every pair: the halves put together equal the whole fill
        for t5 in (None, k5):
            for t3 in (None, k3):
                whole, whole_pos = fref.fill(seq, pos, t5, t3, f5, f3, itd, transcripts, exons, assembly)
                p5, pp5 = (c5.decode(), q5) if t5 is not None else (seq[:b5], pos[:b5])
                s3, ps3 = (c3.decode(), q3) if t3 is not None else (seq[b3 + 1:], pos[b3 + 1:len(seq)])
                assert p5 + seq[b5:b3 + 1] + s3 == whole, (r, t5, t3)
                assert pp5 + pos[b5:b3 + 1] + ps3 == whole_pos[:len(whole)], (r, t5, t3)
    p.close()
    return branches


# the branches of both sides; "^" / "$": the filled or trimmed side reaches the transcript's start / end. A snapped imprecise 5' side always gets its "^":
# its walk starts at the transcript's first base, and an empty walk means the fake base is that base (output_fusions.cpp:886-927).
WANT = {"5:imprecise-snapped^", "5:imprecise-not-snapped", "5:filled", "5:filled^", "5:trim", "5:trim^", "5:no-overlap", "5:no-sequence",
        "3:imprecise-snapped", "3:imprecise-snapped$", "3:imprecise-not-snapped", "3:filled", "3:filled$", "3:trim", "3:trim$", "3:no-overlap", "3:no-sequence"}


def test_per_job(worlds, hostsim_lib):
    branches = per_job(UnsequencedWorld(worlds.get("small")), hostsim_lib)
    assert WANT <= branches, WANT - branches


def test_per_job_rejects_undefined_input(worlds, hostsim_lib):
    """Fewer positions than characters: the reference would read beyond the positions. A cyclic exon chain would never end."""
    p, genes, contigs = _tables(UnsequencedWorld(worlds.get("small")), hostsim_lib)
    ctx = p.context()
    transcripts, exons, nxt, prv = _transcripts(genes, contigs, random.Random(1), n=5)
    ctx.set_fill_transcripts([t["first"] for t in transcripts], [t["last"] for t in transcripts], [t["contig"] for t in transcripts], nxt, prv)
    with pytest.raises(L.ArbError, match="fewer positions than characters"):
        ctx.fill_gaps([b"ACG|TTT"], [[1, 2, 3, -1, 5, 6]], [(0, 0, ctx.FILL_THREE)])
    a, b = transcripts[0]["first"], next(t["first"] for t in transcripts[1:] if t["first"] != transcripts[0]["first"])
    cyc = list(nxt); cyc[a], cyc[b] = b, a
    with pytest.raises(L.ArbError, match="has a cycle"):
        ctx.set_fill_transcripts([t["first"] for t in transcripts], [t["last"] for t in transcripts], [t["contig"] for t in transcripts], cyc, prv)
    p.close()


# ---- the command line against the reference (CPU stand-in)


@pytest.fixture(scope="module")
def cli():
    return _build.build_cli_hostsim()


@pytest.fixture(scope="module")
def fg_root(tmp_path_factory):
    return str(tmp_path_factory.mktemp("fg"))


def changed_rows(fus, ref_dir):
    """Rows whose fusion_transcript -I changed: the reference's output without -I beside ours with it."""
    plain = open(os.path.join(ref_dir, "fusions.tsv"), "rb").read().splitlines()[1:]
    filled = fus.splitlines()[1:]
    assert len(plain) == len(filled)
    return sum(1 for a, b in zip(plain, filled) if a.split(b"\t")[SEQ_COL] != b.split(b"\t")[SEQ_COL])


def parity(cli, w, args, tmp, env=None):
    _, fus, disc = cli_parity(cli, w, NO_BL + tuple(args), tmp, env)
    plain = oracle_run(w, NO_BL + tuple(x for x in args if x != "-I"), os.path.join(tmp, "plain"))
    assert changed_rows(fus, plain.outdir) > 0, "-I changed no row"
    if "-X" in args:
        plain_disc = open(os.path.join(plain.outdir, "fusions.discarded.tsv"), "rb").read().splitlines()[1:]
        assert sum(1 for a, b in zip(plain_disc, disc.splitlines()[1:]) if a.split(b"\t")[SEQ_COL] != b.split(b"\t")[SEQ_COL]) > 0
    return fus, disc


@pytest.mark.parametrize("name,extra", [("small", ()), ("small", ("-X",)), ("l151", ("-X",)), ("zchr", ("-X",)), ("cfg5", ("-X",))],
                         ids=lambda x: x if isinstance(x, str) else " ".join(x))
def test_cli_parity(worlds, cli, tmp_path, name, extra):
    parity(cli, _world(worlds, name), ("-I",) + tuple(extra), str(tmp_path))


def unsequenced_parity(cli, worlds, tmp):
    """Discarded rows on the contig without sequence carry transcripts: their sides on it stay as they are."""
    w = UnsequencedWorld(worlds.get("small"))
    _, disc = parity(cli, w, ("-I", "-X") + w.args, tmp)
    rows = [l.split(b"\t") for l in disc.splitlines()[1:]]
    assert any((r[4].startswith(b"3:") and r[22] != b".") or (r[5].startswith(b"3:") and r[23] != b".") for r in rows)


def test_cli_parity_contig_without_sequence(worlds, cli, tmp_path):
    unsequenced_parity(cli, worlds, str(tmp_path))


def test_cli_parity_with_other_files(worlds, cli, hostsim_lib, fg_root, tmp_path):
    w = worlds.get("small")
    k, t = rules_file(w, hostsim_lib, fg_root, False), rules_file(w, hostsim_lib, fg_root, True)
    pd = domains_file(w, hostsim_lib, fg_root)
    parity(cli, w, ("-I", "-X", "-k", k, "-t", t, "-p", pd), str(tmp_path))


def test_cli_parity_scattered_and_poisoned(worlds, cli, tmp_path):
    parity(cli, worlds.get("small"), ("-I", "-X"), str(tmp_path), env={"ARB_HOSTSIM_ORDER": "2", "ARB_HOSTSIM_POISON": "1"})


def test_g_still_refused(worlds, cli, tmp_path):
    w = worlds.get("small")
    r = subprocess.run([cli, "-x", w.prefix + ".bam", "-g", w.prefix + ".gtf", "-a", w.prefix + ".fa", "-o", str(tmp_path / "f.tsv"), "-G", "x"], capture_output=True, text=True)
    assert r.returncode != 0 and "option -G is not supported by arriba-b200" in r.stderr


def test_no_option_no_fill_stage(worlds, cli, tmp_path):
    """Without -I the writer has no fill stage."""
    w = worlds.get("small")
    r, _, _ = cli_run(cli, w, NO_BL + ("-X",), str(tmp_path), env={"ARB_TRACE": "1"})
    assert "gap filling" not in r.stderr
    r, _, _ = cli_run(cli, w, NO_BL + ("-X", "-I"), str(tmp_path), env={"ARB_TRACE": "1"})
    assert "gap filling" in r.stderr


# ---- two ranks
WORKER = r"""
import os, sys
sys.path[:0] = [{root!r}, os.path.join({root!r}, "tests")]
import torch.distributed as dist
from arriba_b200 import lib as L, sharded
rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"])
dist.init_process_group("gloo")
out = os.path.join({outdir!r}, "rank%d" % rank); os.makedirs(out, exist_ok=True)
p = L.Pipeline({prefix!r} + ".bam", {prefix!r} + ".gtf", {prefix!r} + ".fa", threads=2, lib_path={lib!r}, fill_sequence_gaps=True, extra_info=True,
               output=os.path.join(out, "fusions.tsv"), discarded=os.path.join(out, "fusions.discarded.tsv"))
sharded.run_sharded(p, rank, world)
p.close()
dist.destroy_process_group()
"""


def test_sharded_two_ranks(worlds, hostsim_lib, tmp_path):
    w = worlds.get("small")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = str(tmp_path / "worker.py")
    open(script, "w").write(WORKER.format(root=root, outdir=str(tmp_path), prefix=w.prefix, lib=hostsim_lib))
    env = dict(os.environ, PYTHONPATH=root + os.pathsep + os.path.join(root, "tests"))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port", str(29700 + os.getpid() % 200), script]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    single = str(tmp_path / "single"); os.makedirs(single)
    p = L.Pipeline(w.prefix + ".bam", w.prefix + ".gtf", w.prefix + ".fa", threads=2, lib_path=hostsim_lib, fill_sequence_gaps=True, extra_info=True,
                   output=os.path.join(single, "fusions.tsv"), discarded=os.path.join(single, "fusions.discarded.tsv"))
    p.run_all(); p.close()
    for f in ("fusions.tsv", "fusions.discarded.tsv"):
        assert open(os.path.join(tmp_path, "rank0", f), "rb").read() == open(os.path.join(single, f), "rb").read(), f
    assert b"(" in open(os.path.join(single, "fusions.discarded.tsv"), "rb").read()


# ---- on the H100
@pytest.mark.gpu
def test_per_job_cuda(worlds, cuda_lib):
    branches = per_job(UnsequencedWorld(worlds.get("small")), cuda_lib)
    assert WANT <= branches, WANT - branches


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small", "cfg5"])
def test_parity_cuda(worlds, cuda_lib, tmp_path, name):
    w = _world(worlds, name)
    cli = _build.build_cli()
    parity(cli, w, ("-I",), str(tmp_path / "i"))
    parity(cli, w, ("-I", "-X"), str(tmp_path / "ix"))
    if name == "small":
        unsequenced_parity(cli, worlds, str(tmp_path / "unsequenced"))


# ---- random worlds against the reference: python tests/test_fill_gaps.py SEED N
if __name__ == "__main__":
    import tempfile
    seed, n = int(sys.argv[1]), int(sys.argv[2])
    cli_bin = _build.build_cli_hostsim()
    rng = random.Random(seed)
    root = tempfile.mkdtemp(prefix="fill_gaps_")
    cache = worldutil.WorldCache(os.path.join(root, "worlds"))
    for i in range(n):
        params = dict(scale=0.001, genes=rng.randint(100, 500), breakpoints=rng.randint(50, 250), fragments=rng.randint(5000, 25000), read_length=rng.choice([75, 101, 151]),
                      seed=rng.randint(1, 1 << 30))
        w = cache.get("r%d" % i, **params)
        tmp = os.path.join(root, "run%d" % i)
        parity(cli_bin, w, ("-I", "-X"), tmp)
        print("world %d %s: identical" % (i, params), flush=True)
