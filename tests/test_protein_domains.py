"""Protein domains (-p): the GFF3 file is read like the reference reads it, the device keeps the reference's index as a table per gene (csrc/domains_hd.h) and
fills the retained_protein_domains column of every written row. Both output files, the WARNING lines and the progress lines must equal the reference's; the
column of every candidate must equal tests/protein_domains_ref.py, a plain transcription of the reference that walks the index key by key."""
import os
import random
import subprocess
import sys
import numpy as np
import pytest
import blacklisttools
import protein_domains_ref as pref
from arriba_b200 import lib as L, _build, sharded
from test_genomic_support import contig_names, contig_ids, oracle_run, sv_file
from test_known_fusions import _world, write, rules_file

NO_BL = ("-f", "blacklist")
CB_PSTRAND1, CB_PSTRAND2, CB_PSTRANDS_AMBIGUOUS, CB_TSTART_GENE1 = 16, 32, 64, 128
GF_DUMMY, GF_CODING = 1, 2

# decoded: spaces, ',' and '|' become '_'; "%2C" / "%7C" / "%09" decode and then become '_'; "%25" decodes to '%'; "%2541" to "%41" (no second decode);
# "%G1", a trailing '%' and "%2" stay; bytes >= 0x80 become '_'
NAMES = ["Kinase", "Pkinase_Tyr", "SH2", "SH3_1", "PH", "with space", "a,b", "a|b", "x%2Cy", "x%7Cy", "p%25q", "%2541", "tab%09x", "%G1", "trail%", "trail%2",
         "caf\xe9", "Zinc finger", "zf-C2H2", "PDZ", "PDZ", "Kinase"]


def gene_ids(gtf_path, genes, cids):
    """gene_id (with its version) of every gene of the run, "" for dummy genes: the GTF's genes lined up with the run's like blacklisttools.gene_names does."""
    order, ext = [], {}
    for line in open(gtf_path):
        if line.startswith("#"):
            continue
        f = line.rstrip("\n").split("\t")
        if len(f) < 9 or f[2] != "exon":
            continue
        attrs = {}
        for a in f[8].split(";"):
            a = a.strip()
            if " " in a:
                k, v = a.split(" ", 1); attrs.setdefault(k, v.strip('"'))
        if "gene_id" not in attrs:
            continue
        c = cids.get(f[0][3:] if f[0].startswith("chr") else f[0])
        key = (attrs["gene_id"].split(".")[0], c, f[6] == "+")
        if key not in ext:
            order.append(key); ext[key] = [attrs["gene_id"], int(f[3]) - 1, int(f[4]) - 1]
        else:
            ext[key][1] = min(ext[key][1], int(f[3]) - 1); ext[key][2] = max(ext[key][2], int(f[4]) - 1)
    ids = [""] * len(genes["gene_start"]); g = 0
    real = [x for x in range(len(ids)) if not genes["gene_flags"][x] & GF_DUMMY]
    for key in order:
        if g < len(real) and (key[1], ext[key][1], ext[key][2]) == (int(genes["gene_contig"][real[g]]), int(genes["gene_start"][real[g]]), int(genes["gene_end"][real[g]])):
            ids[real[g]] = ext[key][0]; g += 1
    assert g == len(real), "GTF genes do not line up with the run's"
    return ids


def final_state(w, lib_path):
    """The candidates after every stage, the genes (dummy genes included), their names and IDs."""
    p = L.Pipeline(w.prefix + ".bam", w.prefix + ".gtf", w.prefix + ".fa", threads=2, lib_path=lib_path)
    p.run(); p.events(len(L.EV_NAMES) - 1)
    cand = p.candidates(); genes = p.genes(); p.close()
    cids = contig_ids(w)
    return cand, genes, blacklisttools.gene_names(w.prefix + ".gtf", genes, cids), gene_ids(w.prefix + ".gtf", genes, cids)


def _cname(nm, c, rng):
    bare = nm[c][3:] if nm[c].startswith("chr") else nm[c]
    return rng.choice([bare, "chr" + bare])


def gff3_lines(cand, genes, names, ids, nm, rng, n_genes=150):
    """Domains in the world's coding genes that carry candidates: inside the gene, overlapping, straddling its start or end, outside it, one base long,
    reversed, on another contig; found by ID, by ID with another version, by name; names repeated within and across genes; and the lines the loader skips."""
    gs, ge, gc, gf = genes["gene_start"], genes["gene_end"], genes["gene_contig"], genes["gene_flags"]
    in_cands = set(int(g) for g in cand["gene1"]) | set(int(g) for g in cand["gene2"])
    coding = sorted(g for g in in_cands if gf[g] & GF_CODING and not gf[g] & GF_DUMMY and names[g] is not None)
    pick = rng.sample(coding, min(len(coding), n_genes))
    out = ["##gff-version 3", "# protein domains written from the world's coding genes", ""]

    def line(c_text, a, b, attrs, strand="+"):  # a, b 0-based
        return "\t".join([c_text, "pfam", "protein_domain", str(a + 1), str(b + 1), ".", strand, ".", attrs])

    def attrs(g, name, how):
        gid = ids[g]
        if how == "version":
            gid = pref.strip_ensembl_version_number(gid) + ".77"
        elif how == "name":
            gid = "LOST%d" % g
        parts = ["gene_name=" + names[g], "gene_id=" + gid, "Name=" + name]
        rng.shuffle(parts)
        return ";".join(parts + ["ID=d%d" % rng.randint(0, 10 ** 6)])

    for g in pick:
        s, e, c = int(gs[g]), int(ge[g]), int(gc[g]); n = e - s + 1
        pool = rng.sample(NAMES, 3)
        for _ in range(rng.randint(1, 7)):
            kind = rng.choice(["in", "in", "in", "in", "start", "end", "outside", "point", "reversed"])
            a = s + rng.randint(0, max(0, n - 1)); b = min(e, a + rng.randint(0, max(1, n // 3)))
            if kind == "start":
                a, b = s - rng.randint(1, 200), s + rng.randint(0, max(0, n // 2))
            elif kind == "end":
                a, b = e - rng.randint(0, max(0, n // 2)), e + rng.randint(1, 200)
            elif kind == "outside":
                a = e + rng.randint(1, 500); b = a + rng.randint(0, 300)
            elif kind == "point":
                b = a
            elif kind == "reversed":
                a, b = b + 5, a
            out.append(line(_cname(nm, c, rng), max(a, 0), max(b, 0), attrs(g, rng.choice(pool), rng.choice(["id", "id", "id", "version", "name"])), rng.choice("+-")))
        if rng.random() < 0.1:  # a domain of this gene on another contig
            other = (c + 1) % len(nm)
            out.append(line(_cname(nm, other, rng), s, e, attrs(g, rng.choice(pool), "id")))
    g0, g1 = pick[0], pick[1]
    s0, e0, c0 = int(gs[g0]), int(ge[g0]), int(gc[g0])
    out += [
        line(nm[c0], s0, e0, "gene_name=NOPE;gene_id=NOPE1;Name=X"), line(nm[c0], s0, e0, "gene_name=NOPE;gene_id=NOPE1;Name=Y"),  # unknown gene, warned once
        line(nm[c0], s0, e0, "gene_name=%s;gene_id=ABC.1;Name=dotted" % names[g0]),  # not ENS: the version stays, found by name
        line(nm[c0], s0, e0, "gene_name=NOPE2;gene_id=;Name=empty_id"),  # the last dummy gene, if there is one
        line("chrUn_nowhere", s0, e0, attrs(g0, "X", "id")),  # unknown contig
        line(nm[c0], s0, e0, "gene_id=%s;Name=Z" % ids[g0]), line(nm[c0], s0, e0, "gene_name=%s;Name=Z" % names[g0]), line(nm[c0], s0, e0, "gene_name=%s;gene_id=%s" % (names[g0], ids[g0])),
        line(nm[c0], s0, e0, "gene_name=%s;gene_id=%s;Note=seeName=inside_note" % (names[g1], ids[g1])),  # Name= found inside another attribute's value
        "\t".join([nm[c0], "pfam", "protein_domain", str(s0 + 1), str(e0 + 1), ".", "+"]),  # too few columns
        "\t".join([nm[c0], "pfam", "protein_domain", "1x", str(e0 + 1), ".", "+", ".", attrs(g0, "X", "id")]),  # not an integer
        "\t".join([nm[c0], "pfam", "protein_domain", str(s0 + 1), str(e0 + 1), ".", "", ".", attrs(g0, "X", "id")]),  # empty strand
        "# a comment", "",
    ]
    head, body = out[:3], out[3:]
    rng.shuffle(body)
    return head + body


_FILES = {}


def domains_file(w, lib_path, root, variant="plain", seed=5):
    key = (w.prefix, variant, seed)
    if key not in _FILES:
        cand, genes, names, ids = final_state(w, lib_path)
        lines = gff3_lines(cand, genes, names, ids, contig_names(w), random.Random(seed))
        path = os.path.join(root, "domains_%d_%s%s" % (len(_FILES), variant, ".gff3.gz" if variant == "gz" else ".gff3"))
        write(path, lines, crlf=variant == "crlf")
        _FILES[key] = path
    return _FILES[key]


@pytest.fixture(scope="module")
def cli():
    return _build.build_cli_hostsim()


@pytest.fixture(scope="module")
def pd_root(tmp_path_factory):
    return str(tmp_path_factory.mktemp("pd"))


def warnings_of(text):
    return [l for l in text.splitlines() if l.startswith("WARNING: failed to") or l.startswith("WARNING: unknown contig") or l.startswith("WARNING: unknown gene")
            or l.startswith("WARNING: encountered")]


def progress_of(text):
    """The loading and writing progress lines, in order, without the output paths (the protein domains are loaded after the tags, before any file is written)."""
    lines = [l.split("] ", 1)[1].strip() for l in text.splitlines() if "Loading" in l or "Writing" in l]
    return [l if l.startswith("Loading protein domains") else l.split(" '")[0] for l in lines]


def cli_run(cli, w, args, tmp, env=None, discarded=True):
    out = os.path.join(tmp, "fusions.tsv"); disc = os.path.join(tmp, "fusions.discarded.tsv")
    cmd = [cli, "-x", w.prefix + ".bam", "-g", w.prefix + ".gtf", "-a", w.prefix + ".fa", "-o", out, "-@", "3"] + (["-O", disc] if discarded else []) + list(args)
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=dict(os.environ, **(env or {})), encoding="latin-1")
    assert r.returncode == 0, r.stderr[-2000:]
    return r, open(out, "rb").read(), open(disc, "rb").read() if discarded else None


def cli_parity(cli, w, args, tmp, env=None, discarded=True):
    ref = oracle_run(w, args, os.path.join(tmp, "oracle"))
    r, fus, disc = cli_run(cli, w, args, tmp, env, discarded)
    assert fus == open(os.path.join(ref.outdir, "fusions.tsv"), "rb").read(), "fusions.tsv differs with %s" % (args,)
    if discarded:
        assert disc == open(os.path.join(ref.outdir, "fusions.discarded.tsv"), "rb").read(), "fusions.discarded.tsv differs with %s" % (args,)
    assert warnings_of(r.stderr) == warnings_of(open(os.path.join(ref.outdir, "stderr.txt"), encoding="latin-1").read())
    want = progress_of(open(os.path.join(ref.outdir, "stdout.txt")).read())
    assert progress_of(r.stdout) == (want if discarded else [l for l in want if not l.startswith("Writing discarded")])  # the oracle always writes both files
    return ref, fus, disc


def domain_cells(blob):
    return [l.split(b"\t")[17] for l in blob.splitlines()[1:] if l.split(b"\t")[17] != b"."]


def assert_meaningful(fus, disc):
    """Kept and discarded rows carry the column, some rows have both sides, some several names, some percentages below 100."""
    cells = domain_cells(fus) + domain_cells(disc)
    assert domain_cells(fus) and domain_cells(disc), (len(domain_cells(fus)), len(domain_cells(disc)))
    assert any(not c.startswith(b"|") and not c.endswith(b"|") for c in cells), "no row with domains on both sides"
    assert any(b"," in c for c in cells), "no row with several names"
    assert any(b"(100%)" not in p for c in cells for p in c.replace(b"|", b",").split(b",") if p), "no percentage below 100"


CASES = [("small", "plain", ()), ("small", "gz", ()), ("small", "crlf", ()), ("small", "plain", ("-X",)), ("l151", "plain", ()), ("zchr", "plain", ()), ("cfg5", "plain", ())]


@pytest.mark.parametrize("name,variant,extra", CASES, ids=lambda x: x if isinstance(x, str) else " ".join(x) if isinstance(x, tuple) else None)
def test_cli_parity(worlds, cli, hostsim_lib, pd_root, tmp_path, name, variant, extra):
    w = _world(worlds, name)
    ref, fus, disc = cli_parity(cli, w, tuple(extra) + NO_BL + ("-p", domains_file(w, hostsim_lib, pd_root, variant)), str(tmp_path))
    if name in ("small", "cfg5"):
        assert_meaningful(fus, disc)


def test_cli_parity_with_other_files_and_no_discarded_file(worlds, cli, hostsim_lib, pd_root, tmp_path):
    w = worlds.get("small")
    p = domains_file(w, hostsim_lib, pd_root)
    from test_known_fusions import stage_state
    cand, genes, names, mmg, _ = stage_state(w, hostsim_lib)
    bl = os.path.join(pd_root, "bl.tsv")
    blacklisttools.write(bl, blacklisttools.rule_lines(cand, genes, names, contig_names(w), random.Random(3), mmg, n_candidates=40))
    k, t = rules_file(w, hostsim_lib, pd_root, False), rules_file(w, hostsim_lib, pd_root, True)
    cli_parity(cli, w, ("-b", bl, "-k", k, "-t", t, "-p", p), str(tmp_path / "bkt"))
    cli_parity(cli, w, NO_BL + ("-d", sv_file(w, hostsim_lib, pd_root), "-p", p), str(tmp_path / "d"))
    cli_parity(cli, w, NO_BL + ("-p", p), str(tmp_path / "noO"), discarded=False)


def test_cli_parity_scattered_and_poisoned(worlds, cli, hostsim_lib, pd_root, tmp_path):
    w = worlds.get("small")
    cli_parity(cli, w, NO_BL + ("-X", "-p", domains_file(w, hostsim_lib, pd_root)), str(tmp_path), env={"ARB_HOSTSIM_ORDER": "2", "ARB_HOSTSIM_POISON": "1"})


# ---- per candidate, through the C ABI
def _bits_offset(n):
    """Offset of the bits column in the blob of arb_candidates_export (csrc/exchange.cu, candidate_sections): 64 bytes of sizes, then 16-byte aligned columns."""
    at = 64
    for elem in (4, 4, 2, 2, 4, 4, 1, 1, 4, 4, 4, 1):  # gene1 .. filter
        at += (elem * n + 15) & ~15
    return at


def _flip_bits(ctx, mask, cuda):
    blob, nbytes, sizes = ctx.candidates_export()
    n = sizes[0]
    v = sharded.view(blob, nbytes, cuda)
    at = _bits_offset(n)
    v[at:at + n] ^= mask
    ctx.candidates_import(blob, nbytes, sizes, 1)


def per_candidate(w, lib_path, path, records_hint=None):
    """retained_protein_domains(ids) for every candidate against the transcription, on the real states and with the strand, ambiguity and transcript-start
    bits flipped."""
    cuda = lib_path != _build.HOSTSIM_LIB
    p = L.Pipeline(w.prefix + ".bam", w.prefix + ".gtf", w.prefix + ".fa", threads=2, lib_path=lib_path)
    p.run(); p.events(len(L.EV_NAMES) - 1)
    genes = p.genes(); cids = contig_ids(w)
    names, ids = blacklisttools.gene_names(w.prefix + ".gtf", genes, cids), gene_ids(w.prefix + ".gtf", genes, cids)
    records, _ = pref.load_protein_domains(path, cids, ids, blacklisttools.gene_by_name(names))
    index = pref.make_annotation_index(records)
    ctx = p.context()
    ctx.set_protein_domains([r["contig"] for r in records], [r["start"] for r in records], [r["end"] for r in records], [r["gene"] for r in records],
                            [r["name"] for r in records])
    nonempty = []
    for mask in (0, CB_PSTRAND1 | CB_PSTRAND2, CB_PSTRANDS_AMBIGUOUS, CB_TSTART_GENE1, CB_PSTRAND1):
        before = ctx.candidates()
        if mask:
            _flip_bits(ctx, mask, cuda)
        cand = ctx.candidates()
        assert np.array_equal(cand["bits"], before["bits"] ^ mask) and np.array_equal(cand["gene1"], before["gene1"])
        n = int(cand["n"])
        got = ctx.retained_protein_domains(np.arange(n, dtype=np.uint32))
        want = [pref.column(cand, k, index, records, genes) for k in range(n)]
        bad = [k for k in range(n) if got[k].decode("latin-1") != want[k]]
        assert not bad, [(k, got[k], want[k]) for k in bad[:5]]
        nonempty.append(sum(1 for x in want if x != "."))
        # a subset, in another order
        sub = np.array(random.Random(mask).sample(range(n), min(n, 50)), np.uint32)
        assert ctx.retained_protein_domains(sub) == [got[k] for k in sub.tolist()]
    timings = ctx.timings()
    p.close()
    return nonempty, timings


def test_per_candidate(worlds, hostsim_lib, pd_root):
    w = worlds.get("small")
    nonempty, _ = per_candidate(w, hostsim_lib, domains_file(w, hostsim_lib, pd_root))
    assert nonempty[0] > 20 and nonempty[2] < nonempty[0], nonempty  # ambiguous strands empty every side


def test_per_candidate_few_records(worlds, hostsim_lib, pd_root):
    """Three records: sides on a contig whose id is >= 3 have none, even in the domains' gene (the reference's index has three entries)."""
    w = worlds.get("small")
    cand, genes, names, ids = final_state(w, hostsim_lib)
    nm = contig_names(w)
    g = next(int(x) for x in cand["gene1"] if genes["gene_flags"][x] & GF_CODING and 1 <= int(genes["gene_contig"][x]) <= 2 and names[x] is not None)
    s, e, c = int(genes["gene_start"][g]), int(genes["gene_end"][g]), int(genes["gene_contig"][g])
    lines = ["\t".join([nm[c], "pfam", "protein_domain", str(s + 1 + k * 10), str(e + 1 - k * 10), ".", "+", ".", "gene_name=%s;gene_id=%s;Name=D%d" % (names[g], ids[g], k % 2)])
             for k in range(3)]
    path = os.path.join(pd_root, "few.gff3"); write(path, lines)
    per_candidate(w, hostsim_lib, path)


def test_cli_errors(worlds, cli, hostsim_lib, pd_root, tmp_path):
    """A missing file and a file without a usable line stop both programs with the same ERROR line and exit code; a record on a contig whose id is not below
    the number of records (undefined in the reference) stops the product with an error naming the file."""
    w = worlds.get("small")
    oracle = _build.build_oracle()
    base = ["-x", w.prefix + ".bam", "-g", w.prefix + ".gtf", "-a", w.prefix + ".fa", "-o", str(tmp_path / "o.tsv"), "-f", "blacklist"]
    empty = str(tmp_path / "empty.gff3"); write(empty, ["# nothing", "", "1\tx\ty\t5\t9\t.\t+\t.\tgene_name=NOPE;gene_id=NOPE;Name=A"])
    for path in (str(tmp_path / "missing.gff3"), empty):
        seen = []
        for exe in (oracle, cli):
            r = subprocess.run([exe] + base + ["-p", path], capture_output=True, text=True, timeout=300)
            seen.append((r.returncode, [l for l in r.stderr.splitlines() if l.startswith("ERROR")]))
        assert seen[0] == seen[1] and seen[0][0] != 0 and seen[0][1], seen
    cand, genes, names, ids = final_state(w, hostsim_lib)
    nm = contig_names(w)
    g = next(x for x in range(len(names)) if names[x] is not None and int(genes["gene_contig"][x]) >= 1)
    ub = str(tmp_path / "ub.gff3")
    write(ub, ["\t".join([nm[int(genes["gene_contig"][g])], "pfam", "protein_domain", "10", "20", ".", "+", ".", "gene_name=%s;gene_id=%s;Name=A" % (names[g], ids[g])])])
    r = subprocess.run([cli] + base + ["-p", ub], capture_output=True, text=True, timeout=300)
    assert r.returncode == 1 and "protein domains '%s'" % ub in r.stderr and "line 1" in r.stderr, r.stderr[-2000:]


def C_byref(x):
    import ctypes
    return ctypes.byref(x)


def test_no_option_changes_nothing(worlds, hostsim_lib, pd_root, tmp_path):
    """Without -p both files equal the reference's, the column is '.' everywhere, and the kernel launches do not change between runs; with -p they do."""
    w = worlds.get("small")
    lib = L.load(hostsim_lib)
    res = []
    for pd in (None, None, domains_file(w, hostsim_lib, pd_root)):
        d = str(tmp_path / ("run%d" % len(res))); os.makedirs(d)
        p = L.Pipeline(w.prefix + ".bam", w.prefix + ".gtf", w.prefix + ".fa", threads=2, lib_path=hostsim_lib, protein_domains=pd,
                       output=os.path.join(d, "fusions.tsv"), discarded=os.path.join(d, "fusions.discarded.tsv"))
        k0 = lib.arb_kernel_launches(); p.run_all(); k1 = lib.arb_kernel_launches(); p.close()
        res.append((k1 - k0, open(os.path.join(d, "fusions.tsv"), "rb").read(), open(os.path.join(d, "fusions.discarded.tsv"), "rb").read()))
    assert res[0] == res[1] and res[2][0] > res[0][0]
    assert res[0][1] == open(os.path.join(w.outdir, "fusions.tsv"), "rb").read() and res[0][2] == open(os.path.join(w.outdir, "fusions.discarded.tsv"), "rb").read()
    assert not domain_cells(res[0][1]) and not domain_cells(res[0][2]) and domain_cells(res[2][2])


WORKER = r"""
import os, sys
sys.path.insert(0, {root!r})
import torch.distributed as dist
from arriba_b200 import lib as L, sharded
rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"])
dist.init_process_group("gloo")
out = os.path.join({outdir!r}, "rank%d" % rank); os.makedirs(out, exist_ok=True)
p = L.Pipeline({prefix!r} + ".bam", {prefix!r} + ".gtf", {prefix!r} + ".fa", threads=2, lib_path={lib!r}, protein_domains={pd!r},
               output=os.path.join(out, "fusions.tsv"), discarded=os.path.join(out, "fusions.discarded.tsv"))
sharded.run_sharded(p, rank, world)
p.close()
dist.destroy_process_group()
"""


def test_sharded_two_ranks(worlds, hostsim_lib, pd_root, tmp_path):
    w = worlds.get("small")
    pd = domains_file(w, hostsim_lib, pd_root)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = str(tmp_path / "worker.py")
    open(script, "w").write(WORKER.format(root=root, outdir=str(tmp_path), prefix=w.prefix, lib=hostsim_lib, pd=pd))
    env = dict(os.environ, PYTHONPATH=root + os.pathsep + os.path.join(root, "tests"))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port", str(29500 + os.getpid() % 200), script]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    single = str(tmp_path / "single"); os.makedirs(single)
    p = L.Pipeline(w.prefix + ".bam", w.prefix + ".gtf", w.prefix + ".fa", threads=2, lib_path=hostsim_lib, protein_domains=pd,
                   output=os.path.join(single, "fusions.tsv"), discarded=os.path.join(single, "fusions.discarded.tsv"))
    p.run_all(); p.close()
    for f in ("fusions.tsv", "fusions.discarded.tsv"):
        assert open(os.path.join(tmp_path, "rank0", f), "rb").read() == open(os.path.join(single, f), "rb").read(), f
    assert domain_cells(open(os.path.join(single, "fusions.discarded.tsv"), "rb").read())


# ---- on the H100
def pipeline_parity(w, lib_path, args, pd, tmp, extra_info=False):
    ref = oracle_run(w, args, os.path.join(tmp, "oracle"))
    out = os.path.join(tmp, "fusions.tsv"); disc = os.path.join(tmp, "fusions.discarded.tsv")
    p = L.Pipeline(w.prefix + ".bam", w.prefix + ".gtf", w.prefix + ".fa", threads=8, lib_path=lib_path, protein_domains=pd, output=out, discarded=disc)
    p.run_all(); p.close()
    for f in ("fusions.tsv", "fusions.discarded.tsv"):
        assert open(os.path.join(tmp, f), "rb").read() == open(os.path.join(ref.outdir, f), "rb").read(), f


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small", "cfg5"])
def test_parity_cuda(worlds, cuda_lib, hostsim_lib, pd_root, tmp_path, name):
    w = _world(worlds, name)
    pd = domains_file(w, hostsim_lib, pd_root)
    pipeline_parity(w, cuda_lib, NO_BL + ("-p", pd), pd, str(tmp_path / "lib"))
    cli = _build.build_cli()
    _, fus, disc = cli_parity(cli, w, NO_BL + ("-p", pd), str(tmp_path / "cli"))
    assert_meaningful(fus, disc)
    from test_known_fusions import stage_state
    cand, genes, names, mmg, _ = stage_state(w, hostsim_lib)
    bl = os.path.join(pd_root, "bl_%s.tsv" % name)
    blacklisttools.write(bl, blacklisttools.rule_lines(cand, genes, names, contig_names(w), random.Random(3), mmg, n_candidates=40))
    k, t = rules_file(w, hostsim_lib, pd_root, False), rules_file(w, hostsim_lib, pd_root, True)
    cli_parity(cli, w, ("-X", "-b", bl, "-k", k, "-t", t, "-p", pd), str(tmp_path / "cli_x"))


@pytest.mark.gpu
def test_per_candidate_cuda(worlds, cuda_lib, hostsim_lib, pd_root):
    w = worlds.get("small")
    nonempty, timings = per_candidate(w, cuda_lib, domains_file(w, hostsim_lib, pd_root))
    assert nonempty[0] > 20 and timings.protein_domains_ms > 0
