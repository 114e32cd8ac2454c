"""Cost of -p on the cfg2 workload (bench.py's default world): whole runs (BAM to both files, reference loading excluded) without -p and with seeded GFF3 files
of 10^5 and 10^6 protein domains, alternated in one process. The domains lie in the world's protein-coding genes (found by gene ID or name), overlap each
other, and take their names from a pool of about 5,000 (so names repeat within and across genes). One JSON line with the card's name and power limit, and
per arm: rows_ms (arb_format_discarded_rows, the discarded rows formatted on the device), protein_domains_ms (tables + the column of the rows the host
formats), the host's share of loading the file (parse_s: what the output stage gained, less both device times), and the rows whose column is not '.'.

python tools/protein_domains_bench.py [--reps 3] [--threads 32]"""
import argparse, json, os, random, statistics, sys, tempfile, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench
from arriba_b200 import lib as L, _build
from blacklist_bench import spread


def coding_genes(gtf):
    """(contig, start, end, gene_id, gene_name) of every gene with a CDS line, 1-based, from the GTF's gene and CDS lines."""
    genes, coding = {}, set()
    for line in open(gtf):
        if line.startswith("#"):
            continue
        f = line.rstrip("\n").split("\t")
        if len(f) < 9 or f[2] not in ("gene", "CDS"):
            continue
        attrs = dict(a.strip().split(" ", 1) for a in f[8].split(";") if " " in a.strip())
        gid = attrs.get("gene_id", "").strip('"')
        if f[2] == "CDS":
            coding.add(gid)
        else:
            genes[gid] = (f[0], int(f[3]), int(f[4]), gid, attrs.get("gene_name", '"%s"' % gid).strip('"'))
    return [genes[g] for g in sorted(coding) if g in genes]


def gff3_file(path, genes, n, seed):
    rng = random.Random(seed)
    pool = ["PF%05d_domain%d" % (rng.randrange(100000), k) for k in range(5000)]
    with open(path, "w") as f:
        f.write("##gff-version 3\n")
        x = 0
        while x < n:
            contig, s, e, gid, name = rng.choice(genes)
            names = rng.sample(pool, 3)
            for _ in range(min(n - x, rng.randint(1, 12))):
                a = rng.randint(s, e); b = min(e + rng.choice((0, 0, 0, 50)), a + rng.randint(10, 3000))
                who = "gene_id=%s;gene_name=%s" % (gid, name) if rng.random() < 0.9 else "gene_id=unknown;gene_name=%s" % name
                f.write("%s\tpfam\tprotein_domain\t%d\t%d\t.\t+\t.\t%s;Name=%s\n" % (contig, a, b, who, rng.choice(names)))
                x += 1


def domain_rows(path):
    n = 0
    with open(path, "rb") as f:
        next(f)
        for line in f:
            n += line.split(b"\t", 18)[17] != b"."
    return n


def one_run(prefix, threads, out, pd):
    t0 = time.perf_counter()
    p = L.Pipeline(prefix + ".bam", prefix + ".gtf", prefix + ".fa", threads=threads, output=os.path.join(out, "fusions.tsv"),
                   discarded=os.path.join(out, "fusions.discarded.tsv"), protein_domains=pd)
    p.run(); p.events(len(L.EV_NAMES) - 1); p.write_output()
    t1 = time.perf_counter()
    s = p.stats(); t = p.context().timings()
    r = {"run_s": t1 - t0 - s.seconds[L.STEP_LOAD_REFERENCE], "output_s": s.output_seconds, "rows_ms": t.rows_ms,
         "protein_domains_ms": t.protein_domains_ms if pd else 0.0,
         "domain_rows": domain_rows(os.path.join(out, "fusions.tsv")) + domain_rows(os.path.join(out, "fusions.discarded.tsv"))}
    p.close()
    for f in ("fusions.tsv", "fusions.discarded.tsv"):
        os.remove(os.path.join(out, f))
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3); ap.add_argument("--threads", type=int, default=2 * (len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else 8))
    ap.add_argument("--workload", default="cfg2_10M_2x101_50k")
    a = ap.parse_args()
    _build.build_product()
    prefix = bench.ensure_world(a.workload)
    card = bench.ClockSampler(0).card()
    genes = coding_genes(prefix + ".gtf")
    with tempfile.TemporaryDirectory() as d:
        files = {"none": None}
        for n in (10 ** 5, 10 ** 6):
            files[str(n)] = os.path.join(d, "domains%d.gff3" % n)
            gff3_file(files[str(n)], genes, n, n)
        one_run(prefix, a.threads, d, None)  # warm-up: page cache, device pool, module load
        res = {k: [] for k in files}
        for _ in range(a.reps):
            for k, pd in files.items():
                res[k].append(one_run(prefix, a.threads, d, pd))
    base = res["none"]
    base_output = statistics.median(r["output_s"] for r in base); base_rows = statistics.median(r["rows_ms"] for r in base)
    out = {"workload": a.workload, "coding_genes": len(genes), "reps": a.reps, "threads": a.threads, **card, "arms": {}}
    for k, rs in res.items():
        arm = {"run_s": spread([r["run_s"] for r in rs]), "rows_ms": spread([r["rows_ms"] for r in rs]), "domain_rows": rs[0]["domain_rows"]}
        if k != "none":
            arm["protein_domains_ms"] = spread([r["protein_domains_ms"] for r in rs])
            arm["parse_s"] = spread([r["output_s"] - base_output - r["protein_domains_ms"] / 1e3 - (r["rows_ms"] - base_rows) / 1e3 for r in rs])
        out["arms"][k] = arm
    print(json.dumps(out))


if __name__ == "__main__":
    main()
