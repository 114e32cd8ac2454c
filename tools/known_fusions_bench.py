"""Cost of -k and -t on the cfg2 workload (bench.py's default world): whole runs (BAM to both files, reference loading excluded) without either option and with
seeded files of 10^4 and 10^6 lines for both (half of each written from the run's own candidates, oriented 5'->3', half placed anywhere on the genome),
alternated in one process; one JSON line with the card's name and power limit, known_fusions_ms and tags_ms (key table + search + copies on the device; tags_ms split into
the match passes and the sort, with the number of (row, rule) pairs), the parse time, the number of candidates rescued and the number of rows that carry a tag.

python tools/known_fusions_bench.py [--reps 3] [--threads 32]"""
import argparse, json, os, random, statistics, sys, tempfile, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench
from arriba_b200 import lib as L, _build
from blacklist_bench import contig_table, spread

INTRONIC = L.EV_NAMES.index("intronic")
CB_TSTART_GENE1 = 128


def rules_file(path, cand, lengths, names, n, seed, tags):
    rng = random.Random(seed)
    k_max = len(cand["breakpoint1"])
    with open(path, "w") as f:
        for x in range(n):
            if x % 2 == 0 and k_max:
                k = rng.randrange(k_max)
                w5 = 1 if int(cand["bits"][k]) & CB_TSTART_GENE1 else 2
                c1, c2 = int(cand["contig%d" % w5][k]), int(cand["contig%d" % (3 - w5)][k])
                p1 = int(cand["breakpoint%d" % w5][k]) + rng.choice((0, 0, rng.randint(-3000, 3000)))
                p2 = int(cand["breakpoint%d" % (3 - w5)][k]) + rng.choice((0, 0, rng.randint(-3000, 3000)))
            else:
                c1, c2 = rng.randrange(len(names)), rng.randrange(len(names))
                p1, p2 = rng.randrange(max(lengths[c1], 1)), rng.randrange(max(lengths[c2], 1))
            first = "%s:%d" % (names[c1], max(p1, 0) + 1) if rng.random() < 0.8 else "%s:%d-%d" % (names[c1], max(p1, 0) + 1, max(p1, 0) + rng.randint(2, 50000))
            line = "%s\t%s:%d" % (first, names[c2], max(p2, 0) + 1)
            f.write(line + ("\ttag%d\n" % rng.randrange(1000) if tags else "\n"))


def tagged_rows(path):
    n = 0
    with open(path, "rb") as f:
        next(f)
        for line in f:
            n += line.split(b"\t", 17)[16] != b"."
    return n


def one_run(prefix, threads, out, kf, tags):
    t0 = time.perf_counter()
    p = L.Pipeline(prefix + ".bam", prefix + ".gtf", prefix + ".fa", threads=threads, output=os.path.join(out, "fusions.tsv"),
                   discarded=os.path.join(out, "fusions.discarded.tsv"), known_fusions=kf, tags=tags)
    p.run(); p.events(INTRONIC)
    t_mid = time.perf_counter()
    remaining = int((p.candidates()["filter"] == 0).sum())
    t_mid = time.perf_counter() - t_mid  # the copy of the table is not part of the run
    p.events(len(L.EV_NAMES) - 1); p.write_output()
    t1 = time.perf_counter()
    s = p.stats(); t = p.context().timings()
    r = {"run_s": t1 - t0 - t_mid - s.seconds[L.STEP_LOAD_REFERENCE], "intronic_s": s.event_seconds[INTRONIC], "output_s": s.output_seconds,
         "known_fusions_ms": t.known_fusions_ms if kf else 0.0, "tags_ms": t.tags_ms if tags else 0.0, "remaining": remaining,
         "tags_match_ms": t.tags_match_ms if tags else 0.0, "tags_sort_ms": t.tags_sort_ms if tags else 0.0, "tag_pairs": int(t.tags_pairs) if tags else 0,
         "tagged_rows": tagged_rows(os.path.join(out, "fusions.tsv")) + tagged_rows(os.path.join(out, "fusions.discarded.tsv"))}
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
    names, lengths = contig_table(prefix)
    with tempfile.TemporaryDirectory() as d:
        p = L.Pipeline(prefix + ".bam", prefix + ".gtf", prefix + ".fa", threads=a.threads)
        p.run(); p.events(INTRONIC); cand = p.candidates(); p.close()
        files = {"none": (None, None)}
        for n in (10 ** 4, 10 ** 6):
            kf, tg = os.path.join(d, "kf%d.tsv" % n), os.path.join(d, "tags%d.tsv" % n)
            rules_file(kf, cand, lengths, names, n, n, False); rules_file(tg, cand, lengths, names, n, n + 1, True)
            files[str(n)] = (kf, tg)
        one_run(prefix, a.threads, d, None, None)  # warm-up: page cache, device pool, module load
        res = {k: [] for k in files}
        for _ in range(a.reps):
            for k, (kf, tg) in files.items():
                res[k].append(one_run(prefix, a.threads, d, kf, tg))
    base = res["none"]
    base_intronic = statistics.median(r["intronic_s"] for r in base); base_output = statistics.median(r["output_s"] for r in base)
    out = {"workload": a.workload, "candidates": int(cand["n"]), "reps": a.reps, "threads": a.threads, **card, "arms": {}}
    for k, rs in res.items():
        arm = {"run_s": spread([r["run_s"] for r in rs])}
        if k != "none":
            arm["known_fusions_ms"] = spread([r["known_fusions_ms"] for r in rs]); arm["tags_ms"] = spread([r["tags_ms"] for r in rs])
            # tags_ms = tags_match_ms (key table + both passes over the rows) + tags_sort_ms (sort of the pairs, duplicates removed, per-candidate table)
            arm["tags_match_ms"] = spread([r["tags_match_ms"] for r in rs]); arm["tags_sort_ms"] = spread([r["tags_sort_ms"] for r in rs])
            arm["tag_pairs"] = rs[0]["tag_pairs"]
            # reading + parsing the files and the host side: what the two stages gained, less the device time
            arm["parse_s"] = spread([r["intronic_s"] - base_intronic - r["known_fusions_ms"] / 1e3 + r["output_s"] - base_output - r["tags_ms"] / 1e3 for r in rs])
            arm["rescued"] = rs[0]["remaining"] - base[0]["remaining"]
            arm["tagged_rows"] = rs[0]["tagged_rows"]
        out["arms"][k] = arm
    print(json.dumps(out))


if __name__ == "__main__":
    main()
