"""Cost of -b on the cfg2 workload (bench.py's default world): whole runs (BAM to both files, reference loading excluded) without -b and with seeded blacklists of
10^4 and 10^6 rules (half of each placed around the run's own candidates, half anywhere on the genome), alternated in one process; one JSON line with the
card's name and power limit, blacklist_ms (key table + search + verdicts on the device), the parse time and the number of candidates blacklisted.

python tools/blacklist_bench.py [--reps 3] [--threads 32]"""
import argparse, json, os, random, statistics, sys, tempfile, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench
from arriba_b200 import lib as L, _build

KEYWORDS = ["any", "split_read_donor", "split_read_acceptor", "split_read_any", "discordant_mates", "read_through", "low_support", "filter_spliced", "not_both_spliced"]
SHORT_ANCHOR = L.EV_NAMES.index("short_anchor")


def blacklist_file(path, cand, lengths, names, n, seed):
    rng = random.Random(seed)
    k_max = len(cand["breakpoint1"])
    with open(path, "w") as f:
        for x in range(n):
            if x % 2 == 0 and k_max:
                k = rng.randrange(k_max)
                c1, c2 = int(cand["contig1"][k]), int(cand["contig2"][k])
                p1 = int(cand["breakpoint1"][k]) + rng.randint(-3000, 3000); p2 = int(cand["breakpoint2"][k]) + rng.randint(-3000, 3000)
            else:
                c1, c2 = rng.randrange(len(names)), rng.randrange(len(names))
                p1, p2 = rng.randrange(max(lengths[c1], 1)), rng.randrange(max(lengths[c2], 1))
            second = rng.choice(KEYWORDS) if rng.random() < 0.3 else "%s:%d" % (names[c2], max(p2, 0) + 1)
            first = "%s:%d" % (names[c1], max(p1, 0) + 1) if rng.random() < 0.8 else "%s:%d-%d" % (names[c1], max(p1, 0) + 1, max(p1, 0) + rng.randint(2, 50000))
            f.write("%s\t%s\n" % (first, second))


def contig_table(prefix):
    names, lengths = [], []
    for line in open(prefix + ".fa"):
        if line.startswith(">"):
            names.append(line[1:].split()[0]); lengths.append(0)
        else:
            lengths[-1] += len(line.strip())
    return names, lengths


def one_run(prefix, threads, out, bl):
    t0 = time.perf_counter()
    p = L.Pipeline(prefix + ".bam", prefix + ".gtf", prefix + ".fa", threads=threads, output=os.path.join(out, "fusions.tsv"),
                   discarded=os.path.join(out, "fusions.discarded.tsv"), blacklist=bl)
    p.run_all()
    t1 = time.perf_counter()
    s = p.stats(); t = p.context().timings()
    r = {"run_s": t1 - t0 - s.seconds[L.STEP_LOAD_REFERENCE], "stage_s": s.event_seconds[SHORT_ANCHOR], "blacklist_ms": t.blacklist_ms if bl else 0.0,
         "blacklisted": int((p.candidates()["filter"] == 20).sum())}
    p.close()
    for f in ("fusions.tsv", "fusions.discarded.tsv"):
        os.remove(os.path.join(out, f))
    return r


def spread(v):
    return {"median": statistics.median(v), "min": min(v), "max": max(v)}


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
        p.run(); p.events(0); cand = p.candidates(); p.close()
        files = {"none": None}
        for n in (10 ** 4, 10 ** 6):
            files[str(n)] = os.path.join(d, "bl%d.tsv" % n); blacklist_file(files[str(n)], cand, lengths, names, n, n)
        one_run(prefix, a.threads, d, None)  # warm-up: page cache, device pool, module load
        res = {k: [] for k in files}
        for _ in range(a.reps):
            for k, path in files.items():
                res[k].append(one_run(prefix, a.threads, d, path))
    base_stage = statistics.median(r["stage_s"] for r in res["none"])
    out = {"workload": a.workload, "candidates": int(cand["n"]), "reps": a.reps, "threads": a.threads, **card, "arms": {}}
    for k, rs in res.items():
        arm = {"run_s": spread([r["run_s"] for r in rs]), "stage_s": spread([r["stage_s"] for r in rs])}
        if k != "none":
            arm["blacklist_ms"] = spread([r["blacklist_ms"] for r in rs])
            # reading + parsing the file and the host side of the stage: what the stage gained, less the device time
            arm["parse_s"] = spread([r["stage_s"] - base_stage - r["blacklist_ms"] / 1e3 for r in rs])
            arm["blacklisted"] = rs[0]["blacklisted"]
        out["arms"][k] = arm
    print(json.dumps(out))


if __name__ == "__main__":
    main()
