"""Cost of -I on the cfg2 workload (bench.py's default world): whole runs (BAM to both files, reference loading excluded) without -I, with -I, and with -I -X,
alternated in one process. One JSON line with the card's name and power limit, and per arm: output_s (the writer stage), fill_gaps_ms (CUDA events around the
transcript table and every fill call: copies of the jobs, the plan and emit kernels, the scan), the fill jobs and the characters they wrote, and the rows whose
fusion_transcript differs from a run without -I (for the discarded file of the -I -X arm: an untimed run with -X alone).

python tools/fill_gaps_bench.py [--reps 3] [--threads 32]"""
import argparse, json, os, sys, tempfile, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench
from arriba_b200 import lib as L, _build
from blacklist_bench import spread

SEQ_COL = 27
ARMS = {"none": dict(), "I": dict(fill_sequence_gaps=True), "I_X": dict(fill_sequence_gaps=True, extra_info=True)}


def sequences(path):
    with open(path, "rb") as f:
        next(f)
        return [line.split(b"\t", SEQ_COL + 1)[SEQ_COL] for line in f]


def one_run(prefix, threads, out, kw):
    t0 = time.perf_counter()
    p = L.Pipeline(prefix + ".bam", prefix + ".gtf", prefix + ".fa", threads=threads, output=os.path.join(out, "fusions.tsv"),
                   discarded=os.path.join(out, "fusions.discarded.tsv"), **kw)
    p.run(); p.events(len(L.EV_NAMES) - 1); p.write_output()
    t1 = time.perf_counter()
    s = p.stats(); t = p.context().timings()
    r = {"run_s": t1 - t0 - s.seconds[L.STEP_LOAD_REFERENCE], "output_s": s.output_seconds, "fill_gaps_ms": t.fill_gaps_ms, "jobs": int(t.fill_gaps_jobs),
         "filled_chars": int(t.fill_gaps_chars), "seq": {f: sequences(os.path.join(out, f)) for f in ("fusions.tsv", "fusions.discarded.tsv")}}
    p.close()
    for f in ("fusions.tsv", "fusions.discarded.tsv"):
        os.remove(os.path.join(out, f))
    return r


def changed(a, b):
    assert len(a) == len(b)
    return sum(1 for x, y in zip(a, b) if x != y)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3); ap.add_argument("--threads", type=int, default=2 * (len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else 8))
    ap.add_argument("--workload", default="cfg2_10M_2x101_50k")
    a = ap.parse_args()
    _build.build_product()
    prefix = bench.ensure_world(a.workload)
    card = bench.ClockSampler(0).card()
    with tempfile.TemporaryDirectory() as d:
        one_run(prefix, a.threads, d, {})  # warm-up: page cache, device pool, module load
        x_only = one_run(prefix, a.threads, d, dict(extra_info=True))["seq"]["fusions.discarded.tsv"]  # the discarded rows' columns without -I
        res = {k: [] for k in ARMS}
        for _ in range(a.reps):
            for k, kw in ARMS.items():
                res[k].append(one_run(prefix, a.threads, d, kw))
    base = res["none"][0]["seq"]
    out = {"workload": a.workload, "reps": a.reps, "threads": a.threads, **card, "arms": {}}
    for k, rs in res.items():
        s = rs[0]["seq"]
        arm = {"run_s": spread([r["run_s"] for r in rs]), "output_s": spread([r["output_s"] for r in rs]), "fill_gaps_ms": spread([r["fill_gaps_ms"] for r in rs]),
               "jobs": rs[0]["jobs"], "filled_chars": rs[0]["filled_chars"], "changed_rows_fusions": changed(base["fusions.tsv"], s["fusions.tsv"])}
        if k == "I_X":
            arm["changed_rows_discarded"] = changed(x_only, s["fusions.discarded.tsv"])
        out["arms"][k] = arm
    print(json.dumps(out))


if __name__ == "__main__":
    main()
