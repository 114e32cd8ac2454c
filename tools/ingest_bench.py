"""Where the BAM ingest of the cfg2 workload (bench.py's default world) spends its time: whole ingest steps through the public Pipeline API (the reference
loaded outside the clock), a warm-up, then timed steps. One JSON line with the card's name and power limit, and per timed step:
  - ingest_s and ingest_split (inflate / parse / finalize, host clocks, as bench.py reports them),
  - bam_scan_ms and its laps (CUDA events, arb_timings.rec_*): per-chunk copy and kernels summed over the chunks; sort, counting launches, scans,
    writing launches, coverage and counter download of arb_records_finish,
  - finalize_rest_s: finalize less the device laps of arb_records_finish (the fragment-table build, its download and the host's share).
Also the rate of a plain copy of one page-locked 128 MiB host buffer to the device in the same process: the PCIe floor of the chunk stream.
With --sam (or --sam-bgzf) the SAM text rendering of the same world (tools/synth.cpp --sam-only, written once next to the BAM) is measured too: BAM and SAM
steps alternate, after one warm-up of each, and every format gets its own medians, its input size and the SAM parse lap (rec_text_parse_ms, part of
rec_chunk_kernels_ms).
With --separate-chimeric the world is also written as STAR's --chimOutType SeparateSAMold pair (tools/synth.cpp --separate-chimeric-only: the chimeric
reads in Chimeric.out.sam, SAM text, the rest in Aligned.out.bam), and the pair (-c and -x) is timed against the WithinBAM file, alternating; the pair's
input_bytes is the main file's, chimeric_input_bytes the -c file's.

python tools/ingest_bench.py [--warmup 1] [--steps 3] [--threads N] [--sam | --sam-bgzf | --separate-chimeric]"""
import argparse, json, os, statistics, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench
from arriba_b200 import lib as L, _build

LAPS = ["rec_chunk_copy_ms", "rec_chunk_kernels_ms", "rec_sort_ms", "rec_count_ms", "rec_scan_ms", "rec_write_ms", "rec_download_ms", "rec_text_parse_ms"]
FINISH_LAPS = ["rec_sort_ms", "rec_count_ms", "rec_scan_ms", "rec_write_ms", "rec_download_ms"]


def pinned_h2d_gbps(reps=10):
    import torch
    src = torch.empty(128 << 20, dtype=torch.uint8, pin_memory=True)
    dst = torch.empty(128 << 20, dtype=torch.uint8, device="cuda")
    dst.copy_(src, non_blocking=True); torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        dst.copy_(src, non_blocking=True)
    b.record(); b.synchronize()
    return reps * (128 << 20) / (a.elapsed_time(b) * 1e-3) / 1e9


def one_step(prefix, threads, path=None, chimeric=None):
    p = L.Pipeline(path or prefix + ".bam", prefix + ".gtf", prefix + ".fa", threads=threads, chimeric=chimeric)
    p.step(L.STEP_LOAD_REFERENCE)
    t0 = time.perf_counter()
    p.step(L.STEP_INGEST)
    ingest_s = time.perf_counter() - t0
    s = p.stats(); t = p.context().timings()
    laps = {k: round(getattr(t, k), 2) for k in LAPS}
    finish_ms = sum(laps[k] for k in FINISH_LAPS)
    r = {"ingest_s": round(ingest_s, 3), "ingest_split": {"inflate": round(s.t_inflate, 3), "parse": round(s.t_parse, 3), "finalize": round(s.t_finalize, 3)},
         "bam_scan_ms": round(t.bam_scan_ms, 1), "laps_ms": laps, "finalize_rest_s": round(s.t_finalize - finish_ms * 1e-3, 3),
         "records": int(s.n_records), "fragments": int(s.n_fragments)}
    if chimeric:
        r.update(chimeric_records=int(s.chimeric_records), chimeric_total=int(s.chimeric_total), chimeric_malformed=int(s.chimeric_malformed))
    p.close()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=1); ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--threads", type=int, default=2 * (len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else 8))
    ap.add_argument("--workload", default="cfg2_10M_2x101_50k")
    ap.add_argument("--sam", action="store_true", help="also the plain SAM rendering of the world")
    ap.add_argument("--sam-bgzf", action="store_true", help="also the BGZF-compressed SAM rendering (level 1)")
    ap.add_argument("--separate-chimeric", action="store_true", help="also the SeparateSAMold pair (-c Chimeric.out.sam -x Aligned.out.bam)")
    a = ap.parse_args()
    if not os.path.exists(_build.PRODUCT_LIB):
        _build.build_product()
    prefix = bench.ensure_world(a.workload)
    card = bench.ClockSampler(0).card()
    inputs = {"bam": (prefix + ".bam", None)}
    if a.sam or a.sam_bgzf:
        kind = "sam_bgzf" if a.sam_bgzf else "sam"
        sam_prefix = prefix + "_" + kind
        if not os.path.exists(sam_prefix + ".done"):
            if not os.path.exists(sam_prefix + ".bam"):
                os.symlink(prefix + ".bam", sam_prefix + ".bam")
            subprocess.run([_build.build_tools(), "--prefix", sam_prefix, "--sam-only"] + (["--sam-bgzf", "1"] if a.sam_bgzf else []), check=True)
            open(sam_prefix + ".done", "w").write("ok")
        inputs[kind] = (sam_prefix + ".sam", None)
    if a.separate_chimeric:
        pair_prefix = prefix + "_separate"
        if not os.path.exists(pair_prefix + ".done"):
            if not os.path.exists(pair_prefix + ".bam"):
                os.symlink(prefix + ".bam", pair_prefix + ".bam")
            subprocess.run([_build.build_tools(), "--prefix", pair_prefix, "--separate-chimeric-only"], check=True)
            open(pair_prefix + ".done", "w").write("ok")
        inputs["separate_chimeric"] = (pair_prefix + ".Aligned.out.bam", pair_prefix + ".Chimeric.out.sam")
    for _ in range(a.warmup):
        for path, chimeric in inputs.values():
            one_step(prefix, a.threads, path, chimeric)
    steps = {k: [] for k in inputs}
    for _ in range(a.steps):  # the formats alternate
        for k, (path, chimeric) in inputs.items():
            steps[k].append(one_step(prefix, a.threads, path, chimeric))
    out = {"workload": a.workload, "threads": a.threads, **card, "pinned_h2d_128MiB_GBps": round(pinned_h2d_gbps(), 2)}
    for k, st in steps.items():
        med = lambda f: statistics.median(f(r) for r in st)
        path, chimeric = inputs[k]
        out[k] = {"input_bytes": os.path.getsize(path), **({"chimeric_input_bytes": os.path.getsize(chimeric)} if chimeric else {}),
                  "median": {"ingest_s": med(lambda r: r["ingest_s"]), "finalize_s": med(lambda r: r["ingest_split"]["finalize"]), "bam_scan_ms": med(lambda r: r["bam_scan_ms"]),
                             "laps_ms": {x: med(lambda r: r["laps_ms"][x]) for x in LAPS}},
                  "steps": st}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
