"""What reading the alignments from a pipe costs, on the cfg2 workload (bench.py's default world). Three arms alternate after one warm-up each:
  file      -x the BAM file (the mapped path),
  pipe      the same bytes from an unthrottled producer process through a pipe (-x /dev/fd/N),
  throttled the same through a producer held to --rate MB/s, as an aligner that writes while it aligns would be,
  read_only the unthrottled producer into a reader that only read()s 1 MiB at a time and discards the bytes: what the pipe itself delivers.
The producers start once the pipeline's reference is loaded, right before the ingest.
Per arm and timed step: ingest_s (the reference is loaded outside the clock), the host CPU seconds of this process during the ingest (getrusage: user +
system, all threads; the producer is another process), the rec_* laps of arb_timings with rec_unwrap_ms (the device's assembly of the stream chunks),
rec_h2d_bytes (what the record loop copied up), how often the record store was allocated and its largest size, and for the throttled arm the tail: from
the producer's end of input to the end of the ingest. The gather rate counts the bytes it reads and writes (2 x the inflated payload) over rec_unwrap_ms.
Then one whole run through a pipe writes both TSV files, whose md5 sums are checked against tests/golden/full_size_md5.json. The card's name and power
limit are read in the same call. One JSON line on stdout (and in the file --out names).

python tools/pipe_bench.py [--warmup 1] [--steps 2] [--rate 500] [--threads N] [--out FILE]"""
import argparse, hashlib, json, os, resource, statistics, struct, subprocess, sys, tempfile, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench
from arriba_b200 import lib as L, _build

LAPS = ["rec_chunk_copy_ms", "rec_unwrap_ms", "rec_chunk_kernels_ms", "rec_sort_ms", "rec_count_ms", "rec_scan_ms", "rec_write_ms", "rec_download_ms"]

PRODUCER = r"""
import os, sys, time
path, rate, report = sys.argv[1], float(sys.argv[2]), sys.argv[3]
piece = 1 << 20
t0 = time.monotonic(); sent = 0
with open(path, "rb", buffering=0) as f:
    while True:
        b = f.read(piece)
        if not b:
            break
        mv = memoryview(b)
        while mv:
            n = os.write(1, mv); mv = mv[n:]
        sent += len(b)
        if rate > 0:
            lag = t0 + sent / (rate * 1e6) - time.monotonic()
            if lag > 0:
                time.sleep(lag)
os.close(1)
open(report, "w").write(repr(time.monotonic()))
"""


def inflated_bytes(path):
    """the sum of the BGZF members' ISIZE: the inflated stream the record loop reads"""
    total = 0
    with open(path, "rb") as f:
        size = os.fstat(f.fileno()).st_size; at = 0
        while at + 18 <= size:
            f.seek(at); h = f.read(18)
            bsize = struct.unpack_from("<H", h, 16)[0] + 1
            f.seek(at + bsize - 4); total += struct.unpack("<I", f.read(4))[0]
            at += bsize
    return total


def cpu_s():
    r = resource.getrusage(resource.RUSAGE_SELF)
    return r.ru_utime + r.ru_stime


def start_producer(prefix, rate, report):
    """the producer process writing the BAM into a new pipe; returns (process, read end)"""
    r, w = os.pipe()
    producer = subprocess.Popen([sys.executable, "-c", PRODUCER, prefix + ".bam", str(rate), report], stdout=w)
    os.close(w)
    return producer, r


def read_only_step(prefix):
    producer, r = start_producer(prefix, 0, os.path.join(tempfile.mkdtemp(prefix="pipe_bench_"), "eof"))
    buf = bytearray(1 << 20); n = 0
    c0, t0 = cpu_s(), time.perf_counter()
    while True:
        k = os.readv(r, [buf])
        if k == 0:
            break
        n += k
    out = {"seconds": round(time.perf_counter() - t0, 3), "host_cpu_s": round(cpu_s() - c0, 2), "bytes": n}
    out["GBps"] = round(n / out["seconds"] / 1e9, 2)
    os.close(r); producer.wait()
    return out


def one_step(prefix, threads, arm, rate, outputs=None):
    if arm == "read_only":
        return read_only_step(prefix)
    tmp = tempfile.mkdtemp(prefix="pipe_bench_")
    producer, report, src = None, os.path.join(tmp, "eof"), prefix + ".bam"
    if arm != "file":  # the pipe exists from the start (its path is the pipeline's input); the producer starts after the reference load
        r, w = os.pipe()
        src = "/dev/fd/%d" % r
    kw = {"output": outputs[0], "discarded": outputs[1]} if outputs else {}
    p = L.Pipeline(src, prefix + ".gtf", prefix + ".fa", threads=threads, **kw)
    p.step(L.STEP_LOAD_REFERENCE)
    if arm != "file":
        producer = subprocess.Popen([sys.executable, "-c", PRODUCER, prefix + ".bam", str(rate if arm == "throttled" else 0), report], stdout=w)
        os.close(w)
    c0, t0 = cpu_s(), time.perf_counter()
    p.step(L.STEP_INGEST)
    ingest_s, end = time.perf_counter() - t0, time.monotonic()
    cpu = cpu_s() - c0
    t = p.context().timings(); s = p.stats()
    out = {"ingest_s": round(ingest_s, 3), "host_cpu_s": round(cpu, 2), "laps_ms": {k: round(getattr(t, k), 2) for k in LAPS},
           "rec_h2d_bytes": int(t.rec_h2d_bytes), "store_allocations": int(t.rec_store_grows), "store_peak_bytes": int(t.rec_store_bytes),
           "records": int(s.n_records), "fragments": int(s.n_fragments)}
    if outputs:  # the remaining steps, each once (the input is read once)
        for step in range(L.STEP_INGEST + 1, L.STEP_COUNT):
            p.step(step)
        p.events(len(L.EV_NAMES) - 1); p.write_output()
    p.close()
    if producer:
        os.close(r); producer.wait()
        if arm == "throttled":
            out["tail_s"] = round(end - float(open(report).read()), 3)
    return out


def md5(path):
    h = hashlib.md5()
    with open(path, "rb") as f:
        for b in iter(lambda: f.read(1 << 24), b""):
            h.update(b)
    return h.hexdigest()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=1); ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--rate", type=float, default=500.0, help="MB/s of the throttled producer")
    ap.add_argument("--threads", type=int, default=2 * (len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else 8))
    ap.add_argument("--workload", default="cfg2_10M_2x101_50k")
    ap.add_argument("--skip-outputs", action="store_true", help="no whole run through the pipe")
    ap.add_argument("--out", help="also write the JSON line to this file")
    a = ap.parse_args()
    if not os.path.exists(_build.PRODUCT_LIB):
        _build.build_product()
    prefix = bench.ensure_world(a.workload)
    card = bench.ClockSampler(0).card()
    arms = ["file", "pipe", "throttled", "read_only"]
    for _ in range(a.warmup):
        for arm in arms:
            one_step(prefix, a.threads, arm, a.rate)
    steps = {arm: [] for arm in arms}
    for _ in range(a.steps):  # the arms alternate
        for arm in arms:
            steps[arm].append(one_step(prefix, a.threads, arm, a.rate))
    inflated = inflated_bytes(prefix + ".bam")
    res = {"workload": a.workload, "threads": a.threads, **card, "input_bytes": os.path.getsize(prefix + ".bam"), "inflated_bytes": inflated, "rate_MBps": a.rate}
    for arm, st in steps.items():
        med = lambda f: statistics.median(f(r) for r in st)
        if arm == "read_only":
            res[arm] = {"median": {k: med(lambda r: r[k]) for k in ("seconds", "GBps", "host_cpu_s")}, "steps": st}
            continue
        m = {"ingest_s": med(lambda r: r["ingest_s"]), "host_cpu_s": med(lambda r: r["host_cpu_s"]), "laps_ms": {k: med(lambda r: r["laps_ms"][k]) for k in LAPS},
             "rec_h2d_bytes": st[-1]["rec_h2d_bytes"], "store_allocations": st[-1]["store_allocations"], "store_peak_bytes": st[-1]["store_peak_bytes"]}
        if arm != "file" and m["laps_ms"]["rec_unwrap_ms"] > 0:
            m["unwrap_GBps_read_plus_write"] = round(2 * inflated / (m["laps_ms"]["rec_unwrap_ms"] * 1e-3) / 1e9, 1)
            m["h2d_over_inflated"] = round(m["rec_h2d_bytes"] / inflated, 5)
        if arm == "throttled":
            m["tail_s"] = med(lambda r: r["tail_s"])
        res[arm] = {"median": m, "steps": st}
    if not a.skip_outputs:
        d = tempfile.mkdtemp(prefix="pipe_bench_out_")
        outs = (os.path.join(d, "fusions.tsv"), os.path.join(d, "fusions.discarded.tsv"))
        t0 = time.perf_counter()
        one_step(prefix, a.threads, "pipe", 0, outs)
        golden = json.load(open(os.path.join(ROOT, "tests", "golden", "full_size_md5.json"))).get(a.workload, {})
        got = {os.path.basename(f): md5(f) for f in outs}
        res["outputs_through_pipe"] = {"seconds": round(time.perf_counter() - t0, 1), "md5": got, "golden_match": all(golden.get(k) == v for k, v in got.items()) and bool(golden)}
    line = json.dumps(res)
    print(line)
    if a.out:
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
