#!/usr/bin/env python
"""AddressSanitizer + UndefinedBehaviorSanitizer over the rule functors and the host code: builds a copy of the CPU stand-in (tests/hostsim: the same functors
as the kernels, every device buffer its own malloc) and of the `arriba` front end with -fsanitize=address,undefined and runs worlds through it. An index that
runs past a column is silent on the GPU; here it stops the run. Test infrastructure; nothing of it is linked into the product.
    python tools/sanitizer_check.py OUTDIR PREFIX [ENV=VALUE ...] [PREFIX ...]      # PREFIX.bam / .gtf / .fa; ENV=VALUE pairs apply to the prefix before them
    python tools/sanitizer_check.py OUTDIR PREFIX "ARGS=-I -X" ...                 # ARGS=...: more command-line options for that run (here: gap filling)
    SANITIZE=thread python tools/sanitizer_check.py ...                                # ThreadSanitizer instead: races between the host threads (THREADS=n for -@)"""
import os, subprocess, sys
from concurrent.futures import ThreadPoolExecutor
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from arriba_b200 import _build as B  # noqa: E402


SAN = os.environ.get("SANITIZE", "address,undefined")


def build(out):
    obj = os.path.join(out, "obj"); os.makedirs(obj, exist_ok=True)
    flags = ["-O1", "-g", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fsanitize=" + SAN, "-fno-omit-frame-pointer", "-DARB_HOSTSIM", "-I", os.path.join(ROOT, "include")]
    jobs = [["g++", "-x", "c++"] + flags + ["-c", os.path.join(B.CSRC, s), "-o", os.path.join(obj, s + ".o")] for s in B.CU_SOURCES]
    jobs += [["g++"] + flags + ["-c", os.path.join(B.CSRC, s), "-o", os.path.join(obj, s.replace("/", "_") + ".o")] for s in B.CPP_SOURCES]
    with ThreadPoolExecutor(8) as ex:
        list(ex.map(B._run, jobs))
    lib = os.path.join(out, "libarriba_b200_hostsim.so")
    B._run(["g++", "-shared", "-fsanitize=" + SAN, "-o", lib] + [os.path.join(obj, s.replace("/", "_") + ".o") for s in B.CU_SOURCES + B.CPP_SOURCES] + ["-lz", "-lpthread"])
    exe = os.path.join(out, "arriba_sanitized")
    B._run(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=" + SAN, "-o", exe, os.path.join(B.CSRC, "host", "cli_main.cpp"), "-I", os.path.join(ROOT, "include"),
            "-L", out, "-l:libarriba_b200_hostsim.so", "-Wl,-rpath," + out, "-lpthread"])
    return exe


def main():
    out = sys.argv[1]; os.makedirs(out, exist_ok=True)
    exe = build(out)
    runs = []
    for a in sys.argv[2:]:
        if "=" in a and runs:
            k, v = a.split("=", 1); runs[-1][1][k] = v
        else:
            runs.append((a, {}))
    bad = 0
    for i, (prefix, extra) in enumerate(runs):
        extra = dict(extra); args = extra.pop("ARGS", "").split()
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:halt_on_error=1", UBSAN_OPTIONS="print_stacktrace=1:halt_on_error=1", TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0", **extra)
        r = subprocess.run([exe, "-x", prefix + ".bam", "-g", prefix + ".gtf", "-a", prefix + ".fa", "-o", os.path.join(out, "%d.tsv" % i), "-O", os.path.join(out, "%d.discarded.tsv" % i), "-f", "blacklist", "-@", os.environ.get("THREADS", "5")] + args,
                           env=env, stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, text=True)
        reports = [l for l in r.stderr.splitlines() if "AddressSanitizer" in l or "runtime error" in l or "WARNING: ThreadSanitizer" in l]
        print("%s %s %s: exit code %d, sanitizer reports %d" % (prefix, " ".join(args), extra, r.returncode, len(reports)), flush=True)
        for l in reports[:5]:
            print("   ", l)
        bad += bool(reports) or r.returncode != 0
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
