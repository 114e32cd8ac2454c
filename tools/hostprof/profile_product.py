"""PC samples of the host stages of the PRODUCT library on a GPU box (tools/hostprof/pcsample.c; there is no perf in the image).
  here:      python tools/hostprof/profile_product.py build                 # host objects with -g, linked with the product's CUDA objects -> build/product_g/
  GPU box:   LD_PRELOAD=build/libpcsample.so python tools/hostprof/profile_product.py run WORKLOAD OUTDIR
  here:      python tools/hostprof/report.py OUTDIR/ingest.pcs build/product_g/libarriba_b200_g.so"""
import ctypes, os, sys, time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from arriba_b200 import _build as B, lib  # noqa: E402

LIB_G = os.path.join(ROOT, "build", "product_g", "libarriba_b200_g.so")


def build():
    B.build_product()
    objdir = os.path.join(ROOT, "build", "product_g"); os.makedirs(objdir, exist_ok=True)
    flags = B.GXX_FLAGS + ["-g", "-fno-omit-frame-pointer", "-I", os.path.join(B.ROOT, "include")]
    jobs = [["g++"] + flags + ["-c", os.path.join(B.CSRC, s), "-o", os.path.join(objdir, s.replace("/", "_") + ".o")] for s in B.CPP_SOURCES]
    with ThreadPoolExecutor(8) as ex:
        list(ex.map(B._run, jobs))
    objs = [os.path.join(ROOT, "build", "product", s + ".o") for s in B.CU_SOURCES] + [os.path.join(objdir, s.replace("/", "_") + ".o") for s in B.CPP_SOURCES]
    B._run([B.nvcc_path(), "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB_G] + objs + ["-lcudart", "-lz", "-lpthread"])
    B._run(["gcc", "-O2", "-shared", "-fPIC", "-o", os.path.join(ROOT, "build", "libpcsample.so"), os.path.join(ROOT, "tools", "hostprof", "pcsample.c"), "-ldl"])
    print(LIB_G)


def run(workload, outdir):
    import bench
    os.makedirs(outdir, exist_ok=True)
    prefix = bench.ensure_world(workload)
    prof = ctypes.CDLL(None)
    if not hasattr(prof, "pcsample_reset"):
        raise SystemExit("run under LD_PRELOAD=build/libpcsample.so")
    threads = int(os.environ.get("ARB_PROFILE_THREADS", "32"))
    for rep in range(2):   # the second pass is the one that counts (pools and page cache warm)
        p = lib.Pipeline(prefix + ".bam", prefix + ".gtf", prefix + ".fa", threads=threads, lib_path=LIB_G, output="/tmp/hostprof_fusions.tsv", discarded="/tmp/hostprof_fusions.discarded.tsv")   # not into gpurun_out/: a gigabyte
        p.step(lib.STEP_LOAD_REFERENCE)

        def sampled(name, f):
            prof.pcsample_reset(); t = time.time(); f()
            print("%-10s %.2f s" % (name, time.time() - t), flush=True)
            if rep == 1:
                prof.pcsample_dump(os.path.join(outdir, name + ".pcs").encode())
        sampled("ingest", lambda: p.step(lib.STEP_INGEST))
        for s in range(lib.STEP_INGEST + 1, lib.STEP_COUNT):
            p.step(s)
        sampled("events", lambda: p.events(len(lib.EV_NAMES) - 1))
        sampled("output", p.write_output)
        p.close()


if __name__ == "__main__":
    if sys.argv[1] == "build":
        build()
    else:
        run(sys.argv[2], sys.argv[3])
