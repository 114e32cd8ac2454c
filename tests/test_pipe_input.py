"""Input from a pipe (-x /dev/stdin, a FIFO, -c from a FIFO): the same bytes must give the same outcome as in a regular file -- the fragment table,
coverage windows and front-end stages against the oracle's dumps, both output files, warnings, progress lines, ERROR texts and exit codes. The streams
are written by a thread in pieces of random size (1 B to ~200 kB, with short pauses), so headers, blocks and records straddle the reads."""
import contextlib, ctypes as C, os, random, re, subprocess, sys, threading, time
import numpy as np
import pytest
import bamtools, samtext, worldutil
from arriba_b200 import lib as L, _build
from test_sam_input import world, sam_of, check_front_end_sam, run_outputs, warnings_of, progress_of
from test_chimeric_file import pair, totals
from test_z_bam_corpus import transcoded_world
from test_genomic_support import sv_file
from test_blacklist import blacklist_file
from test_known_fusions import rules_file
from test_protein_domains import domains_file


# ---- the producer
def _write_pieces(fd, data, seed):
    rng = random.Random(seed)
    at = 0
    try:
        while at < len(data):
            n = rng.choice((rng.randint(1, 64), rng.randint(1, 4096), rng.randint(1, 200000)))
            at += os.write(fd, data[at:at + n])
            if rng.random() < 0.02:
                time.sleep(0.002)
    except BrokenPipeError:  # the reader stopped early (an error): released, not blocked
        pass
    finally:
        os.close(fd)


@contextlib.contextmanager
def fifo_of(data, tmp, name="in", seed=1):
    """a FIFO that a thread fills with `data`; on exit the writer is released even if nothing opened the read end"""
    path = os.path.join(str(tmp), name + ".fifo")
    os.mkfifo(path)
    t = threading.Thread(target=lambda: _write_pieces(os.open(path, os.O_WRONLY), data, seed), daemon=True)
    t.start()
    try:
        yield path
    finally:
        if t.is_alive():  # no reader yet, or one that did not read to the end: a reader of our own lets open() return, then the write fails
            with contextlib.suppress(OSError):
                os.close(os.open(path, os.O_RDONLY | os.O_NONBLOCK))
        t.join(60)
        assert not t.is_alive(), "the writer of %s is still blocked" % path
        os.remove(path)


def input_of(worlds, tmp_root, name, kind):
    """(world whose oracle run the input means, input path)"""
    w = world(worlds, name)
    if kind == "bam":
        return w, w.prefix + ".bam"  # synth: stored BGZF
    if kind.startswith("transcoded"):
        t = transcoded_world(worlds, tmp_root, 7 if kind == "transcoded" else 8, kind == "transcoded", **({} if name == "small" else {"name": name}))[1]
        return t, t.prefix + ".bam"
    return w, sam_of(w, kind)


FRONT_END = [  # world, input, threads, test hooks
    ("small", "bam", 2, {}), ("small", "bam", 1, {"ARB_CHUNK_BYTES": "1"}), ("small", "transcoded", 3, {"ARB_CHUNK_BYTES": "300"}),
    ("small", "transcoded_noeof", 2, {}), ("small", "plain", 2, {"ARB_CHUNK_BYTES": "300"}), ("small", "longheader_crlf_bgzf", 2, {"ARB_CHUNK_BYTES": "1"}),
    ("small", "bam", 2, {"ARB_KEY_HASH_BITS": "4"}), ("l151", "bam", 4, {"ARB_CHUNK_BYTES": "70000"}), ("l151", "crlf_bgzf_nolf", 3, {}),
    ("zchr", "plain", 2, {"ARB_KEY_HASH_BITS": "4"}), ("zchr", "bam", 2, {"ARB_CHUNK_BYTES": "70000"}),
]


def _id(x):
    return x if isinstance(x, str) else str(x) if isinstance(x, int) else "-".join("%s=%s" % kv for kv in x.items()) or "default"


@pytest.fixture(scope="module")
def corpus_root(tmp_path_factory):
    return tmp_path_factory.mktemp("pipe_corpus")


@pytest.mark.parametrize("name,kind,threads,hooks", FRONT_END, ids=_id)
def test_front_end_stream_hostsim(worlds, corpus_root, hostsim_lib, monkeypatch, tmp_path, name, kind, threads, hooks):
    for k, v in hooks.items():
        monkeypatch.setenv(k, v)
    w, path = input_of(worlds, corpus_root, name, kind)
    with fifo_of(open(path, "rb").read(), tmp_path) as fifo:
        check_front_end_sam(w, fifo, hostsim_lib, threads)


@pytest.mark.parametrize("name,kind", [("small", "transcoded"), ("l151", "plain")])
def test_outputs_stream_hostsim(worlds, corpus_root, hostsim_lib, tmp_path, name, kind):
    w, path = input_of(worlds, corpus_root, name, kind)
    with fifo_of(open(path, "rb").read(), tmp_path, seed=3) as fifo:
        fus, disc = run_outputs(fifo, w, hostsim_lib, str(tmp_path))
    assert fus == open(os.path.join(w.outdir, "fusions.tsv"), "rb").read()
    assert disc == open(os.path.join(w.outdir, "fusions.discarded.tsv"), "rb").read()


def test_store_grows_without_a_size_hostsim(worlds, hostsim_lib, monkeypatch, tmp_path):
    """without a total the store starts from the first chunk and grows by a quarter: many times with small chunks; the outputs do not change"""
    monkeypatch.setenv("ARB_CHUNK_BYTES", "70000")
    w = world(worlds, "cfg5")
    out, disc = str(tmp_path / "fusions.tsv"), str(tmp_path / "fusions.discarded.tsv")
    with fifo_of(open(w.prefix + ".bam", "rb").read(), tmp_path) as fifo:
        p = L.Pipeline(fifo, w.prefix + ".gtf", w.prefix + ".fa", threads=3, lib_path=hostsim_lib, output=out, discarded=disc)
        p.run()  # every step once (run_all would read the input again)
        tm = p.context().timings()
        assert tm.rec_store_grows >= 5 and tm.rec_store_bytes > 0, (tm.rec_store_grows, tm.rec_store_bytes)
        p.events(len(L.EV_NAMES) - 1); p.write_output(); p.close()
    assert open(out, "rb").read() == open(os.path.join(w.outdir, "fusions.tsv"), "rb").read()
    assert open(disc, "rb").read() == open(os.path.join(w.outdir, "fusions.discarded.tsv"), "rb").read()


# ---- the command line
@pytest.fixture(scope="module")
def cli():
    return _build.build_cli_hostsim()


def run_cli(cli, x, w, out, args=(), **kw):
    os.makedirs(out, exist_ok=True)
    return subprocess.run([cli, "-x", x, "-g", w.prefix + ".gtf", "-a", w.prefix + ".fa", "-o", os.path.join(out, "fusions.tsv"), "-O", os.path.join(out, "fusions.discarded.tsv"),
                           "-@", "3"] + list(args), capture_output=True, timeout=900, **kw)


def same_run(a, b, out_a, out_b):
    """identical exit code, ERROR and WARNING lines, progress lines (paths aside) and, on success, output files"""
    ea, eb = a.stderr.decode("latin-1"), b.stderr.decode("latin-1")
    assert a.returncode == b.returncode, (ea[-2000:], eb[-2000:])
    errors = lambda t: [l for l in t.splitlines() if l.startswith("ERROR:")]
    assert errors(ea) == errors(eb)
    assert warnings_of(ea) == warnings_of(eb)
    assert progress_of(a.stdout.decode("latin-1")) == progress_of(b.stdout.decode("latin-1"))
    if a.returncode == 0:
        for f in ("fusions.tsv", "fusions.discarded.tsv"):
            assert open(os.path.join(out_a, f), "rb").read() == open(os.path.join(out_b, f), "rb").read(), f


@pytest.mark.parametrize("name,kind", [("small", "bam"), ("small", "transcoded_noeof"), ("small", "crlf"), ("small", "longheader_bgzf")])
def test_cli_stdin_hostsim(worlds, corpus_root, cli, tmp_path, name, kind):
    w, path = input_of(worlds, corpus_root, name, kind)
    data = open(path, "rb").read()
    want = run_cli(cli, path, w, str(tmp_path / "file"), ("-f", "blacklist"))
    assert want.returncode == 0, want.stderr[-2000:]
    piped = run_cli(cli, "/dev/stdin", w, str(tmp_path / "pipe"), ("-f", "blacklist"), input=data)
    same_run(piped, want, str(tmp_path / "pipe"), str(tmp_path / "file"))
    with open(path, "rb") as f:  # stdin redirected from the file: a regular file, mapped as before
        redirected = run_cli(cli, "/dev/stdin", w, str(tmp_path / "redirect"), ("-f", "blacklist"), stdin=f)
    same_run(redirected, want, str(tmp_path / "redirect"), str(tmp_path / "file"))
    for f in ("fusions.tsv", "fusions.discarded.tsv"):
        assert open(os.path.join(str(tmp_path / "pipe"), f), "rb").read() == open(os.path.join(w.outdir, f), "rb").read(), f


def test_cli_stdin_with_every_input_file_hostsim(worlds, cli, hostsim_lib, tmp_path_factory, tmp_path):
    w = world(worlds, "small")
    root = str(tmp_path_factory.mktemp("files"))
    args = ("-b", blacklist_file(w, hostsim_lib, root), "-k", rules_file(w, hostsim_lib, root, False), "-t", rules_file(w, hostsim_lib, root, True),
            "-p", domains_file(w, hostsim_lib, root), "-d", sv_file(w, hostsim_lib, root))
    want = run_cli(cli, w.prefix + ".bam", w, str(tmp_path / "file"), args)
    assert want.returncode == 0, want.stderr[-2000:]
    piped = run_cli(cli, "/dev/stdin", w, str(tmp_path / "pipe"), args, input=open(w.prefix + ".bam", "rb").read())
    same_run(piped, want, str(tmp_path / "pipe"), str(tmp_path / "file"))


@pytest.mark.parametrize("c_from,x_from", [("fifo", "file"), ("fifo", "fifo"), ("file", "stdin")])
def test_chimeric_file_from_a_pipe_hostsim(worlds, cli, tmp_path, c_from, x_from):
    w, c = pair(worlds, "small", ("both",), "bgzf")
    want = subprocess.run([cli, "-c", c, "-x", w.prefix + ".bam", "-g", w.prefix + ".gtf", "-a", w.prefix + ".fa", "-o", str(tmp_path / "f.tsv"), "-f", "blacklist"],
                          capture_output=True, timeout=900)
    assert want.returncode == 0
    with contextlib.ExitStack() as stack:
        cp = stack.enter_context(fifo_of(open(c, "rb").read(), tmp_path, "c", 5)) if c_from == "fifo" else c
        xp = w.prefix + ".bam"; stdin = None
        if x_from == "fifo":
            xp = stack.enter_context(fifo_of(open(xp, "rb").read(), tmp_path, "x", 6))
        elif x_from == "stdin":
            xp, stdin = "/dev/stdin", open(xp, "rb").read()
        r = subprocess.run([cli, "-c", cp, "-x", xp, "-g", w.prefix + ".gtf", "-a", w.prefix + ".fa", "-o", str(tmp_path / "fusions.tsv"), "-O", str(tmp_path / "fusions.discarded.tsv"),
                            "-f", "blacklist", "-@", "3"], capture_output=True, timeout=900, input=stdin)
    assert r.returncode == 0, r.stderr[-2000:]
    for f in ("fusions.tsv", "fusions.discarded.tsv"):
        assert open(str(tmp_path / f), "rb").read() == open(os.path.join(w.outdir, f), "rb").read(), f
    err, out = r.stderr.decode("latin-1"), r.stdout.decode("latin-1")
    assert warnings_of(err) == warnings_of(open(os.path.join(w.outdir, "stderr.txt"), encoding="latin-1").read())
    assert totals(out) == totals(want.stdout.decode("latin-1")) and len(totals(out)) == 2


# ---- errors: a stream and the same bytes in a file stop with the same ERROR and exit code, and the writer is released
def _blocks(raw):
    """(start, size) of every BGZF member"""
    out, at = [], 0
    while at < len(raw):
        size = int.from_bytes(raw[at + 16:at + 18], "little") + 1
        out.append((at, size)); at += size
    return out


def _error_cases(w):
    import gzip, struct
    bam = open(w.prefix + ".bam", "rb").read()
    blocks = _blocks(bam)
    text, refs, bodies = bamtools.read_bam(w.prefix + ".bam")
    mid = blocks[len(blocks) // 2]
    cases = {
        "empty": b"",
        "gzip": gzip.compress(open(sam_of(w), "rb").read()[:100000]),
        "cram": b"CRAM\x03\x00" + bytes(range(256)) * 4,
        "garbage": bytes(range(256)) * 16,
        "cut_in_block_header": bam[:mid[0] + 9],
        "cut_in_payload": bam[:mid[0] + mid[1] // 2],
        "cut_in_record": bam[:mid[0]] + bamtools.EOF_BLOCK,  # whole blocks, the last record unfinished
        "one_byte": bam[:1],
    }
    cases["bad_cigar"] = damaged_bam(w.prefix + ".bam", os.path.dirname(w.prefix), "cigar", 1 / 3)
    cases["beyond_contig"] = damaged_bam(w.prefix + ".bam", os.path.dirname(w.prefix), "beyond", 1 / 3)
    cases["framing_after_record_error"] = damaged_bam(w.prefix + ".bam", os.path.dirname(w.prefix), "cigar", 1 / 10, framing_late=True)
    return cases


def damaged_bam(src, d, kind, at, framing_late=False):
    """the BAM `src` re-framed with one record damaged (kind "cigar": its CIGAR does not fit; "beyond": it ends past its contig) at fraction `at` of the
    records; framing_late: the BC subfield of the third block from the end damaged as well, so that the record error comes first in the file"""
    import struct
    text, refs, bodies = bamtools.read_bam(src)
    i = int(len(bodies) * at)
    r = bamtools.split_record(bodies[i])
    if kind == "cigar":
        r["cigar"] = struct.pack("<I", (r["l_seq"] + 5) << 4)
    else:
        r["pos"] = refs[r["tid"]][1] - 3
    new = list(bodies); new[i] = bamtools.join_record(r)
    path = os.path.join(d, "err_%s_%d.bam" % (kind, i))
    bamtools.write_bam(path, text, refs, new, random.Random(4))
    data = bytearray(open(path, "rb").read())
    if framing_late:
        data[_blocks(bytes(data))[-3][0] + 12] ^= 0xFF  # the 'B' of the BC subfield
    return bytes(data)


def test_errors_stream_vs_file_hostsim(worlds, cli, tmp_path):
    w = world(worlds, "small")
    for name, data in _error_cases(w).items():
        path = str(tmp_path / (name + ".bam")); open(path, "wb").write(data)
        want = run_cli(cli, path, w, str(tmp_path / name / "file"), ("-f", "blacklist"))
        assert want.returncode != 0, name
        piped = run_cli(cli, "/dev/stdin", w, str(tmp_path / name / "pipe"), ("-f", "blacklist"), input=data)
        same_run(piped, want, "", "")
        with fifo_of(data, tmp_path, name) as fifo:
            fed = run_cli(cli, fifo, w, str(tmp_path / name / "fifo"), ("-f", "blacklist"))
        same_run(fed, want, "", "")


@pytest.mark.parametrize("chunk", ["300", "70000"])
def test_framing_error_after_record_error_small_chunks_hostsim(worlds, cli, monkeypatch, tmp_path, chunk):
    """with small chunks the record error's chunk is scanned long before the damaged block is read: the framing error must still be the only outcome"""
    monkeypatch.setenv("ARB_CHUNK_BYTES", chunk)
    w = world(worlds, "small")
    data = damaged_bam(w.prefix + ".bam", str(tmp_path), "cigar", 1 / 10, framing_late=True)
    path = str(tmp_path / "x.bam"); open(path, "wb").write(data)
    want = run_cli(cli, path, w, str(tmp_path / "file"), ("-f", "blacklist"))
    assert want.returncode == 1 and want.stderr.decode().splitlines()[-1] == "ERROR: failed to load alignments"
    same_run(run_cli(cli, "/dev/stdin", w, str(tmp_path / "pipe"), ("-f", "blacklist"), input=data), want, "", "")
    with fifo_of(data, tmp_path) as fifo:
        same_run(run_cli(cli, fifo, w, str(tmp_path / "fifo"), ("-f", "blacklist")), want, "", "")


@pytest.mark.parametrize("damaged", ["x", "c_and_x"])
def test_framing_error_after_record_error_with_chimeric_file_hostsim(worlds, cli, monkeypatch, tmp_path, damaged):
    """-c with a piped -x: a record error early (in -x, or in a piped -c) and a damaged block late in -x. As for the files, only the framing error is
    reported: no progress line, no warning of the -c file's call"""
    monkeypatch.setenv("ARB_CHUNK_BYTES", "70000")
    w, c = pair(worlds, "small", ("both",), "bam")
    x_data = damaged_bam(w.prefix + ".bam", str(tmp_path), "cigar", 1 / 10, framing_late=True)
    c_data = damaged_bam(c, str(tmp_path), "beyond", 1 / 2) if damaged == "c_and_x" else open(c, "rb").read()
    x_path, c_path = str(tmp_path / "x.bam"), str(tmp_path / "c.bam")
    open(x_path, "wb").write(x_data); open(c_path, "wb").write(c_data)
    want = run_cli(cli, x_path, w, str(tmp_path / "file"), ("-f", "blacklist", "-c", c_path))
    assert want.returncode == 1 and want.stderr.decode().splitlines()[-1] == "ERROR: failed to load alignments"
    assert "Reading chimeric alignments" not in want.stdout.decode()
    with fifo_of(c_data, tmp_path, "c", 5) as c_fifo:
        piped = run_cli(cli, "/dev/stdin", w, str(tmp_path / "pipe"), ("-f", "blacklist", "-c", c_fifo if damaged == "c_and_x" else c_path), input=x_data)
    same_run(piped, want, "", "")
    assert "Reading chimeric alignments" not in piped.stdout.decode() and "WARNING" not in piped.stderr.decode()


def test_directory_is_refused_hostsim(worlds, cli, tmp_path):
    w = world(worlds, "small")
    r = run_cli(cli, str(tmp_path), w, str(tmp_path / "out"), ("-f", "blacklist"))
    assert r.returncode == 1 and b"ERROR: failed to open SAM file" in r.stderr


# ---- the device's assembly of a stream chunk (arb_records_bgzf_stage) against a plain assembly
class Block(C.Structure):
    _fields_ = [("src", C.c_uint64), ("bytes", C.c_uint64), ("dst", C.c_uint64)]


def _stage_case(rng, n_blocks, sizes):
    """raw bytes (stored-like and 'inflated' payloads at unaligned offsets, gaps between them) and the block table; the payloads in order"""
    raw, table, payloads, dst = bytearray(rng.randbytes(rng.randint(0, 7))), [], [], 0
    for _ in range(n_blocks):
        n = rng.choice(sizes)
        raw += rng.randbytes(rng.randint(0, 30))  # a header, or nothing
        data = bytes(b if b != 10 else 11 for b in rng.randbytes(n))  # no LF: the text chunk below keeps it all as a carry
        table.append((len(raw), n, dst)); raw += data; payloads.append(data); dst += n
    if rng.random() < 0.5:  # some payloads live behind the raw blocks, as the host's inflated copies do
        order = list(range(len(table))); rng.shuffle(order)
        for k in order[:len(order) // 2]:
            s, n, d = table[k]; table[k] = (len(raw), n, d); raw += payloads[k]
    return bytes(raw), table, b"".join(payloads)


def check_stage(lib_path):
    ctx = L.Context(lib_path=lib_path)
    lib = ctx.lib
    lib.arb_records_bgzf_stage.argtypes = [C.c_void_p, C.c_char_p, C.c_uint64, C.POINTER(Block), C.c_uint32]
    lib.arb_selftest_staged_chunk.argtypes = [C.c_void_p, C.c_char_p, C.c_uint64]
    lib.arb_records_text_chunk.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_int, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    lib.arb_records_begin.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_int, C.c_uint64]
    rng = random.Random(11)
    cases = [(1, [1]), (3, [0, 1, 2, 3]), (40, [0, 1, 5, 16, 17, 31, 100]), (6, [65536, 1, 0, 4095]), (300, list(range(0, 70))), (2, [65536]), (0, [1])]
    for n_blocks, sizes in cases:
        ctx._check(lib.arb_records_begin(ctx.h, None, 0, None, None, None, 0, 0, 0, 0))
        carry = b""
        for round_ in range(3):
            raw, table, want = _stage_case(rng, n_blocks, sizes)
            blocks = (Block * max(1, len(table)))(*[Block(*t) for t in table])
            ctx._check(lib.arb_records_bgzf_stage(ctx.h, raw, len(raw), blocks, len(table)))
            got = C.create_string_buffer(len(carry) + len(want))
            ctx._check(lib.arb_selftest_staged_chunk(ctx.h, got, len(carry) + len(want)))
            assert got.raw == carry + want, (n_blocks, sizes, round_)
            # the text chunk finds no LF: everything behind `first` is carried into the next stage
            first = rng.randint(0, len(want)) if want else 0
            n, cy, err = C.c_uint64(), C.c_uint64(), C.c_uint64()
            ctx._check(lib.arb_records_text_chunk(ctx.h, None, len(want), first, 0, 0, C.byref(n), C.byref(cy), C.byref(err)))
            carry = (carry + want)[first if not carry else 0:]
            assert cy.value == len(carry)
    assert ctx.timings().rec_unwrap_ms >= 0
    ctx.close()


def test_stage_assembly_hostsim(hostsim_lib):
    check_stage(hostsim_lib)


# ---- one sample on two ranks, rank 0 reading a FIFO
WORKER = r"""
import os, sys
sys.path.insert(0, {root!r})
import torch.distributed as dist
from arriba_b200 import lib as L, sharded
rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"])
dist.init_process_group("gloo")
out = os.path.join({outdir!r}, "rank%d" % rank); os.makedirs(out, exist_ok=True)
p = L.Pipeline({fifo!r} if rank == 0 else "/nonexistent.bam", {prefix!r} + ".gtf", {prefix!r} + ".fa", threads=2, lib_path={lib!r},
               output=os.path.join(out, "fusions.tsv"), discarded=os.path.join(out, "fusions.discarded.tsv"))
sharded.run_sharded(p, rank, world)
p.close()
dist.destroy_process_group()
"""


def test_sharded_two_ranks_hostsim(worlds, hostsim_lib, tmp_path):
    w = world(worlds, "small")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with fifo_of(open(w.prefix + ".bam", "rb").read(), tmp_path) as fifo:
        script = str(tmp_path / "worker.py")
        open(script, "w").write(WORKER.format(root=root, outdir=str(tmp_path), fifo=fifo, prefix=w.prefix, lib=hostsim_lib))
        env = dict(os.environ, PYTHONPATH=root + os.pathsep + os.path.join(root, "tests"))
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port", str(29500 + os.getpid() % 200), script]
        r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    for f in ("fusions.tsv", "fusions.discarded.tsv"):
        assert open(os.path.join(tmp_path, "rank0", f), "rb").read() == open(os.path.join(w.outdir, f), "rb").read(), f


# ---- on the H100
GPU_FRONT_END = [("small", "bam", {}), ("small", "transcoded", {"ARB_CHUNK_BYTES": "1"}), ("small", "bgzf", {"ARB_CHUNK_BYTES": "70000"}),
                 ("l151", "bam", {"ARB_CHUNK_BYTES": "70000"}), ("l151", "transcoded", {}), ("l151", "crlf_bgzf", {"ARB_CHUNK_BYTES": "1"})]


@pytest.mark.gpu
@pytest.mark.parametrize("name,kind,hooks", GPU_FRONT_END, ids=_id)
def test_front_end_stream_cuda(worlds, corpus_root, cuda_lib, monkeypatch, tmp_path, name, kind, hooks):
    for k, v in hooks.items():
        monkeypatch.setenv(k, v)
    w, path = input_of(worlds, corpus_root, name, kind)
    with fifo_of(open(path, "rb").read(), tmp_path) as fifo:
        check_front_end_sam(w, fifo, cuda_lib, 8)


@pytest.mark.gpu
def test_outputs_stream_cuda(worlds, cuda_lib, tmp_path):
    w = world(worlds, "l151")
    with fifo_of(open(w.prefix + ".bam", "rb").read(), tmp_path) as fifo:
        p = L.Pipeline(fifo, w.prefix + ".gtf", w.prefix + ".fa", threads=8, lib_path=cuda_lib, output=str(tmp_path / "fusions.tsv"), discarded=str(tmp_path / "fusions.discarded.tsv"))
        p.run()
        tm = p.context().timings()
        inflated = sum(len(m) for m in bamtools.bgzf_members(open(w.prefix + ".bam", "rb").read()))
        assert tm.rec_unwrap_ms > 0 and abs(tm.rec_h2d_bytes - inflated) <= 0.001 * inflated, (tm.rec_h2d_bytes, inflated)
        p.events(len(L.EV_NAMES) - 1); p.write_output(); p.close()
    for f in ("fusions.tsv", "fusions.discarded.tsv"):
        assert open(str(tmp_path / f), "rb").read() == open(os.path.join(w.outdir, f), "rb").read(), f


@pytest.fixture(scope="module")
def cuda_cli():
    return _build.build_cli()


@pytest.mark.gpu
def test_cli_stdin_cuda(worlds, cuda_cli, tmp_path):
    w = world(worlds, "small")
    want = run_cli(cuda_cli, w.prefix + ".bam", w, str(tmp_path / "file"), ("-f", "blacklist"))
    assert want.returncode == 0, want.stderr[-2000:]
    piped = run_cli(cuda_cli, "/dev/stdin", w, str(tmp_path / "pipe"), ("-f", "blacklist"), input=open(w.prefix + ".bam", "rb").read())
    same_run(piped, want, str(tmp_path / "pipe"), str(tmp_path / "file"))


@pytest.mark.gpu
def test_errors_stream_vs_file_cuda(worlds, cuda_cli, tmp_path):
    w = world(worlds, "small")
    cases = _error_cases(w)
    for name in ("empty", "cut_in_payload", "cut_in_record", "framing_after_record_error", "bad_cigar"):
        path = str(tmp_path / (name + ".bam")); open(path, "wb").write(cases[name])
        want = run_cli(cuda_cli, path, w, str(tmp_path / name / "file"), ("-f", "blacklist"))
        piped = run_cli(cuda_cli, "/dev/stdin", w, str(tmp_path / name / "pipe"), ("-f", "blacklist"), input=cases[name])
        same_run(piped, want, "", "")


@pytest.mark.gpu
def test_stage_assembly_cuda(cuda_lib):
    check_stage(cuda_lib)
