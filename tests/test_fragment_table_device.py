"""The fragment table that the device builds from the ingest's worker pools (csrc/fragtable.cu): slot normalisation, name order, columns and multimapper
flags against the oracle's ingest stage, on files whose read names are long and share most of their bytes, as real Illumina names do (the name sort then
needs several words of every name), with few records over many workers, and in small chunks."""
import os
import random
import pytest
import bamtools
import worldutil
from test_ingest import check_front_end

PREFIX = b"A00123:456:HXXXXXXXX:1:1101:"   # 28 bytes shared by every name, then the synthetic name: 30-byte common prefixes and names that begin others


def renamed_world(worlds, root, keep_records=None):
    base = worlds.get("l151", read_length=151, seed=7, extra=("--shuffle", "--varnames"))
    d = os.path.join(str(root), "renamed_%s" % keep_records); os.makedirs(d, exist_ok=True)
    prefix = os.path.join(d, "w")
    for ext in (".fa", ".gtf"):
        if not os.path.exists(prefix + ext):
            os.symlink(base.prefix + ext, prefix + ext)
    text, refs, bodies = bamtools.read_bam(base.prefix + ".bam")
    if keep_records is not None:
        bodies = bodies[:keep_records]
    out = []
    for b in bodies:
        r = bamtools.split_record(b)
        r["qname"] = PREFIX + b"00" + r["qname"]
        out.append(bamtools.join_record(r))
    bamtools.write_bam(prefix + ".bam", text, refs, out, random.Random(3))
    worldutil.run_oracle(prefix, os.path.join(d, "oracle"))
    return worldutil.World(prefix, os.path.join(d, "oracle"))


@pytest.fixture(scope="module")
def renamed(worlds, tmp_path_factory):
    root = tmp_path_factory.mktemp("fragment_table")
    return {"all": renamed_world(worlds, root), "few": renamed_world(worlds, root, keep_records=40)}


def test_names_share_long_prefixes(renamed):
    names = bytes(renamed["all"].stage("ingest")["names"])
    assert names.count(PREFIX + b"00") > 1000


@pytest.mark.parametrize("which,threads,chunk_bytes", [("all", 5, None), ("all", 3, "70000"), ("few", 64, None)])
def test_fragment_table_hostsim(renamed, hostsim_lib, monkeypatch, which, threads, chunk_bytes):
    if chunk_bytes:
        monkeypatch.setenv("ARB_CHUNK_BYTES", chunk_bytes)
    check_front_end(renamed[which], hostsim_lib, threads=threads)


@pytest.mark.gpu
@pytest.mark.parametrize("which,threads", [("all", 8), ("few", 64)])
def test_fragment_table_cuda(renamed, cuda_lib, which, threads):
    check_front_end(renamed[which], cuda_lib, threads=threads)
