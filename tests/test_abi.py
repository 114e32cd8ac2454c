"""The C-ABI shared library must load and export every symbol include/arriba_b200.h declares (no compute calls: runs without a GPU)."""
import ctypes, os, re
import pytest
from arriba_b200 import _build, lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "arriba_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(arb_[a-z_0-9]+)\s*\(", text)))


def test_header_declares_the_expected_surface():
    syms = declared_symbols()
    for must in ("arb_ctx_create", "arb_push_chunk", "arb_run_read_filters", "arb_find_fusions", "arb_merge_adjacent", "arb_estimate_evalues",
                 "arb_build_kmer_index", "arb_homolog_pairs", "arb_filter_mismappers", "arb_pipeline_run", "arb_pipeline_write_output"):
        assert must in syms


def test_product_library_exports_every_declared_symbol():
    path = _build.build_product()  # cross-compiles for sm_90a; works without a GPU
    lib = ctypes.CDLL(path)
    missing = [s for s in declared_symbols() if not hasattr(lib, s)]
    assert not missing, missing
    lib.arb_backend.restype = ctypes.c_char_p
    assert lib.arb_backend() == b"cuda-sm_90a"


def test_struct_layouts_match_the_binding(hostsim_lib):
    L.load(hostsim_lib)  # raises on mismatch


def test_product_refuses_to_run_without_a_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    lib = L.load(_build.build_product())
    h = ctypes.c_void_p()
    assert lib.arb_ctx_create(ctypes.byref(h), 0) != 0
    assert b"no CPU fallback" in lib.arb_last_error(None)


def test_cli_reports_usage_errors_like_the_reference(tmp_path):
    import subprocess
    cli = _build.build_cli()
    r = subprocess.run([cli, "-x", "/nonexistent.bam"], capture_output=True, text=True)
    assert r.returncode == 1 and "ERROR: file not found/readable: /nonexistent.bam" in r.stderr
    r = subprocess.run([cli, "-g", __file__, "-a", __file__, "-o", str(tmp_path / "o.tsv")], capture_output=True, text=True)
    assert r.returncode == 1 and "ERROR: missing mandatory option -x" in r.stderr
    r = subprocess.run([cli, "-x", __file__, "-g", __file__, "-a", __file__, "-o", str(tmp_path / "o.tsv")], capture_output=True, text=True)
    assert r.returncode == 1 and "filter 'blacklist' enabled, but missing option -b" in r.stderr
