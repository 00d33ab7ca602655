"""CPU-only: include/cvb200_lsh.h (exact Hamming k-NN over frame hashes) -- libcvb200_lsh.so exports exactly the symbols the header
declares, libcvb200.so's exports are unchanged, a C program calls every one of them, the generated Rust bindings match the header, the
Python wrappers reject wrong shapes and dtypes, and without a CUDA device the search fails cleanly (no CPU fallback)."""
import importlib.util
import os
import re
import subprocess

import numpy as np
import pytest

import cv_b200
from cv_b200._lib import (ABI_SYMBOLS, CVB_ENODEV, FILTER_ABI_SYMBOLS, IMAGE_ABI_SYMBOLS, LSH_ABI_SYMBOLS, OPT_ABI_SYMBOLS,
                          PINHOLE_ABI_SYMBOLS, SFM_ABI_SYMBOLS, TRI_ABI_SYMBOLS, lsh_lib_path)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "cvb200_lsh.h")


def _ensure_built():
    if not (os.path.exists(cv_b200.lib_path()) and os.path.exists(lsh_lib_path())):
        import __graft_entry__ as g
        g.build()


def _declared():
    plain = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return set(re.findall(r"\b(cvb_[a-z0-9_]+)\s*\(", plain))


def _exported(path):
    out = subprocess.run(["nm", "-D", "--defined-only", path], capture_output=True, text=True, check=True).stdout
    return {ln.split()[-1] for ln in out.splitlines() if re.search(r" T cvb_", ln)}


def test_library_exports_exactly_the_header_symbols():
    _ensure_built()
    assert _declared() == set(LSH_ABI_SYMBOLS), _declared() ^ set(LSH_ABI_SYMBOLS)
    others = (set(ABI_SYMBOLS) | set(SFM_ABI_SYMBOLS) | set(TRI_ABI_SYMBOLS) | set(OPT_ABI_SYMBOLS) | set(PINHOLE_ABI_SYMBOLS) |
              set(IMAGE_ABI_SYMBOLS) | set(FILTER_ABI_SYMBOLS))
    assert not set(LSH_ABI_SYMBOLS) & others
    assert _exported(lsh_lib_path()) == set(LSH_ABI_SYMBOLS)
    assert _exported(cv_b200.lib_path()) == set(ABI_SYMBOLS) | set(SFM_ABI_SYMBOLS) | set(TRI_ABI_SYMBOLS)   # unchanged
    L = cv_b200._lib.load_lsh_library()
    for s in LSH_ABI_SYMBOLS:
        assert hasattr(L, s), s


def test_limits_match_the_python_constants():
    from cv_b200.knn import MAX_K, MAX_WORDS
    text = open(HEADER).read()
    assert int(re.search(r"#define\s+CVB_LSH_MAX_WORDS\s+(\d+)", text).group(1)) == MAX_WORDS == 128
    assert int(re.search(r"#define\s+CVB_LSH_MAX_K\s+(\d+)", text).group(1)) == MAX_K == 1024


def _build_smoke():
    out = os.path.join(ROOT, "tests", "csrc", "_build")
    os.makedirs(out, exist_ok=True)
    exe = os.path.join(out, "abi_smoke_lsh")
    libdir = os.path.join(ROOT, "cv_b200")
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", os.path.join(ROOT, "tests", "csrc", "abi_smoke_lsh.c"),
                           "-I" + os.path.join(ROOT, "include"), "-L" + libdir, "-lcvb200_lsh", "-lcvb200", "-Wl,-rpath," + libdir,
                           "-o", exe])
    return exe


def test_c_program_compiles_against_lsh_header_and_calls_every_entry_point():
    _ensure_built()
    exe = _build_smoke()
    src = open(os.path.join(ROOT, "tests", "csrc", "abi_smoke_lsh.c")).read()
    for sym in _declared():
        assert re.search(r"\b" + sym + r"\s*\(", src), f"{sym} is not called by abi_smoke_lsh.c"
    r = subprocess.run([exe, "0"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.gpu
def test_c_program_lsh_gpu_workflow():
    _ensure_built()
    r = subprocess.run([_build_smoke(), "1"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "GPU workflow ok" in r.stdout, r.stdout + r.stderr


def test_rust_lsh_bindings_are_generated_from_the_current_header():
    """cv-b200-sys/src/lsh.rs is what scripts/gen_rust_sys.py produces from include/cvb200_lsh.h, and the shim's lsh.rs what it
    assembles from INTEGRATION.md section 2i; every symbol is declared once with the header's arity; the shim calls only declared externs
    and keeps the reference's method names."""
    spec = importlib.util.spec_from_file_location("gen_rust_sys", os.path.join(ROOT, "scripts", "gen_rust_sys.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    header = open(HEADER).read()
    text, _ = gen.generate_lsh(header)
    assert open(gen.LSH_OUT).read() == text, "stale: python scripts/gen_rust_sys.py"
    assert open(gen.LSH_SHIM_OUT).read() == gen.generate_shim_lsh(), "stale: python scripts/gen_rust_sys.py"
    assert open(gen.SHIM_OUT).read() == gen.generate_shim(), "stale: python scripts/gen_rust_sys.py"
    assert "pub mod lsh;" in open(gen.OUT).read() and "pub mod lsh;" in open(gen.SHIM_OUT).read()
    assert '#[link(name = "cvb200_lsh")]' in text
    assert "pub const CVB_LSH_MAX_WORDS: u32 = 128;" in text and "pub const CVB_LSH_MAX_K: u32 = 1024;" in text
    declared = re.findall(r"pub fn (cvb_\w+)\((.*?)\)(?: -> [^;]+)?;", text)
    assert sorted(n for n, _ in declared) == sorted(LSH_ABI_SYMBOLS)
    plain = gen.strip_comments(header)
    for name, params in declared:
        cargs = re.search(r"\b" + name + r"\s*\(([^;{]*?)\)\s*;", plain, flags=re.S).group(1)
        assert cargs.count(",") == params.count(","), name
    shim = open(gen.LSH_SHIM_OUT).read()
    assert set(re.findall(r"\b(cvb_[a-z0-9_]+)\s*\(", shim)) == {"cvb_hash_knn"}
    for f in ("pub struct CudaFrameIndex<V>", "pub fn insert(&mut self, key: BitArray<512>, value: V)",
              "pub fn knn_values(&self, query: &BitArray<512>, num: usize) -> Vec<(u32, &V)>"):
        assert f in shim, f


def test_wrappers_check_types_and_shapes():
    from cv_b200.knn import hash_knn
    good = np.zeros((2, 16), np.uint8)
    with pytest.raises(TypeError):
        hash_knn(good.astype(np.int8), good, 1)
    with pytest.raises(TypeError):
        hash_knn(good, good.view(np.uint32), 1)
    for bad in (np.zeros(16, np.uint8), np.zeros((2, 2, 16), np.uint8), np.zeros((2, 0), np.uint8), np.zeros((2, 6), np.uint8),
                np.zeros((2, 516), np.uint8)):
        with pytest.raises(ValueError):
            hash_knn(bad, good, 1)
        with pytest.raises(ValueError):
            hash_knn(good, bad, 1)
    with pytest.raises(ValueError):
        hash_knn(good, np.zeros((2, 12), np.uint8), 1)
    with pytest.raises(ValueError):
        cv_b200.FrameHashIndex(words=0)
    with pytest.raises(ValueError):
        cv_b200.FrameHashIndex(words=129)


def test_search_reports_no_device():
    _ensure_built()
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    q = np.zeros((1, 512), np.uint8)
    with pytest.raises(cv_b200.CvbError) as e:
        cv_b200.hash_knn(q, q, 1)
    assert e.value.code == CVB_ENODEV
