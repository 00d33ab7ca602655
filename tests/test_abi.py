"""CPU-only: the C-ABI library builds, loads and exports every symbol include/cvb200.h declares;
the product path fails loudly (no CPU fallback) when no CUDA device is present."""
import os
import re

import pytest

import cv_b200
from cv_b200._lib import ABI_SYMBOLS, load_library

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ensure_built():
    if not os.path.exists(cv_b200.lib_path()):
        import __graft_entry__ as g
        g.build()


def test_library_exports_every_header_symbol():
    _ensure_built()
    L = load_library()
    header = open(os.path.join(ROOT, "include", "cvb200.h")).read()
    declared = set(re.findall(r"\b(cvb_[a-z0-9_]+)\s*\(", header))
    assert declared == set(ABI_SYMBOLS), declared ^ set(ABI_SYMBOLS)
    for s in declared:
        assert hasattr(L, s), s
    assert b"sm_90a" in L.cvb_version()


def _build_abi_smoke():
    import subprocess
    out = os.path.join(ROOT, "tests", "csrc", "_build")
    os.makedirs(out, exist_ok=True)
    exe = os.path.join(out, "abi_smoke")
    libdir = os.path.join(ROOT, "cv_b200")
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", os.path.join(ROOT, "tests", "csrc", "abi_smoke.c"),
                           "-I" + os.path.join(ROOT, "include"), "-L" + libdir, "-lcvb200", "-lm", "-Wl,-rpath," + libdir, "-o", exe])
    return exe


def test_c_program_compiles_against_header_and_calls_every_entry_point():
    """tests/csrc/abi_smoke.c includes include/cvb200.h and calls every declared function: a C compiler (-Werror) checks the
    prototypes that a Rust / cgo binding transcribes; without a GPU every call must fail cleanly (no crash, no CPU fallback)."""
    import subprocess
    _ensure_built()
    exe = _build_abi_smoke()
    src = open(os.path.join(ROOT, "tests", "csrc", "abi_smoke.c")).read()
    header = open(os.path.join(ROOT, "include", "cvb200.h")).read()
    for sym in set(re.findall(r"\b(cvb_[a-z0-9_]+)\s*\(", header)):
        assert re.search(r"\b" + sym + r"\s*\(", src), f"{sym} is not called by abi_smoke.c"
    r = subprocess.run([exe, "0"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.gpu
def test_c_program_gpu_workflow():
    import subprocess
    _ensure_built()
    r = subprocess.run([_build_abi_smoke(), "1"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "GPU workflow ok" in r.stdout, r.stdout + r.stderr


def test_struct_layouts_match_header():
    import ctypes as C
    from cv_b200._lib import KP_DTYPE, AkazeCfg
    assert C.sizeof(AkazeCfg) == 80
    assert KP_DTYPE.itemsize == 28
    from cv_b200.geom import ArrsacCfg, Pose, Rng
    from cv_b200.pair import Intrinsics
    assert C.sizeof(Pose) == 96 and C.sizeof(Rng) == 40 and C.sizeof(ArrsacCfg) == 40 and C.sizeof(Intrinsics) == 40


def test_no_cpu_fallback_without_gpu():
    _ensure_built()
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(cv_b200.CvbError):
        cv_b200.Context(0)
    with pytest.raises(cv_b200.CvbError):
        import numpy as np
        cv_b200.Akaze().extract_from_gray_float_image(np.zeros((64, 64), np.float32))


def test_product_never_imports_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "cv_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                src = open(os.path.join(dirpath, f), errors="ignore").read()
                assert "oracle" not in src.lower(), os.path.join(dirpath, f)


def test_rust_bindings_are_generated_from_the_current_header():
    """bindings/rust: the sys crate is what scripts/gen_rust_sys.py produces from include/cvb200.h (and the shim what it assembles from
    INTEGRATION.md); every exported symbol is declared exactly once with the header's parameter count; repr(C) structs keep the
    header's field order.  (No Rust toolchain in the image: this is the drift check the bindings get instead of a compile.)"""
    import importlib.util
    import re
    spec = importlib.util.spec_from_file_location("gen_rust_sys", os.path.join(ROOT, "scripts", "gen_rust_sys.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    header = open(os.path.join(ROOT, "include", "cvb200.h")).read()
    text, protos = gen.generate(header)
    assert open(gen.OUT).read() == text, "stale: python scripts/gen_rust_sys.py"
    assert open(gen.SHIM_OUT).read() == gen.generate_shim(), "stale: python scripts/gen_rust_sys.py"
    from cv_b200._lib import ABI_SYMBOLS
    declared = re.findall(r"pub fn (cvb_\w+)\((.*?)\)(?: -> [^;]+)?;", text)
    assert sorted(n for n, _ in declared) == sorted(ABI_SYMBOLS)
    plain = gen.strip_comments(header)
    for name, params in declared:
        cargs = re.search(r"\b" + name + r"\s*\(([^;{]*?)\)\s*;", plain, flags=re.S).group(1)
        cn = 0 if cargs.strip() in ("", "void") else cargs.count(",") + 1
        rn = 0 if not params.strip() else params.count(",") + 1
        assert cn == rn, (name, cn, rn)
    # struct layout: field names in header order, pointer-free PODs
    for cname, fields in gen.parse(header)[2]:
        body = re.search(r"pub struct " + cname + r" \{(.*?)\n\}", text, flags=re.S).group(1)
        assert [f for f, _ in fields] == re.findall(r"pub (\w+):", body), cname
    # every extern the safe shim calls exists in the sys crate
    shim = open(gen.SHIM_OUT).read()
    called = set(re.findall(r"\b(cvb_[a-z0-9_]+)\s*\(", shim))
    assert called and called <= set(ABI_SYMBOLS), sorted(called - set(ABI_SYMBOLS))
