"""CPU-only: include/cvb200_filter.h (akaze::image on the device) -- libcvb200_filter.so exports exactly the symbols the header declares,
libcvb200.so's exports are unchanged, a C program calls every one of them, the generated Rust bindings match the header, gaussian_kernel
(host arithmetic) equals the oracle bit for bit, and without a CUDA device every filter fails cleanly (no CPU fallback)."""
import importlib.util
import os
import re
import subprocess

import numpy as np
import pytest

import cv_b200
from cv_b200._lib import (ABI_SYMBOLS, CVB_EINVAL, FILTER_ABI_SYMBOLS, IMAGE_ABI_SYMBOLS, OPT_ABI_SYMBOLS, PINHOLE_ABI_SYMBOLS,
                          SFM_ABI_SYMBOLS, TRI_ABI_SYMBOLS, filter_lib_path)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "cvb200_filter.h")


def _ensure_built():
    if not (os.path.exists(cv_b200.lib_path()) and os.path.exists(filter_lib_path())):
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
    assert _declared() == set(FILTER_ABI_SYMBOLS), _declared() ^ set(FILTER_ABI_SYMBOLS)
    others = (set(ABI_SYMBOLS) | set(SFM_ABI_SYMBOLS) | set(TRI_ABI_SYMBOLS) | set(OPT_ABI_SYMBOLS) | set(PINHOLE_ABI_SYMBOLS) |
              set(IMAGE_ABI_SYMBOLS))
    assert not set(FILTER_ABI_SYMBOLS) & others
    assert _exported(filter_lib_path()) == set(FILTER_ABI_SYMBOLS)
    assert _exported(cv_b200.lib_path()) == set(ABI_SYMBOLS) | set(SFM_ABI_SYMBOLS) | set(TRI_ABI_SYMBOLS)   # unchanged
    L = cv_b200._lib.load_filter_library()
    for s in FILTER_ABI_SYMBOLS:
        assert hasattr(L, s), s


def test_tap_cap_matches_the_python_constant():
    from cv_b200.filter import MAX_TAPS
    assert int(re.search(r"#define\s+CVB_FILTER_MAX_TAPS\s+(\d+)", open(HEADER).read()).group(1)) == MAX_TAPS == 1023


def _build_smoke():
    out = os.path.join(ROOT, "tests", "csrc", "_build")
    os.makedirs(out, exist_ok=True)
    exe = os.path.join(out, "abi_smoke_filter")
    libdir = os.path.join(ROOT, "cv_b200")
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", os.path.join(ROOT, "tests", "csrc", "abi_smoke_filter.c"),
                           "-I" + os.path.join(ROOT, "include"), "-L" + libdir, "-lcvb200_filter", "-lcvb200", "-lm",
                           "-Wl,-rpath," + libdir, "-o", exe])
    return exe


def test_c_program_compiles_against_filter_header_and_calls_every_entry_point():
    _ensure_built()
    exe = _build_smoke()
    src = open(os.path.join(ROOT, "tests", "csrc", "abi_smoke_filter.c")).read()
    for sym in _declared():
        assert re.search(r"\b" + sym + r"\s*\(", src), f"{sym} is not called by abi_smoke_filter.c"
    r = subprocess.run([exe, "0"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.gpu
def test_c_program_filter_gpu_workflow():
    _ensure_built()
    r = subprocess.run([_build_smoke(), "1"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "GPU workflow ok" in r.stdout, r.stdout + r.stderr


def test_rust_filter_bindings_are_generated_from_the_current_header():
    """cv-b200-sys/src/filter.rs is what scripts/gen_rust_sys.py produces from include/cvb200_filter.h, and the shim's filter.rs what it
    assembles from INTEGRATION.md section 2h; every symbol is declared once with the header's arity; the shim calls only declared externs
    and keeps the reference's function names."""
    spec = importlib.util.spec_from_file_location("gen_rust_sys", os.path.join(ROOT, "scripts", "gen_rust_sys.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    header = open(HEADER).read()
    text, _ = gen.generate_filter(header)
    assert open(gen.FILTER_OUT).read() == text, "stale: python scripts/gen_rust_sys.py"
    assert open(gen.FILTER_SHIM_OUT).read() == gen.generate_shim_filter(), "stale: python scripts/gen_rust_sys.py"
    assert open(gen.SHIM_OUT).read() == gen.generate_shim(), "stale: python scripts/gen_rust_sys.py"
    assert "pub mod filter;" in open(gen.OUT).read() and "pub mod filter;" in open(gen.SHIM_OUT).read()
    assert '#[link(name = "cvb200_filter")]' in text and "pub const CVB_FILTER_MAX_TAPS: u32 = 1023;" in text
    declared = re.findall(r"pub fn (cvb_\w+)\((.*?)\)(?: -> [^;]+)?;", text)
    assert sorted(n for n, _ in declared) == sorted(FILTER_ABI_SYMBOLS)
    plain = gen.strip_comments(header)
    for name, params in declared:
        cargs = re.search(r"\b" + name + r"\s*\(([^;{]*?)\)\s*;", plain, flags=re.S).group(1)
        assert cargs.count(",") == params.count(","), name
    shim = open(gen.FILTER_SHIM_OUT).read()
    called = set(re.findall(r"\b(cvb_[a-z0-9_]+)\s*\(", shim))
    assert called == {"cvb_gaussian_kernel", "cvb_horizontal_filter", "cvb_vertical_filter", "cvb_separable_filter", "cvb_gaussian_blur",
                      "cvb_half_size"}
    for f in ("pub fn gaussian_kernel(r: f32, kernel_size: usize) -> Vec<f32>",
              "pub fn horizontal_filter(ctx: &Ctx, image: &GrayImageBuffer, kernel: &[f32]) -> GrayImageBuffer",
              "pub fn vertical_filter(ctx: &Ctx, image: &GrayImageBuffer, kernel: &[f32]) -> GrayImageBuffer",
              "pub fn separable_filter(ctx: &Ctx, image: &GrayImageBuffer, h_kernel: &[f32], v_kernel: &[f32]) -> GrayImageBuffer",
              "pub fn gaussian_blur(ctx: &Ctx, image: &GrayFloatImage, r: f32) -> GrayFloatImage",
              "pub fn half_size(ctx: &Ctx, image: &GrayFloatImage) -> GrayFloatImage"):
        assert f in shim, f


RADII = [0.5, 1.0, 1.6, 3.0, 10.0, 100.0]
SIZES = [1, 3, 5, 7, 9, 71, 1023]


@pytest.mark.parametrize("r", RADII)
def test_gaussian_kernel_equals_the_oracle_bit_for_bit(r):
    from oracle import pyoracle as O
    for ks in SIZES:
        got = cv_b200.gaussian_kernel(r, ks)
        want = O.gaussian_kernel(r, ks)
        assert got.dtype == np.float32 and got.tobytes() == want.tobytes(), (r, ks)


def test_gaussian_kernel_known_answer_and_sizes():
    """image.rs:395-412; an even size is the reference's assert; sigma 0 gives NaN taps, as in the reference"""
    known = np.array([0.10628852, 0.14032133, 0.16577007, 0.17524014, 0.16577007, 0.14032133, 0.10628852], np.float32)
    assert np.abs(cv_b200.gaussian_kernel(3.0, 7) - known).max() < 1e-4
    for ks in (0, 2, 4, 70):
        with pytest.raises(cv_b200.CvbError) as e:
            cv_b200.gaussian_kernel(1.0, ks)
        assert e.value.code == CVB_EINVAL
    assert np.isnan(cv_b200.gaussian_kernel(0.0, 5)).all()
    assert cv_b200.gaussian_kernel(1.0, 1).tolist() == [1.0]
    assert len(cv_b200.gaussian_kernel(1.0, 2049)) == 2049   # host arithmetic: no cap


def test_wrappers_check_types_and_shapes():
    from cv_b200 import filter as F
    with pytest.raises(TypeError):
        F.horizontal_filter(np.zeros((4, 4), np.float64), [1.0])
    with pytest.raises(TypeError):
        F.half_size(np.zeros((4, 4), np.uint8))
    for bad in (np.zeros(4, np.float32), np.zeros((2, 2, 2, 2), np.float32), np.zeros((0, 4), np.float32)):
        with pytest.raises(ValueError):
            F.gaussian_blur(bad, 1.0)
    with pytest.raises(ValueError):
        F.vertical_filter(np.zeros((4, 4), np.float32), np.ones((3, 1), np.float32))


def test_filters_report_no_device():
    _ensure_built()
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from cv_b200._lib import CVB_ENODEV
    img = np.zeros((2, 16, 16), np.float32)
    k = cv_b200.gaussian_kernel(1.0, 7)
    for call in (lambda: cv_b200.horizontal_filter(img, k), lambda: cv_b200.vertical_filter(img[0], k),
                 lambda: cv_b200.separable_filter(img, k, k), lambda: cv_b200.gaussian_blur(img, 1.6), lambda: cv_b200.half_size(img)):
        with pytest.raises(cv_b200.CvbError) as e:
            call()
        assert e.value.code == CVB_ENODEV
