"""CPU-only: include/cvb200_sfm.h (the K1 camera and cv-sfm's frame ingestion) -- the library exports every symbol it declares, a C
program calls every one of them, the struct layout matches, the generated Rust bindings match the header, and without a CUDA device
every new entry point fails cleanly (no CPU fallback)."""
import ctypes as C
import importlib.util
import os
import re
import subprocess

import pytest

import cv_b200
from cv_b200._lib import ABI_SYMBOLS, SFM_ABI_SYMBOLS, load_library

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "cvb200_sfm.h")


def _ensure_built():
    if not os.path.exists(cv_b200.lib_path()):
        import __graft_entry__ as g
        g.build()


def _declared():
    plain = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)      # the comments cite the cvb200.h entry points
    return set(re.findall(r"\b(cvb_[a-z0-9_]+)\s*\(", plain))


def test_library_exports_every_sfm_header_symbol():
    _ensure_built()
    L = load_library()
    assert _declared() == set(SFM_ABI_SYMBOLS), _declared() ^ set(SFM_ABI_SYMBOLS)
    assert not set(SFM_ABI_SYMBOLS) & set(ABI_SYMBOLS)
    for s in SFM_ABI_SYMBOLS:
        assert hasattr(L, s), s


def _build_smoke():
    out = os.path.join(ROOT, "tests", "csrc", "_build")
    os.makedirs(out, exist_ok=True)
    exe = os.path.join(out, "abi_smoke_sfm")
    libdir = os.path.join(ROOT, "cv_b200")
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", os.path.join(ROOT, "tests", "csrc", "abi_smoke_sfm.c"),
                           "-I" + os.path.join(ROOT, "include"), "-L" + libdir, "-lcvb200", "-lm", "-Wl,-rpath," + libdir, "-o", exe])
    return exe


def test_c_program_compiles_against_sfm_header_and_calls_every_entry_point():
    _ensure_built()
    exe = _build_smoke()
    src = open(os.path.join(ROOT, "tests", "csrc", "abi_smoke_sfm.c")).read()
    for sym in _declared():
        assert re.search(r"\b" + sym + r"\s*\(", src), f"{sym} is not called by abi_smoke_sfm.c"
    r = subprocess.run([exe, "0"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.gpu
def test_c_program_sfm_gpu_workflow():
    _ensure_built()
    r = subprocess.run([_build_smoke(), "1"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "GPU workflow ok" in r.stdout, r.stdout + r.stderr


def test_intrinsics_k1_layout_matches_header():
    from cv_b200.pair import Intrinsics, IntrinsicsK1
    body = re.search(r"typedef struct \{([^}]*)\} cvb_intrinsics_k1;", open(HEADER).read()).group(1)
    assert re.findall(r"\w+", body.replace("double", "")) == [f for f, _ in IntrinsicsK1._fields_] == ["fx", "fy", "cx", "cy", "skew", "k1"]
    assert C.sizeof(IntrinsicsK1) == 48 and IntrinsicsK1.k1.offset == 40 and C.sizeof(Intrinsics) == 40


def test_rust_sfm_bindings_are_generated_from_the_current_header():
    """bindings/rust: cv-b200-sys/src/sfm.rs is what scripts/gen_rust_sys.py produces from include/cvb200_sfm.h and the shim's sfm.rs what
    it assembles from INTEGRATION.md section 2c; every symbol is declared once with the header's parameter count; the shim calls only
    declared externs."""
    spec = importlib.util.spec_from_file_location("gen_rust_sys", os.path.join(ROOT, "scripts", "gen_rust_sys.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    header = open(HEADER).read()
    text, _ = gen.generate_sfm(header)
    assert open(gen.SFM_OUT).read() == text, "stale: python scripts/gen_rust_sys.py"
    assert open(gen.SFM_SHIM_OUT).read() == gen.generate_shim_sfm(), "stale: python scripts/gen_rust_sys.py"
    assert "pub mod sfm;" in open(gen.OUT).read() and "mod sfm;" in open(gen.SHIM_OUT).read()
    declared = re.findall(r"pub fn (cvb_\w+)\((.*?)\)(?: -> [^;]+)?;", text)
    assert sorted(n for n, _ in declared) == sorted(SFM_ABI_SYMBOLS)
    plain = gen.strip_comments(header)
    for name, params in declared:
        cargs = re.search(r"\b" + name + r"\s*\(([^;{]*?)\)\s*;", plain, flags=re.S).group(1)
        assert cargs.count(",") + 1 == params.count(",") + 1, name
    body = re.search(r"pub struct cvb_intrinsics_k1 \{(.*?)\n\}", text, flags=re.S).group(1)
    assert re.findall(r"pub (\w+):", body) == ["fx", "fy", "cx", "cy", "skew", "k1"]
    shim = open(gen.SFM_SHIM_OUT).read()
    called = set(re.findall(r"\b(cvb_[a-z0-9_]+)\s*\(", shim))
    assert {"cvb_two_view_frames_k1", "cvb_frame_features_batch"} <= called <= set(ABI_SYMBOLS) | set(SFM_ABI_SYMBOLS)


def test_new_entry_points_report_no_device():
    _ensure_built()
    import numpy as np
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from cv_b200._lib import CVB_ENODEV
    cam = cv_b200.CameraIntrinsicsK1Distortion(cv_b200.CameraIntrinsics((1000.0, 1000.0), (960.0, 540.0)), -0.28)
    with pytest.raises(cv_b200.CvbError) as e:
        cv_b200.frame_features(cv_b200.Akaze(), np.zeros((1, 32, 32), np.float32), np.zeros((1, 32, 32, 3), np.uint8), cam)
    assert e.value.code == CVB_ENODEV
    with pytest.raises(cv_b200.CvbError) as e:
        cv_b200.two_view_frames(cv_b200.Akaze(), np.zeros((2, 32, 32), np.float32), cam, cv_b200.Arrsac(1e-7, cv_b200.Xoshiro256PlusPlus(0)))
    assert e.value.code == CVB_ENODEV
