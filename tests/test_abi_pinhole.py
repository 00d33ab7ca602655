"""CPU-only: include/cvb200_pinhole.h (cv-pinhole's reprojection error and EssentialMatrix) -- libcvb200_pinhole.so exports exactly the
symbols the header declares, libcvb200.so's exports are unchanged, a C program calls every one of them, the generated Rust bindings match
the header, and without a CUDA device every entry point fails cleanly (no CPU fallback)."""
import importlib.util
import os
import re
import subprocess

import numpy as np
import pytest

import cv_b200
from cv_b200._lib import ABI_SYMBOLS, OPT_ABI_SYMBOLS, PINHOLE_ABI_SYMBOLS, SFM_ABI_SYMBOLS, TRI_ABI_SYMBOLS, pinhole_lib_path

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "cvb200_pinhole.h")


def _ensure_built():
    if not (os.path.exists(cv_b200.lib_path()) and os.path.exists(pinhole_lib_path())):
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
    assert _declared() == set(PINHOLE_ABI_SYMBOLS), _declared() ^ set(PINHOLE_ABI_SYMBOLS)
    assert not set(PINHOLE_ABI_SYMBOLS) & (set(ABI_SYMBOLS) | set(SFM_ABI_SYMBOLS) | set(TRI_ABI_SYMBOLS) | set(OPT_ABI_SYMBOLS))
    assert _exported(pinhole_lib_path()) == set(PINHOLE_ABI_SYMBOLS)
    assert _exported(cv_b200.lib_path()) == set(ABI_SYMBOLS) | set(SFM_ABI_SYMBOLS) | set(TRI_ABI_SYMBOLS)   # unchanged
    L = cv_b200._lib.load_pinhole_library()
    for s in PINHOLE_ABI_SYMBOLS:
        assert hasattr(L, s), s


def _build_smoke():
    out = os.path.join(ROOT, "tests", "csrc", "_build")
    os.makedirs(out, exist_ok=True)
    exe = os.path.join(out, "abi_smoke_pinhole")
    libdir = os.path.join(ROOT, "cv_b200")
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", os.path.join(ROOT, "tests", "csrc", "abi_smoke_pinhole.c"),
                           "-I" + os.path.join(ROOT, "include"), "-L" + libdir, "-lcvb200_pinhole", "-lcvb200", "-lm",
                           "-Wl,-rpath," + libdir, "-o", exe])
    return exe


def test_c_program_compiles_against_pinhole_header_and_calls_every_entry_point():
    _ensure_built()
    exe = _build_smoke()
    src = open(os.path.join(ROOT, "tests", "csrc", "abi_smoke_pinhole.c")).read()
    for sym in _declared():
        assert re.search(r"\b" + sym + r"\s*\(", src), f"{sym} is not called by abi_smoke_pinhole.c"
    r = subprocess.run([exe, "0"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.gpu
def test_c_program_pinhole_gpu_workflow():
    _ensure_built()
    r = subprocess.run([_build_smoke(), "1"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "GPU workflow ok" in r.stdout, r.stdout + r.stderr


def test_rust_pinhole_bindings_are_generated_from_the_current_header():
    """cv-b200-sys/src/pinhole.rs is what scripts/gen_rust_sys.py produces from include/cvb200_pinhole.h, and the shim's pinhole.rs what it
    assembles from INTEGRATION.md section 2f; every symbol is declared once with the header's arity; the shim calls only declared externs."""
    spec = importlib.util.spec_from_file_location("gen_rust_sys", os.path.join(ROOT, "scripts", "gen_rust_sys.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    header = open(HEADER).read()
    text, _ = gen.generate_pinhole(header)
    assert open(gen.PINHOLE_OUT).read() == text, "stale: python scripts/gen_rust_sys.py"
    assert open(gen.PINHOLE_SHIM_OUT).read() == gen.generate_shim_pinhole(), "stale: python scripts/gen_rust_sys.py"
    assert "pub mod pinhole;" in open(gen.OUT).read() and "pub mod pinhole;" in open(gen.SHIM_OUT).read()
    assert '#[link(name = "cvb200_pinhole")]' in text
    declared = re.findall(r"pub fn (cvb_\w+)\((.*?)\)(?: -> [^;]+)?;", text)
    assert sorted(n for n, _ in declared) == sorted(PINHOLE_ABI_SYMBOLS)
    plain = gen.strip_comments(header)
    for name, params in declared:
        cargs = re.search(r"\b" + name + r"\s*\(([^;{]*?)\)\s*;", plain, flags=re.S).group(1)
        assert cargs.count(",") == params.count(","), name
    shim = open(gen.PINHOLE_SHIM_OUT).read()
    called = set(re.findall(r"\b(cvb_[a-z0-9_]+)\s*\(", shim))
    assert set(PINHOLE_ABI_SYMBOLS) - {"cvb_pose_reprojection_error_dev"} <= called <= set(ABI_SYMBOLS) | set(TRI_ABI_SYMBOLS) | set(PINHOLE_ABI_SYMBOLS)
    for f in ("pub fn pose_reprojection_error(", "pub fn pose_reprojection_error_batch(", "pub fn average_pose_reprojection_error(",
              "pub fn from_matches_batch(", "pub fn recondition_batch(", "pub fn possible_rotations_unscaled_translation_batch("):
        assert f in shim, f


def test_new_entry_points_report_no_device():
    _ensure_built()
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from cv_b200._lib import CVB_ENODEV
    eye = (np.eye(3), np.array([1.0, 0.0, 0.0]))
    a = np.tile([0.0, 0.0, 1.0], (8, 1))
    E = cv_b200.EssentialMatrix.from_pose(eye)
    for call in (lambda: cv_b200.pose_reprojection_error(eye, a[0], a[0], cv_b200.LinearEigenTriangulator()),
                 lambda: cv_b200.average_pose_reprojection_error_batch([eye], a, a, cv_b200.AngularL1Triangulator()),
                 lambda: cv_b200.EightPoint().from_matches(a, a),
                 lambda: E.residuals(a, a),
                 lambda: E.recondition(1e-12, 1000),
                 lambda: E.possible_unscaled_poses(1e-6, 50)):
        with pytest.raises(cv_b200.CvbError) as e:
            call()
        assert e.value.code == CVB_ENODEV
