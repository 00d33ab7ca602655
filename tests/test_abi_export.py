"""CPU-only: include/cvb200_export.h (cv-sfm's reconstruction export) -- libcvb200_export.so exports exactly the symbols the header
declares, libcvb200.so's exports are unchanged, a C program calls every one of them, the generated Rust bindings match the header, the
defaults are cv-sfm's, the host validator refuses malformed snapshots, constraints and first views, and without a CUDA device the calls
fail cleanly."""
import ctypes as C
import importlib.util
import os
import re
import subprocess

import numpy as np
import pytest

import cv_b200
from cv_b200._lib import (ABI_SYMBOLS, BATCH_ABI_SYMBOLS, CONSTRAINTS_ABI_SYMBOLS, CVB_EINVAL, CVB_ENODEV, EXPORT_ABI_SYMBOLS,
                          FILTER_ABI_SYMBOLS, IMAGE_ABI_SYMBOLS, INIT_ABI_SYMBOLS, LSH_ABI_SYMBOLS, OPT_ABI_SYMBOLS, PINHOLE_ABI_SYMBOLS,
                          RECONSTRUCTION_ABI_SYMBOLS, SFM_ABI_SYMBOLS, STAGES_ABI_SYMBOLS, TRI_ABI_SYMBOLS, export_lib_path)
from cv_b200.constraints import CONSTRAINT_DTYPE
from cv_b200.export import CAMERA_DTYPE, NORMALIZE_RESULT_DTYPE, check_export

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "cvb200_export.h")


def _ensure_built():
    if not (os.path.exists(cv_b200.lib_path()) and os.path.exists(export_lib_path())):
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
    assert _declared() == set(EXPORT_ABI_SYMBOLS), _declared() ^ set(EXPORT_ABI_SYMBOLS)
    others = (set(ABI_SYMBOLS) | set(SFM_ABI_SYMBOLS) | set(TRI_ABI_SYMBOLS) | set(OPT_ABI_SYMBOLS) | set(PINHOLE_ABI_SYMBOLS) |
              set(IMAGE_ABI_SYMBOLS) | set(FILTER_ABI_SYMBOLS) | set(LSH_ABI_SYMBOLS) | set(STAGES_ABI_SYMBOLS) | set(BATCH_ABI_SYMBOLS) |
              set(INIT_ABI_SYMBOLS) | set(CONSTRAINTS_ABI_SYMBOLS) | set(RECONSTRUCTION_ABI_SYMBOLS))
    assert not set(EXPORT_ABI_SYMBOLS) & others
    assert _exported(export_lib_path()) == set(EXPORT_ABI_SYMBOLS)
    assert _exported(cv_b200.lib_path()) == set(ABI_SYMBOLS) | set(SFM_ABI_SYMBOLS) | set(TRI_ABI_SYMBOLS)   # unchanged
    L = cv_b200._lib.load_export_library()
    for s in EXPORT_ABI_SYMBOLS:
        assert hasattr(L, s), s


def _build_smoke():
    out = os.path.join(ROOT, "tests", "csrc", "_build")
    os.makedirs(out, exist_ok=True)
    exe = os.path.join(out, "abi_smoke_export")
    libdir = os.path.join(ROOT, "cv_b200")
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", os.path.join(ROOT, "tests", "csrc", "abi_smoke_export.c"),
                           "-I" + os.path.join(ROOT, "include"), "-L" + libdir, "-lcvb200_export", "-lcvb200", "-Wl,-rpath," + libdir,
                           "-lm", "-o", exe])
    return exe


def test_c_program_compiles_against_export_header_and_calls_every_entry_point():
    _ensure_built()
    exe = _build_smoke()
    src = open(os.path.join(ROOT, "tests", "csrc", "abi_smoke_export.c")).read()
    for sym in _declared():
        assert re.search(r"\b" + sym + r"\s*\(", src), f"{sym} is not called by abi_smoke_export.c"
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: test_c_program_export_gpu_workflow runs the program")
    r = subprocess.run([exe, "0"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.gpu
def test_c_program_export_gpu_workflow():
    _ensure_built()
    r = subprocess.run([_build_smoke(), "1"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "GPU workflow ok" in r.stdout, r.stdout + r.stderr


def test_rust_export_bindings_are_generated_from_the_current_header():
    """cv-b200-sys/src/export.rs is what scripts/gen_rust_sys.py produces from include/cvb200_export.h, and the shim's export.rs what it
    assembles from INTEGRATION.md section 2o; every symbol is declared once with the header's arity."""
    spec = importlib.util.spec_from_file_location("gen_rust_sys", os.path.join(ROOT, "scripts", "gen_rust_sys.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    header = open(HEADER).read()
    text, _ = gen.generate_export(header)
    assert open(gen.EXPORT_OUT).read() == text, "stale: python scripts/gen_rust_sys.py"
    assert open(gen.EXPORT_SHIM_OUT).read() == gen.generate_shim_export(), "stale: python scripts/gen_rust_sys.py"
    assert "pub mod export;" in open(gen.OUT).read() and "pub mod export;" in open(gen.SHIM_OUT).read()
    shim = open(gen.EXPORT_SHIM_OUT).read()
    assert "pub fn export_reconstruction(ctx: &Ctx" in shim and "pub fn normalize_reconstruction(ctx: &Ctx" in shim
    assert '#[link(name = "cvb200_export")]' in text and "pub struct cvb_export_camera {" in text
    assert "pub const CVB_EXPORT_AT_INFINITY: u32 = 3;" in text
    declared = re.findall(r"pub fn (cvb_\w+)\((.*?)\)(?: -> [^;]+)?;", text)
    assert sorted(n for n, _ in declared) == sorted(EXPORT_ABI_SYMBOLS)
    plain = gen.strip_comments(header)
    for name, params in declared:
        cargs = re.search(r"\b" + name + r"\s*\(([^;{]*?)\)\s*;", plain, flags=re.S).group(1)
        assert cargs.count(",") == params.count(","), name
    r = subprocess.run(["python", os.path.join(ROOT, "scripts", "gen_rust_sys.py"), "--check"], capture_output=True, text=True)
    assert r.returncode == 0 and "up to date" in r.stdout, r.stdout


def test_defaults_are_cv_sfm_settings():
    """cvb_export_cfg_default, the Python ExportSettings and the oracle's ExportCfg hold cv-sfm's defaults (cv-sfm/src/settings.rs); the
    record layouts agree with the header."""
    _ensure_built()
    from oracle.pyoracle_export import ExportCfg
    want = dict(robust_observation_incidence_minimum_cosine_distance=1e-3, robust_minimum_observations=3)
    c = cv_b200.ExportSettings()
    C.memset(C.addressof(c), 0, C.sizeof(c))
    cv_b200._lib.load_export_library().cvb_export_cfg_default(C.addressof(c))
    for s in (c, cv_b200.ExportSettings(), ExportCfg()):
        assert {k: getattr(s, k) for k in want} == want
    assert C.sizeof(c) == 16 and C.sizeof(ExportCfg) == 16
    assert CAMERA_DTYPE.itemsize == 80 and NORMALIZE_RESULT_DTYPE.itemsize == 16


def test_export_reports_no_device():
    _ensure_built()
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(cv_b200.CvbError) as e:
        cv_b200.Context(0)
    assert e.value.code == CVB_ENODEV


def _inputs():
    # views 0..3; landmark 0 in views 0-2, landmark 1 in views 0 and 3, landmark 2 only in view 1; two constraints
    vo = [0, 2, 4, 5, 6]
    vl = [1, 0, 2, 0, 0, 1]
    lo = [0, 3, 5, 6]
    obs = [[0, 1], [1, 1], [2, 0], [0, 0], [3, 0], [1, 0]]
    cons = np.zeros(2, CONSTRAINT_DTYPE)
    cons["views"] = [[0, 1, 2], [1, 2, 3]]
    return vo, vl, lo, obs, cons


def test_host_validator_accepts_consistent_inputs():
    _ensure_built()
    vo, vl, lo, obs, cons = _inputs()
    for first in range(4):
        assert check_export(vo, vl, lo, obs, cons, first) == 0
    assert check_export(vo, vl, lo, obs) == 0


@pytest.mark.parametrize("kind", ["offset_start", "view_offsets_decrease", "landmark_out_of_range", "feature_of_other_landmark",
                                  "view_observed_twice", "no_views", "constraint_view_out_of_range", "constraint_views_repeated",
                                  "null_constraints", "first_view_equal_V", "first_view_above_V"])
def test_host_validator_rejects_malformed_inputs(kind):
    _ensure_built()
    vo, vl, lo, obs, cons = _inputs()
    first = 0
    if kind == "offset_start":
        vo = [1, 2, 4, 5, 6]
    elif kind == "view_offsets_decrease":
        vo = [0, 3, 2, 5, 6]
    elif kind == "landmark_out_of_range":
        vl[0] = 7
    elif kind == "feature_of_other_landmark":
        obs[1] = [1, 0]
    elif kind == "view_observed_twice":
        obs[1] = [0, 1]
    elif kind == "no_views":
        vo, vl, lo, obs, cons = [0], [], [0], [], cons[:0]
    elif kind == "constraint_view_out_of_range":
        cons[1]["views"][2] = 4
    elif kind == "constraint_views_repeated":
        cons[0]["views"][1] = 2
    elif kind == "null_constraints":
        u = (lambda a: np.ascontiguousarray(a, np.uint32))
        a = [u(vo), u(vl), u(lo), u(obs).reshape(-1)]
        assert cv_b200._lib.load_export_library().cvb_export_check(4, a[0].ctypes.data, a[1].ctypes.data, 3, a[2].ctypes.data,
                                                                    a[3].ctypes.data, None, 2, 0) == CVB_EINVAL
        return
    elif kind == "first_view_equal_V":
        first = 4
    elif kind == "first_view_above_V":
        first = 1 << 31
    assert check_export(vo, vl, lo, obs, cons, first) == CVB_EINVAL
