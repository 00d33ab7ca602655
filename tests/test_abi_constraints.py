"""CPU-only: include/cvb200_constraints.h (cv-sfm's three-view constraints) -- libcvb200_constraints.so exports exactly the symbols the header
declares, libcvb200.so's exports are unchanged, a C program calls every one of them, the generated Rust bindings match the header, the
defaults are cv-sfm's, the host validator refuses every kind of malformed snapshot, and without a CUDA device the calls fail cleanly."""
import ctypes as C
import importlib.util
import os
import re
import subprocess

import numpy as np
import pytest

import cv_b200
from cv_b200._lib import (ABI_SYMBOLS, BATCH_ABI_SYMBOLS, CONSTRAINTS_ABI_SYMBOLS, CVB_EINVAL, CVB_ENODEV, FILTER_ABI_SYMBOLS,
                          IMAGE_ABI_SYMBOLS, INIT_ABI_SYMBOLS, LSH_ABI_SYMBOLS, OPT_ABI_SYMBOLS, PINHOLE_ABI_SYMBOLS, SFM_ABI_SYMBOLS,
                          STAGES_ABI_SYMBOLS, TRI_ABI_SYMBOLS, constraints_lib_path)
from cv_b200.constraints import check_snapshot

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "cvb200_constraints.h")


def _ensure_built():
    if not (os.path.exists(cv_b200.lib_path()) and os.path.exists(constraints_lib_path())):
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
    assert _declared() == set(CONSTRAINTS_ABI_SYMBOLS), _declared() ^ set(CONSTRAINTS_ABI_SYMBOLS)
    others = (set(ABI_SYMBOLS) | set(SFM_ABI_SYMBOLS) | set(TRI_ABI_SYMBOLS) | set(OPT_ABI_SYMBOLS) | set(PINHOLE_ABI_SYMBOLS) |
              set(IMAGE_ABI_SYMBOLS) | set(FILTER_ABI_SYMBOLS) | set(LSH_ABI_SYMBOLS) | set(STAGES_ABI_SYMBOLS) | set(BATCH_ABI_SYMBOLS) |
              set(INIT_ABI_SYMBOLS))
    assert not set(CONSTRAINTS_ABI_SYMBOLS) & others
    assert _exported(constraints_lib_path()) == set(CONSTRAINTS_ABI_SYMBOLS)
    assert _exported(cv_b200.lib_path()) == set(ABI_SYMBOLS) | set(SFM_ABI_SYMBOLS) | set(TRI_ABI_SYMBOLS)   # unchanged
    L = cv_b200._lib.load_constraints_library()
    for s in CONSTRAINTS_ABI_SYMBOLS:
        assert hasattr(L, s), s


def _build_smoke():
    out = os.path.join(ROOT, "tests", "csrc", "_build")
    os.makedirs(out, exist_ok=True)
    exe = os.path.join(out, "abi_smoke_constraints")
    libdir = os.path.join(ROOT, "cv_b200")
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", os.path.join(ROOT, "tests", "csrc", "abi_smoke_constraints.c"),
                           "-I" + os.path.join(ROOT, "include"), "-L" + libdir, "-lcvb200_constraints", "-lcvb200", "-Wl,-rpath," + libdir,
                           "-lm", "-o", exe])
    return exe


def test_c_program_compiles_against_constraints_header_and_calls_every_entry_point():
    _ensure_built()
    exe = _build_smoke()
    src = open(os.path.join(ROOT, "tests", "csrc", "abi_smoke_constraints.c")).read()
    for sym in _declared():
        assert re.search(r"\b" + sym + r"\s*\(", src), f"{sym} is not called by abi_smoke_constraints.c"
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: test_c_program_constraints_gpu_workflow runs the program")
    r = subprocess.run([exe, "0"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.gpu
def test_c_program_constraints_gpu_workflow():
    _ensure_built()
    r = subprocess.run([_build_smoke(), "1"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "GPU workflow ok" in r.stdout, r.stdout + r.stderr


def test_rust_constraints_bindings_are_generated_from_the_current_header():
    """cv-b200-sys/src/constraints.rs is what scripts/gen_rust_sys.py produces from include/cvb200_constraints.h, and the shim's
    constraints.rs what it assembles from INTEGRATION.md section 2m; every symbol is declared once with the header's arity."""
    spec = importlib.util.spec_from_file_location("gen_rust_sys", os.path.join(ROOT, "scripts", "gen_rust_sys.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    header = open(HEADER).read()
    text, _ = gen.generate_constraints(header)
    assert open(gen.CONSTRAINTS_OUT).read() == text, "stale: python scripts/gen_rust_sys.py"
    assert open(gen.CONSTRAINTS_SHIM_OUT).read() == gen.generate_shim_constraints(), "stale: python scripts/gen_rust_sys.py"
    assert "pub mod constraints;" in open(gen.OUT).read() and "pub mod constraints;" in open(gen.SHIM_OUT).read()
    assert "pub fn view_constraints(ctx: &Ctx" in open(gen.CONSTRAINTS_SHIM_OUT).read()
    assert '#[link(name = "cvb200_constraints")]' in text and "pub struct cvb_constraints_cfg {" in text
    assert "pub const CVB_CONSTRAINTS_MAX_LANDMARKS: u32 = 512;" in text
    declared = re.findall(r"pub fn (cvb_\w+)\((.*?)\)(?: -> [^;]+)?;", text)
    assert sorted(n for n, _ in declared) == sorted(CONSTRAINTS_ABI_SYMBOLS)
    plain = gen.strip_comments(header)
    for name, params in declared:
        cargs = re.search(r"\b" + name + r"\s*\(([^;{]*?)\)\s*;", plain, flags=re.S).group(1)
        assert cargs.count(",") == params.count(","), name
    r = subprocess.run(["python", os.path.join(ROOT, "scripts", "gen_rust_sys.py"), "--check"], capture_output=True, text=True)
    assert r.returncode == 0 and "up to date" in r.stdout, r.stdout


def test_defaults_are_cv_sfm_settings():
    """cvb_constraints_cfg_default, the Python ConstraintSettings and the oracle's ConstraintsCfg hold cv-sfm's defaults
    (cv-sfm/src/settings.rs:332-350, 453-483)."""
    _ensure_built()
    from oracle.pyoracle_constraints import ConstraintsCfg
    want = dict(robust_observation_incidence_minimum_cosine_distance=1e-3, robust_view_bearing_pair_minimum_cosine_distance=1e-2,
                robust_minimum_observations=3, robust_view_num_robust_bearing_pair=3, optimization_robust_covisibility_minimum_landmarks=16,
                optimization_minimum_landmarks=24, optimization_maximum_landmarks=64, optimization_maximum_three_view_constraints=64,
                optimization_minimum_new_constraints=4, constraint_patience=4096)
    c = cv_b200.ConstraintSettings()
    C.memset(C.addressof(c), 0, C.sizeof(c))
    cv_b200._lib.load_constraints_library().cvb_constraints_cfg_default(C.addressof(c))
    for s in (c, cv_b200.ConstraintSettings(), ConstraintsCfg()):
        assert {k: getattr(s, k) for k in want} == want
    assert C.sizeof(c) == 48 and C.sizeof(ConstraintsCfg) == 48


def test_constraints_report_no_device():
    _ensure_built()
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(cv_b200.CvbError) as e:
        cv_b200.Context(0)
    assert e.value.code == CVB_ENODEV


def _snap():
    # views 0..2; landmark 0 in all three, landmark 1 in views 0 and 2, landmark 2 only in view 1
    vo = [0, 2, 4, 6]
    vl = [1, 0, 2, 0, 0, 1]
    lo = [0, 3, 5, 6]
    obs = [[0, 1], [1, 1], [2, 0], [0, 0], [2, 1], [1, 0]]
    return vo, vl, lo, obs


def test_host_validator_accepts_a_consistent_snapshot():
    _ensure_built()
    vo, vl, lo, obs = _snap()
    assert check_snapshot(vo, vl, lo, obs, [0, 1, 2, 2]) == 0


@pytest.mark.parametrize("kind", ["offset_start", "view_offsets_decrease", "landmark_offsets_decrease", "landmark_out_of_range",
                                  "view_out_of_range", "feature_out_of_range", "feature_of_other_landmark", "view_observed_twice",
                                  "missing_observation", "query_out_of_range", "no_views"])
def test_host_validator_rejects_malformed_snapshots(kind):
    _ensure_built()
    vo, vl, lo, obs = _snap()
    q = [0, 1]
    if kind == "offset_start":
        vo = [1, 2, 4, 6]
    elif kind == "view_offsets_decrease":
        vo = [0, 3, 2, 6]
    elif kind == "landmark_offsets_decrease":
        lo = [0, 4, 3, 6]
    elif kind == "landmark_out_of_range":
        vl[0] = 7
    elif kind == "view_out_of_range":
        obs[0] = [3, 1]
    elif kind == "feature_out_of_range":
        obs[0] = [0, 2]
    elif kind == "feature_of_other_landmark":
        obs[1] = [1, 0]
    elif kind == "view_observed_twice":
        obs[1] = [0, 1]
    elif kind == "missing_observation":
        lo, obs = [0, 3, 4, 5], obs[:4] + obs[5:]
    elif kind == "query_out_of_range":
        q = [0, 3]
    elif kind == "no_views":
        vo = [0]
    assert check_snapshot(vo, vl, lo, obs, q) == CVB_EINVAL
