"""CPU-only: include/cvb200_register.h (cv-sfm's frame registration) -- libcvb200_register.so exports exactly the symbols the header
declares, libcvb200.so's exports are unchanged, a C program calls every one of them, the defaults are cv-sfm's, the host validator refuses
malformed snapshots and view matches, and without a CUDA device the calls fail cleanly."""
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
                          RECONSTRUCTION_ABI_SYMBOLS, REGISTER_ABI_SYMBOLS, SFM_ABI_SYMBOLS, STAGES_ABI_SYMBOLS, TRI_ABI_SYMBOLS,
                          register_lib_path)
from cv_b200.register import MATCH_DTYPE, RESULT_DTYPE, STATS_DTYPE, check_register
from oracle.pyoracle_register import MATCH_DTYPE as O_MATCH, RESULT_DTYPE as O_RESULT, STATS_DTYPE as O_STATS, RegisterCfg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "cvb200_register.h")


def _ensure_built():
    if not (os.path.exists(cv_b200.lib_path()) and os.path.exists(register_lib_path())):
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
    assert _declared() == set(REGISTER_ABI_SYMBOLS), _declared() ^ set(REGISTER_ABI_SYMBOLS)
    others = (set(ABI_SYMBOLS) | set(SFM_ABI_SYMBOLS) | set(TRI_ABI_SYMBOLS) | set(OPT_ABI_SYMBOLS) | set(PINHOLE_ABI_SYMBOLS) |
              set(IMAGE_ABI_SYMBOLS) | set(FILTER_ABI_SYMBOLS) | set(LSH_ABI_SYMBOLS) | set(STAGES_ABI_SYMBOLS) | set(BATCH_ABI_SYMBOLS) |
              set(INIT_ABI_SYMBOLS) | set(CONSTRAINTS_ABI_SYMBOLS) | set(RECONSTRUCTION_ABI_SYMBOLS) | set(EXPORT_ABI_SYMBOLS))
    assert not set(REGISTER_ABI_SYMBOLS) & others
    assert _exported(register_lib_path()) == set(REGISTER_ABI_SYMBOLS)
    assert _exported(cv_b200.lib_path()) == set(ABI_SYMBOLS) | set(SFM_ABI_SYMBOLS) | set(TRI_ABI_SYMBOLS)   # unchanged
    L = cv_b200._lib.load_register_library()
    for s in REGISTER_ABI_SYMBOLS:
        assert hasattr(L, s), s


def _build_smoke():
    out = os.path.join(ROOT, "tests", "csrc", "_build")
    os.makedirs(out, exist_ok=True)
    exe = os.path.join(out, "abi_smoke_register")
    libdir = os.path.join(ROOT, "cv_b200")
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", os.path.join(ROOT, "tests", "csrc", "abi_smoke_register.c"),
                           "-I" + os.path.join(ROOT, "include"), "-L" + libdir, "-lcvb200_register", "-lcvb200", "-Wl,-rpath," + libdir,
                           "-lm", "-o", exe])
    return exe


def test_c_program_compiles_against_register_header_and_calls_every_entry_point():
    _ensure_built()
    exe = _build_smoke()
    src = open(os.path.join(ROOT, "tests", "csrc", "abi_smoke_register.c")).read()
    for sym in _declared():
        assert re.search(r"\b" + sym + r"\s*\(", src), f"{sym} is not called by abi_smoke_register.c"
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: test_c_program_register_gpu_workflow runs the program")
    r = subprocess.run([exe, "0"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.gpu
def test_c_program_register_gpu_workflow():
    _ensure_built()
    r = subprocess.run([_build_smoke(), "1"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr


def test_rust_register_bindings_are_generated_from_the_current_header():
    """cv-b200-sys/src/register.rs is what scripts/gen_rust_sys.py produces from include/cvb200_register.h, and the shim's register.rs
    what it assembles from INTEGRATION.md section 2p; every symbol is declared once with the header's arity."""
    spec = importlib.util.spec_from_file_location("gen_rust_sys", os.path.join(ROOT, "scripts", "gen_rust_sys.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    header = open(HEADER).read()
    text, _ = gen.generate_register(header)
    assert open(gen.REGISTER_OUT).read() == text, "stale: python scripts/gen_rust_sys.py"
    assert open(gen.REGISTER_SHIM_OUT).read() == gen.generate_shim_register(), "stale: python scripts/gen_rust_sys.py"
    assert "pub mod register;" in open(gen.OUT).read() and "pub mod register;" in open(gen.SHIM_OUT).read()
    assert "pub fn register_frame(ctx: &Ctx" in open(gen.REGISTER_SHIM_OUT).read()
    assert '#[link(name = "cvb200_register")]' in text and "pub struct cvb_register_stats {" in text
    assert "pub filter_matches: [u32; 16]," in text and "pub const CVB_REGISTER_NONE: u32 = 0xffffffff;" in text
    declared = re.findall(r"pub fn (cvb_\w+)\((.*?)\)(?: -> [^;]+)?;", text)
    assert sorted(n for n, _ in declared) == sorted(REGISTER_ABI_SYMBOLS)
    plain = gen.strip_comments(header)
    for name, params in declared:
        cargs = re.search(r"\b" + name + r"\s*\(([^;{]*?)\)\s*;", plain, flags=re.S).group(1)
        assert cargs.count(",") == params.count(","), name
    r = subprocess.run(["python", os.path.join(ROOT, "scripts", "gen_rust_sys.py"), "--check"], capture_output=True, text=True)
    assert r.returncode == 0 and "up to date" in r.stdout, r.stdout


def test_defaults_are_cv_sfm_settings():
    _ensure_built()
    want = dict(single_view_optimization_rate=1e-3, maximum_sine_distance=0.1, maximum_cosine_distance=1e-5,
                robust_observation_incidence_minimum_cosine_distance=1e-3, single_view_match_better_by=24,
                single_view_initial_features=8192, single_view_minimum_landmarks=32, single_view_optimization_num_matches=2048,
                single_view_filter_loop_iterations=5, single_view_patience=100000, single_view_minimum_robust_landmarks=64,
                robust_minimum_observations=3)
    c = cv_b200.RegisterSettings()
    C.CDLL(register_lib_path())   # the library loads
    lib_cfg = cv_b200.RegisterSettings()
    cv_b200._lib.load_register_library().cvb_register_cfg_default(C.addressof(lib_cfg))
    for s in (c, lib_cfg, RegisterCfg()):
        assert {k: getattr(s, k) for k in want} == want
    assert C.sizeof(c) == 64 and C.sizeof(RegisterCfg) == 64
    assert MATCH_DTYPE == O_MATCH and RESULT_DTYPE == O_RESULT and STATS_DTYPE == O_STATS
    assert MATCH_DTYPE.itemsize == 12 and RESULT_DTYPE.itemsize == 112 and STATS_DTYPE.itemsize == 112


def test_register_reports_no_device():
    _ensure_built()
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(cv_b200.CvbError) as e:
        cv_b200.Context(0)
    assert e.value.code == CVB_ENODEV


def _inputs():
    # views 0..2; landmark 0 in views 0-2, landmark 1 in views 0 and 2, landmark 2 only in view 1
    vo = [0, 2, 4, 6]
    vl = [1, 0, 2, 0, 0, 1]
    lo = [0, 3, 5, 6]
    obs = [[0, 1], [1, 1], [2, 0], [0, 0], [2, 1], [1, 0]]
    return vo, vl, lo, obs


def test_host_validator_accepts_consistent_inputs():
    _ensure_built()
    vo, vl, lo, obs = _inputs()
    assert check_register(vo, vl, lo, obs, [0, 1, 2, 2]) == 0
    assert check_register(vo, vl, lo, obs, []) == 0


@pytest.mark.parametrize("kind", ["view_out_of_range", "offsets_not_monotone", "offsets_not_from_zero", "landmark_out_of_range",
                                  "csr_disagree", "view_observed_twice"])
def test_host_validator_rejects_malformed_inputs(kind):
    _ensure_built()
    vo, vl, lo, obs = _inputs()
    vm = [0, 1]
    if kind == "view_out_of_range":
        vm = [3]
    elif kind == "offsets_not_monotone":
        vo = [0, 3, 2, 6]
    elif kind == "offsets_not_from_zero":
        lo = [1, 3, 5, 6]
    elif kind == "landmark_out_of_range":
        vl = [1, 0, 3, 0, 0, 1]
    elif kind == "csr_disagree":
        obs = [[0, 1], [1, 1], [2, 1], [0, 0], [2, 0], [1, 0]]
        obs[2] = [2, 1]
        obs[4] = [2, 1]
    elif kind == "view_observed_twice":
        vl = [0, 0, 2, 0, 0, 1]
    assert check_register(vo, vl, lo, obs, vm) == CVB_EINVAL


def test_python_entry_refuses_mismatched_new_frame():
    _ensure_built()

    class _Ctx:
        handle = None

    with pytest.raises(ValueError):
        cv_b200.register_frame(_Ctx(), np.zeros((1, 12)), [0, 0], [], np.zeros((0, 3)), np.zeros((0, 64), np.uint8), [0], [],
                               np.zeros((2, 64), np.uint8), np.zeros((1, 3)), [0], None)
