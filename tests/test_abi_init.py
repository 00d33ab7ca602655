"""CPU-only: include/cvb200_init.h (cv-sfm's three-view initialisation) -- libcvb200_init.so exports exactly the symbols the header
declares, libcvb200.so's exports are unchanged, a C program calls every one of them, the generated Rust bindings match the header, the
defaults are cv-sfm's, and without a CUDA device the calls fail cleanly (no CPU fallback).  Also the Python wrapper's tensor checks."""
import ctypes as C
import importlib.util
import os
import re
import subprocess

import pytest

import cv_b200
from cv_b200._lib import (ABI_SYMBOLS, BATCH_ABI_SYMBOLS, CVB_ENODEV, FILTER_ABI_SYMBOLS, IMAGE_ABI_SYMBOLS, INIT_ABI_SYMBOLS,
                          LSH_ABI_SYMBOLS, OPT_ABI_SYMBOLS, PINHOLE_ABI_SYMBOLS, SFM_ABI_SYMBOLS, STAGES_ABI_SYMBOLS, TRI_ABI_SYMBOLS,
                          init_lib_path)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "cvb200_init.h")


def _ensure_built():
    if not (os.path.exists(cv_b200.lib_path()) and os.path.exists(init_lib_path())):
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
    assert _declared() == set(INIT_ABI_SYMBOLS), _declared() ^ set(INIT_ABI_SYMBOLS)
    others = (set(ABI_SYMBOLS) | set(SFM_ABI_SYMBOLS) | set(TRI_ABI_SYMBOLS) | set(OPT_ABI_SYMBOLS) | set(PINHOLE_ABI_SYMBOLS) |
              set(IMAGE_ABI_SYMBOLS) | set(FILTER_ABI_SYMBOLS) | set(LSH_ABI_SYMBOLS) | set(STAGES_ABI_SYMBOLS) | set(BATCH_ABI_SYMBOLS))
    assert not set(INIT_ABI_SYMBOLS) & others
    assert _exported(init_lib_path()) == set(INIT_ABI_SYMBOLS)
    assert _exported(cv_b200.lib_path()) == set(ABI_SYMBOLS) | set(SFM_ABI_SYMBOLS) | set(TRI_ABI_SYMBOLS)   # unchanged
    L = cv_b200._lib.load_init_library()
    for s in INIT_ABI_SYMBOLS:
        assert hasattr(L, s), s


def _build_smoke():
    out = os.path.join(ROOT, "tests", "csrc", "_build")
    os.makedirs(out, exist_ok=True)
    exe = os.path.join(out, "abi_smoke_init")
    libdir = os.path.join(ROOT, "cv_b200")
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", os.path.join(ROOT, "tests", "csrc", "abi_smoke_init.c"),
                           "-I" + os.path.join(ROOT, "include"), "-L" + libdir, "-lcvb200_init", "-lcvb200", "-Wl,-rpath," + libdir,
                           "-lm", "-o", exe])
    return exe


def test_c_program_compiles_against_init_header_and_calls_every_entry_point():
    _ensure_built()
    exe = _build_smoke()
    src = open(os.path.join(ROOT, "tests", "csrc", "abi_smoke_init.c")).read()
    for sym in _declared():
        assert re.search(r"\b" + sym + r"\s*\(", src), f"{sym} is not called by abi_smoke_init.c"
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: test_c_program_init_gpu_workflow runs the program")
    r = subprocess.run([exe, "0"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.gpu
def test_c_program_init_gpu_workflow():
    _ensure_built()
    r = subprocess.run([_build_smoke(), "1"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "GPU workflow ok" in r.stdout, r.stdout + r.stderr


def test_rust_init_bindings_are_generated_from_the_current_header():
    """cv-b200-sys/src/init.rs is what scripts/gen_rust_sys.py produces from include/cvb200_init.h, and the shim's init.rs what it
    assembles from INTEGRATION.md section 2l; every symbol is declared once with the header's arity."""
    spec = importlib.util.spec_from_file_location("gen_rust_sys", os.path.join(ROOT, "scripts", "gen_rust_sys.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    header = open(HEADER).read()
    text, _ = gen.generate_init(header)
    assert open(gen.INIT_OUT).read() == text, "stale: python scripts/gen_rust_sys.py"
    assert open(gen.INIT_SHIM_OUT).read() == gen.generate_shim_init(), "stale: python scripts/gen_rust_sys.py"
    assert "pub mod init;" in open(gen.OUT).read() and "pub mod init;" in open(gen.SHIM_OUT).read()
    assert "pub unsafe fn init_reconstruction_dev(ctx: &Ctx" in open(gen.INIT_SHIM_OUT).read()
    assert '#[link(name = "cvb200_init")]' in text and "pub struct cvb_init_cfg {" in text and "pub const CVB_INIT_ACCEPTED: i32 = 1;" in text
    declared = re.findall(r"pub fn (cvb_\w+)\((.*?)\)(?: -> [^;]+)?;", text)
    assert sorted(n for n, _ in declared) == sorted(INIT_ABI_SYMBOLS)
    plain = gen.strip_comments(header)
    for name, params in declared:
        cargs = re.search(r"\b" + name + r"\s*\(([^;{]*?)\)\s*;", plain, flags=re.S).group(1)
        assert cargs.count(",") == params.count(","), name
    r = subprocess.run(["python", os.path.join(ROOT, "scripts", "gen_rust_sys.py"), "--check"], capture_output=True, text=True)
    assert r.returncode == 0 and "up to date" in r.stdout, r.stdout


def test_defaults_are_cv_sfm_settings():
    """cvb_init_cfg_default, the Python InitSettings and the oracle's InitCfg all hold cv-sfm's defaults (cv-sfm/src/settings.rs)."""
    _ensure_built()
    from oracle.pyoracle_init import InitCfg
    want = dict(two_view_minimum_robust_matches=256, robust_observation_incidence_minimum_cosine_distance=1e-3,
                three_view_minimum_relative_scales=16, three_view_optimization_landmarks=1024,
                robust_view_bearing_pair_minimum_cosine_distance=1e-2, robust_view_num_robust_bearing_pair=3,
                three_view_filter_loop_iterations=8, three_view_patience=65536, maximum_cosine_distance=1e-5, maximum_sine_distance=0.1,
                three_view_minimum_robust_matches=32)
    c = cv_b200.InitSettings()
    cv_b200._lib.load_init_library().cvb_init_cfg_default(C.addressof(c))
    for s in (c, cv_b200.InitSettings(), InitCfg()):
        assert {k: getattr(s, k) for k in want} == want
    assert C.sizeof(c) == 64 and C.sizeof(InitCfg) == 64


def test_init_reports_no_device():
    _ensure_built()
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(cv_b200.CvbError) as e:
        cv_b200.Context(0)
    assert e.value.code == CVB_ENODEV


def test_init_reconstruction_checks_its_tensors():
    import torch
    feats = dict(descriptors=torch.zeros((3, 8, 64), dtype=torch.uint8), counts=torch.zeros(3, dtype=torch.int32),
                 bearings=torch.zeros((3, 8, 3), dtype=torch.float64))
    with pytest.raises(ValueError):
        cv_b200.init_reconstruction(feats, 0, [1, 2], None, [None, None])      # host tensors: the call works on device tensors
    with pytest.raises(ValueError):
        cv_b200.init_reconstruction(feats, 0, [1, 2], None, [None, None], triangulator=cv_b200.RelativeDltTriangulator())
    with pytest.raises(ValueError):
        cv_b200.pair.init_reconstruction_dev(None, feats["bearings"], 0, [1, 2], None)    # host bearings
