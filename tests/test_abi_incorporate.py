"""CPU-only: include/cvb200_incorporate.h (cv-sfm's frame incorporation) -- libcvb200_incorporate.so exports exactly the symbols the
header declares, libcvb200.so's exports are unchanged, a C program calls every one of them, the generated Rust is in sync, the result
records match the header's layout, and without a CUDA device the calls fail cleanly.  The host validator's refusals are in
tests/test_oracle_incorporate.py."""
import importlib.util
import os
import re
import subprocess

import numpy as np
import pytest

import cv_b200
from cv_b200._lib import (ABI_SYMBOLS, BATCH_ABI_SYMBOLS, CONSTRAINTS_ABI_SYMBOLS, CVB_ENODEV, EXPORT_ABI_SYMBOLS, FILTER_ABI_SYMBOLS,
                          IMAGE_ABI_SYMBOLS, INCORPORATE_ABI_SYMBOLS, INIT_ABI_SYMBOLS, LSH_ABI_SYMBOLS, OPT_ABI_SYMBOLS, PINHOLE_ABI_SYMBOLS,
                          RECONSTRUCTION_ABI_SYMBOLS, REGISTER_ABI_SYMBOLS, SFM_ABI_SYMBOLS, STAGES_ABI_SYMBOLS, TRI_ABI_SYMBOLS,
                          incorporate_lib_path)
from cv_b200.incorporate import COUNTS_DTYPE, RESULT_DTYPE
from oracle.pyoracle_incorporate import COUNTS_DTYPE as O_COUNTS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "cvb200_incorporate.h")


def _ensure_built():
    if not (os.path.exists(cv_b200.lib_path()) and os.path.exists(incorporate_lib_path())):
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
    assert _declared() == set(INCORPORATE_ABI_SYMBOLS), _declared() ^ set(INCORPORATE_ABI_SYMBOLS)
    others = (set(ABI_SYMBOLS) | set(SFM_ABI_SYMBOLS) | set(TRI_ABI_SYMBOLS) | set(OPT_ABI_SYMBOLS) | set(PINHOLE_ABI_SYMBOLS) |
              set(IMAGE_ABI_SYMBOLS) | set(FILTER_ABI_SYMBOLS) | set(LSH_ABI_SYMBOLS) | set(STAGES_ABI_SYMBOLS) | set(BATCH_ABI_SYMBOLS) |
              set(INIT_ABI_SYMBOLS) | set(CONSTRAINTS_ABI_SYMBOLS) | set(RECONSTRUCTION_ABI_SYMBOLS) | set(EXPORT_ABI_SYMBOLS) |
              set(REGISTER_ABI_SYMBOLS))
    assert not set(INCORPORATE_ABI_SYMBOLS) & others
    assert _exported(incorporate_lib_path()) == set(INCORPORATE_ABI_SYMBOLS)
    assert _exported(cv_b200.lib_path()) == set(ABI_SYMBOLS) | set(SFM_ABI_SYMBOLS) | set(TRI_ABI_SYMBOLS)   # unchanged
    L = cv_b200._lib.load_incorporate_library()
    for s in INCORPORATE_ABI_SYMBOLS:
        assert hasattr(L, s), s


def _build_smoke():
    out = os.path.join(ROOT, "tests", "csrc", "_build")
    os.makedirs(out, exist_ok=True)
    exe = os.path.join(out, "abi_smoke_incorporate")
    libdir = os.path.join(ROOT, "cv_b200")
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", os.path.join(ROOT, "tests", "csrc", "abi_smoke_incorporate.c"),
                           "-I" + os.path.join(ROOT, "include"), "-L" + libdir, "-lcvb200_incorporate", "-lcvb200_register",
                           "-lcvb200_constraints", "-lcvb200_reconstruction", "-lcvb200", "-Wl,-rpath," + libdir, "-lm", "-o", exe])
    return exe


def test_c_program_compiles_against_incorporate_header_and_calls_every_entry_point():
    _ensure_built()
    exe = _build_smoke()
    src = open(os.path.join(ROOT, "tests", "csrc", "abi_smoke_incorporate.c")).read()
    for sym in _declared():
        assert re.search(r"\b" + sym + r"\s*\(", src), f"{sym} is not called by abi_smoke_incorporate.c"
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: test_c_program_incorporate_gpu_workflow runs the program")
    r = subprocess.run([exe, "0"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.gpu
def test_c_program_incorporate_gpu_workflow():
    _ensure_built()
    r = subprocess.run([_build_smoke(), "1"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr


def test_rust_incorporate_bindings_are_generated_from_the_current_header():
    """cv-b200-sys/src/incorporate.rs is what scripts/gen_rust_sys.py produces from include/cvb200_incorporate.h, and the shim's
    incorporate.rs what it assembles from INTEGRATION.md section 2q; every symbol is declared once with the header's arity."""
    spec = importlib.util.spec_from_file_location("gen_rust_sys", os.path.join(ROOT, "scripts", "gen_rust_sys.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    header = open(HEADER).read()
    text, _ = gen.generate_incorporate(header)
    assert open(gen.INCORPORATE_OUT).read() == text, "stale: python scripts/gen_rust_sys.py"
    assert open(gen.INCORPORATE_SHIM_OUT).read() == gen.generate_shim_incorporate(), "stale: python scripts/gen_rust_sys.py"
    assert "pub mod incorporate;" in open(gen.OUT).read() and "pub mod incorporate;" in open(gen.SHIM_OUT).read()
    shim = open(gen.INCORPORATE_SHIM_OUT).read()
    assert "pub fn incorporate_frame(ctx: &Ctx" in shim and "pub fn apply_optimization(ctx: &Ctx" in shim
    assert '#[link(name = "cvb200_incorporate")]' in text and "pub struct cvb_incorporate_result {" in text
    assert "pub const CVB_INCORPORATE_NONE: u32 = 0xffffffff;" in text
    declared = re.findall(r"pub fn (cvb_\w+)\((.*?)\)(?: -> [^;]+)?;", text)
    assert sorted(n for n, _ in declared) == sorted(INCORPORATE_ABI_SYMBOLS)
    plain = gen.strip_comments(header)
    for name, params in declared:
        cargs = re.search(r"\b" + name + r"\s*\(([^;{]*?)\)\s*;", plain, flags=re.S).group(1)
        assert cargs.count(",") == params.count(","), name
    r = subprocess.run(["python", os.path.join(ROOT, "scripts", "gen_rust_sys.py"), "--check"], capture_output=True, text=True)
    assert r.returncode == 0 and "up to date" in r.stdout, r.stdout


def test_result_layouts():
    assert COUNTS_DTYPE == O_COUNTS and COUNTS_DTYPE.itemsize == 24
    assert RESULT_DTYPE.itemsize == 304
    assert [RESULT_DTYPE.fields[k][1] for k in ("counts", "reg", "reg_stats", "con", "recon", "reserved")] == [8, 32, 144, 256, 264, 296]


def test_incorporate_reports_no_device():
    _ensure_built()
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(cv_b200.CvbError) as e:
        cv_b200.Context(0)
    assert e.value.code == CVB_ENODEV


def test_python_entry_refuses_mismatched_new_frame():
    _ensure_built()

    class _Ctx:
        handle = None

    snap = dict(poses=np.zeros((1, 12)), view_offsets=[0, 0], view_landmarks=[], bearings=np.zeros((0, 3)),
                descriptors=np.zeros((0, 64), np.uint8), colors=None, landmark_offsets=[0], observations=np.zeros((0, 2)), constraints=None)
    with pytest.raises(ValueError):
        cv_b200.incorporate_frame(_Ctx(), snap, np.zeros((2, 64), np.uint8), np.zeros((1, 3)), [0], None)
