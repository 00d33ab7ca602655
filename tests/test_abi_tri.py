"""CPU-only: include/cvb200_tri.h (cv-geom's triangulators) -- the library exports exactly the symbols it declares, a C program calls every
one of them, the struct layout matches, the generated Rust bindings match the header, and without a CUDA device every new entry point
fails cleanly (no CPU fallback)."""
import ctypes as C
import importlib.util
import os
import re
import subprocess

import numpy as np
import pytest

import cv_b200
from cv_b200._lib import ABI_SYMBOLS, SFM_ABI_SYMBOLS, TRI_ABI_SYMBOLS, load_library

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "cvb200_tri.h")


def _ensure_built():
    if not os.path.exists(cv_b200.lib_path()):
        import __graft_entry__ as g
        g.build()


def _declared():
    plain = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return set(re.findall(r"\b(cvb_[a-z0-9_]+)\s*\(", plain))


def _exported():
    out = subprocess.run(["nm", "-D", "--defined-only", cv_b200.lib_path()], capture_output=True, text=True, check=True).stdout
    return {ln.split()[-1] for ln in out.splitlines() if re.search(r" T cvb_", ln)}


def test_library_exports_exactly_the_header_symbols():
    _ensure_built()
    L = load_library()
    assert _declared() == set(TRI_ABI_SYMBOLS), _declared() ^ set(TRI_ABI_SYMBOLS)
    assert not set(TRI_ABI_SYMBOLS) & (set(ABI_SYMBOLS) | set(SFM_ABI_SYMBOLS))
    for s in TRI_ABI_SYMBOLS:
        assert hasattr(L, s), s
    # every exported cvb_ symbol is declared by one of the three headers
    assert _exported() == set(ABI_SYMBOLS) | set(SFM_ABI_SYMBOLS) | set(TRI_ABI_SYMBOLS)


def _build_smoke():
    out = os.path.join(ROOT, "tests", "csrc", "_build")
    os.makedirs(out, exist_ok=True)
    exe = os.path.join(out, "abi_smoke_tri")
    libdir = os.path.join(ROOT, "cv_b200")
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", os.path.join(ROOT, "tests", "csrc", "abi_smoke_tri.c"),
                           "-I" + os.path.join(ROOT, "include"), "-L" + libdir, "-lcvb200", "-lm", "-Wl,-rpath," + libdir, "-o", exe])
    return exe


def test_c_program_compiles_against_tri_header_and_calls_every_entry_point():
    _ensure_built()
    exe = _build_smoke()
    src = open(os.path.join(ROOT, "tests", "csrc", "abi_smoke_tri.c")).read()
    for sym in _declared():
        assert re.search(r"\b" + sym + r"\s*\(", src), f"{sym} is not called by abi_smoke_tri.c"
    r = subprocess.run([exe, "0"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.gpu
def test_c_program_tri_gpu_workflow():
    _ensure_built()
    r = subprocess.run([_build_smoke(), "1"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "GPU workflow ok" in r.stdout, r.stdout + r.stderr


def test_triangulator_layout_and_defaults_match_header():
    from cv_b200.triangulation import TriangulatorCfg
    text = open(HEADER).read()
    body = re.search(r"typedef struct \{([^}]*)\} cvb_triangulator;", text).group(1)
    assert re.findall(r"\w+", re.sub(r"int32_t|uint32_t|double", "", body)) == [f for f, _ in TriangulatorCfg._fields_] == \
        ["method", "max_iterations", "epsilon", "optimization_rate"]
    assert C.sizeof(TriangulatorCfg) == 24 and TriangulatorCfg.epsilon.offset == 8
    consts = dict((k, int(v)) for k, v in re.findall(r"#define\s+(CVB_TRI_\w+)\s+(\d+)", text))
    classes = [cv_b200.LinearEigenTriangulator, cv_b200.SineL1Triangulator, cv_b200.MeanMeanTriangulator, cv_b200.RelativeDltTriangulator,
               cv_b200.AngularL1Triangulator, cv_b200.AngularLInfinityTriangulator]
    assert [c.method for c in classes] == [consts[k] for k in ("CVB_TRI_LINEAR_EIGEN", "CVB_TRI_SINE_L1", "CVB_TRI_MEAN_MEAN",
                                                                "CVB_TRI_RELATIVE_DLT", "CVB_TRI_ANGULAR_L1", "CVB_TRI_ANGULAR_LINF")]
    # the Python defaults are the library's (and the reference's Default impls)
    _ensure_built()
    L = load_library()
    L.cvb_triangulator_default.argtypes = [C.POINTER(TriangulatorCfg), C.c_int32]
    L.cvb_triangulator_default.restype = None
    for cls in classes:
        want = TriangulatorCfg()
        L.cvb_triangulator_default(C.byref(want), cls.method)
        assert bytes(cls().cfg) == bytes(want), cls
    s = cv_b200.SineL1Triangulator().cfg
    assert (s.epsilon, s.max_iterations, s.optimization_rate) == (1e-12, 1000, 1.0)
    # relative-only classes have only the relative methods
    assert not hasattr(cv_b200.AngularL1Triangulator(), "triangulate_batch")
    assert hasattr(cv_b200.MeanMeanTriangulator(), "triangulate_relative_batch")


def test_rust_tri_bindings_are_generated_from_the_current_header():
    """cv-b200-sys/src/tri.rs is what scripts/gen_rust_sys.py produces from include/cvb200_tri.h, and the shim's tri.rs what it assembles
    from INTEGRATION.md section 2d; every symbol and #define is declared once; the shim calls only declared externs."""
    spec = importlib.util.spec_from_file_location("gen_rust_sys", os.path.join(ROOT, "scripts", "gen_rust_sys.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    header = open(HEADER).read()
    text, _ = gen.generate_tri(header)
    assert open(gen.TRI_OUT).read() == text, "stale: python scripts/gen_rust_sys.py"
    assert open(gen.TRI_SHIM_OUT).read() == gen.generate_shim_tri(), "stale: python scripts/gen_rust_sys.py"
    assert "pub mod tri;" in open(gen.OUT).read() and "mod tri;" in open(gen.SHIM_OUT).read()
    declared = re.findall(r"pub fn (cvb_\w+)\((.*?)\)(?: -> [^;]+)?;", text)
    assert sorted(n for n, _ in declared) == sorted(TRI_ABI_SYMBOLS)
    plain = gen.strip_comments(header)
    for name, params in declared:
        cargs = re.search(r"\b" + name + r"\s*\(([^;{]*?)\)\s*;", plain, flags=re.S).group(1)
        assert cargs.count(",") == params.count(","), name
    for k, v in re.findall(r"#define\s+(CVB_TRI_\w+)\s+(\d+)", header):
        assert f"pub const {k}: i32 = {v};" in text, k
    body = re.search(r"pub struct cvb_triangulator \{(.*?)\n\}", text, flags=re.S).group(1)
    assert re.findall(r"pub (\w+):", body) == ["method", "max_iterations", "epsilon", "optimization_rate"]
    shim = open(gen.TRI_SHIM_OUT).read()
    called = set(re.findall(r"\b(cvb_[a-z0-9_]+)\s*\(", shim))
    assert {"cvb_triangulate_observations", "cvb_triangulate_relative"} <= called <= set(ABI_SYMBOLS) | set(TRI_ABI_SYMBOLS)


def test_new_entry_points_report_no_device():
    _ensure_built()
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from cv_b200._lib import CVB_ENODEV
    eye = (np.eye(3), np.zeros(3))
    for call in (lambda: cv_b200.SineL1Triangulator().triangulate_batch([eye, eye], np.eye(3)[:2], [0, 2]),
                 lambda: cv_b200.AngularL1Triangulator().triangulate_relative(eye, np.eye(3)[2], np.eye(3)[2]),
                 lambda: cv_b200.observation_losses([eye] * 3, np.eye(3), [0, 3], triangulator=cv_b200.MeanMeanTriangulator())):
        with pytest.raises(cv_b200.CvbError) as e:
            call()
        assert e.value.code == CVB_ENODEV
