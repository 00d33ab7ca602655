"""CPU-only: include/cvb200_stages.h (AKAZE's staged surface) -- libcvb200_stages.so exports exactly the symbols the header declares,
libcvb200.so's exports are unchanged, a C program calls every one of them, the generated Rust bindings match the header, the Python
wrappers reject bad input, and without a CUDA device the calls fail cleanly (no CPU fallback)."""
import importlib.util
import os
import re
import subprocess

import numpy as np
import pytest

import cv_b200
from cv_b200._lib import (ABI_SYMBOLS, CVB_ENODEV, EVOLUTION_DTYPE, FILTER_ABI_SYMBOLS, IMAGE_ABI_SYMBOLS, LSH_ABI_SYMBOLS,
                          OPT_ABI_SYMBOLS, PINHOLE_ABI_SYMBOLS, SFM_ABI_SYMBOLS, STAGES_ABI_SYMBOLS, TRI_ABI_SYMBOLS, stages_lib_path)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "cvb200_stages.h")


def _ensure_built():
    if not (os.path.exists(cv_b200.lib_path()) and os.path.exists(stages_lib_path())):
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
    assert _declared() == set(STAGES_ABI_SYMBOLS), _declared() ^ set(STAGES_ABI_SYMBOLS)
    others = (set(ABI_SYMBOLS) | set(SFM_ABI_SYMBOLS) | set(TRI_ABI_SYMBOLS) | set(OPT_ABI_SYMBOLS) | set(PINHOLE_ABI_SYMBOLS) |
              set(IMAGE_ABI_SYMBOLS) | set(FILTER_ABI_SYMBOLS) | set(LSH_ABI_SYMBOLS))
    assert not set(STAGES_ABI_SYMBOLS) & others
    assert _exported(stages_lib_path()) == set(STAGES_ABI_SYMBOLS)
    assert _exported(cv_b200.lib_path()) == set(ABI_SYMBOLS) | set(SFM_ABI_SYMBOLS) | set(TRI_ABI_SYMBOLS)   # unchanged
    L = cv_b200._lib.load_stages_library()
    for s in STAGES_ABI_SYMBOLS:
        assert hasattr(L, s), s


def test_evolution_struct_matches_the_python_dtype():
    body = re.search(r"typedef struct \{(.*?)\} cvb_akaze_evolution;", open(HEADER).read(), flags=re.S).group(1)
    fields = re.findall(r"\b(uint32_t|double)\s+(\w+);", body)
    assert [f for _, f in fields] == list(EVOLUTION_DTYPE.names)
    assert [{"uint32_t": "<u4", "double": "<f8"}[t] for t, _ in fields] == [EVOLUTION_DTYPE[n].str for n in EVOLUTION_DTYPE.names]
    assert EVOLUTION_DTYPE.itemsize == 40


def _build_smoke():
    out = os.path.join(ROOT, "tests", "csrc", "_build")
    os.makedirs(out, exist_ok=True)
    exe = os.path.join(out, "abi_smoke_stages")
    libdir = os.path.join(ROOT, "cv_b200")
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", os.path.join(ROOT, "tests", "csrc", "abi_smoke_stages.c"),
                           "-I" + os.path.join(ROOT, "include"), "-L" + libdir, "-lcvb200_stages", "-lcvb200", "-Wl,-rpath," + libdir,
                           "-lm", "-o", exe])
    return exe


def test_c_program_compiles_against_stages_header_and_calls_every_entry_point():
    _ensure_built()
    exe = _build_smoke()
    src = open(os.path.join(ROOT, "tests", "csrc", "abi_smoke_stages.c")).read()
    for sym in _declared():
        assert re.search(r"\b" + sym + r"\s*\(", src), f"{sym} is not called by abi_smoke_stages.c"
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: test_c_program_stages_gpu_workflow runs the program")
    r = subprocess.run([exe, "0"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.gpu
def test_c_program_stages_gpu_workflow():
    _ensure_built()
    r = subprocess.run([_build_smoke(), "1"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "GPU workflow ok" in r.stdout, r.stdout + r.stderr


def test_rust_stages_bindings_are_generated_from_the_current_header():
    """cv-b200-sys/src/stages.rs is what scripts/gen_rust_sys.py produces from include/cvb200_stages.h, and the shim's stages.rs what it
    assembles from INTEGRATION.md section 2j; every symbol is declared once with the header's arity; the shim keeps the reference's
    method signatures with CudaEvolutions in place of [EvolutionStep]."""
    spec = importlib.util.spec_from_file_location("gen_rust_sys", os.path.join(ROOT, "scripts", "gen_rust_sys.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    header = open(HEADER).read()
    text, _ = gen.generate_stages(header)
    assert open(gen.STAGES_OUT).read() == text, "stale: python scripts/gen_rust_sys.py"
    assert open(gen.STAGES_SHIM_OUT).read() == gen.generate_shim_stages(), "stale: python scripts/gen_rust_sys.py"
    assert open(gen.SHIM_OUT).read() == gen.generate_shim(), "stale: python scripts/gen_rust_sys.py"
    assert "pub mod stages;" in open(gen.OUT).read() and "pub mod stages;" in open(gen.SHIM_OUT).read()
    assert '#[link(name = "cvb200_stages")]' in text and "pub struct cvb_akaze_evolution {" in text
    declared = re.findall(r"pub fn (cvb_\w+)\((.*?)\)(?: -> [^;]+)?;", text)
    assert sorted(n for n, _ in declared) == sorted(STAGES_ABI_SYMBOLS)
    plain = gen.strip_comments(header)
    for name, params in declared:
        cargs = re.search(r"\b" + name + r"\s*\(([^;{]*?)\)\s*;", plain, flags=re.S).group(1)
        assert cargs.count(",") == params.count(","), name
    shim = open(gen.STAGES_SHIM_OUT).read()
    for f in ("pub struct CudaEvolutions",
              "pub fn create_scale_space(&self, img: &akaze::image::GrayFloatImage) -> CudaEvolutions",
              "pub fn find_image_keypoints(&self, evolutions: &mut CudaEvolutions) -> Vec<akaze::KeyPoint>",
              "pub fn extract_descriptors(&self, evolutions: &CudaEvolutions, keypoints: &[akaze::KeyPoint]) -> (Vec<akaze::KeyPoint>, Vec<BitArray<64>>)"):
        assert f in shim, f
    r = subprocess.run(["python", os.path.join(ROOT, "scripts", "gen_rust_sys.py"), "--check"], capture_output=True, text=True)
    assert r.returncode == 0 and "up to date" in r.stdout, r.stdout


def test_wrappers_check_types_and_shapes():
    ak = cv_b200.Akaze()
    with pytest.raises(TypeError):
        ak.create_scale_space(np.zeros((40, 40), np.float64))
    with pytest.raises(ValueError):
        ak.create_scale_space(np.zeros((1, 2, 40, 40), np.float32))


def test_scale_space_reports_no_device():
    _ensure_built()
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(cv_b200.CvbError) as e:
        cv_b200.Akaze().create_scale_space(np.zeros((64, 64), np.float32))
    assert e.value.code == CVB_ENODEV
