"""CPU-only: include/cvb200_batch.h (batched device ARRSAC) -- libcvb200_batch.so exports exactly the symbols the header declares,
libcvb200.so's exports are unchanged, a C program calls every one of them, the generated Rust bindings match the header, and without a
CUDA device the calls fail cleanly (no CPU fallback).  Also the host logic of Arrsac.model_inliers_batch: CSR packing and argument
checks."""
import importlib.util
import os
import re
import subprocess

import numpy as np
import pytest

import cv_b200
from cv_b200._lib import (ABI_SYMBOLS, ARRSAC_BATCH_MAX, BATCH_ABI_SYMBOLS, CVB_ENODEV, FILTER_ABI_SYMBOLS, IMAGE_ABI_SYMBOLS,
                          LSH_ABI_SYMBOLS, OPT_ABI_SYMBOLS, PINHOLE_ABI_SYMBOLS, SFM_ABI_SYMBOLS, STAGES_ABI_SYMBOLS, TRI_ABI_SYMBOLS,
                          batch_lib_path)
from cv_b200.geom import pack_arrsac_batch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "cvb200_batch.h")


def _ensure_built():
    if not (os.path.exists(cv_b200.lib_path()) and os.path.exists(batch_lib_path())):
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
    assert _declared() == set(BATCH_ABI_SYMBOLS), _declared() ^ set(BATCH_ABI_SYMBOLS)
    others = (set(ABI_SYMBOLS) | set(SFM_ABI_SYMBOLS) | set(TRI_ABI_SYMBOLS) | set(OPT_ABI_SYMBOLS) | set(PINHOLE_ABI_SYMBOLS) |
              set(IMAGE_ABI_SYMBOLS) | set(FILTER_ABI_SYMBOLS) | set(LSH_ABI_SYMBOLS) | set(STAGES_ABI_SYMBOLS))
    assert not set(BATCH_ABI_SYMBOLS) & others
    assert _exported(batch_lib_path()) == set(BATCH_ABI_SYMBOLS)
    assert _exported(cv_b200.lib_path()) == set(ABI_SYMBOLS) | set(SFM_ABI_SYMBOLS) | set(TRI_ABI_SYMBOLS)   # unchanged
    L = cv_b200._lib.load_batch_library()
    for s in BATCH_ABI_SYMBOLS:
        assert hasattr(L, s), s


def test_batch_maximum_matches_the_header():
    m = re.search(r"#define CVB_ARRSAC_BATCH_MAX (\d+)", open(HEADER).read())
    assert int(m.group(1)) == ARRSAC_BATCH_MAX >= 64


def _build_smoke():
    out = os.path.join(ROOT, "tests", "csrc", "_build")
    os.makedirs(out, exist_ok=True)
    exe = os.path.join(out, "abi_smoke_batch")
    libdir = os.path.join(ROOT, "cv_b200")
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", os.path.join(ROOT, "tests", "csrc", "abi_smoke_batch.c"),
                           "-I" + os.path.join(ROOT, "include"), "-L" + libdir, "-lcvb200_batch", "-lcvb200", "-Wl,-rpath," + libdir,
                           "-lm", "-o", exe])
    return exe


def test_c_program_compiles_against_batch_header_and_calls_every_entry_point():
    _ensure_built()
    exe = _build_smoke()
    src = open(os.path.join(ROOT, "tests", "csrc", "abi_smoke_batch.c")).read()
    for sym in _declared():
        assert re.search(r"\b" + sym + r"\s*\(", src), f"{sym} is not called by abi_smoke_batch.c"
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: test_c_program_batch_gpu_workflow runs the program")
    r = subprocess.run([exe, "0"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.gpu
def test_c_program_batch_gpu_workflow():
    _ensure_built()
    r = subprocess.run([_build_smoke(), "1"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "GPU workflow ok" in r.stdout, r.stdout + r.stderr


def test_rust_batch_bindings_are_generated_from_the_current_header():
    """cv-b200-sys/src/batch.rs is what scripts/gen_rust_sys.py produces from include/cvb200_batch.h, and the shim's batch.rs what it
    assembles from INTEGRATION.md section 2k; every symbol is declared once with the header's arity."""
    spec = importlib.util.spec_from_file_location("gen_rust_sys", os.path.join(ROOT, "scripts", "gen_rust_sys.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    header = open(HEADER).read()
    text, _ = gen.generate_batch(header)
    assert open(gen.BATCH_OUT).read() == text, "stale: python scripts/gen_rust_sys.py"
    assert open(gen.BATCH_SHIM_OUT).read() == gen.generate_shim_batch(), "stale: python scripts/gen_rust_sys.py"
    assert "pub mod batch;" in open(gen.OUT).read() and "pub mod batch;" in open(gen.SHIM_OUT).read()
    assert "pub fn model_inliers_batch(&mut self, _e: &eight_point::EightPoint, problems: &[Vec<FeatureMatch>], rngs: &mut [cvb_rng])" in \
        open(gen.BATCH_SHIM_OUT).read()
    assert '#[link(name = "cvb200_batch")]' in text and "pub const CVB_ARRSAC_BATCH_MAX: u32 = 64;" in text
    declared = re.findall(r"pub fn (cvb_\w+)\((.*?)\)(?: -> [^;]+)?;", text)
    assert sorted(n for n, _ in declared) == sorted(BATCH_ABI_SYMBOLS)
    plain = gen.strip_comments(header)
    for name, params in declared:
        cargs = re.search(r"\b" + name + r"\s*\(([^;{]*?)\)\s*;", plain, flags=re.S).group(1)
        assert cargs.count(",") == params.count(","), name
    r = subprocess.run(["python", os.path.join(ROOT, "scripts", "gen_rust_sys.py"), "--check"], capture_output=True, text=True)
    assert r.returncode == 0 and "up to date" in r.stdout, r.stdout


def test_csr_packing_keeps_each_problems_rows_in_order():
    rng = np.random.default_rng(0)
    probs = [(rng.normal(size=(n, 3)), rng.normal(size=(n, 3))) for n in (5, 0, 12, 1)]
    kind, row0, a, b, offs = pack_arrsac_batch(cv_b200.EightPoint(), probs)
    assert (kind, row0) == (0, 5) and offs.dtype == np.uint32 and list(offs) == [0, 5, 5, 17, 18]
    for i, (pa, pb) in enumerate(probs):
        assert np.array_equal(a[offs[i]:offs[i + 1]], pa) and np.array_equal(b[offs[i]:offs[i + 1]], pb)
    kind, row0, a, b, offs = pack_arrsac_batch(cv_b200.NisterStewenius(corrected=True), probs)
    assert (kind, row0) == (2, 6)
    w = [(rng.normal(size=(4, 3)), rng.normal(size=(4, 4)))]
    kind, row0, a, b, offs = pack_arrsac_batch(cv_b200.LambdaTwist(), w)
    assert kind == 1 and b.shape == (4, 4) and list(offs) == [0, 4]


def test_packing_rejects_bad_problems():
    rng = np.random.default_rng(1)
    with pytest.raises(ValueError):
        pack_arrsac_batch(cv_b200.EightPoint(), [(rng.normal(size=(5, 3)), rng.normal(size=(4, 3)))])     # row counts differ
    with pytest.raises(ValueError):
        pack_arrsac_batch(cv_b200.LambdaTwist(), [(rng.normal(size=(5, 3)), rng.normal(size=(5, 3)))])    # world points need 4 columns
    with pytest.raises(TypeError):
        pack_arrsac_batch(object(), [])


def test_batch_reports_no_device():
    _ensure_built()
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(cv_b200.CvbError) as e:
        cv_b200.Arrsac(1e-6, cv_b200.Xoshiro256PlusPlus(0))
    assert e.value.code == CVB_ENODEV


def test_two_view_option_result_applies_the_minimum_robust_matches_rule():
    from cv_b200.pair import TWO_VIEW_MINIMUM_ROBUST_MATCHES, two_view_option_result
    assert TWO_VIEW_MINIMUM_ROBUST_MATCHES == 256                      # cv-sfm's default (settings.rs:393-395)
    pairs = np.arange(20, dtype=np.uint32).reshape(10, 2)            # 10 matches (center, option)
    inl = np.array([1, 4, 7, 0, 0], np.uint32)
    R, t = np.eye(3).ravel(), np.array([1.0, 0.0, 0.0])
    r = two_view_option_result(pairs, 10, R, t, inl, 3, 1, 3)
    assert np.array_equal(r[2], [[2, 3], [8, 9], [14, 15]]) and r[2].dtype == np.int64 and np.array_equal(r[0], np.eye(3))
    assert two_view_option_result(pairs, 10, R, t, inl, 3, 1, 4) is None          # fewer inliers than the minimum: None
    assert two_view_option_result(pairs, 10, R, t, inl, 3, 0, 0) is None          # no consensus: None


def test_init_two_view_options_checks_its_tensors():
    import torch
    feats = dict(descriptors=torch.zeros((3, 8, 64), dtype=torch.uint8), counts=torch.zeros(3, dtype=torch.int32),
                 bearings=torch.zeros((3, 8, 3), dtype=torch.float64))
    with pytest.raises(ValueError):
        cv_b200.init_two_view_options(feats, 0, [1, 2], None, [None, None])      # host tensors: the call works on device tensors
