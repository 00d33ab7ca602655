"""CPU-only: include/cvb200_image.h (8- and 16-bit frames into the extractor) -- libcvb200_image.so exports exactly the symbols the header
declares, libcvb200.so's exports are unchanged, a C program calls every one of them, the generated Rust bindings match the header, and
without a CUDA device every entry point fails cleanly (no CPU fallback)."""
import importlib.util
import os
import re
import subprocess

import numpy as np
import pytest

import cv_b200
from cv_b200._lib import (ABI_SYMBOLS, IMAGE_ABI_SYMBOLS, OPT_ABI_SYMBOLS, PINHOLE_ABI_SYMBOLS, SFM_ABI_SYMBOLS, TRI_ABI_SYMBOLS,
                          image_lib_path)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "cvb200_image.h")


def _ensure_built():
    if not (os.path.exists(cv_b200.lib_path()) and os.path.exists(image_lib_path())):
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
    assert _declared() == set(IMAGE_ABI_SYMBOLS), _declared() ^ set(IMAGE_ABI_SYMBOLS)
    others = set(ABI_SYMBOLS) | set(SFM_ABI_SYMBOLS) | set(TRI_ABI_SYMBOLS) | set(OPT_ABI_SYMBOLS) | set(PINHOLE_ABI_SYMBOLS)
    assert not set(IMAGE_ABI_SYMBOLS) & others
    assert _exported(image_lib_path()) == set(IMAGE_ABI_SYMBOLS)
    assert _exported(cv_b200.lib_path()) == set(ABI_SYMBOLS) | set(SFM_ABI_SYMBOLS) | set(TRI_ABI_SYMBOLS)   # unchanged
    L = cv_b200._lib.load_image_library()
    for s in IMAGE_ABI_SYMBOLS:
        assert hasattr(L, s), s


def test_pixel_format_codes_match_the_python_and_oracle_tables():
    from cv_b200.image import FORMATS
    from oracle import pyoracle_image as OI
    codes = dict(re.findall(r"#define\s+CVB_PIXEL_([A-Z0-9_]+)\s+(\d+)", open(HEADER).read()))
    for kind, (code, ch, dt) in FORMATS.items():
        assert int(codes[kind.upper()]) == code
        assert OI.FORMATS[code] == (ch, dt)
    assert int(codes["RGB32F"]) == 8 and int(codes["RGBA32F"]) == 9


def _build_smoke():
    out = os.path.join(ROOT, "tests", "csrc", "_build")
    os.makedirs(out, exist_ok=True)
    exe = os.path.join(out, "abi_smoke_image")
    libdir = os.path.join(ROOT, "cv_b200")
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", os.path.join(ROOT, "tests", "csrc", "abi_smoke_image.c"),
                           "-I" + os.path.join(ROOT, "include"), "-L" + libdir, "-lcvb200_image", "-lcvb200", "-lm",
                           "-Wl,-rpath," + libdir, "-o", exe])
    return exe


def test_c_program_compiles_against_image_header_and_calls_every_entry_point():
    _ensure_built()
    exe = _build_smoke()
    src = open(os.path.join(ROOT, "tests", "csrc", "abi_smoke_image.c")).read()
    for sym in _declared():
        assert re.search(r"\b" + sym + r"\s*\(", src), f"{sym} is not called by abi_smoke_image.c"
    r = subprocess.run([exe, "0"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.gpu
def test_c_program_image_gpu_workflow():
    _ensure_built()
    r = subprocess.run([_build_smoke(), "1"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "GPU workflow ok" in r.stdout, r.stdout + r.stderr


def test_rust_image_bindings_are_generated_from_the_current_header():
    """cv-b200-sys/src/image.rs is what scripts/gen_rust_sys.py produces from include/cvb200_image.h, and the shim's dynamic.rs what it
    assembles from INTEGRATION.md section 2g; every symbol is declared once with the header's arity; the shim calls only declared externs."""
    spec = importlib.util.spec_from_file_location("gen_rust_sys", os.path.join(ROOT, "scripts", "gen_rust_sys.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    header = open(HEADER).read()
    text, _ = gen.generate_image(header)
    assert open(gen.IMAGE_OUT).read() == text, "stale: python scripts/gen_rust_sys.py"
    assert open(gen.IMAGE_SHIM_OUT).read() == gen.generate_shim_image(), "stale: python scripts/gen_rust_sys.py"
    assert open(gen.SHIM_OUT).read() == gen.generate_shim(), "stale: python scripts/gen_rust_sys.py"
    assert "pub mod image;" in open(gen.OUT).read() and "pub mod dynamic;" in open(gen.SHIM_OUT).read()
    assert '#[link(name = "cvb200_image")]' in text
    assert len(re.findall(r"pub const CVB_PIXEL_\w+: cvb_pixel_format = \d+;", text)) == 10
    declared = re.findall(r"pub fn (cvb_\w+)\((.*?)\)(?: -> [^;]+)?;", text)
    assert sorted(n for n, _ in declared) == sorted(IMAGE_ABI_SYMBOLS)
    plain = gen.strip_comments(header)
    for name, params in declared:
        cargs = re.search(r"\b" + name + r"\s*\(([^;{]*?)\)\s*;", plain, flags=re.S).group(1)
        assert cargs.count(",") == params.count(","), name
    shim = open(gen.IMAGE_SHIM_OUT).read()
    called = set(re.findall(r"\b(cvb_[a-z0-9_]+)\s*\(", shim))
    assert {"cvb_akaze_extract_dynamic_batch", "cvb_frame_features_dynamic_batch"} <= called
    assert called <= set(ABI_SYMBOLS) | set(SFM_ABI_SYMBOLS) | set(IMAGE_ABI_SYMBOLS)
    for f in ("pub fn extract_dynamic(", "pub fn kps_descriptors_dynamic(", "pub fn pixel_format("):
        assert f in shim, f


def test_new_entry_points_report_no_device():
    _ensure_built()
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from cv_b200._lib import CVB_ENODEV
    im = cv_b200.DynamicImage.luma8(np.zeros((32, 32), np.uint8))
    cam = cv_b200.CameraIntrinsicsK1Distortion(cv_b200.CameraIntrinsics((1000.0, 1000.0), (16.0, 16.0)), -0.28)
    for call in (lambda: cv_b200.Akaze().extract(im),
                 lambda: cv_b200.Akaze().extract_batch([im, im]),
                 lambda: cv_b200.frame_features(cv_b200.Akaze(), im, cam),
                 lambda: cv_b200.two_view_frames(cv_b200.Akaze(), [im, im], cam, cv_b200.Arrsac(1e-7, cv_b200.Xoshiro256PlusPlus(0)))):
        with pytest.raises(cv_b200.CvbError) as e:
            call()
        assert e.value.code == CVB_ENODEV
