"""CPU-only: include/cvb200_try_init.h (cv-sfm's reconstruction creation) -- libcvb200_try_init.so exports exactly the symbols the header
declares, libcvb200.so's exports are unchanged, the result record matches the header's layout, and without a CUDA device the calls fail
cleanly.  The host validator's refusals are in tests/test_oracle_try_init.py."""
import os
import re
import subprocess

import pytest

import cv_b200
from cv_b200._lib import ABI_SYMBOLS, MERGE_ABI_SYMBOLS, SFM_ABI_SYMBOLS, TRI_ABI_SYMBOLS, TRY_INIT_ABI_SYMBOLS, CVB_ENODEV, try_init_lib_path
from cv_b200.try_init import RESULT_DTYPE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "cvb200_try_init.h")


def _ensure_built():
    if not (os.path.exists(cv_b200.lib_path()) and os.path.exists(try_init_lib_path())):
        import __graft_entry__ as g
        g.build()


def _exported(path):
    out = subprocess.run(["nm", "-D", "--defined-only", path], capture_output=True, text=True, check=True).stdout
    return {ln.split()[-1] for ln in out.splitlines() if re.search(r" T cvb_", ln)}


def test_library_exports_exactly_the_header_symbols():
    _ensure_built()
    plain = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    assert set(re.findall(r"\b(cvb_[a-z0-9_]+)\s*\(", plain)) == set(TRY_INIT_ABI_SYMBOLS)
    assert not set(TRY_INIT_ABI_SYMBOLS) & set(MERGE_ABI_SYMBOLS)
    assert _exported(try_init_lib_path()) == set(TRY_INIT_ABI_SYMBOLS)
    assert _exported(cv_b200.lib_path()) == set(ABI_SYMBOLS) | set(SFM_ABI_SYMBOLS) | set(TRI_ABI_SYMBOLS)   # unchanged
    L = cv_b200._lib.load_try_init_library()
    for s in TRY_INIT_ABI_SYMBOLS:
        assert hasattr(L, s), s


def test_c_program_compiles_against_the_header():
    _ensure_built()
    out = os.path.join(ROOT, "tests", "csrc", "_build")
    os.makedirs(out, exist_ok=True)
    src = os.path.join(out, "try_init_layout.c")
    with open(src, "w") as f:
        f.write('#include <stddef.h>\n#include <stdio.h>\n#include "cvb200_try_init.h"\nint main(void) {\n'
                '    printf("%zu %zu %zu %zu\\n", sizeof(cvb_try_init_result), offsetof(cvb_try_init_result, frames),\n'
                '           offsetof(cvb_try_init_result, init), offsetof(cvb_try_init_result, counts));\n'
                '    return cvb_try_init_check(1, 1, 1, 0, 0, 1, NULL, 0, NULL, 0, NULL, 0) == CVB_EINVAL ? 0 : 1;\n}\n')
    exe = os.path.join(out, "try_init_layout")
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", src, "-I" + os.path.join(ROOT, "include"),
                           "-L" + os.path.join(ROOT, "cv_b200"), "-lcvb200_try_init", "-lcvb200", "-Wl,-rpath," + os.path.join(ROOT, "cv_b200"),
                           "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stdout + r.stderr
    sizes = [int(x) for x in r.stdout.split()]
    assert sizes == [RESULT_DTYPE.itemsize] + [RESULT_DTYPE.fields[k][1] for k in ("frames", "init", "counts")]


def _build_smoke():
    out = os.path.join(ROOT, "tests", "csrc", "_build")
    os.makedirs(out, exist_ok=True)
    exe = os.path.join(out, "abi_smoke_try_init")
    libdir = os.path.join(ROOT, "cv_b200")
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", os.path.join(ROOT, "tests", "csrc", "abi_smoke_try_init.c"),
                           "-I" + os.path.join(ROOT, "include"), "-L" + libdir, "-lcvb200_try_init", "-lcvb200_init",
                           "-lcvb200", "-Wl,-rpath," + libdir, "-lm", "-o", exe])
    return exe


def test_c_program_calls_every_entry_point():
    _ensure_built()
    exe = _build_smoke()
    src = open(os.path.join(ROOT, "tests", "csrc", "abi_smoke_try_init.c")).read()
    for sym in TRY_INIT_ABI_SYMBOLS:
        assert re.search(r"\b" + sym + r"\s*\(", src), f"{sym} is not called by abi_smoke_try_init.c"
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: test_c_program_try_init_gpu_workflow runs the program")
    r = subprocess.run([exe, "0"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.gpu
def test_c_program_try_init_gpu_workflow():
    _ensure_built()
    r = subprocess.run([_build_smoke(), "1"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr


def test_rust_try_init_bindings_are_generated_from_the_current_header():
    """cv-b200-sys/src/try_init.rs is what scripts/gen_rust_sys.py produces from include/cvb200_try_init.h, and the shim's try_init.rs what
    it assembles from INTEGRATION.md section 2s; every symbol is declared once with the header's arity."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("gen_rust_sys", os.path.join(ROOT, "scripts", "gen_rust_sys.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    header = open(HEADER).read()
    text, _ = gen.generate_try_init(header)
    assert open(gen.TRY_INIT_OUT).read() == text, "stale: python scripts/gen_rust_sys.py"
    assert open(gen.TRY_INIT_SHIM_OUT).read() == gen.generate_shim_try_init(), "stale: python scripts/gen_rust_sys.py"
    assert "pub mod try_init;" in open(gen.OUT).read() and "pub mod try_init;" in open(gen.SHIM_OUT).read()
    assert "pub fn try_init(ctx: &Ctx" in open(gen.TRY_INIT_SHIM_OUT).read()
    assert '#[link(name = "cvb200_try_init")]' in text and "pub struct cvb_try_init_result {" in text
    assert "pub const CVB_TRY_INIT_NO_FRAME: u32 = 0xffffffff;" in text
    declared = re.findall(r"pub fn (cvb_\w+)\((.*?)\)(?: -> [^;]+)?;", text)
    assert sorted(n for n, _ in declared) == sorted(TRY_INIT_ABI_SYMBOLS)
    plain = gen.strip_comments(header)
    for name, params in declared:
        cargs = re.search(r"\b" + name + r"\s*\(([^;{]*?)\)\s*;", plain, flags=re.S).group(1)
        assert cargs.count(",") == params.count(","), name


def test_layout():
    assert RESULT_DTYPE.itemsize == 264 and RESULT_DTYPE.fields["init"][1] == 16 and RESULT_DTYPE.fields["counts"][1] == 240


def test_try_init_reports_no_device():
    _ensure_built()
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(cv_b200.CvbError) as e:
        cv_b200.Context(0)
    assert e.value.code == CVB_ENODEV
