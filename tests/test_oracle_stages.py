"""CPU-only: the numerics behind include/cvb200_stages.h's describe call at caller keypoints.

- Full-range sin / cos: the oracle's (oracle/ref_stages.c) and the device source's (cv_b200/csrc/device_libm.cuh, compiled as host
  code) equal the host glibc sinf / cosf bit for bit on samples from every binade of both signs, subnormals, +-0, +-inf and NaN.
  (scripts/sweep_sincos.py checks all 2^32 inputs of both against the host libm: 0 mismatches; these samples keep it so.)
- The describe oracle on the extractor oracle's sorted keypoints reproduces the extractor oracle's keypoints and descriptors.
- NaN-coordinate, NaN-angle, huge-angle and rounding-tie keypoints match a NumPy restatement of get_mldb_descriptor
  (descriptors.rs:55-202) that rounds half away from zero and uses Rust's saturating float -> isize cast.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import pyoracle as O
from oracle import pyoracle_stages as OS
from tests.common import kitti_frame

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIBM = C.CDLL("libm.so.6")
for _f in ("sinf", "cosf"):
    getattr(_LIBM, _f).argtypes = [C.c_float]
    getattr(_LIBM, _f).restype = C.c_float


def _libm(xs):
    return (np.array([_LIBM.sinf(float(v)) for v in xs], np.float32), np.array([_LIBM.cosf(float(v)) for v in xs], np.float32))


def _samples():
    rng = np.random.default_rng(7)
    bits = []
    for e in range(256):   # every binade (255: inf / NaN) with its end points and random mantissas
        mant = np.concatenate([[0, 1, 0x7fffff, 0x400000], rng.integers(0, 1 << 23, 28)]).astype(np.uint32)
        bits.append((np.uint32(e) << np.uint32(23)) | mant)
    bits = np.concatenate(bits)
    bits = np.concatenate([bits, bits | np.uint32(0x80000000)])
    extra = np.array([120.0, -120.0, 119.99999, 1e6, 1e30, 360.0, 2 * np.pi, np.pi, 1.5707964], np.float32).view(np.uint32)
    return np.concatenate([bits, extra]).view(np.float32)


def _same(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.all((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b)))


def test_oracle_sin_cos_equal_host_libm_over_the_whole_range():
    xs = _samples()
    s, c = OS.sincos_array(xs)
    hs, hc = _libm(xs)
    assert _same(s, hs) and _same(c, hc)
    assert np.isnan(s[np.isinf(xs)]).all() and np.isnan(c[np.isnan(xs)]).all()


def test_device_sin_cos_compiled_for_the_host_equal_host_libm():
    out = os.path.join(ROOT, "tests", "csrc", "_build")
    os.makedirs(out, exist_ok=True)
    exe = os.path.join(out, "dlm_host")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc, "-std=c++17", "-O2", "-Xcompiler", "-ffp-contract=off", "-o", exe,
                           os.path.join(ROOT, "tests", "csrc", "dlm_host.cu")])
    xs = _samples()
    r = subprocess.run([exe], input=xs.tobytes(), capture_output=True, check=True)
    got = np.frombuffer(r.stdout, np.float32).reshape(-1, 2)
    hs, hc = _libm(xs)
    assert _same(got[:, 0], hs) and _same(got[:, 1], hc)


@pytest.fixture(scope="module")
def kitti():
    A = O.Akaze(detector_threshold=0.01)
    kps, desc = A.extract(kitti_frame("0000000000"))
    return A, kps, desc


def test_describe_of_sorted_keypoints_reproduces_extract(kitti):
    A, kps, desc = kitti
    got_k, got_d = OS.describe(A, A.stage("sorted"))
    assert got_k.tobytes() == kps.tobytes() and np.array_equal(got_d, desc) and len(desc) == 399


def test_describe_rejects_invalid_keypoints(kitti):
    A, kps, _ = kitti
    bad = kps[:3].copy()
    bad["class_id"][1] = A.num_evolutions()
    with pytest.raises(ValueError, match="invalid keypoint 1"):
        OS.describe(A, bad)
    bad = kps[:3].copy()
    bad["octave"][2] = 32
    with pytest.raises(ValueError, match="invalid keypoint 2"):
        OS.describe(A, bad)


def _as_isize(v):
    v = np.float32(v)
    if np.isnan(v):
        return 0
    if v >= np.float32(2.0 ** 63):
        return 2 ** 63 - 1
    if v <= np.float32(-2.0 ** 63):
        return -2 ** 63
    return int(v)


def _round_away(v):
    """f32::round: half away from zero (np.round rounds half to even); exact through float64 for every float32"""
    v = float(v)
    return np.float32(np.copysign(np.floor(abs(v) + 0.5), v))


def _mldb_numpy(planes, kp, nch=3, pattern=10, rnd=_round_away):
    """get_mldb_descriptor (descriptors.rs:55-202) in float32 scalar steps; None when a sample leaves the level."""
    f = np.float32
    Lt, Lx, Ly = planes[int(kp["class_id"])]
    H, W = Lt.shape
    ratio = f(1 << int(kp["octave"]))
    scale = f(rnd(f(0.5) * kp["size"] / ratio))
    xf, yf = f(kp["x"] / ratio), f(kp["y"] / ratio)
    co, si = f(_LIBM.cosf(float(kp["angle"]))), f(_LIBM.sinf(float(kp["angle"])))
    bits = []
    with np.errstate(all="ignore"):
        for mult in (f(1.0), f(2.0) / f(3.0), f(1.0) / f(2.0)):
            step = int(np.ceil(f(pattern) * mult))
            vals = []
            for i in range(-pattern, pattern, step):
                for j in range(-pattern, pattern, step):
                    di = dx = dy = f(0)
                    ns = 0
                    for k in range(i, i + step):
                        for l in range(j, j + step):
                            lf, kf = f(l), f(k)
                            sy = yf + (lf * co * scale + kf * si * scale)
                            sx = xf + (-lf * si * scale + kf * co * scale)
                            y1, x1 = _as_isize(rnd(sy)), _as_isize(rnd(sx))
                            if not (0 <= x1 < W and 0 <= y1 < H):
                                return None
                            di = f(di + Lt[y1, x1])
                            rx, ry = Lx[y1, x1], Ly[y1, x1]
                            if nch == 2:
                                dx = f(dx + np.sqrt(rx * rx + ry * ry))
                            elif nch == 3:
                                dx = f(dx + (-rx * si + ry * co))
                                dy = f(dy + (rx * co + ry * si))
                            ns += 1
                    vals.append((di / f(ns), dx / f(ns), dy / f(ns)))
            for pos in range(nch):
                for a in range(len(vals)):
                    for b in range(a + 1, len(vals)):
                        bits.append(1 if vals[a][pos] > vals[b][pos] else 0)
    out = np.zeros(512, np.uint8)
    out[:len(bits)] = bits
    return np.packbits(out, bitorder="little")


def test_caller_keypoints_match_a_numpy_restatement_with_rusts_cast(kitti):
    A, kps, _ = kitti
    planes = [(A.plane(i, "Lt"), A.plane(i, "Lx"), A.plane(i, "Ly")) for i in range(A.num_evolutions())]
    base = kps[np.argsort(-kps["size"])[:2]]
    cases = []
    for kp in base:
        for field, v in (("x", np.nan), ("y", np.nan), ("angle", np.nan), ("angle", np.inf), ("angle", 1e6), ("angle", 1e30),
                         ("angle", -1e30), ("angle", 200.0), ("size", np.nan), ("x", np.inf), ("y", -np.inf)):
            k = kp.copy()
            k[field] = v
            cases.append(k)
    cases = np.array(cases, O.KP_DTYPE)
    got_k, got_d = OS.describe(A, cases)
    want = [(k, d) for k in cases for d in [_mldb_numpy(planes, k)] if d is not None]
    assert got_k.tobytes() == np.array([k for k, _ in want], O.KP_DTYPE).tobytes()
    assert np.array_equal(got_d, np.array([d for _, d in want]).reshape(-1, 64))
    kept = {(int(np.isnan(k["x"])), int(np.isnan(k["angle"]))) for k in got_k}
    assert (1, 0) in kept and (0, 1) in kept   # NaN positions read row / column 0 and are kept
    assert not np.isinf(got_k["x"]).any() and not np.isinf(got_k["y"]).any()


def test_rounding_ties_go_away_from_zero(kitti):
    """angle 0 and positions / scales at exact .5: every sample position is a tie, as is 0.5 * size; f32::round takes them away from
    zero, and the restatement with half-to-even rounding gives other descriptors, so these cases tell the two apart"""
    A, _, _ = kitti
    planes = [(A.plane(i, "Lt"), A.plane(i, "Lx"), A.plane(i, "Ly")) for i in range(A.num_evolutions())]
    ties = np.zeros(6, O.KP_DTYPE)
    ties["x"] = [100.5, 101.5, 200.5, 300.0, 64.5, 65.5]
    ties["y"] = [80.5, 81.5, 120.0, 150.5, 90.5, 91.5]
    ties["size"] = [5.0, 5.0, 7.0, 6.0, 4.0, 9.0]
    got_k, got_d = OS.describe(A, ties)
    assert got_k.tobytes() == ties.tobytes()
    want = np.array([_mldb_numpy(planes, k) for k in ties])
    assert np.array_equal(got_d, want)
    half_even = np.array([_mldb_numpy(planes, k, rnd=lambda v: np.float32(np.round(v))) for k in ties])
    assert not np.array_equal(half_even, want)
