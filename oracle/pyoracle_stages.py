"""ctypes binding of the CPU oracle of include/cvb200_stages.h's describe call (oracle/ref_stages.c in
oracle/_build/libcvb_oracle_stages.so, built by oracle/stages.mk): akaze's extract_descriptors at caller keypoints on the planes of
the extractor oracle's last extract, with full-range glibc sinf / cosf and Rust's saturating float -> isize cast.

TEST INFRASTRUCTURE ONLY, like oracle/pyoracle.py.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from . import pyoracle as O

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "libcvb_oracle_stages.so")

_L = None


def build(force=False):
    srcs = [os.path.join(_HERE, f) for f in ("ref_stages.c", "ref_libm.h", "ref_akaze.h", "stages.mk")]
    if not force and os.path.exists(_LIB_PATH) and all(os.path.getmtime(_LIB_PATH) >= os.path.getmtime(s) for s in srcs):
        return _LIB_PATH
    subprocess.check_call(["make", "-s", "-C", _HERE, "-f", "stages.mk"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


def _lib():
    global _L
    if _L is None:
        build()
        L = C.CDLL(_LIB_PATH)
        vp, i32 = C.c_void_p, C.c_int
        L.ref_describe.argtypes = [vp, vp, vp, vp, vp, i32, i32, i32, vp, i32, vp, vp, C.POINTER(i32)]
        L.ref_describe.restype = i32
        for f in ("ref_full_sinf", "ref_full_cosf"):
            getattr(L, f).argtypes = [C.c_float]
            getattr(L, f).restype = C.c_float
        _L = L
    return _L


def sinf(x):
    return np.float32(_lib().ref_full_sinf(float(np.float32(x))))


def cosf(x):
    return np.float32(_lib().ref_full_cosf(float(np.float32(x))))


def sincos_array(xs):
    """(sin, cos) of every float32 of xs, bit for bit as the oracle computes them."""
    xs = np.ascontiguousarray(xs, np.float32).reshape(-1)
    L = _lib()
    s = np.array([L.ref_full_sinf(float(v)) for v in xs], np.float32)
    c = np.array([L.ref_full_cosf(float(v)) for v in xs], np.float32)
    return s, c


def _plane_ptr(A, i, plane):
    return C.cast(O.lib().ref_akaze_plane(A._h, i, O.PLANES[plane]), C.c_void_p).value


def describe(A, keypoints, channels=3, pattern=10):
    """extract_descriptors(&evolutions, keypoints) on the planes of oracle extractor A's last extract: (kept keypoints in input
    order, [n, 64] uint8 descriptors).  Raises ValueError naming the first invalid keypoint (class_id >= E or octave >= 32)."""
    kps = np.ascontiguousarray(keypoints, dtype=O.KP_DTYPE).reshape(-1)
    E = A.num_evolutions()
    arrs = {p: (C.c_void_p * max(E, 1))(*[_plane_ptr(A, i, p) for i in range(E)]) for p in ("Lt", "Lx", "Ly")}
    info = [A.evolution_info(i) for i in range(E)]
    w = np.array([d["w"] for d in info] or [0], np.int32)
    h = np.array([d["h"] for d in info] or [0], np.int32)
    kp_out = np.zeros(max(len(kps), 1), O.KP_DTYPE)
    desc = np.zeros((max(len(kps), 1), 64), np.uint8)
    n = C.c_int()
    kin = kps if len(kps) else np.zeros(1, O.KP_DTYPE)
    rc = _lib().ref_describe(arrs["Lt"], arrs["Lx"], arrs["Ly"], w.ctypes.data, h.ctypes.data, E, channels, pattern, kin.ctypes.data,
                             len(kps), kp_out.ctypes.data, desc.ctypes.data, C.byref(n))
    if rc < 0:
        raise ValueError(f"invalid keypoint {-1 - rc}")
    return kp_out[:n.value].copy(), desc[:n.value].copy()
