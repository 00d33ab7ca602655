"""ctypes binding of the CPU oracle of include/cvb200_filter.h (oracle/ref_filter.c in oracle/_build/libcvb_oracle_filter.so, built by
oracle/filter.mk): akaze::image's horizontal / vertical / separable filters with their zero-weighted tail taps, and gaussian_blur over
them.  gaussian_kernel and half_size are oracle/pyoracle.py's (oracle/ref_akaze.c).

TEST INFRASTRUCTURE ONLY, like oracle/pyoracle.py.  Images are float32 [H, W] or batches [B, H, W]; each plane is filtered on its own.
"""
import ctypes as C
import math
import os
import subprocess

import numpy as np

from . import pyoracle as O

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "libcvb_oracle_filter.so")

_L = None


def build(force=False):
    srcs = [os.path.join(_HERE, f) for f in ("ref_filter.c", "filter.mk")]
    if not force and os.path.exists(_LIB_PATH) and all(os.path.getmtime(_LIB_PATH) >= os.path.getmtime(s) for s in srcs):
        return _LIB_PATH
    subprocess.check_call(["make", "-s", "-C", _HERE, "-f", "filter.mk"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


def _lib():
    global _L
    if _L is None:
        build()
        L = C.CDLL(_LIB_PATH)
        vp = C.c_void_p
        for f in (L.ref_filter_horizontal, L.ref_filter_vertical):
            f.argtypes = [vp, C.c_int, C.c_int, vp, C.c_int, vp]
        _L = L
    return _L


def _planes(fn, img, kernel):
    img = np.ascontiguousarray(img, np.float32)
    k = np.ascontiguousarray(kernel, np.float32).reshape(-1)
    flat = img.reshape((-1,) + img.shape[-2:])
    out = np.empty_like(flat)
    h, w = flat.shape[1:]
    for b in range(len(flat)):
        assert fn(flat[b].ctypes.data, w, h, k.ctypes.data, len(k), out[b].ctypes.data) == 0
    return out.reshape(img.shape)


def horizontal_filter(img, kernel):
    return _planes(_lib().ref_filter_horizontal, img, kernel)


def vertical_filter(img, kernel):
    return _planes(_lib().ref_filter_vertical, img, kernel)


def separable_filter(img, h_kernel, v_kernel):
    """image.rs:333-340: H, rounded to f32, then V"""
    return vertical_filter(horizontal_filter(img, h_kernel), v_kernel)


def gaussian_kernel(r, ks):
    return O.gaussian_kernel(np.float32(r), ks)


def blur_size(r):
    """image.rs:385-386 in f32: 2 * ceil(2 r) + 1"""
    return 2 * int(math.ceil(np.float32(2.0) * np.float32(r))) + 1


def gaussian_blur(img, r):
    k = gaussian_kernel(r, blur_size(r))
    return separable_filter(img, k, k)


def half_size(img):
    img = np.ascontiguousarray(img, np.float32)
    flat = img.reshape((-1,) + img.shape[-2:])
    out = np.stack([O.half_size(p) for p in flat])
    return out.reshape(img.shape[:-2] + out.shape[-2:])
