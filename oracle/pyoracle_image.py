"""ctypes binding of the CPU oracle of include/cvb200_image.h (oracle/ref_image.c in oracle/_build/libcvb_oracle_image.so, built by
oracle/image.mk): GrayFloatImage::from_dynamic of the eight integer DynamicImage variants and DynamicImage::to_rgb8() of the 8-bit ones.

TEST INFRASTRUCTURE ONLY, like oracle/pyoracle.py.  Pixels are numpy arrays of the format's dtype with the channels last ([..., H, W]
for luma, [..., H, W, C] otherwise); the result has the leading shape without the channel axis.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "libcvb_oracle_image.so")

# cvb_pixel_format codes: (channels, dtype)
FORMATS = {0: (1, np.uint8), 1: (2, np.uint8), 2: (3, np.uint8), 3: (4, np.uint8),
           4: (1, np.uint16), 5: (2, np.uint16), 6: (3, np.uint16), 7: (4, np.uint16)}

_L = None


def build(force=False):
    srcs = [os.path.join(_HERE, f) for f in ("ref_image.c", "ref_image.h", "image.mk")]
    if not force and os.path.exists(_LIB_PATH) and all(os.path.getmtime(_LIB_PATH) >= os.path.getmtime(s) for s in srcs):
        return _LIB_PATH
    subprocess.check_call(["make", "-s", "-C", _HERE, "-f", "image.mk"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


def _lib():
    global _L
    if _L is None:
        build()
        L = C.CDLL(_LIB_PATH)
        vp = C.c_void_p
        L.ref_rgb_to_luma.argtypes = [C.c_uint32] * 3
        L.ref_rgb_to_luma.restype = C.c_uint32
        L.ref_from_dynamic.argtypes = [C.c_uint32, vp, C.c_size_t, vp]
        L.ref_to_rgb8.argtypes = [C.c_uint32, vp, C.c_size_t, vp]
        _L = L
    return _L


def _pixels(fmt, pixels):
    ch, dt = FORMATS[fmt]
    p = np.ascontiguousarray(pixels)
    if p.dtype != dt:
        raise TypeError(f"format {fmt} takes {np.dtype(dt).name}")
    shape = p.shape if ch == 1 else p.shape[:-1]
    if ch > 1 and p.shape[-1] != ch:
        raise ValueError(f"format {fmt} takes {ch} channels")
    return p, shape


def rgb_to_luma(r, g, b):
    return int(_lib().ref_rgb_to_luma(int(r), int(g), int(b)))


def from_dynamic(fmt, pixels):
    p, shape = _pixels(fmt, pixels)
    out = np.empty(shape, np.float32)
    assert _lib().ref_from_dynamic(fmt, p.ctypes.data, out.size, out.ctypes.data) == 0
    return out


def to_rgb8(fmt, pixels):
    if fmt > 3:
        raise ValueError("to_rgb8 is restated for the 8-bit formats only")
    p, shape = _pixels(fmt, pixels)
    out = np.empty(shape + (3,), np.uint8)
    assert _lib().ref_to_rgb8(fmt, p.ctypes.data, int(np.prod(shape)), out.ctypes.data) == 0
    return out
