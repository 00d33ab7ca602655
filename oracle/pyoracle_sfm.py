"""ctypes binding of the CPU oracle of include/cvb200_sfm.h (oracle/_build/libcvb_oracle_sfm.so, built by oracle/sfm.mk): the camera with
radial distortion (cv-pinhole CameraIntrinsicsK1Distortion) and cv-sfm's per-frame feature ingestion (VSlam::kps_descriptors).

TEST INFRASTRUCTURE ONLY, like oracle/pyoracle.py, whose AKAZE extractor kps_descriptors runs.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "libcvb_oracle_sfm.so")
_lib = None


def build(force=False):
    srcs = [os.path.join(_HERE, f) for f in ("ref_sfm.c", "sfm.mk")]
    if not force and os.path.exists(_LIB_PATH) and all(os.path.getmtime(_LIB_PATH) >= os.path.getmtime(s) for s in srcs):
        return _LIB_PATH
    subprocess.check_call(["make", "-s", "-C", _HERE, "-f", "sfm.mk"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB_PATH)
        dp = C.POINTER(C.c_double)
        L.ref_calibrate_k1.argtypes = [C.c_double] * 8 + [dp]
        L.ref_uncalibrate_k1.argtypes = [C.c_double] * 6 + [dp, dp]
        L.ref_bicubic_rgb8.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_float, C.c_void_p]
        L.ref_kps_features.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, dp, dp, C.c_void_p]
        _lib = L
    return _lib


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def calibrate_k1(fx, fy, cx, cy, skew, k1, px, py):
    """CameraIntrinsicsK1Distortion::calibrate (cv-pinhole/src/lib.rs:191-202)"""
    out = np.zeros(3)
    lib().ref_calibrate_k1(fx, fy, cx, cy, skew, k1, px, py, _dp(out))
    return out


def uncalibrate_k1(fx, fy, cx, cy, skew, k1, bearing):
    """CameraIntrinsicsK1Distortion::uncalibrate (cv-pinhole/src/lib.rs:224-239): pixel (2,) or None"""
    b = np.ascontiguousarray(bearing, np.float64)
    out = np.zeros(2)
    return out if lib().ref_uncalibrate_k1(fx, fy, cx, cy, skew, k1, _dp(b), _dp(out)) else None


def bicubic_rgb8(rgb, x, y):
    """cv-sfm/src/bicubic.rs interpolate_bicubic on an [h, w, 3] u8 image at (x, y) f32 -> (3,) u8, black outside the border rule"""
    rgb = np.ascontiguousarray(rgb, np.uint8)
    out = np.zeros(3, np.uint8)
    lib().ref_bicubic_rgb8(rgb.ctypes.data, rgb.shape[1], rgb.shape[0], float(np.float32(x)), float(np.float32(y)), out.ctypes.data)
    return out


def kps_descriptors(akaze, image, rgb, K):
    """VSlam::kps_descriptors (cv-sfm/src/lib.rs:2195-2235) on the oracle extractor (a pyoracle.Akaze): image [h, w] f32 luma,
    rgb [h, w, 3] u8, K = (fx, fy, cx, cy, skew, k1).  Returns (keypoints, descriptors, bearings [n, 3], responses [n],
    colors [n, 3] u8) in AKAZE's order, which is the reference's order after its unstable sort by descending response."""
    kps, desc = akaze.extract(image)
    rgb = np.ascontiguousarray(rgb, np.uint8)
    xy = np.ascontiguousarray(np.stack([kps["x"], kps["y"]], 1), np.float32)
    Kd = np.ascontiguousarray(K, np.float64)
    bearings = np.zeros((len(kps), 3)); colors = np.zeros((len(kps), 3), np.uint8)
    lib().ref_kps_features(xy.ctypes.data, len(kps), rgb.ctypes.data, rgb.shape[1], rgb.shape[0], _dp(Kd), _dp(bearings), colors.ctypes.data)
    return kps, desc, bearings, kps["response"].copy(), colors
