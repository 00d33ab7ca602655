"""ctypes binding of the CPU oracle of include/cvb200_pinhole.h (oracle/ref_pinhole.c in oracle/_build/libcvb_oracle_pinhole.so, built by
oracle/pinhole.mk): cv-pinhole's pose reprojection error over any relative triangulator, and the EssentialMatrix model (from_matches,
residual, recondition, possible_rotations_unscaled_translation).

TEST INFRASTRUCTURE ONLY, like oracle/pyoracle.py.  Triangulators are oracle.pyoracle_tri.Triangulator; poses are POSE_DTYPE arrays or
lists of (R, t); matrices are [m, 3, 3].  Rows the reference returns None for have ok = False and hold NaN.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from .pyoracle_tri import Triangulator, _f64, _poses

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "libcvb_oracle_pinhole.so")

_L = None


def build(force=False):
    srcs = [os.path.join(_HERE, f) for f in ("ref_pinhole.c", "ref_pinhole.h", "ref_triangulation.c", "ref_triangulation.h", "ref_geom.c",
                                             "ref_geom.h", "ref_optimize.c", "pinhole.mk")]
    if not force and os.path.exists(_LIB_PATH) and all(os.path.getmtime(_LIB_PATH) >= os.path.getmtime(s) for s in srcs):
        return _LIB_PATH
    subprocess.check_call(["make", "-s", "-C", _HERE, "-f", "pinhole.mk"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


def _lib():
    global _L
    if _L is None:
        build()
        L = C.CDLL(_LIB_PATH)
        vp, u32, f64, i32, T = C.c_void_p, C.c_uint32, C.c_double, C.c_int, C.POINTER(Triangulator)
        L.ref_pose_reprojection_error_batch.argtypes = [T, vp, u32, vp, vp, u32, vp, vp, vp]
        L.ref_pose_reprojection_error_batch.restype = None
        L.ref_eight_point_essential_batch.argtypes = [vp, vp, vp, u32, f64, i32, vp, vp]
        L.ref_eight_point_essential_batch.restype = None
        L.ref_residuals_essential.argtypes = [vp, u32, vp, vp, u32, vp]
        L.ref_residuals_essential.restype = None
        L.ref_essential_recondition_batch.argtypes = [vp, u32, f64, i32, vp, vp]
        L.ref_essential_recondition_batch.restype = None
        L.ref_essential_decompose_batch.argtypes = [vp, u32, f64, i32, vp, vp, vp, vp]
        L.ref_essential_decompose_batch.restype = None
        _L = L
    return _L


def _sweeps(iterations):
    return min(int(iterations), 0x7fffffff)


def _mats(E):
    return np.ascontiguousarray(np.asarray(E, np.float64).reshape(-1, 9))


def pose_reprojection_error_batch(tri, poses, a, b):
    """poses: 1 or n CameraToCamera poses -> (err[n, 4] (a.x a.y b.x b.y), avg[n], ok[n] bool)"""
    p = _poses(poses); a = _f64(a, 3); b = _f64(b, 3)
    n = len(a)
    err = np.zeros((n, 4)); avg = np.zeros(n); ok = np.zeros(n, np.uint8)
    _lib().ref_pose_reprojection_error_batch(C.byref(tri), p.ctypes.data, len(p), a.ctypes.data, b.ctypes.data, n, err.ctypes.data,
                                             avg.ctypes.data, ok.ctypes.data)
    return err, avg, ok.astype(bool)


def eight_point_essential_batch(a, b, samples, epsilon=1e-12, iterations=1000):
    """EightPoint { epsilon, iterations }::from_matches per sample of 8 indices -> (E[H, 3, 3], ok[H] bool)"""
    a = _f64(a, 3); b = _f64(b, 3); s = np.ascontiguousarray(samples, np.uint32).reshape(-1, 8)
    E = np.zeros((len(s), 9)); ok = np.zeros(len(s), np.uint8)
    _lib().ref_eight_point_essential_batch(a.ctypes.data, b.ctypes.data, s.ctypes.data, len(s), epsilon, _sweeps(iterations), E.ctypes.data,
                                           ok.ctypes.data)
    return E.reshape(-1, 3, 3), ok.astype(bool)


def residuals_essential(Es, a, b):
    """EssentialMatrix::residual of every (E, match) -> [m, n]"""
    E = _mats(Es); a = _f64(a, 3); b = _f64(b, 3)
    out = np.zeros((len(E), len(a)))
    _lib().ref_residuals_essential(E.ctypes.data, len(E), a.ctypes.data, b.ctypes.data, len(a), out.ctypes.data)
    return out


def essential_recondition_batch(Es, epsilon, max_iterations):
    """EssentialMatrix::recondition -> (E[m, 3, 3], ok[m] bool)"""
    E = _mats(Es)
    out = np.zeros((len(E), 9)); ok = np.zeros(len(E), np.uint8)
    _lib().ref_essential_recondition_batch(E.ctypes.data, len(E), epsilon, _sweeps(max_iterations), out.ctypes.data, ok.ctypes.data)
    return out.reshape(-1, 3, 3), ok.astype(bool)


def essential_decompose_batch(Es, epsilon, max_iterations):
    """possible_rotations_unscaled_translation -> (rot_a[m, 3, 3], rot_b[m, 3, 3], t[m, 3], ok[m] bool)"""
    E = _mats(Es)
    m = len(E)
    ra = np.zeros((m, 9)); rb = np.zeros((m, 9)); t = np.zeros((m, 3)); ok = np.zeros(m, np.uint8)
    _lib().ref_essential_decompose_batch(E.ctypes.data, m, epsilon, _sweeps(max_iterations), ra.ctypes.data, rb.ctypes.data, t.ctypes.data,
                                         ok.ctypes.data)
    return ra.reshape(-1, 3, 3), rb.reshape(-1, 3, 3), t, ok.astype(bool)
