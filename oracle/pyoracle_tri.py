"""ctypes binding of the CPU oracle of include/cvb200_tri.h (oracle/ref_triangulation.c in oracle/_build/libcvb_oracle_tri.so, built by
oracle/tri.mk): the triangulators of cv-geom/src/triangulation.rs, and cv-sfm's observation losses / tri-landmark robustness with a
chosen triangulator.

TEST INFRASTRUCTURE ONLY, like oracle/pyoracle.py.  Poses are POSE_DTYPE arrays (rotation row-major, translation) or lists of (R, t).
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "libcvb_oracle_tri.so")

LINEAR_EIGEN, SINE_L1, MEAN_MEAN, RELATIVE_DLT, ANGULAR_L1, ANGULAR_LINF = range(6)
POSE_DTYPE = np.dtype([("r", "<f8", (9,)), ("t", "<f8", (3,))])


class Triangulator(C.Structure):
    """ref_triangulator (== cvb_triangulator)"""
    _fields_ = [("method", C.c_int32), ("max_iterations", C.c_uint32), ("epsilon", C.c_double), ("optimization_rate", C.c_double)]


_L = None


def build(force=False):
    srcs = [os.path.join(_HERE, f) for f in ("ref_triangulation.c", "ref_triangulation.h", "ref_geom.c", "ref_geom.h", "ref_optimize.c", "tri.mk")]
    if not force and os.path.exists(_LIB_PATH) and all(os.path.getmtime(_LIB_PATH) >= os.path.getmtime(s) for s in srcs):
        return _LIB_PATH
    subprocess.check_call(["make", "-s", "-C", _HERE, "-f", "tri.mk"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


def _lib():
    global _L
    if _L is None:
        build()
        L = C.CDLL(_LIB_PATH)
        vp, u32, f64, T = C.c_void_p, C.c_uint32, C.c_double, C.POINTER(Triangulator)
        L.ref_triangulator_default.argtypes = [T, C.c_int32]
        L.ref_triangulator_default.restype = None
        L.ref_triangulate_observations_batch.argtypes = [T, vp, vp, vp, u32, vp, vp, vp]
        L.ref_triangulate_observations_batch.restype = None
        L.ref_triangulate_relative_batch.argtypes = [T, vp, u32, vp, vp, u32, vp, vp]
        L.ref_triangulate_relative_batch.restype = None
        L.ref_observation_losses_tri.argtypes = [T, vp, vp, u32, vp]
        L.ref_observation_losses_tri.restype = None
        L.ref_is_tri_landmark_robust_tri.argtypes = [T, vp, vp, vp, vp, vp, f64, f64]
        _L = L
    return _L


def triangulator(method, epsilon=None, max_iterations=None, optimization_rate=None):
    """the reference's Default of `method`, with the given builder settings"""
    t = Triangulator()
    _lib().ref_triangulator_default(C.byref(t), method)
    if epsilon is not None:
        t.epsilon = epsilon
    if max_iterations is not None:
        t.max_iterations = max_iterations
    if optimization_rate is not None:
        t.optimization_rate = optimization_rate
    return t


def _poses(poses):
    if isinstance(poses, np.ndarray) and poses.dtype == POSE_DTYPE:
        return np.ascontiguousarray(poses)
    out = np.zeros(len(poses), POSE_DTYPE)
    for i, (R, t) in enumerate(poses):
        out[i]["r"] = np.asarray(R, np.float64).reshape(9)
        out[i]["t"] = np.asarray(t, np.float64).reshape(3)
    return out


def _f64(a, cols):
    return np.ascontiguousarray(np.asarray(a, np.float64).reshape(-1, cols))


def triangulate_observations_batch(tri, poses, bearings, offsets):
    """-> (xyzw[L, 4], ok[L] bool, SineL1 iterations[L] uint32)"""
    p = _poses(poses); b = _f64(bearings, 3); off = np.ascontiguousarray(offsets, np.uint32)
    L = len(off) - 1
    out = np.zeros((L, 4)); ok = np.zeros(L, np.uint8); it = np.zeros(L, np.uint32)
    _lib().ref_triangulate_observations_batch(C.byref(tri), p.ctypes.data, b.ctypes.data, off.ctypes.data, L, out.ctypes.data, ok.ctypes.data,
                                              it.ctypes.data)
    return out, ok.astype(bool), it


def triangulate_relative_batch(tri, poses, a, b):
    """poses: 1 or n CameraToCamera poses -> (xyzw[n, 4], ok[n] bool)"""
    p = _poses(poses); a = _f64(a, 3); b = _f64(b, 3)
    n = len(a)
    out = np.zeros((n, 4)); ok = np.zeros(n, np.uint8)
    _lib().ref_triangulate_relative_batch(C.byref(tri), p.ctypes.data, len(p), a.ctypes.data, b.ctypes.data, n, out.ctypes.data, ok.ctypes.data)
    return out, ok.astype(bool)


def triangulate_relative(tri, pose, a, b):
    out, ok = triangulate_relative_batch(tri, [pose], [a], [b])
    return out[0] if ok[0] else None


def observation_losses(tri, poses, bearings, offsets):
    """observation_loss of every observation of L landmarks, landmark by landmark"""
    p = _poses(poses); b = _f64(bearings, 3); off = np.asarray(offsets, np.int64)
    out = np.zeros(len(b))
    L = _lib()
    for l in range(len(off) - 1):
        o0, o1 = int(off[l]), int(off[l + 1])
        if o1 > o0:
            L.ref_observation_losses_tri(C.byref(tri), p[o0:o1].ctypes.data, b[o0:o1].ctypes.data, o1 - o0, out[o0:o1].ctypes.data)
    return out


def tri_landmarks_robust(tri, first_pose, second_pose, observations, max_cos, inc_min_cos):
    p = _poses([first_pose, second_pose]); o = _f64(observations, 9)
    L = _lib()
    return np.array([bool(L.ref_is_tri_landmark_robust_tri(C.byref(tri), p[0:1].ctypes.data, p[1:2].ctypes.data, o[i, 0:3].ctypes.data,
                                                           o[i, 3:6].ctypes.data, o[i, 6:9].ctypes.data, max_cos, inc_min_cos))
                     for i in range(len(o))], bool)
