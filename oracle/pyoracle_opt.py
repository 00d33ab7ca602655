"""ctypes binding of the CPU oracle of include/cvb200_opt.h (oracle/ref_optimize_l1.c in oracle/_build/libcvb_oracle_opt.so, built by
oracle/opt.mk): cv-optimize's L1 (Weiszfeld) pose optimizers, single_view_simple_optimize_l1 and three_view_simple_optimize_l1.

TEST INFRASTRUCTURE ONLY, like oracle/pyoracle.py.  Poses are (R[3,3], t[3]) pairs.  `order` picks the summation order of the
per-iteration sums: LANDMARK_ORDER (the reference's) or DEVICE_ORDER (the kernels').
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "libcvb_oracle_opt.so")

LANDMARK_ORDER, DEVICE_ORDER = 0, 1


class Pose(C.Structure):
    """ref_pose (== cvb_pose)"""
    _fields_ = [("R", C.c_double * 9), ("t", C.c_double * 3)]

    def numpy(self):
        return np.array(self.R, dtype=np.float64).reshape(3, 3), np.array(self.t, dtype=np.float64)


def _pose(R, t):
    p = Pose()
    p.R[:] = list(np.asarray(R, np.float64).reshape(9))
    p.t[:] = list(np.asarray(t, np.float64).reshape(3))
    return p


_L = None


def build(force=False):
    srcs = [os.path.join(_HERE, f) for f in ("ref_optimize_l1.c", "ref_optimize_l1.h", "ref_optimize.c", "ref_geom.c", "ref_geom.h", "opt.mk")]
    if not force and os.path.exists(_LIB_PATH) and all(os.path.getmtime(_LIB_PATH) >= os.path.getmtime(s) for s in srcs):
        return _LIB_PATH
    subprocess.check_call(["make", "-s", "-C", _HERE, "-f", "opt.mk"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


def _lib():
    global _L
    if _L is None:
        build()
        L = C.CDLL(_LIB_PATH)
        vp, u32, f64 = C.c_void_p, C.c_uint32, C.c_double
        L.ref_single_view_optimize_l1.argtypes = [C.POINTER(Pose), f64, f64, u32, vp, vp, u32, C.c_int]
        L.ref_single_view_optimize_l1.restype = u32
        L.ref_three_view_optimize_l1.argtypes = [C.POINTER(Pose), f64, f64, u32, vp, u32, C.c_int]
        L.ref_three_view_optimize_l1.restype = u32
        _L = L
    return _L


def single_view_optimize_l1(pose, epsilon, rate, iterations, bearings, world, order=LANDMARK_ORDER):
    """single_view_simple_optimize_l1 -> (R, t, pose updates applied); bearings[n, 3], world[n, 4] homogeneous"""
    p = _pose(*pose)
    b = np.ascontiguousarray(bearings, np.float64).reshape(-1, 3); w = np.ascontiguousarray(world, np.float64).reshape(-1, 4)
    if len(b) != len(w):
        raise ValueError("bearings / world disagree")
    upd = _lib().ref_single_view_optimize_l1(C.byref(p), epsilon, rate, iterations, b.ctypes.data, w.ctypes.data, len(b), order)
    R, t = p.numpy()
    return R, t, int(upd)


def three_view_optimize_l1(poses, epsilon, rate, iterations, obs, order=LANDMARK_ORDER):
    """three_view_simple_optimize_l1 -> ([(R, t) centre -> first, (R, t) centre -> second], pose updates applied); obs[n, 3, 3]"""
    arr = (Pose * 2)(_pose(*poses[0]), _pose(*poses[1]))
    o = np.ascontiguousarray(obs, np.float64).reshape(-1, 9)
    upd = _lib().ref_three_view_optimize_l1(arr, epsilon, rate, iterations, o.ctypes.data, len(o), order)
    return [arr[0].numpy(), arr[1].numpy()], int(upd)
