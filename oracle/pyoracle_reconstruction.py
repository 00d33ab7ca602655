"""ctypes binding of the CPU oracle of include/cvb200_reconstruction.h (oracle/ref_reconstruction.c in
oracle/_build/libcvb_oracle_reconstruction.so, built by oracle/reconstruction.mk): cv-sfm's optimize_reconstruction
(cv-sfm/src/lib.rs:2343-2355), restated step by step.

TEST INFRASTRUCTURE ONLY, like oracle/pyoracle.py.  The inputs are those of cv_b200.optimize_reconstruction (host arrays); the outputs
are in the same form."""
import ctypes as C
import os
import subprocess

import numpy as np

from .pyoracle_tri import LINEAR_EIGEN, Triangulator, triangulator

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "libcvb_oracle_reconstruction.so")

POSE_DTYPE = np.dtype([("r", "<f8", (9,)), ("t", "<f8", (3,))])
CONSTRAINT_DTYPE = np.dtype([("views", "<u4", (3,)), ("landmarks", "<u4"), ("poses", POSE_DTYPE, (2,))])
RESULT_DTYPE = np.dtype([("status", "<i4"), ("round", "<u4"), ("step", "<u4"), ("views_removed", "<u4"), ("robust_before", "<u4"),
                         ("robust_after", "<u4"), ("observations_split", "<u4"), ("small_angle_updates", "<u4")])


class ReconCfg(C.Structure):
    """ref_recon_cfg (== cvb_recon_cfg), with cv-sfm's defaults (cv-sfm/src/settings.rs)"""
    _fields_ = [("graph_optimization_rate", C.c_double), ("maximum_sine_distance", C.c_double), ("maximum_cosine_distance", C.c_double),
                ("robust_observation_incidence_minimum_cosine_distance", C.c_double), ("optimization_iterations", C.c_uint32),
                ("reconstruction_optimization_iterations", C.c_uint32), ("robust_minimum_observations", C.c_uint32),
                ("minimum_robust_landmarks", C.c_uint32)]

    def __init__(self, **kw):
        d = dict(graph_optimization_rate=0.001, maximum_sine_distance=0.1, maximum_cosine_distance=1e-5,
                 robust_observation_incidence_minimum_cosine_distance=1e-3, optimization_iterations=1024,
                 reconstruction_optimization_iterations=1, robust_minimum_observations=3, minimum_robust_landmarks=32)
        d.update(kw)
        super().__init__(**d)


_L = None


def build(force=False):
    srcs = [os.path.join(_HERE, f) for f in ("ref_reconstruction.c", "ref_triangulation.c", "ref_triangulation.h", "ref_geom.c", "ref_geom.h",
                                             "ref_optimize.c", "reconstruction.mk")]
    if not force and os.path.exists(_LIB_PATH) and all(os.path.getmtime(_LIB_PATH) >= os.path.getmtime(s) for s in srcs):
        return _LIB_PATH
    subprocess.check_call(["make", "-s", "-C", _HERE, "-f", "reconstruction.mk"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


def _lib():
    global _L
    if _L is None:
        build()
        L = C.CDLL(_LIB_PATH)
        vp, u32 = C.c_void_p, C.c_uint32
        L.ref_optimize_reconstruction.argtypes = [C.POINTER(ReconCfg), C.POINTER(Triangulator), u32, vp, vp, vp, u32, vp, vp, vp, u32, vp, vp,
                                                  vp, vp, C.c_int]
        L.ref_optimize_reconstruction.restype = C.c_int
        _L = L
    return _L


def optimize_reconstruction(poses, view_offsets, bearings, landmark_offsets, observations, constraints, cfg=None, tri=None, threads=0):
    """Returns dict(result RESULT_DTYPE scalar, poses [V, 12], view_state uint8 [V], obs_state uint8 [n_observations]).  constraints: a
    CONSTRAINT_DTYPE array in the reconstruction's order.  threads: OpenMP threads over views and landmarks (0: OpenMP's default)."""
    cfg = cfg if cfg is not None else ReconCfg()
    tri = tri if tri is not None else triangulator(LINEAR_EIGEN)
    P = np.ascontiguousarray(poses, np.float64).reshape(-1, 12)
    u = (lambda a: np.ascontiguousarray(a, np.uint32).reshape(-1))
    vo, lo, ob = u(view_offsets), u(landmark_offsets), u(observations)
    bear = np.ascontiguousarray(bearings, np.float64).reshape(-1)
    cons = np.ascontiguousarray(constraints, CONSTRAINT_DTYPE).reshape(-1)
    V, Lm = len(vo) - 1, len(lo) - 1
    res = np.zeros(1, RESULT_DTYPE)
    pout = np.zeros((max(V, 1), 12))
    vs = np.zeros(max(V, 1), np.uint8)
    os_ = np.zeros(max(int(lo[-1]), 1), np.uint8)
    ptr = (lambda a: a.ctypes.data if a.size else None)
    rc = _lib().ref_optimize_reconstruction(C.byref(cfg), C.byref(tri), V, P.ctypes.data, ptr(vo), ptr(bear), Lm, ptr(lo), ptr(ob), ptr(cons),
                                            len(cons), res.ctypes.data, pout.ctypes.data, vs.ctypes.data, os_.ctypes.data, int(threads))
    assert rc == 0
    return dict(result=res[0], poses=pout[:V].copy(), view_state=vs[:V].copy(), obs_state=os_[:int(lo[-1])].copy())
