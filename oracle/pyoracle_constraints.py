"""ctypes binding of the CPU oracle of include/cvb200_constraints.h (oracle/ref_constraints.c in
oracle/_build/libcvb_oracle_constraints.so, built by oracle/constraints.mk): cv-sfm's generate_view_constraints and record_view_constraints'
acceptance (cv-sfm/src/lib.rs:2092-2109, 2438-2516), restated one query at a time.

TEST INFRASTRUCTURE ONLY, like oracle/pyoracle.py.  The inputs are those of cv_b200.generate_view_constraints (host arrays); the outputs
are in the same form."""
import ctypes as C
import os
import subprocess

import numpy as np

from .pyoracle_tri import LINEAR_EIGEN, Triangulator, triangulator

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "libcvb_oracle_constraints.so")

POSE_DTYPE = np.dtype([("r", "<f8", (9,)), ("t", "<f8", (3,))])
CONSTRAINT_DTYPE = np.dtype([("views", "<u4", (3,)), ("landmarks", "<u4"), ("poses", POSE_DTYPE, (2,))])
RESULT_DTYPE = np.dtype([("n_constraints", "<u4"), ("accepted", "<i4")])
STATS_DTYPE = np.dtype([("robust_landmarks", "<u4"), ("coviews", "<u4"), ("triples", "<u4"), ("unique_triples", "<u4"), ("candidates", "<u4"),
                        ("few_landmarks", "<u4"), ("few_bearing_pairs", "<u4"), ("updates", "<u4")])


class ConstraintsCfg(C.Structure):
    """ref_constraints_cfg (== cvb_constraints_cfg), with cv-sfm's defaults (cv-sfm/src/settings.rs)"""
    _fields_ = [("robust_observation_incidence_minimum_cosine_distance", C.c_double),
                ("robust_view_bearing_pair_minimum_cosine_distance", C.c_double), ("robust_minimum_observations", C.c_uint32),
                ("robust_view_num_robust_bearing_pair", C.c_uint32), ("optimization_robust_covisibility_minimum_landmarks", C.c_uint32),
                ("optimization_minimum_landmarks", C.c_uint32), ("optimization_maximum_landmarks", C.c_uint32),
                ("optimization_maximum_three_view_constraints", C.c_uint32), ("optimization_minimum_new_constraints", C.c_uint32),
                ("constraint_patience", C.c_uint32)]

    def __init__(self, **kw):
        d = dict(robust_observation_incidence_minimum_cosine_distance=1e-3, robust_view_bearing_pair_minimum_cosine_distance=1e-2,
                 robust_minimum_observations=3, robust_view_num_robust_bearing_pair=3, optimization_robust_covisibility_minimum_landmarks=16,
                 optimization_minimum_landmarks=24, optimization_maximum_landmarks=64, optimization_maximum_three_view_constraints=64,
                 optimization_minimum_new_constraints=4, constraint_patience=4096)
        d.update(kw)
        super().__init__(**d)


_L = None


def build(force=False):
    srcs = [os.path.join(_HERE, f) for f in ("ref_constraints.c", "ref_triangulation.c", "ref_triangulation.h", "ref_geom.c", "ref_geom.h",
                                             "ref_optimize.c", "constraints.mk")]
    if not force and os.path.exists(_LIB_PATH) and all(os.path.getmtime(_LIB_PATH) >= os.path.getmtime(s) for s in srcs):
        return _LIB_PATH
    subprocess.check_call(["make", "-s", "-C", _HERE, "-f", "constraints.mk"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


def _lib():
    global _L
    if _L is None:
        build()
        L = C.CDLL(_LIB_PATH)
        vp, u32 = C.c_void_p, C.c_uint32
        L.ref_view_constraints.argtypes = [C.POINTER(ConstraintsCfg), C.POINTER(Triangulator), u32, vp, vp, vp, vp, u32, vp, vp, vp, u32, vp,
                                           vp, vp, C.c_int]
        L.ref_view_constraints.restype = C.c_int
        _L = L
    return _L


def view_constraints(poses, view_offsets, view_landmarks, bearings, landmark_offsets, observations, queries, cfg=None, tri=None, threads=0):
    """Returns dict(constraints (per query, CONSTRAINT_DTYPE), results RESULT_DTYPE [Q], stats STATS_DTYPE [Q]).  threads: OpenMP
    threads over landmarks and queries (0: OpenMP's default)."""
    cfg = cfg if cfg is not None else ConstraintsCfg()
    tri = tri if tri is not None else triangulator(LINEAR_EIGEN)
    P = np.ascontiguousarray(poses, np.float64).reshape(-1, 12)
    u = (lambda a: np.ascontiguousarray(a, np.uint32).reshape(-1))
    vo, vl, lo, ob, q = u(view_offsets), u(view_landmarks), u(landmark_offsets), u(observations), u(queries)
    bear = np.ascontiguousarray(bearings, np.float64).reshape(-1)
    Q, maxc = len(q), cfg.optimization_maximum_three_view_constraints
    out = np.zeros(max(Q * maxc, 1), CONSTRAINT_DTYPE)
    res = np.zeros(max(Q, 1), RESULT_DTYPE)
    st = np.zeros(max(Q, 1), STATS_DTYPE)
    ptr = (lambda a: a.ctypes.data if a.size else None)
    rc = _lib().ref_view_constraints(C.byref(cfg), C.byref(tri), len(vo) - 1, P.ctypes.data, ptr(vo), ptr(vl), ptr(bear), len(lo) - 1, ptr(lo),
                                     ptr(ob), ptr(q), Q, out.ctypes.data, res.ctypes.data, st.ctypes.data, int(threads))
    assert rc == 0
    res = res[:Q].copy()
    return dict(constraints=[out[i * maxc:i * maxc + res[i]["n_constraints"]].copy() for i in range(Q)], results=res, stats=st[:Q].copy())
