"""ctypes binding of the CPU oracle of include/cvb200_register.h (oracle/ref_register.c in oracle/_build/libcvb_oracle_register.so, built by
oracle/register.mk): cv-sfm's register_frame / register_frame_subset (cv-sfm/src/lib.rs:1452-1812), restated loop for loop.

TEST INFRASTRUCTURE ONLY, like oracle/pyoracle.py.  The inputs are those of cv_b200.register_frame (host arrays, an oracle ArrsacCfg and
Rng from oracle.pyoracle, advanced in place); the outputs are in the same form."""
import ctypes as C
import os
import subprocess

import numpy as np

from .pyoracle import ArrsacCfg, Rng
from .pyoracle_tri import LINEAR_EIGEN, Triangulator, triangulator

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "libcvb_oracle_register.so")

STATUS_NAMES = ["ok", "few_robust_landmarks", "no_consensus", "filter_half", "final_half", "final_robust_half", "few_matches", "panic"]
NONE = 0xFFFFFFFF
MATCH_DTYPE = np.dtype([("feature", "<u4"), ("landmark_a", "<u4"), ("landmark_b", "<u4")])
RESULT_DTYPE = np.dtype([("status", "<i4"), ("iteration", "<u4"), ("n_matches", "<u4"), ("n_inliers", "<u4"),
                         ("pose", [("r", "<f8", (9,)), ("t", "<f8", (3,))])])
STATS_DTYPE = np.dtype([("subsets", "<u4"), ("matches", "<u4"), ("claimed", "<u4"), ("matches_3d", "<u4"), ("inliers", "<u4"),
                        ("final_robust", "<u4"), ("final_matches", "<u4"), ("iterations", "<u4"), ("filter_matches", "<u4", (16,)),
                        ("final_stage_matches", "<u4"), ("reserved", "<u4", (3,))])


class RegisterCfg(C.Structure):
    """ref_register_cfg (== cvb_register_cfg), with cv-sfm's defaults (cv-sfm/src/settings.rs)"""
    _fields_ = [("single_view_optimization_rate", C.c_double), ("maximum_sine_distance", C.c_double),
                ("maximum_cosine_distance", C.c_double), ("robust_observation_incidence_minimum_cosine_distance", C.c_double),
                ("single_view_match_better_by", C.c_uint32), ("single_view_initial_features", C.c_uint32),
                ("single_view_minimum_landmarks", C.c_uint32), ("single_view_optimization_num_matches", C.c_uint32),
                ("single_view_filter_loop_iterations", C.c_uint32), ("single_view_patience", C.c_uint32),
                ("single_view_minimum_robust_landmarks", C.c_uint32), ("robust_minimum_observations", C.c_uint32)]

    def __init__(self, **kw):
        d = dict(single_view_optimization_rate=1e-3, maximum_sine_distance=0.1, maximum_cosine_distance=1e-5,
                 robust_observation_incidence_minimum_cosine_distance=1e-3, single_view_match_better_by=24,
                 single_view_initial_features=8192, single_view_minimum_landmarks=32, single_view_optimization_num_matches=2048,
                 single_view_filter_loop_iterations=5, single_view_patience=100000, single_view_minimum_robust_landmarks=64,
                 robust_minimum_observations=3)
        d.update(kw)
        super().__init__(**d)


_L = None


def build(force=False):
    srcs = [os.path.join(_HERE, f) for f in ("ref_register.c", "ref_match.c", "ref_triangulation.c", "ref_triangulation.h", "ref_geom.c",
                                             "ref_geom.h", "ref_optimize.c", "register.mk")]
    if not force and os.path.exists(_LIB_PATH) and all(os.path.getmtime(_LIB_PATH) >= os.path.getmtime(s) for s in srcs):
        return _LIB_PATH
    subprocess.check_call(["make", "-s", "-C", _HERE, "-f", "register.mk"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


def _lib():
    global _L
    if _L is None:
        build()
        L = C.CDLL(_LIB_PATH)
        vp, u32 = C.c_void_p, C.c_uint32
        L.ref_register_frame.argtypes = [C.POINTER(RegisterCfg), C.POINTER(Triangulator), C.POINTER(ArrsacCfg), C.POINTER(Rng), u32, vp, vp,
                                         vp, vp, vp, u32, vp, vp, vp, vp, u32, vp, u32, vp, vp, vp, vp]
        L.ref_register_frame.restype = C.c_int
        _L = L
    return _L


def _ptr(a):
    return a.ctypes.data if a.size else None


def register_frame(poses, view_offsets, view_landmarks, bearings, descriptors, landmark_offsets, observations, new_descriptors, new_bearings,
                   view_matches, arrsac_cfg, rng, cfg=None, tri=None):
    """dict(status name, result RESULT_DTYPE record, pose (R, t) or None, matches MATCH_DTYPE [n] ascending by feature, inliers (the last
    subset's consensus inliers, indices into its matches_3d), stats STATS_DTYPE record); rng (an oracle Rng) is advanced like the reference's generator."""
    cfg = cfg if cfg is not None else RegisterCfg()
    tri = tri if tri is not None else triangulator(LINEAR_EIGEN)
    u = (lambda a: np.ascontiguousarray(a, np.uint32).reshape(-1))
    P = np.ascontiguousarray(poses, np.float64).reshape(-1, 12)
    vo, vl, lo, ob, vm = u(view_offsets), u(view_landmarks), u(landmark_offsets), u(observations), u(view_matches)
    bear = np.ascontiguousarray(bearings, np.float64).reshape(-1)
    desc = np.ascontiguousarray(descriptors, np.uint8).reshape(-1)
    nd = np.ascontiguousarray(new_descriptors, np.uint8).reshape(-1, 64)
    nb = np.ascontiguousarray(new_bearings, np.float64).reshape(-1, 3)
    V, Lm, N = len(vo) - 1, len(lo) - 1, len(nd)
    res = np.zeros(1, RESULT_DTYPE)
    out = np.zeros(max(N, 1), MATCH_DTYPE)
    st = np.zeros(1, STATS_DTYPE)
    inl = np.zeros(max(N, 1), np.uint32)
    assert _lib().ref_register_frame(C.byref(cfg), C.byref(tri), C.byref(arrsac_cfg), C.byref(rng), V, _ptr(P), _ptr(vo), _ptr(vl), _ptr(bear),
                                     _ptr(desc), Lm, _ptr(lo), _ptr(ob), _ptr(nd), _ptr(nb), N, _ptr(vm), len(vm), res.ctypes.data,
                                     out.ctypes.data, inl.ctypes.data, st.ctypes.data) == 0
    r = res[0]
    status = STATUS_NAMES[int(r["status"])]
    pose = (r["pose"]["r"].reshape(3, 3).copy(), r["pose"]["t"].copy()) if status == "ok" else None
    return dict(status=status, result=r, pose=pose, matches=out[:int(r["n_matches"])].copy(), inliers=inl[:int(r["n_inliers"])].copy(),
                stats=st[0])
