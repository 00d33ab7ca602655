"""ctypes binding of the CPU oracle of include/cvb200_init.h (oracle/ref_init.c in oracle/_build/libcvb_oracle_init.so, built by
oracle/init.mk): cv-sfm's init_reconstruction from the two-view options on (cv-sfm/src/lib.rs:986-1303), restated pair by pair.

TEST INFRASTRUCTURE ONLY, like oracle/pyoracle.py.  The inputs are host copies of what cvb_init_reconstruction_dev takes: bearings
[frames, cap, 3] f64, and per option f pairs [F, cap, 2], n_pairs [F], model [F, 12] (rotation row-major, translation), inliers [F, cap],
n_inliers [F], found [F].  `options_from_matches` builds them from plain per-option match lists.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from .pyoracle_tri import LINEAR_EIGEN, Triangulator, triangulator

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "libcvb_oracle_init.so")

NONE, ACCEPTED, NONE_BEARING_PAIRS = 0, 1, 2
(PAIR_NOT_EVALUATED, PAIR_ACCEPTED, PAIR_BEARING_PAIRS, PAIR_FEW_SCALES, PAIR_FEW_MATCHES, PAIR_HALF_MATCHES, PAIR_HALF_ROBUST,
 PAIR_FEW_ROBUST) = range(8)

POSE_DTYPE = np.dtype([("r", "<f8", (9,)), ("t", "<f8", (3,))])
RESULT_DTYPE = np.dtype([("status", "<i4"), ("pair", "<u4"), ("first", "<u4"), ("second", "<u4"), ("n_pairs", "<u4"), ("n_combined", "<u4"),
                         ("n_first_matches", "<u4"), ("n_second_matches", "<u4"), ("first_pose", POSE_DTYPE), ("second_pose", POSE_DTYPE)])
STATS_DTYPE = np.dtype([("outcome", "<i4"), ("first", "<u4"), ("second", "<u4"), ("scales", "<u4"), ("median_scale", "<f8"),
                        ("bearing_pairs", "<u8"), ("common", "<u4"), ("opti", "<u4"), ("updates", "<u4"), ("robust", "<u4")])


class InitCfg(C.Structure):
    """ref_init_cfg (== cvb_init_cfg), with cv-sfm's defaults (cv-sfm/src/settings.rs)"""
    _fields_ = [("robust_observation_incidence_minimum_cosine_distance", C.c_double),
                ("robust_view_bearing_pair_minimum_cosine_distance", C.c_double), ("maximum_cosine_distance", C.c_double),
                ("maximum_sine_distance", C.c_double), ("two_view_minimum_robust_matches", C.c_uint32),
                ("three_view_minimum_relative_scales", C.c_uint32), ("three_view_optimization_landmarks", C.c_uint32),
                ("robust_view_num_robust_bearing_pair", C.c_uint32), ("three_view_filter_loop_iterations", C.c_uint32),
                ("three_view_patience", C.c_uint32), ("three_view_minimum_robust_matches", C.c_uint32), ("reserved", C.c_uint32)]

    def __init__(self, **kw):
        d = dict(robust_observation_incidence_minimum_cosine_distance=1e-3, robust_view_bearing_pair_minimum_cosine_distance=1e-2,
                 maximum_cosine_distance=1e-5, maximum_sine_distance=0.1, two_view_minimum_robust_matches=256,
                 three_view_minimum_relative_scales=16, three_view_optimization_landmarks=1024, robust_view_num_robust_bearing_pair=3,
                 three_view_filter_loop_iterations=8, three_view_patience=65536, three_view_minimum_robust_matches=32)
        d.update(kw)
        super().__init__(**d)


_L = None


def build(force=False):
    srcs = [os.path.join(_HERE, f) for f in ("ref_init.c", "ref_triangulation.c", "ref_triangulation.h", "ref_geom.c", "ref_geom.h",
                                             "ref_optimize.c", "init.mk")]
    if not force and os.path.exists(_LIB_PATH) and all(os.path.getmtime(_LIB_PATH) >= os.path.getmtime(s) for s in srcs):
        return _LIB_PATH
    subprocess.check_call(["make", "-s", "-C", _HERE, "-f", "init.mk"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


def _lib():
    global _L
    if _L is None:
        build()
        L = C.CDLL(_LIB_PATH)
        vp, u32 = C.c_void_p, C.c_uint32
        L.ref_init_reconstruction.argtypes = [C.POINTER(InitCfg), C.POINTER(Triangulator), vp, u32, u32, vp, u32, vp, vp, vp, vp, vp, vp, vp,
                                              vp, vp, vp, vp]
        L.ref_init_reconstruction.restype = C.c_int
        _L = L
    return _L


def options_from_matches(F, cap, matches, poses, found=None):
    """Device-layout option arrays from per-option match lists: matches[f] = [[center feature, option feature], ...] (all inliers, in
    order), poses[f] = (R, t).  Returns (pairs, n_pairs, model, inliers, n_inliers, found)."""
    pairs = np.zeros((F, cap, 2), np.uint32)
    inl = np.zeros((F, cap), np.uint32)
    n = np.zeros(F, np.uint32)
    model = np.zeros((F, 12), np.float64)
    for f in range(F):
        m = np.asarray(matches[f], np.uint32).reshape(-1, 2)
        n[f] = len(m)
        pairs[f, :len(m)] = m
        inl[f, :len(m)] = np.arange(len(m))
        R, t = poses[f]
        model[f, :9] = np.asarray(R, np.float64).reshape(9)
        model[f, 9:] = np.asarray(t, np.float64)
    fnd = np.ones(F, np.int32) if found is None else np.asarray(found, np.int32)
    return pairs, n.copy(), model, inl, n, fnd


def init_reconstruction(bearings, center, options, pairs, n_pairs, model, inliers, n_inliers, found, cfg=None, tri=None):
    """Returns dict(result (RESULT_DTYPE record), combined [n, 3], first_matches [n, 2], second_matches [n, 2], stats [F(F-1)/2])."""
    bearings = np.ascontiguousarray(bearings, np.float64)
    frames, cap = bearings.shape[0], bearings.shape[1]
    opts = np.ascontiguousarray(options, np.uint32)
    F = len(opts)
    pairs = np.ascontiguousarray(pairs, np.uint32).reshape(max(F, 1) if F else 0, cap, 2) if F else np.zeros((1, cap, 2), np.uint32)
    n_pairs = np.ascontiguousarray(n_pairs, np.uint32) if F else np.zeros(1, np.uint32)
    model = np.ascontiguousarray(model, np.float64).reshape(-1, 12) if F else np.zeros((1, 12))
    inliers = np.ascontiguousarray(inliers, np.uint32).reshape(-1, cap) if F else np.zeros((1, cap), np.uint32)
    n_inliers = np.ascontiguousarray(n_inliers, np.uint32) if F else np.zeros(1, np.uint32)
    found = np.ascontiguousarray(found, np.int32) if F else np.zeros(1, np.int32)
    assert center < frames and all(o < frames for o in opts)
    cfg = cfg if cfg is not None else InitCfg()
    tri = tri if tri is not None else triangulator(LINEAR_EIGEN)
    res = np.zeros(1, RESULT_DTYPE)
    comb = np.zeros((cap, 3), np.uint32)
    fm = np.zeros((cap, 2), np.uint32)
    sm = np.zeros((cap, 2), np.uint32)
    stats = np.zeros(max(F * (F - 1) // 2, 1), STATS_DTYPE)
    rc = _lib().ref_init_reconstruction(C.byref(cfg), C.byref(tri), bearings.ctypes.data, cap, int(center),
                                        opts.ctypes.data if F else None, F, pairs.ctypes.data, n_pairs.ctypes.data, model.ctypes.data,
                                        inliers.ctypes.data, n_inliers.ctypes.data, found.ctypes.data, res.ctypes.data, comb.ctypes.data,
                                        fm.ctypes.data, sm.ctypes.data, stats.ctypes.data)
    assert rc == 0
    r = res[0]
    return dict(result=r, combined=comb[:r["n_combined"]].copy(), first_matches=fm[:r["n_first_matches"]].copy(),
                second_matches=sm[:r["n_second_matches"]].copy(), stats=stats[:F * (F - 1) // 2].copy())
