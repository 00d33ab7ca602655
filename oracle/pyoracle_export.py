"""ctypes binding of the CPU oracle of include/cvb200_export.h (oracle/ref_export.c in oracle/_build/libcvb_oracle_export.so, built by
oracle/export.mk): cv-sfm's triangulate_landmark_robust, normalize_reconstruction and export_reconstruction (cv-sfm/src/lib.rs:2241-2340,
2907-3000), restated loop for loop.

TEST INFRASTRUCTURE ONLY, like oracle/pyoracle.py.  The inputs are those of cv_b200.robust_landmarks, cv_b200.normalize_reconstruction and
cv_b200.export_reconstruction (host arrays); the outputs are in the same form."""
import ctypes as C
import os
import subprocess

import numpy as np

from .pyoracle_reconstruction import CONSTRAINT_DTYPE
from .pyoracle_tri import LINEAR_EIGEN, Triangulator, triangulator

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "libcvb_oracle_export.so")

CAMERA_DTYPE = np.dtype([("optical_center", "<f8", (3,)), ("up_direction", "<f8", (3,)), ("forward_direction", "<f8", (3,)),
                         ("focal_length", "<f8")])
NORMALIZE_RESULT_DTYPE = np.dtype([("normalized", "<i4"), ("robust_points", "<u4"), ("mean_distance", "<f8")])


class ExportCfg(C.Structure):
    """ref_export_cfg (== cvb_export_cfg), with cv-sfm's defaults (cv-sfm/src/settings.rs)"""
    _fields_ = [("robust_observation_incidence_minimum_cosine_distance", C.c_double), ("robust_minimum_observations", C.c_uint32)]

    def __init__(self, **kw):
        d = dict(robust_observation_incidence_minimum_cosine_distance=1e-3, robust_minimum_observations=3)
        d.update(kw)
        super().__init__(**d)


_L = None


def build(force=False):
    srcs = [os.path.join(_HERE, f) for f in ("ref_export.c", "ref_triangulation.c", "ref_triangulation.h", "ref_geom.c", "ref_geom.h",
                                             "ref_optimize.c", "export.mk")]
    if not force and os.path.exists(_LIB_PATH) and all(os.path.getmtime(_LIB_PATH) >= os.path.getmtime(s) for s in srcs):
        return _LIB_PATH
    subprocess.check_call(["make", "-s", "-C", _HERE, "-f", "export.mk"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


def _lib():
    global _L
    if _L is None:
        build()
        L = C.CDLL(_LIB_PATH)
        vp, u32, cfg, tri = C.c_void_p, C.c_uint32, C.POINTER(ExportCfg), C.POINTER(Triangulator)
        L.ref_robust_landmarks.argtypes = [cfg, tri, u32, vp, vp, vp, vp, u32, vp, vp, vp, vp, C.c_int]
        L.ref_export_reconstruction.argtypes = [cfg, tri, u32, vp, vp, vp, vp, vp, u32, vp, vp, vp, vp, vp, vp, vp, C.c_int]
        L.ref_normalize_reconstruction.argtypes = [cfg, tri, u32, vp, vp, vp, vp, u32, vp, vp, vp, u32, u32, vp, vp, vp]
        for f in (L.ref_robust_landmarks, L.ref_export_reconstruction, L.ref_normalize_reconstruction):
            f.restype = C.c_int
        _L = L
    return _L


def _ptr(a):
    return a.ctypes.data if a.size else None


def _snap(poses, view_offsets, view_landmarks, bearings, landmark_offsets, observations):
    u = (lambda a: np.ascontiguousarray(a, np.uint32).reshape(-1))
    P = np.ascontiguousarray(poses, np.float64).reshape(-1, 12)
    return P, u(view_offsets), u(view_landmarks), np.ascontiguousarray(bearings, np.float64).reshape(-1), u(landmark_offsets), u(observations)


def robust_landmarks(poses, view_offsets, view_landmarks, bearings, landmark_offsets, observations, cfg=None, tri=None, threads=0):
    """dict(points [L, 4], state uint8 [L]).  threads: OpenMP threads over the landmarks (0: OpenMP's default)."""
    cfg = cfg if cfg is not None else ExportCfg()
    tri = tri if tri is not None else triangulator(LINEAR_EIGEN)
    P, vo, vl, bear, lo, ob = _snap(poses, view_offsets, view_landmarks, bearings, landmark_offsets, observations)
    V, Lm = len(vo) - 1, len(lo) - 1
    pts = np.zeros((max(Lm, 1), 4))
    st = np.zeros(max(Lm, 1), np.uint8)
    assert _lib().ref_robust_landmarks(C.byref(cfg), C.byref(tri), V, _ptr(P), _ptr(vo), _ptr(vl), _ptr(bear), Lm, _ptr(lo), _ptr(ob),
                                       pts.ctypes.data, st.ctypes.data, int(threads)) == 0
    return dict(points=pts[:Lm].copy(), state=st[:Lm].copy())


def export_reconstruction(poses, view_offsets, view_landmarks, bearings, landmark_offsets, observations, colors, cfg=None, tri=None,
                          threads=0):
    """dict(points [n, 3], colors uint8 [n, 3], cameras CAMERA_DTYPE [V], mean_distance [V]).  threads: OpenMP threads over the landmarks
    and the views (0: OpenMP's default)."""
    cfg = cfg if cfg is not None else ExportCfg()
    tri = tri if tri is not None else triangulator(LINEAR_EIGEN)
    P, vo, vl, bear, lo, ob = _snap(poses, view_offsets, view_landmarks, bearings, landmark_offsets, observations)
    col = np.ascontiguousarray(colors, np.uint8).reshape(-1)
    V, Lm = len(vo) - 1, len(lo) - 1
    pts = np.zeros((max(Lm, 1), 3))
    pcol = np.zeros((max(Lm, 1), 3), np.uint8)
    n = C.c_uint32(0)
    cams = np.zeros(max(V, 1), CAMERA_DTYPE)
    mean = np.zeros(max(V, 1))
    assert _lib().ref_export_reconstruction(C.byref(cfg), C.byref(tri), V, _ptr(P), _ptr(vo), _ptr(vl), _ptr(bear), _ptr(col), Lm, _ptr(lo),
                                            _ptr(ob), pts.ctypes.data, pcol.ctypes.data, C.addressof(n), cams.ctypes.data, mean.ctypes.data,
                                            int(threads)) == 0
    return dict(points=pts[:n.value].copy(), colors=pcol[:n.value].copy(), cameras=cams[:V].copy(), mean_distance=mean[:V].copy())


def normalize_reconstruction(poses, view_offsets, view_landmarks, bearings, landmark_offsets, observations, constraints, first_view=0,
                             cfg=None, tri=None):
    """dict(result NORMALIZE_RESULT_DTYPE scalar, poses [V, 12], constraints CONSTRAINT_DTYPE [C])"""
    cfg = cfg if cfg is not None else ExportCfg()
    tri = tri if tri is not None else triangulator(LINEAR_EIGEN)
    P, vo, vl, bear, lo, ob = _snap(poses, view_offsets, view_landmarks, bearings, landmark_offsets, observations)
    cons = np.ascontiguousarray(constraints, CONSTRAINT_DTYPE).reshape(-1)
    V, Lm = len(vo) - 1, len(lo) - 1
    res = np.zeros(1, NORMALIZE_RESULT_DTYPE)
    pout = np.zeros((max(V, 1), 12))
    cout = np.zeros(max(len(cons), 1), CONSTRAINT_DTYPE)
    assert _lib().ref_normalize_reconstruction(C.byref(cfg), C.byref(tri), V, _ptr(P), _ptr(vo), _ptr(vl), _ptr(bear), Lm, _ptr(lo), _ptr(ob),
                                               _ptr(cons), len(cons), int(first_view), pout.ctypes.data, cout.ctypes.data,
                                               res.ctypes.data) == 0
    return dict(result=res[0], poses=pout[:V].copy(), constraints=cout[:len(cons)].copy())
