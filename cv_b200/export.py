"""cv-sfm's reconstruction export on the device (include/cvb200_export.h): VSlam::triangulate_landmark_robust for every landmark
(cv-sfm/src/lib.rs:2907-3000), normalize_reconstruction (lib.rs:2241-2283) and export_reconstruction (lib.rs:2285-2340), each one call on
a reconstruction snapshot.  The PLY file itself is written on the host by cv_b200.formats.export_ply."""
import ctypes as C

import numpy as np

from ._lib import load_export_library
from .constraints import CONSTRAINT_DTYPE, _poses, _u32
from .formats import export_ply

# landmark states of include/cvb200_export.h
POINT, NOT_ROBUST, TRI_FAILED, AT_INFINITY = 0, 1, 2, 3
# cvb_export_camera (cv-sfm/src/export.rs's ExportCamera) and cvb_normalize_result
CAMERA_DTYPE = np.dtype([("optical_center", "<f8", (3,)), ("up_direction", "<f8", (3,)), ("forward_direction", "<f8", (3,)),
                         ("focal_length", "<f8")])
NORMALIZE_RESULT_DTYPE = np.dtype([("normalized", "<i4"), ("robust_points", "<u4"), ("mean_distance", "<f8")])


class ExportSettings(C.Structure):
    """cvb_export_cfg: the cv-sfm settings these calls read, with their defaults (cv-sfm/src/settings.rs).  vslam-sandbox exports with
    robust_minimum_observations set from --export-robust-minimum-observations (default 3)."""
    _fields_ = [("robust_observation_incidence_minimum_cosine_distance", C.c_double), ("robust_minimum_observations", C.c_uint32)]

    def __init__(self, **kw):
        d = dict(robust_observation_incidence_minimum_cosine_distance=1e-3, robust_minimum_observations=3)
        d.update(kw)
        super().__init__(**d)


def _ptr(a):
    return a.ctypes.data if a.size else None


def _snapshot(poses, view_offsets, view_landmarks, bearings, landmark_offsets, observations):
    P = _poses(poses)
    vo, vl, lo, ob = _u32(view_offsets), _u32(view_landmarks), _u32(landmark_offsets), _u32(observations).reshape(-1)
    bear = np.ascontiguousarray(bearings, np.float64).reshape(-1)
    return P, vo, vl, bear, lo, ob


def _defaults(settings, triangulator):
    from .triangulation import LinearEigenTriangulator
    return (settings if settings is not None else ExportSettings(),
            triangulator if triangulator is not None else LinearEigenTriangulator())


def check_export(view_offsets, view_landmarks, landmark_offsets, observations, constraints=None, first_view=0):
    """cvb_export_check on the host (no device): 0, or CVB_EINVAL for a malformed snapshot or constraints, or first_view >= V."""
    vo, vl, lo, ob = _u32(view_offsets), _u32(view_landmarks), _u32(landmark_offsets), _u32(observations).reshape(-1)
    cons = np.ascontiguousarray(constraints if constraints is not None else np.zeros(0, CONSTRAINT_DTYPE), CONSTRAINT_DTYPE).reshape(-1)
    return load_export_library().cvb_export_check(max(len(vo) - 1, 0), _ptr(vo), _ptr(vl), max(len(lo) - 1, 0), _ptr(lo), _ptr(ob),
                                                  _ptr(cons), len(cons), int(first_view))


def robust_landmarks(ctx, poses, view_offsets, view_landmarks, bearings, landmark_offsets, observations, settings=None, triangulator=None):
    """triangulate_landmark_robust of every landmark (cvb_robust_landmarks).  The snapshot is laid out as for
    cv_b200.generate_view_constraints; settings: ExportSettings; triangulator: LinearEigen, SineL1 or MeanMean (default LinearEigen).
    Returns dict(points float64 [L, 4] (the homogeneous WorldPoint of POINT and AT_INFINITY landmarks, else zero), state uint8 [L])."""
    settings, tri = _defaults(settings, triangulator)
    P, vo, vl, bear, lo, ob = _snapshot(poses, view_offsets, view_landmarks, bearings, landmark_offsets, observations)
    V, Lm = len(vo) - 1, len(lo) - 1
    pts = np.zeros((max(Lm, 1), 4))
    st = np.zeros(max(Lm, 1), np.uint8)
    ctx.check(load_export_library().cvb_robust_landmarks(ctx.handle, C.addressof(settings), C.addressof(tri.cfg), V, _ptr(P), _ptr(vo), _ptr(vl),
                                                         _ptr(bear), Lm, _ptr(lo), _ptr(ob), pts.ctypes.data, st.ctypes.data))
    return dict(points=pts[:Lm].copy(), state=st[:Lm].copy())


def normalize_reconstruction(ctx, poses, view_offsets, view_landmarks, bearings, landmark_offsets, observations, constraints, first_view=0,
                             settings=None, triangulator=None):
    """cv-sfm's normalize_reconstruction (cvb_normalize_reconstruction): the first view moved to the origin and the reconstruction scaled
    so that its mean robust point distance is one.  constraints: a CONSTRAINT_DTYPE array; first_view: the index of the view the
    reconstruction's slot map yields first.  Returns dict(result: a NORMALIZE_RESULT_DTYPE record (normalized, robust_points,
    mean_distance), poses [V, 12], constraints CONSTRAINT_DTYPE [C]); when the mean is not normal they are the inputs unchanged."""
    settings, tri = _defaults(settings, triangulator)
    P, vo, vl, bear, lo, ob = _snapshot(poses, view_offsets, view_landmarks, bearings, landmark_offsets, observations)
    cons = np.ascontiguousarray(constraints, CONSTRAINT_DTYPE).reshape(-1)
    V, Lm = len(vo) - 1, len(lo) - 1
    res = np.zeros(1, NORMALIZE_RESULT_DTYPE)
    pout = np.zeros((max(V, 1), 12))
    cout = np.zeros(max(len(cons), 1), CONSTRAINT_DTYPE)
    ctx.check(load_export_library().cvb_normalize_reconstruction(
        ctx.handle, C.addressof(settings), C.addressof(tri.cfg), V, _ptr(P), _ptr(vo), _ptr(vl), _ptr(bear), Lm, _ptr(lo), _ptr(ob),
        _ptr(cons), len(cons), int(first_view), pout.ctypes.data, cout.ctypes.data, res.ctypes.data))
    return dict(result=res[0], poses=pout[:V].copy(), constraints=cout[:len(cons)].copy())


def write_ply(path, points, colors, cameras, camera_faces=True):
    """Writes export_reconstruction's outputs as cv-sfm/src/export.rs does (cameras first, then the points) with formats.export_ply."""
    cams = [dict(optical_center=c["optical_center"], up_direction=c["up_direction"], forward_direction=c["forward_direction"],
                 focal_length=c["focal_length"]) for c in cameras]
    with open(path, "w") as f:
        export_ply(f, list(zip(points, colors)), cams, camera_faces)


def export_reconstruction(ctx, poses, view_offsets, view_landmarks, bearings, landmark_offsets, observations, colors, path=None,
                          camera_faces=True, settings=None, triangulator=None):
    """cv-sfm's export_reconstruction (cvb_export_reconstruction).  colors: uint8 [n_features, 3] on the view CSR.  Returns
    dict(points float64 [n, 3], colors uint8 [n, 3], cameras CAMERA_DTYPE [V], mean_distance float64 [V]); given a path, also writes the
    PLY file there (write_ply)."""
    settings, tri = _defaults(settings, triangulator)
    P, vo, vl, bear, lo, ob = _snapshot(poses, view_offsets, view_landmarks, bearings, landmark_offsets, observations)
    col = np.ascontiguousarray(colors, np.uint8).reshape(-1)
    V, Lm = len(vo) - 1, len(lo) - 1
    pts = np.zeros((max(Lm, 1), 3))
    pcol = np.zeros((max(Lm, 1), 3), np.uint8)
    n = C.c_uint32(0)
    cams = np.zeros(max(V, 1), CAMERA_DTYPE)
    mean = np.zeros(max(V, 1))
    ctx.check(load_export_library().cvb_export_reconstruction(
        ctx.handle, C.addressof(settings), C.addressof(tri.cfg), V, _ptr(P), _ptr(vo), _ptr(vl), _ptr(bear), _ptr(col), Lm, _ptr(lo), _ptr(ob),
        pts.ctypes.data, pcol.ctypes.data, C.addressof(n), cams.ctypes.data, mean.ctypes.data))
    out = dict(points=pts[:n.value].copy(), colors=pcol[:n.value].copy(), cameras=cams[:V].copy(), mean_distance=mean[:V].copy())
    if path is not None:
        write_ply(path, out["points"], out["colors"], out["cameras"], camera_faces)
    return out


__all__ = ["ExportSettings", "robust_landmarks", "normalize_reconstruction", "export_reconstruction", "write_ply", "check_export",
           "CAMERA_DTYPE", "NORMALIZE_RESULT_DTYPE", "POINT", "NOT_ROBUST", "TRI_FAILED", "AT_INFINITY"]
