"""cv-sfm's frame registration on the device (include/cvb200_register.h): VSlam::register_frame / register_frame_subset
(cv-sfm/src/lib.rs:1452-1812) for one new frame against one reconstruction snapshot, from the frame's descriptors and bearings to the
refined WorldToCamera pose and its landmark matches, in one call."""
import ctypes as C

import numpy as np

from ._lib import load_register_library
from .constraints import _poses, _u32

# result statuses of include/cvb200_register.h, one per `return None` of the reference and its panic
STATUS_NAMES = ["ok", "few_robust_landmarks", "no_consensus", "filter_half", "final_half", "final_robust_half", "few_matches", "panic"]
NONE = 0xFFFFFFFF
POSE_F64 = np.dtype([("r", "<f8", (9,)), ("t", "<f8", (3,))])
MATCH_DTYPE = np.dtype([("feature", "<u4"), ("landmark_a", "<u4"), ("landmark_b", "<u4")])
RESULT_DTYPE = np.dtype([("status", "<i4"), ("iteration", "<u4"), ("n_matches", "<u4"), ("n_inliers", "<u4"), ("pose", POSE_F64)])
STATS_DTYPE = np.dtype([("subsets", "<u4"), ("matches", "<u4"), ("claimed", "<u4"), ("matches_3d", "<u4"), ("inliers", "<u4"),
                        ("final_robust", "<u4"), ("final_matches", "<u4"), ("iterations", "<u4"), ("filter_matches", "<u4", (16,)),
                        ("final_stage_matches", "<u4"), ("reserved", "<u4", (3,))])


class RegisterSettings(C.Structure):
    """cvb_register_cfg: the cv-sfm settings register_frame reads, with their defaults (cv-sfm/src/settings.rs)."""
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


def _ptr(a):
    return a.ctypes.data if a.size else None


def check_register(view_offsets, view_landmarks, landmark_offsets, observations, view_matches):
    """cvb_register_check on the host (no device): 0, or CVB_EINVAL for a malformed snapshot or a view match out of range."""
    vo, vl, lo, ob, vm = _u32(view_offsets), _u32(view_landmarks), _u32(landmark_offsets), _u32(observations).reshape(-1), _u32(view_matches)
    return load_register_library().cvb_register_check(max(len(vo) - 1, 0), _ptr(vo), _ptr(vl), max(len(lo) - 1, 0), _ptr(lo), _ptr(ob),
                                                      _ptr(vm), len(vm))


def register_frame(ctx, poses, view_offsets, view_landmarks, bearings, descriptors, landmark_offsets, observations, new_descriptors,
                   new_bearings, view_matches, arrsac, settings=None, triangulator=None, stats=False):
    """cv-sfm's register_frame (cvb_register_frame).  The snapshot is laid out as for cv_b200.generate_view_constraints, plus
    descriptors uint8 [n_features, 64] on the view CSR; new_descriptors uint8 [N, 64] and new_bearings [N, 3] are the new frame's;
    view_matches: the view indices to match against.  arrsac: a cv_b200.Arrsac (VSlam's single_view_consensus), whose generator advances
    as the reference's would; triangulator: LinearEigen, SineL1 or MeanMean (default LinearEigen).

    Returns (status name, pose (R [3, 3], t [3]) or None, matches MATCH_DTYPE [n] ascending by feature, landmark_b = NONE for a single
    landmark), with two more elements when stats is true: the STATS_DTYPE record and the last subset's consensus inliers (indices into
    its matches_3d, in the consensus' order).  'filter_half' carries no iteration here; it is in the statistics' `iterations` (the
    iteration that failed is iterations - 1)."""
    from .triangulation import LinearEigenTriangulator
    settings = settings if settings is not None else RegisterSettings()
    tri = triangulator if triangulator is not None else LinearEigenTriangulator()
    P, vo, vl, lo, ob = _poses(poses), _u32(view_offsets), _u32(view_landmarks), _u32(landmark_offsets), _u32(observations).reshape(-1)
    bear = np.ascontiguousarray(bearings, np.float64).reshape(-1)
    desc = np.ascontiguousarray(descriptors, np.uint8).reshape(-1)
    nd = np.ascontiguousarray(new_descriptors, np.uint8).reshape(-1, 64)
    nb = np.ascontiguousarray(new_bearings, np.float64).reshape(-1, 3)
    if len(nd) != len(nb):
        raise ValueError("one bearing per new descriptor expected")
    vm = _u32(view_matches).reshape(-1)
    V, Lm, N = len(vo) - 1, len(lo) - 1, len(nd)
    res = np.zeros(1, RESULT_DTYPE)
    matches = np.zeros(max(N, 1), MATCH_DTYPE)
    st = np.zeros(1, STATS_DTYPE)
    inl = np.zeros(max(N, 1), np.uint32)
    ctx.check(load_register_library().cvb_register_frame(
        ctx.handle, C.addressof(settings), C.addressof(tri.cfg), C.addressof(arrsac.cfg), C.addressof(arrsac.rng.state), V, _ptr(P), _ptr(vo),
        _ptr(vl), _ptr(bear), _ptr(desc), Lm, _ptr(lo), _ptr(ob), _ptr(nd), _ptr(nb), N, _ptr(vm), len(vm), res.ctypes.data,
        matches.ctypes.data, inl.ctypes.data if stats else None, st.ctypes.data if stats else None))
    r = res[0]
    status = STATUS_NAMES[int(r["status"])]
    pose = (r["pose"]["r"].reshape(3, 3).copy(), r["pose"]["t"].copy()) if status == "ok" else None
    out = (status, pose, matches[:int(r["n_matches"])].copy())
    return out + (st[0], inl[:int(r["n_inliers"])].copy()) if stats else out


__all__ = ["RegisterSettings", "register_frame", "check_register", "STATUS_NAMES", "MATCH_DTYPE", "RESULT_DTYPE", "STATS_DTYPE", "NONE"]
