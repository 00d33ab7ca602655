"""cv-sfm's three-view constraints on the device (include/cvb200_constraints.h): VSlam::generate_view_constraints
(cv-sfm/src/lib.rs:2438-2516) and record_view_constraints' acceptance (lib.rs:2092-2109) for many query views of one reconstruction
snapshot in one call, and the warp-per-problem adaptive three-view optimiser they run on."""
import ctypes as C

import numpy as np

from ._lib import CONSTRAINTS_MAX_LANDMARKS, load_constraints_library

POSE_DTYPE = np.dtype([("r", "<f8", (9,)), ("t", "<f8", (3,))])
# cvb_view_constraint, cvb_view_constraints_result and cvb_view_constraints_stats
CONSTRAINT_DTYPE = np.dtype([("views", "<u4", (3,)), ("landmarks", "<u4"), ("poses", POSE_DTYPE, (2,))])
RESULT_DTYPE = np.dtype([("n_constraints", "<u4"), ("accepted", "<i4")])
STATS_DTYPE = np.dtype([("robust_landmarks", "<u4"), ("coviews", "<u4"), ("triples", "<u4"), ("unique_triples", "<u4"), ("candidates", "<u4"),
                        ("few_landmarks", "<u4"), ("few_bearing_pairs", "<u4"), ("updates", "<u4")])


class ConstraintSettings(C.Structure):
    """cvb_constraints_cfg: the cv-sfm settings generate_view_constraints and record_view_constraints read, with their defaults
    (cv-sfm/src/settings.rs:332-350, 453-483)."""
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
                 optimization_minimum_new_constraints=4, constraint_patience=1 << 12)
        d.update(kw)
        super().__init__(**d)


def _u32(a):
    return np.ascontiguousarray(a, np.uint32)


def _poses(p):
    p = np.asarray(p)
    if p.dtype == POSE_DTYPE:
        return np.ascontiguousarray(p)
    return np.ascontiguousarray(p, np.float64).reshape(-1, 12)


def check_snapshot(view_offsets, view_landmarks, landmark_offsets, observations, queries):
    """cvb_view_constraints_check on the host (no device): 0, or CVB_EINVAL for a malformed snapshot or queries."""
    vo, vl, lo, ob, q = _u32(view_offsets), _u32(view_landmarks), _u32(landmark_offsets), _u32(observations).reshape(-1), _u32(queries)
    L = load_constraints_library()
    return L.cvb_view_constraints_check(max(len(vo) - 1, 0), vo.ctypes.data if len(vo) else None, vl.ctypes.data if len(vl) else None,
                                        max(len(lo) - 1, 0), lo.ctypes.data if len(lo) else None, ob.ctypes.data if len(ob) else None,
                                        q.ctypes.data if len(q) else None, len(q))


def generate_view_constraints(ctx, poses, view_offsets, view_landmarks, bearings, landmark_offsets, observations, queries, settings=None,
                              triangulator=None, stats=False):
    """cv-sfm's generate_view_constraints for every view in `queries` of one reconstruction snapshot, on the device (cvb_view_constraints).

    poses: [V, 12] float64 WorldToCamera (rotation row-major, translation), views numbered in ascending ViewKey order; view_offsets
    [V + 1] and view_landmarks: View.landmarks as CSR (one landmark index per feature); bearings [n_features, 3] on the same CSR;
    landmark_offsets [L + 1] and observations [n_observations, 2]: Landmark.observations as CSR of (view, feature), in the order the
    reference's map would give them; queries: view indices (duplicates allowed).  settings: ConstraintSettings (cv-sfm's defaults);
    triangulator: LinearEigen, SineL1 or MeanMean (default LinearEigen).

    Returns dict(constraints: per query a CONSTRAINT_DTYPE array in the reference's evaluation order, results: RESULT_DTYPE [Q]
    (n_constraints, accepted = record_view_constraints' return), stats: STATS_DTYPE [Q] or None).  A call over every view is
    regenerate_reconstruction's constraint pass; incorporate_reconstruction removes views between its calls, which
    cv_b200.incorporate_reconstruction does by repeating the call after each refusal.  Unpinned, as the reference leaves these orders undefined: coviews ascending, stable sorts, no shuffle of the landmarks,
    observations in the given order."""
    from .triangulation import LinearEigenTriangulator
    settings = settings if settings is not None else ConstraintSettings()
    tri = triangulator if triangulator is not None else LinearEigenTriangulator()
    P = _poses(poses)
    vo, vl, lo, ob, q = _u32(view_offsets), _u32(view_landmarks), _u32(landmark_offsets), _u32(observations).reshape(-1), _u32(queries)
    bear = np.ascontiguousarray(bearings, np.float64).reshape(-1)
    V, Lm, Q, maxc = len(vo) - 1, len(lo) - 1, len(q), settings.optimization_maximum_three_view_constraints
    out = np.zeros(max(Q * maxc, 1), CONSTRAINT_DTYPE)
    res = np.zeros(max(Q, 1), RESULT_DTYPE)
    st = np.zeros(max(Q, 1), STATS_DTYPE) if stats else None
    L = load_constraints_library()
    ptr = (lambda a: a.ctypes.data if a.size else None)
    ctx.check(L.cvb_view_constraints(ctx.handle, C.addressof(settings), C.addressof(tri.cfg), V, ptr(P), ptr(vo), ptr(vl), ptr(bear), Lm,
                                     ptr(lo), ptr(ob), ptr(q), Q, out.ctypes.data, res.ctypes.data, st.ctypes.data if stats else None))
    res = res[:Q].copy()
    cons = [out[i * maxc:i * maxc + res[i]["n_constraints"]].copy() for i in range(Q)]
    return dict(constraints=cons, results=res, stats=st[:Q].copy() if stats else None)


def three_view_adaptive_optimize_l2_dev(ctx, poses, obs, offsets, iterations):
    """three_view_adaptive_optimize_l2 of B problems on the device, one warp each (cvb_three_view_adaptive_optimize_l2_dev): poses [B, 2, 12]
    float64 (CUDA, CameraToCamera centre -> first / second), obs [n, 9] float64 (CUDA, centre / first / second bearings), offsets [B + 1]
    int32 (CUDA).  At most CONSTRAINTS_MAX_LANDMARKS rows per problem.  Returns (poses [B, 2, 12], updates [B]) as CUDA tensors."""
    import torch
    for t in (poses, obs, offsets):
        if not t.is_cuda or not t.is_contiguous():
            raise ValueError("poses, obs and offsets must be contiguous CUDA tensors")
    if poses.dtype != torch.float64 or obs.dtype != torch.float64 or offsets.dtype != torch.int32:
        raise ValueError("poses and obs are float64, offsets int32")
    B = offsets.shape[0] - 1
    out = torch.empty_like(poses)
    upd = torch.zeros(max(B, 1), dtype=torch.int32, device=poses.device)
    L = load_constraints_library()
    torch.cuda.synchronize(poses.device)
    ctx.check(L.cvb_three_view_adaptive_optimize_l2_dev(ctx.handle, poses.data_ptr(), B, obs.data_ptr(), offsets.data_ptr(), int(iterations),
                                                        out.data_ptr(), upd.data_ptr()))
    return out, upd[:B]


__all__ = ["ConstraintSettings", "generate_view_constraints", "check_snapshot", "three_view_adaptive_optimize_l2_dev",
           "CONSTRAINTS_MAX_LANDMARKS"]
