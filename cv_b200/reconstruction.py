"""cv-sfm's reconstruction optimisation on the device (include/cvb200_reconstruction.h): VSlam::optimize_reconstruction
(cv-sfm/src/lib.rs:2343-2355) -- the three-view pose graph of apply_constraints and filter_non_robust_observations -- as a pure function of
a reconstruction snapshot and its constraints, and regenerate_reconstruction (lib.rs:2418-2435), which builds those constraints with
generate_view_constraints first, all on the device."""
import ctypes as C

import numpy as np

from ._lib import load_constraints_library, load_reconstruction_library
from .constraints import CONSTRAINT_DTYPE, ConstraintSettings, _poses, _u32

# cvb_recon_result; the statuses, view states and observation states of include/cvb200_reconstruction.h
RESULT_DTYPE = np.dtype([("status", "<i4"), ("round", "<u4"), ("step", "<u4"), ("views_removed", "<u4"), ("robust_before", "<u4"),
                         ("robust_after", "<u4"), ("observations_split", "<u4"), ("small_angle_updates", "<u4")])
KEPT, REMOVED_CONSTRAINTS, REMOVED_FILTER, PANIC = 0, 1, 2, 3
VIEW_KEPT, VIEW_NO_EDGES, VIEW_NON_FINITE = 0, 1, 2
OBS_KEPT, OBS_SPLIT, OBS_DROPPED = 0, 1, 2


class ReconstructionSettings(C.Structure):
    """cvb_recon_cfg: the cv-sfm settings optimize_reconstruction reads, with their defaults (cv-sfm/src/settings.rs)."""
    _fields_ = [("graph_optimization_rate", C.c_double), ("maximum_sine_distance", C.c_double), ("maximum_cosine_distance", C.c_double),
                ("robust_observation_incidence_minimum_cosine_distance", C.c_double), ("optimization_iterations", C.c_uint32),
                ("reconstruction_optimization_iterations", C.c_uint32), ("robust_minimum_observations", C.c_uint32),
                ("minimum_robust_landmarks", C.c_uint32)]

    def __init__(self, **kw):
        d = dict(graph_optimization_rate=0.001, maximum_sine_distance=0.1, maximum_cosine_distance=1e-5,
                 robust_observation_incidence_minimum_cosine_distance=1e-3, optimization_iterations=1 << 10,
                 reconstruction_optimization_iterations=1, robust_minimum_observations=3, minimum_robust_landmarks=32)
        d.update(kw)
        super().__init__(**d)


def check_reconstruction(view_offsets, view_landmarks, landmark_offsets, observations, constraints):
    """cvb_optimize_reconstruction_check on the host (no device): 0, or CVB_EINVAL for a malformed snapshot or constraints."""
    vo, vl, lo, ob = _u32(view_offsets), _u32(view_landmarks), _u32(landmark_offsets), _u32(observations).reshape(-1)
    cons = np.ascontiguousarray(constraints, CONSTRAINT_DTYPE).reshape(-1)
    ptr = (lambda a: a.ctypes.data if a.size else None)
    return load_reconstruction_library().cvb_optimize_reconstruction_check(max(len(vo) - 1, 0), ptr(vo), ptr(vl), max(len(lo) - 1, 0), ptr(lo),
                                                                          ptr(ob), ptr(cons), len(cons))


def optimize_reconstruction(ctx, poses, view_offsets, view_landmarks, bearings, landmark_offsets, observations, constraints, settings=None,
                            triangulator=None):
    """cv-sfm's optimize_reconstruction of one reconstruction snapshot on the device (cvb_optimize_reconstruction).

    The snapshot is laid out as for cv_b200.generate_view_constraints; constraints: a CONSTRAINT_DTYPE array in the order of the
    reconstruction's constraint map (unpinned upstream; their `landmarks` field is ignored).  settings: ReconstructionSettings (cv-sfm's
    defaults); triangulator: LinearEigen, SineL1 or MeanMean (default LinearEigen).

    Returns dict(result: a RESULT_DTYPE record (status KEPT / REMOVED_CONSTRAINTS / REMOVED_FILTER / PANIC, where it stopped, views removed,
    robust landmarks before and after the last filter, observations split, updates through the small-angle exp map), poses [V, 12],
    view_state uint8 [V] (VIEW_*), obs_state uint8 [n_observations] (OBS_*, on the input observation CSR)).  With these the caller replays
    the slot-map edits of the reference."""
    from .triangulation import LinearEigenTriangulator
    settings = settings if settings is not None else ReconstructionSettings()
    tri = triangulator if triangulator is not None else LinearEigenTriangulator()
    P = _poses(poses)
    vo, vl, lo, ob = _u32(view_offsets), _u32(view_landmarks), _u32(landmark_offsets), _u32(observations).reshape(-1)
    bear = np.ascontiguousarray(bearings, np.float64).reshape(-1)
    cons = np.ascontiguousarray(constraints, CONSTRAINT_DTYPE).reshape(-1)
    V, Lm = len(vo) - 1, len(lo) - 1
    n_obs = int(lo[-1]) if len(lo) else 0
    res = np.zeros(1, RESULT_DTYPE)
    pout = np.zeros((max(V, 1), 12))
    vs = np.zeros(max(V, 1), np.uint8)
    os_ = np.zeros(max(n_obs, 1), np.uint8)
    ptr = (lambda a: a.ctypes.data if a.size else None)
    ctx.check(load_reconstruction_library().cvb_optimize_reconstruction(
        ctx.handle, C.addressof(settings), C.addressof(tri.cfg), V, ptr(P), ptr(vo), ptr(vl), ptr(bear), Lm, ptr(lo), ptr(ob), ptr(cons),
        len(cons), res.ctypes.data, pout.ctypes.data, vs.ctypes.data, os_.ctypes.data))
    return dict(result=res[0], poses=pout[:V].copy(), view_state=vs[:V].copy(), obs_state=os_[:n_obs].copy())


def regenerate_reconstruction(ctx, poses, view_offsets, view_landmarks, bearings, landmark_offsets, observations, settings=None,
                              constraint_settings=None, triangulator=None):
    """cv-sfm's regenerate_reconstruction (lib.rs:2418-2435) on the device: generate_view_constraints for every view
    (cvb_view_constraints_dev), the constraints of the accepted views kept in view order (record_view_constraints inserts them so), then
    optimize_reconstruction (cvb_optimize_reconstruction_dev).  The constraints stay on the device; only their count is read back.

    Inputs as optimize_reconstruction's, without the constraints; constraint_settings: ConstraintSettings.  Returns optimize_reconstruction's
    dict plus n_constraints."""
    import torch
    from .triangulation import LinearEigenTriangulator
    settings = settings if settings is not None else ReconstructionSettings()
    cset = constraint_settings if constraint_settings is not None else ConstraintSettings()
    tri = triangulator if triangulator is not None else LinearEigenTriangulator()
    dev = torch.device("cuda", ctx.device)
    host = (np.ascontiguousarray(_poses(poses)).view(np.float64).reshape(-1), _u32(view_offsets), _u32(view_landmarks),
            np.ascontiguousarray(bearings, np.float64).reshape(-1), _u32(landmark_offsets), _u32(observations).reshape(-1))
    P, vo, vl, bear, lo, ob = (torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in host)
    V, Lm, nf, n_obs = len(host[1]) - 1, len(host[4]) - 1, int(host[1][-1]), int(host[4][-1])
    maxc = cset.optimization_maximum_three_view_constraints
    csz = CONSTRAINT_DTYPE.itemsize
    cons = torch.zeros(max(V * maxc, 1) * csz, dtype=torch.uint8, device=dev)
    cres = torch.zeros(max(V, 1) * 2, dtype=torch.int32, device=dev)
    queries = np.arange(V, dtype=np.uint32)
    ptr = (lambda t: t.data_ptr() if t.numel() else None)
    torch.cuda.synchronize(dev)
    ctx.check(load_constraints_library().cvb_view_constraints_dev(
        ctx.handle, C.addressof(cset), C.addressof(tri.cfg), V, ptr(P), ptr(vo), ptr(vl), ptr(bear), nf, Lm, ptr(lo), ptr(ob), n_obs,
        queries.ctypes.data, V, cons.data_ptr(), cres.data_ptr(), None))
    r = cres[:2 * V].view(V, 2)
    keep = (torch.arange(maxc, device=dev)[None, :] < r[:, :1]) & (r[:, 1:] != 0)
    kept = cons[:V * maxc * csz].view(V * maxc, csz)[keep.reshape(-1)].contiguous()
    Cn = kept.shape[0]
    res = torch.zeros(RESULT_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    pout = torch.zeros(max(V, 1) * 12, dtype=torch.float64, device=dev)
    vs = torch.zeros(max(V, 1), dtype=torch.uint8, device=dev)
    os_ = torch.zeros(max(n_obs, 1), dtype=torch.uint8, device=dev)
    torch.cuda.synchronize(dev)
    ctx.check(load_reconstruction_library().cvb_optimize_reconstruction_dev(
        ctx.handle, C.addressof(settings), C.addressof(tri.cfg), V, ptr(P), ptr(vo), ptr(vl), ptr(bear), nf, Lm, ptr(lo), ptr(ob), n_obs,
        ptr(kept), Cn, res.data_ptr(), pout.data_ptr(), vs.data_ptr(), os_.data_ptr()))
    return dict(result=res.cpu().numpy().view(RESULT_DTYPE)[0], poses=pout.cpu().numpy().reshape(-1, 12)[:V].copy(),
                view_state=vs.cpu().numpy()[:V].copy(), obs_state=os_.cpu().numpy()[:n_obs].copy(), n_constraints=Cn)


__all__ = ["ReconstructionSettings", "optimize_reconstruction", "regenerate_reconstruction", "check_reconstruction", "RESULT_DTYPE", "KEPT",
           "REMOVED_CONSTRAINTS", "REMOVED_FILTER", "PANIC", "VIEW_KEPT", "VIEW_NO_EDGES", "VIEW_NON_FINITE", "OBS_KEPT", "OBS_SPLIT",
           "OBS_DROPPED"]
