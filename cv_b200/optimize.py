"""Host-side mirror of the steps that follow the consensus stage in cv-sfm, over the C ABI (include/cvb200.h, and
include/cvb200_opt.h for the L1 optimizers):

  single_view_simple_optimize_l1   <- cv-optimize/src/single_view_optimizer.rs:16-78
  single_view_simple_optimize_l2   <- cv-optimize/src/single_view_optimizer.rs:80-135
  three_view_simple_optimize_l1    <- cv-optimize/src/three_view_optimizer.rs:23-124
  three_view_simple_optimize_l2    <- cv-optimize/src/three_view_optimizer.rs:126-201
  three_view_adaptive_optimize_l2  <- cv-optimize/src/three_view_optimizer.rs:203-272
  observation_losses               <- VSlam::observation_loss, cv-sfm/src/lib.rs:2570-2620
  tri_landmarks_robust             <- VSlam::is_tri_landmark_robust, cv-sfm/src/lib.rs:1320-1360

Every function has a `_batch` form: the refinement loops are sequential in the iteration count, so the GPU earns its
keep by running many independent problems (frames, tracks, candidate view triples) in one launch, one CTA each.
Poses are (R[3,3], t[3]) pairs like everywhere else in this package."""
import ctypes as C

import numpy as np

from ._lib import default_context, load_opt_library
from .geom import POSE_DTYPE, _f64, _poses_in
from .triangulation import _lib as _tri_lib


def _lib(ctx):
    ctx = ctx or default_context(0)
    L = ctx.lib
    if not getattr(L, "_opt_bound", False):
        vp, u32, f64 = C.c_void_p, C.c_uint32, C.c_double
        L.cvb_single_view_optimize_l2.argtypes = [vp, vp, u32, f64, u32, vp, vp, vp, vp, vp]
        L.cvb_three_view_optimize_l2.argtypes = [vp, vp, u32, C.c_int32, f64, u32, vp, vp, vp, vp]
        L.cvb_observation_losses.argtypes = [vp, vp, vp, vp, u32, vp]
        L.cvb_tri_landmarks_robust.argtypes = [vp, vp, vp, vp, u32, f64, f64, vp]
        L._opt_bound = True
    return ctx, L


def _l1_lib(ctx):
    """the context and libcvb200_opt.so (include/cvb200_opt.h); errors are reported through the context as for every entry point"""
    ctx = ctx or default_context(0)
    L = load_opt_library()
    if not getattr(L, "_l1_bound", False):
        vp, u32, f64 = C.c_void_p, C.c_uint32, C.c_double
        L.cvb_single_view_optimize_l1.argtypes = [vp, vp, u32, f64, f64, u32, vp, vp, vp, vp, vp]
        L.cvb_three_view_optimize_l1.argtypes = [vp, vp, u32, f64, f64, u32, vp, vp, vp, vp]
        L._l1_bound = True
    return ctx, L


def _poses_out(arr):
    return [(arr[i]["r"].reshape(3, 3).copy(), arr[i]["t"].copy()) for i in range(len(arr))]


def single_view_simple_optimize_l2_batch(poses, optimization_rate, iterations, bearings, world, offsets, ctx=None):
    """B problems: poses[b] with landmarks offsets[b]..offsets[b+1] of (bearings[n,3], world[n,4]) -> ([(R, t)], updates[B])"""
    ctx, L = _lib(ctx)
    p = _poses_in(poses); b = _f64(bearings, 3); w = _f64(world, 4)
    off = np.ascontiguousarray(offsets, np.uint32)
    nb = len(off) - 1
    if nb != len(p) or off[-1] != len(b) or len(b) != len(w):
        raise ValueError("offsets / poses / landmark arrays disagree")
    out = np.zeros(nb, POSE_DTYPE); upd = np.zeros(nb, np.uint32)
    ctx.check(L.cvb_single_view_optimize_l2(ctx.handle, p.ctypes.data, nb, optimization_rate, iterations, b.ctypes.data, w.ctypes.data,
                                            off.ctypes.data, out.ctypes.data, upd.ctypes.data))
    return _poses_out(out), upd


def single_view_simple_optimize_l2(pose, optimization_rate, iterations, landmarks, ctx=None):
    """landmarks = (bearings[n,3], world[n,4]) FeatureWorldMatches -> refined (R, t)"""
    bearings, world = landmarks
    if len(bearings) == 0:
        return pose
    out, _ = single_view_simple_optimize_l2_batch([pose], optimization_rate, iterations, bearings, world, [0, len(bearings)], ctx)
    return out[0]


def three_view_optimize_l2_batch(poses, optimization_rate, iterations, observations, offsets, adaptive=False, ctx=None):
    """B problems: poses[b] = [(R, t) centre->first, (R, t) centre->second]; observations[n,3,3] = (centre, first, second) bearings"""
    ctx, L = _lib(ctx)
    flat = [q for pair in poses for q in pair]
    p = _poses_in(flat)
    o = np.ascontiguousarray(observations, np.float64).reshape(-1, 9)
    off = np.ascontiguousarray(offsets, np.uint32)
    nb = len(off) - 1
    if 2 * nb != len(p) or off[-1] != len(o):
        raise ValueError("offsets / poses / observation arrays disagree")
    out = np.zeros(2 * nb, POSE_DTYPE); upd = np.zeros(nb, np.uint32)
    ctx.check(L.cvb_three_view_optimize_l2(ctx.handle, p.ctypes.data, nb, int(bool(adaptive)), optimization_rate, iterations, o.ctypes.data,
                                           off.ctypes.data, out.ctypes.data, upd.ctypes.data))
    po = _poses_out(out)
    return [[po[2 * i], po[2 * i + 1]] for i in range(nb)], upd


def three_view_simple_optimize_l2(poses, optimization_rate, iterations, landmarks, ctx=None):
    if len(landmarks) == 0:
        return list(poses)
    return three_view_optimize_l2_batch([poses], optimization_rate, iterations, landmarks, [0, len(landmarks)], False, ctx)[0][0]


def three_view_adaptive_optimize_l2(poses, iterations, landmarks, ctx=None):
    if len(landmarks) == 0:
        return list(poses)
    return three_view_optimize_l2_batch([poses], 0.0, iterations, landmarks, [0, len(landmarks)], True, ctx)[0][0]


def single_view_simple_optimize_l1_batch(poses, epsilon, optimization_rate, iterations, bearings, world, offsets, ctx=None):
    """B problems of single_view_simple_optimize_l1: poses[b] with landmarks offsets[b]..offsets[b+1] of (bearings[n,3], world[n,4])
    -> ([(R, t)], updates[B])"""
    ctx, L = _l1_lib(ctx)
    p = _poses_in(poses); b = _f64(bearings, 3); w = _f64(world, 4)
    off = np.ascontiguousarray(offsets, np.uint32)
    nb = len(off) - 1
    if nb != len(p) or off[-1] != len(b) or len(b) != len(w):
        raise ValueError("offsets / poses / landmark arrays disagree")
    out = np.zeros(nb, POSE_DTYPE); upd = np.zeros(nb, np.uint32)
    ctx.check(L.cvb_single_view_optimize_l1(ctx.handle, p.ctypes.data, nb, epsilon, optimization_rate, iterations, b.ctypes.data,
                                            w.ctypes.data, off.ctypes.data, out.ctypes.data, upd.ctypes.data))
    return _poses_out(out), upd


def single_view_simple_optimize_l1(pose, epsilon, optimization_rate, iterations, landmarks, ctx=None):
    """landmarks = (bearings[n,3], world[n,4]) FeatureWorldMatches -> refined (R, t); the reference's Weiszfeld iteration, epsilon
    has no default there either"""
    bearings, world = landmarks
    if len(bearings) == 0:
        return pose
    out, _ = single_view_simple_optimize_l1_batch([pose], epsilon, optimization_rate, iterations, bearings, world, [0, len(bearings)], ctx)
    return out[0]


def three_view_simple_optimize_l1_batch(poses, epsilon, optimization_rate, iterations, observations, offsets, ctx=None):
    """B problems of three_view_simple_optimize_l1: poses[b] = [(R, t) centre->first, (R, t) centre->second];
    observations[n,3,3] = (centre, first, second) bearings -> ([[(R, t), (R, t)]], updates[B])"""
    ctx, L = _l1_lib(ctx)
    flat = [q for pair in poses for q in pair]
    p = _poses_in(flat)
    o = np.ascontiguousarray(observations, np.float64).reshape(-1, 9)
    off = np.ascontiguousarray(offsets, np.uint32)
    nb = len(off) - 1
    if 2 * nb != len(p) or off[-1] != len(o):
        raise ValueError("offsets / poses / observation arrays disagree")
    out = np.zeros(2 * nb, POSE_DTYPE); upd = np.zeros(nb, np.uint32)
    ctx.check(L.cvb_three_view_optimize_l1(ctx.handle, p.ctypes.data, nb, epsilon, optimization_rate, iterations, o.ctypes.data,
                                           off.ctypes.data, out.ctypes.data, upd.ctypes.data))
    po = _poses_out(out)
    return [[po[2 * i], po[2 * i + 1]] for i in range(nb)], upd


def three_view_simple_optimize_l1(poses, epsilon, optimization_rate, iterations, landmarks, ctx=None):
    if len(landmarks) == 0:
        return list(poses)
    return three_view_simple_optimize_l1_batch([poses], epsilon, optimization_rate, iterations, landmarks, [0, len(landmarks)], ctx)[0][0]


def observation_losses(poses, bearings, offsets, ctx=None, triangulator=None):
    """observation_loss of every observation of L landmarks (observation lists as in LinearEigenTriangulator.triangulate_batch).
    triangulator: VSlam's triangulator for the landmarks of three or more observations (a LinearEigen, SineL1 or MeanMean
    Triangulator from cv_b200.triangulation); None is LinearEigenTriangulator's default."""
    ctx, L = _lib(ctx)
    p = _poses_in(poses); b = _f64(bearings, 3)
    off = np.ascontiguousarray(offsets, np.uint32)
    out = np.zeros(len(b), np.float64)
    if triangulator is None:
        ctx.check(L.cvb_observation_losses(ctx.handle, p.ctypes.data, b.ctypes.data, off.ctypes.data, len(off) - 1, out.ctypes.data))
    else:
        ctx, L = _tri_lib(ctx)
        ctx.check(L.cvb_observation_losses_tri(ctx.handle, C.byref(triangulator.cfg), p.ctypes.data, b.ctypes.data, off.ctypes.data,
                                               len(off) - 1, out.ctypes.data))
    return out


def tri_landmarks_robust(first_pose, second_pose, observations, maximum_cosine_distance, incidence_minimum_cosine_distance, ctx=None,
                         triangulator=None):
    """is_tri_landmark_robust for n (centre, first, second) bearing triples of one view triple -> bool[n].  triangulator: as in
    observation_losses."""
    ctx, L = _lib(ctx)
    p = _poses_in([first_pose, second_pose])
    o = np.ascontiguousarray(observations, np.float64).reshape(-1, 9)
    out = np.zeros(len(o), np.uint8)
    if triangulator is None:
        ctx.check(L.cvb_tri_landmarks_robust(ctx.handle, p[0:1].ctypes.data, p[1:2].ctypes.data, o.ctypes.data, len(o), maximum_cosine_distance,
                                             incidence_minimum_cosine_distance, out.ctypes.data))
    else:
        ctx, L = _tri_lib(ctx)
        ctx.check(L.cvb_tri_landmarks_robust_tri(ctx.handle, C.byref(triangulator.cfg), p[0:1].ctypes.data, p[1:2].ctypes.data, o.ctypes.data,
                                                 len(o), maximum_cosine_distance, incidence_minimum_cosine_distance, out.ctypes.data))
    return out.astype(bool)
