"""Host-side mirror of the reference's geometric-verification surfaces over the C ABI.

  EightPoint.estimate / LambdaTwist.estimate   <- sample_consensus::Estimator impls
      (eight-point/src/lib.rs:70-84, lambda-twist/src/lib.rs:330-347), batched over many minimal samples
  residuals_camera_to_camera / _world_to_camera <- sample_consensus::Model::residual
      (cv-core/src/pose.rs:249-296, 194-202)
  LinearEigenTriangulator and cv-geom's other triangulators: cv_b200/triangulation.py
  Arrsac.model / model_inliers                  <- arrsac::Arrsac as sample_consensus::Consensus
      (call sites akaze/tests/estimate_pose.rs:63-67, lambda-twist/tests/consensus.rs:20,59-61)
  Arrsac.model_inliers_batch                    <- many independent model_inliers calls, one generator each, in one set of launches
      (include/cvb200_batch.h; e.g. the candidate frames of cv-sfm's init_reconstruction, cv-sfm/src/lib.rs:966-985)
  Xoshiro256PlusPlus / Pcg64                     <- rand_xoshiro / rand_pcg generators handed to Arrsac::new
"""
import ctypes as C

import numpy as np

from ._lib import default_context


class Pose(C.Structure):
    """cvb_pose == IsometryMatrix3<f64> (rotation row-major, translation)"""
    _fields_ = [("r", C.c_double * 9), ("t", C.c_double * 3)]


class Rng(C.Structure):
    _fields_ = [("kind", C.c_int32), ("s", C.c_uint64 * 4)]


class ArrsacCfg(C.Structure):
    _fields_ = [("inlier_threshold", C.c_double), ("initialization_hypotheses", C.c_uint32), ("initialization_blocks", C.c_uint32),
                ("max_candidate_hypotheses", C.c_uint32), ("estimations_per_block", C.c_uint32), ("block_size", C.c_uint32),
                ("likelihood_ratio_threshold", C.c_float), ("initial_epsilon", C.c_float), ("initial_delta", C.c_float)]


POSE_DTYPE = np.dtype([("r", "<f8", (9,)), ("t", "<f8", (3,))])


def _f64(a, cols):
    a = np.ascontiguousarray(a, dtype=np.float64)
    if a.ndim != 2 or a.shape[1] != cols:
        raise ValueError(f"expected [N, {cols}] float64")
    return a


def _same_len(a, b, what="a, b"):
    if len(a) != len(b):
        raise ValueError(f"{what} must have the same number of rows ({len(a)} != {len(b)})")


def _poses_in(poses):
    """accepts a POSE_DTYPE array or a list of (R[3,3], t[3])"""
    if isinstance(poses, np.ndarray) and poses.dtype == POSE_DTYPE:
        return np.ascontiguousarray(poses)
    out = np.zeros(len(poses), POSE_DTYPE)
    for i, (R, t) in enumerate(poses):
        out[i]["r"] = np.asarray(R, np.float64).reshape(9)
        out[i]["t"] = np.asarray(t, np.float64).reshape(3)
    return out


def _lib(ctx):
    ctx = ctx or default_context(0)
    L = ctx.lib
    if not getattr(L, "_geom_bound", False):
        vp, u32 = C.c_void_p, C.c_uint32
        L.cvb_arrsac_default_cfg.argtypes = [C.POINTER(ArrsacCfg), C.c_double]
        L.cvb_arrsac_default_cfg.restype = None
        L.cvb_rng_seed_xoshiro256pp.argtypes = [C.POINTER(Rng), C.c_uint64]
        L.cvb_rng_seed_xoshiro256pp.restype = None
        L.cvb_rng_seed_pcg64.argtypes = [C.POINTER(Rng), C.c_char_p]
        L.cvb_rng_seed_pcg64.restype = None
        L.cvb_rng_next_u32.argtypes = [C.POINTER(Rng)]
        L.cvb_rng_next_u32.restype = u32
        L.cvb_eight_point_batch.argtypes = [vp, vp, vp, u32, vp, u32, vp, vp]
        L.cvb_p3p_batch.argtypes = [vp, vp, vp, u32, vp, u32, vp, vp]
        L.cvb_five_point_batch.argtypes = [vp, vp, vp, u32, vp, u32, C.c_int32, vp, vp]
        L.cvb_arrsac_five_point.argtypes = [vp, C.POINTER(ArrsacCfg), vp, vp, u32, C.POINTER(Rng), C.c_int32, C.POINTER(Pose), vp, u32,
                                            C.POINTER(u32), C.POINTER(C.c_int32)]
        L.cvb_residuals_camera_to_camera.argtypes = [vp, vp, u32, vp, vp, u32, vp]
        L.cvb_residuals_world_to_camera.argtypes = [vp, vp, u32, vp, vp, u32, vp]
        L.cvb_arrsac_eight_point.argtypes = [vp, C.POINTER(ArrsacCfg), vp, vp, u32, C.POINTER(Rng), C.POINTER(Pose), vp, u32,
                                             C.POINTER(u32), C.POINTER(C.c_int32)]
        L.cvb_arrsac_p3p.argtypes = L.cvb_arrsac_eight_point.argtypes
        L._geom_bound = True
    return ctx, L


class Xoshiro256PlusPlus:
    """rand_xoshiro::Xoshiro256PlusPlus::seed_from_u64 (== rand 0.8 SmallRng on 64-bit targets)."""

    def __init__(self, seed, ctx=None):
        _, L = _lib(ctx)
        self.state = Rng()
        L.cvb_rng_seed_xoshiro256pp(C.byref(self.state), seed)
        self._L = L

    def next_u32(self):
        return self._L.cvb_rng_next_u32(C.byref(self.state))


class Pcg64(Xoshiro256PlusPlus):
    """rand_pcg::Pcg64::from_seed([u8; 32])"""

    def __init__(self, seed_bytes, ctx=None):
        _, L = _lib(ctx)
        self.state = Rng()
        L.cvb_rng_seed_pcg64(C.byref(self.state), bytes(seed_bytes))
        self._L = L


class EightPoint:
    """eight_point::EightPoint: MIN_SAMPLES = 8, up to 4 CameraToCamera poses per sample."""
    MIN_SAMPLES = 8

    def estimate_batch(self, a, b, samples, ctx=None):
        ctx, L = _lib(ctx)
        a, b = _f64(a, 3), _f64(b, 3)
        _same_len(a, b)
        s = np.ascontiguousarray(samples, np.uint32).reshape(-1, 8)
        poses = np.zeros((len(s), 4), POSE_DTYPE)
        cnt = np.zeros(len(s), np.uint8)
        ctx.check(L.cvb_eight_point_batch(ctx.handle, a.ctypes.data, b.ctypes.data, len(a), s.ctypes.data, len(s), poses.ctypes.data,
                                          cnt.ctypes.data))
        return poses, cnt

    def estimate(self, a, b, ctx=None):
        """Estimator::estimate on exactly the first 8 matches."""
        poses, cnt = self.estimate_batch(a, b, np.arange(8, dtype=np.uint32)[None], ctx)
        return [(poses[0, k]["r"].reshape(3, 3).copy(), poses[0, k]["t"].copy()) for k in range(cnt[0])]

    def from_matches(self, a, b, epsilon=1e-12, iterations=1000, ctx=None):
        """EightPoint { epsilon, iterations }::from_matches (eight-point/src/lib.rs:43-58) on the first 8 matches -> EssentialMatrix or
        None.  To recondition the result, see EssentialMatrix.recondition.  Batched over samples: cv_b200.pinhole.eight_point_essential_batch."""
        from .pinhole import EssentialMatrix, eight_point_essential_batch
        if len(a) < 8:
            raise ValueError("from_matches needs 8 matches")
        E, ok = eight_point_essential_batch(a, b, np.arange(8, dtype=np.uint32)[None], epsilon, iterations, ctx)
        return EssentialMatrix(E[0]) if ok[0] else None


class NisterStewenius:
    """nister_stewenius::NisterStewenius: MIN_SAMPLES = 5, up to 40 CameraToCamera poses per sample
    (nister-stewenius/src/lib.rs:303-330).  `corrected=False` reproduces the reference bit for bit in structure,
    including its off-by-one eigenvector rows (lib.rs:229); `corrected=True` reads (x, y, z, 1) from rows 6..9."""
    MIN_SAMPLES = 5

    def __init__(self, corrected=False):
        self.row0 = 6 if corrected else 5

    def estimate_batch(self, a, b, samples, ctx=None):
        ctx, L = _lib(ctx)
        a, b = _f64(a, 3), _f64(b, 3)
        _same_len(a, b)
        s = np.ascontiguousarray(samples, np.uint32).reshape(-1, 5)
        poses = np.zeros((len(s), 40), POSE_DTYPE)
        cnt = np.zeros(len(s), np.uint8)
        ctx.check(L.cvb_five_point_batch(ctx.handle, a.ctypes.data, b.ctypes.data, len(a), s.ctypes.data, len(s), self.row0,
                                         poses.ctypes.data, cnt.ctypes.data))
        return poses, cnt

    def estimate(self, a, b, ctx=None):
        poses, cnt = self.estimate_batch(a, b, np.arange(5, dtype=np.uint32)[None], ctx)
        return [(poses[0, k]["r"].reshape(3, 3).copy(), poses[0, k]["t"].copy()) for k in range(cnt[0])]


class LambdaTwist:
    """lambda_twist::LambdaTwist: MIN_SAMPLES = 3, up to 4 WorldToCamera poses per sample."""
    MIN_SAMPLES = 3

    def estimate_batch(self, bearings, world, samples, ctx=None):
        ctx, L = _lib(ctx)
        a, b = _f64(bearings, 3), _f64(world, 4)
        _same_len(a, b, "bearings, world")
        s = np.ascontiguousarray(samples, np.uint32).reshape(-1, 3)
        poses = np.zeros((len(s), 4), POSE_DTYPE)
        cnt = np.zeros(len(s), np.uint8)
        ctx.check(L.cvb_p3p_batch(ctx.handle, a.ctypes.data, b.ctypes.data, len(a), s.ctypes.data, len(s), poses.ctypes.data, cnt.ctypes.data))
        return poses, cnt

    def estimate(self, bearings, world, ctx=None):
        poses, cnt = self.estimate_batch(bearings, world, np.arange(3, dtype=np.uint32)[None], ctx)
        return [(poses[0, k]["r"].reshape(3, 3).copy(), poses[0, k]["t"].copy()) for k in range(cnt[0])]


def residuals_camera_to_camera(poses, a, b, ctx=None):
    """CameraToCamera::residual for every (pose, FeatureMatch): [M, N] float64."""
    ctx, L = _lib(ctx)
    p = _poses_in(poses); a, b = _f64(a, 3), _f64(b, 3)
    _same_len(a, b)
    out = np.zeros((len(p), len(a)), np.float64)
    ctx.check(L.cvb_residuals_camera_to_camera(ctx.handle, p.ctypes.data, len(p), a.ctypes.data, b.ctypes.data, len(a), out.ctypes.data))
    return out


def residuals_world_to_camera(poses, bearings, world, ctx=None):
    """WorldToCamera::residual for every (pose, FeatureWorldMatch): [M, N] float64."""
    ctx, L = _lib(ctx)
    p = _poses_in(poses); a, b = _f64(bearings, 3), _f64(world, 4)
    _same_len(a, b, "bearings, world")
    out = np.zeros((len(p), len(a)), np.float64)
    ctx.check(L.cvb_residuals_world_to_camera(ctx.handle, p.ctypes.data, len(p), a.ctypes.data, b.ctypes.data, len(a), out.ctypes.data))
    return out


class Arrsac:
    """arrsac::Arrsac::new(inlier_threshold, rng) with the builder setters used by the reference."""

    def __init__(self, inlier_threshold, rng, ctx=None):
        self.ctx, self._L = _lib(ctx)
        self.cfg = ArrsacCfg()
        self._L.cvb_arrsac_default_cfg(C.byref(self.cfg), inlier_threshold)
        self.rng = rng

    def initialization_hypotheses(self, n):
        self.cfg.initialization_hypotheses = n; return self

    def initialization_blocks(self, n):
        self.cfg.initialization_blocks = n; return self

    def max_candidate_hypotheses(self, n):
        self.cfg.max_candidate_hypotheses = n; return self

    def estimations_per_block(self, n):
        self.cfg.estimations_per_block = n; return self

    def block_size(self, n):
        self.cfg.block_size = n; return self

    def model_inliers(self, estimator, a, b):
        """Consensus::model_inliers: (R, t, inlier indices) or None.  estimator: EightPoint (a, b bearings) or
        LambdaTwist (a bearings, b homogeneous world points)."""
        two_view = isinstance(estimator, (EightPoint, NisterStewenius))
        a = _f64(a, 3); b = _f64(b, 3 if two_view else 4)
        _same_len(a, b)
        n = len(a)
        model = Pose(); inl = np.zeros(max(n, 1), np.uint32); cnt = C.c_uint32(); found = C.c_int32()
        if isinstance(estimator, NisterStewenius):
            self.ctx.check(self._L.cvb_arrsac_five_point(self.ctx.handle, C.byref(self.cfg), a.ctypes.data, b.ctypes.data, n,
                                                         C.byref(self.rng.state), estimator.row0, C.byref(model), inl.ctypes.data, n,
                                                         C.byref(cnt), C.byref(found)))
        else:
            fn = self._L.cvb_arrsac_eight_point if two_view else self._L.cvb_arrsac_p3p
            self.ctx.check(fn(self.ctx.handle, C.byref(self.cfg), a.ctypes.data, b.ctypes.data, n, C.byref(self.rng.state), C.byref(model),
                              inl.ctypes.data, n, C.byref(cnt), C.byref(found)))
        if not found.value:
            return None
        return np.array(model.r).reshape(3, 3), np.array(model.t), inl[:cnt.value].copy()

    def model_inliers_batch(self, estimator, problems, rngs):
        """model_inliers of every problem in one batched device run: problems is a list of (a, b) as model_inliers takes them, rngs
        one generator per problem (each advanced as model_inliers would advance it; self.rng is not used).  Returns a list with one
        (R, t, inlier indices) or None per problem; problem i equals model_inliers(estimator, *problems[i]) with rngs[i].

        The reference runs such problems one after the other on ONE shared generator; a batch cannot know where each would start,
        so parity with that shared-generator sequence is unpinned (include/cvb200_batch.h)."""
        from ._lib import ARRSAC_BATCH_MAX, load_batch_library
        B = len(problems)
        if len(rngs) != B:
            raise ValueError(f"one generator per problem ({len(rngs)} != {B})")
        if B > ARRSAC_BATCH_MAX:
            raise ValueError(f"at most {ARRSAC_BATCH_MAX} problems per batch")
        if B == 0:
            return []
        kind, row0, a, b, offsets = pack_arrsac_batch(estimator, problems)
        BL = load_batch_library()
        states = (Rng * B)(*[r.state for r in rngs])
        models = (Pose * B)()
        inl = np.zeros(max(int(offsets[-1]), 1), np.uint32)
        cnt = np.zeros(B, np.uint32)
        found = np.zeros(B, np.int32)
        self.ctx.check(BL.cvb_arrsac_batch(self.ctx.handle, C.addressof(self.cfg), kind, row0, a.ctypes.data, b.ctypes.data,
                                           offsets.ctypes.data, B, C.addressof(states), C.addressof(models), inl.ctypes.data,
                                           cnt.ctypes.data, found.ctypes.data))
        out = []
        for i in range(B):
            C.memmove(C.addressof(rngs[i].state), C.addressof(states[i]), C.sizeof(Rng))
            if not found[i]:
                out.append(None)
                continue
            o = int(offsets[i])
            out.append((np.array(models[i].r).reshape(3, 3), np.array(models[i].t), inl[o:o + cnt[i]].copy()))
        return out

    def model(self, estimator, a, b):
        r = self.model_inliers(estimator, a, b)
        return None if r is None else (r[0], r[1])


def pack_arrsac_batch(estimator, problems):
    """(kind, eigenvector_row0, a, b, offsets) of cvb_arrsac_batch: the problems' rows packed one after the other, offsets in CSR form."""
    if isinstance(estimator, EightPoint):
        kind, row0, bc = 0, 5, 3
    elif isinstance(estimator, LambdaTwist):
        kind, row0, bc = 1, 5, 4
    elif isinstance(estimator, NisterStewenius):
        kind, row0, bc = 2, estimator.row0, 3
    else:
        raise TypeError("estimator must be EightPoint, LambdaTwist or NisterStewenius")
    As, Bs = [], []
    for pa, pb in problems:
        pa, pb = _f64(pa, 3), _f64(pb, bc)
        _same_len(pa, pb)
        As.append(pa); Bs.append(pb)
    offsets = np.zeros(len(problems) + 1, np.uint32)
    offsets[1:] = np.cumsum([len(x) for x in As])
    a = np.ascontiguousarray(np.concatenate(As) if As else np.zeros((0, 3)), np.float64)
    b = np.ascontiguousarray(np.concatenate(Bs) if Bs else np.zeros((0, bc)), np.float64)
    return kind, row0, a, b, offsets
