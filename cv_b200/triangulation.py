"""The triangulators of cv-geom (cv-geom/src/triangulation.rs) on the device, over include/cvb200_tri.h.

  LinearEigenTriangulator       <- :39-130   TriangulatorObservations (+ TriangulatorRelative through the blanket impl)
  SineL1Triangulator            <- :163-276  TriangulatorObservations (+ TriangulatorRelative)
  MeanMeanTriangulator          <- :389-442  TriangulatorObservations (+ TriangulatorRelative)
  RelativeDltTriangulator       <- :279-363  TriangulatorRelative only
  AngularL1Triangulator         <- :469-530  TriangulatorRelative only
  AngularLInfinityTriangulator  <- :555-606  TriangulatorRelative only

Constructor arguments are the reference's builder settings with its Default values (SineL1's rate is 1.0 although the setter's doc
comment says 0.01; RelativeDlt's epsilon / max_iterations are 1e-12 / 1000 although its doc comments say 1e-9 / 100).
Points come back homogeneous and normalised as Projective::from_homogeneous does (w >= 0, |xyz| = 1); a row whose `ok` is False is
the reference's None and holds zeros.  There is no CPU fallback: without a Hopper GPU every call raises CvbError (CVB_ENODEV).
"""
import ctypes as C

import numpy as np

from .geom import _f64, _lib as _geom_lib, _poses_in, _same_len

CVB_TRI_LINEAR_EIGEN, CVB_TRI_SINE_L1, CVB_TRI_MEAN_MEAN, CVB_TRI_RELATIVE_DLT, CVB_TRI_ANGULAR_L1, CVB_TRI_ANGULAR_LINF = range(6)


class TriangulatorCfg(C.Structure):
    """cvb_triangulator"""
    _fields_ = [("method", C.c_int32), ("max_iterations", C.c_uint32), ("epsilon", C.c_double), ("optimization_rate", C.c_double)]


def _lib(ctx):
    ctx, L = _geom_lib(ctx)
    if not getattr(L, "_tri_bound", False):
        vp, u32, T = C.c_void_p, C.c_uint32, C.POINTER(TriangulatorCfg)
        L.cvb_triangulator_default.argtypes = [T, C.c_int32]
        L.cvb_triangulator_default.restype = None
        L.cvb_triangulate_observations.argtypes = [vp, T, vp, vp, vp, u32, vp, vp]
        L.cvb_triangulate_relative.argtypes = [vp, T, vp, u32, vp, vp, u32, vp, vp]
        L.cvb_observation_losses_tri.argtypes = [vp, T, vp, vp, vp, u32, vp]
        L.cvb_tri_landmarks_robust_tri.argtypes = [vp, T, vp, vp, vp, u32, C.c_double, C.c_double, vp]
        L._tri_bound = True
    return ctx, L


class _Triangulator:
    method = None

    def __init__(self, epsilon=0.0, max_iterations=0, optimization_rate=0.0):
        self.cfg = TriangulatorCfg(self.method, int(max_iterations), float(epsilon), float(optimization_rate))

    def __repr__(self):
        c = self.cfg
        return f"{type(self).__name__}(epsilon={c.epsilon!r}, max_iterations={c.max_iterations}, optimization_rate={c.optimization_rate!r})"

    def triangulate_relative_batch(self, poses, a, b, ctx=None):
        """TriangulatorRelative::triangulate_relative for n (CameraToCamera pose, a, b) triples.  poses: one pose for every triple
        (a (R, t) pair, or a list / POSE_DTYPE array of length 1) or one per triple -> (xyzw[n, 4] CameraPoints, ok[n] bool)"""
        ctx, L = _lib(ctx)
        if isinstance(poses, tuple) and len(poses) == 2 and np.asarray(poses[0]).shape == (3, 3):
            poses = [poses]
        p = _poses_in(poses); a = _f64(a, 3); b = _f64(b, 3)
        _same_len(a, b)
        n = len(a)
        if len(p) not in (1, n):
            raise ValueError(f"expected 1 or {n} poses, got {len(p)}")
        out = np.zeros((n, 4), np.float64); ok = np.zeros(n, np.uint8)
        ctx.check(L.cvb_triangulate_relative(ctx.handle, C.byref(self.cfg), p.ctypes.data, len(p), a.ctypes.data, b.ctypes.data, n,
                                             out.ctypes.data, ok.ctypes.data))
        return out, ok.astype(bool)

    def triangulate_relative(self, pose, a, b, ctx=None):
        """pose: (R, t) CameraToCamera from a's camera to b's -> homogeneous CameraPoint in a's camera, or None"""
        out, ok = self.triangulate_relative_batch([pose], np.reshape(a, (1, 3)), np.reshape(b, (1, 3)), ctx)
        return out[0] if ok[0] else None


class _ObservationsTriangulator(_Triangulator):
    def triangulate_batch(self, poses, bearings, offsets, ctx=None):
        """TriangulatorObservations::triangulate_observations for L landmarks: landmark l has the observations offsets[l] ..
        offsets[l + 1] - 1 of (poses (WorldToCamera), bearings[n, 3]) -> (xyzw[L, 4] WorldPoints, ok[L] bool)"""
        ctx, L = _lib(ctx)
        p = _poses_in(poses); b = _f64(bearings, 3)
        off = np.ascontiguousarray(offsets, np.uint32)
        _same_len(p, b, "poses, bearings")
        if len(off) < 1 or off[0] != 0 or (np.diff(off.astype(np.int64)) < 0).any() or off[-1] > len(p):
            raise ValueError("offsets must start at 0, be non-decreasing and end within the observations")
        nl = len(off) - 1
        out = np.zeros((nl, 4), np.float64); ok = np.zeros(nl, np.uint8)
        ctx.check(L.cvb_triangulate_observations(ctx.handle, C.byref(self.cfg), p.ctypes.data, b.ctypes.data, off.ctypes.data, nl,
                                                 out.ctypes.data, ok.ctypes.data))
        return out, ok.astype(bool)

    def triangulate_observations(self, pairs, ctx=None):
        """pairs: [((R, t), bearing), ...] -> homogeneous WorldPoint or None"""
        poses = [p for p, _ in pairs]
        out, ok = self.triangulate_batch(poses, np.array([b for _, b in pairs], np.float64).reshape(-1, 3), [0, len(pairs)], ctx)
        return out[0] if ok[0] else None


class LinearEigenTriangulator(_ObservationsTriangulator):
    """cv_geom::triangulation::LinearEigenTriangulator; epsilon / max_iterations of its symmetric eigen solver"""
    method = CVB_TRI_LINEAR_EIGEN

    def __init__(self, epsilon=1e-12, max_iterations=1000):
        super().__init__(epsilon, max_iterations)


class SineL1Triangulator(_ObservationsTriangulator):
    """cv_geom::triangulation::SineL1Triangulator: LinearEigen's point refined by gradient steps on the sine-L1 epipolar error"""
    method = CVB_TRI_SINE_L1

    def __init__(self, epsilon=1e-12, max_iterations=1000, optimization_rate=1.0):
        super().__init__(epsilon, max_iterations, optimization_rate)


class MeanMeanTriangulator(_ObservationsTriangulator):
    """cv_geom::triangulation::MeanMeanTriangulator"""
    method = CVB_TRI_MEAN_MEAN


class RelativeDltTriangulator(_Triangulator):
    """cv_geom::triangulation::RelativeDltTriangulator; epsilon / max_iterations of its SVD"""
    method = CVB_TRI_RELATIVE_DLT

    def __init__(self, epsilon=1e-12, max_iterations=1000):
        super().__init__(epsilon, max_iterations)


class AngularL1Triangulator(_Triangulator):
    """cv_geom::triangulation::AngularL1Triangulator"""
    method = CVB_TRI_ANGULAR_L1


class AngularLInfinityTriangulator(_Triangulator):
    """cv_geom::triangulation::AngularLInfinityTriangulator"""
    method = CVB_TRI_ANGULAR_LINF
