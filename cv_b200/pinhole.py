"""cv-pinhole (cv-pinhole/src/lib.rs, essential.rs).

  CameraIntrinsics, CameraIntrinsicsK1Distortion  <- lib.rs:32-240: pixel <-> unit bearing.  Scalar per-keypoint host work in the
      reference (SURVEY.md section 8a row C1, "negligible; keep on host"); vectorised here over all keypoints in f64 with the reference's
      operation order.
  pose_reprojection_error, average_pose_reprojection_error  <- lib.rs:314-372, on the device over any of cv-geom's triangulators
  EssentialMatrix  <- essential.rs:56-275, on the device (From<CameraToCamera> is host numpy)

The device functions run over include/cvb200_pinhole.h (cv_b200/libcvb200_pinhole.so); there is no CPU fallback: without a Hopper GPU
they raise CvbError (CVB_ENODEV).  Batch forms return an `ok` flag per row: False where the reference returns None, and those rows hold
NaN.  epsilon / max_iterations bound the device's Jacobi sweeps; max_iterations = 0 gives no result (nalgebra reads 0 as unbounded).
"""
import ctypes as C
from dataclasses import dataclass

import numpy as np

from ._lib import default_context, load_pinhole_library
from .geom import _f64, _poses_in, _same_len
from .triangulation import TriangulatorCfg


@dataclass
class CameraIntrinsics:
    focals: tuple            # (fx, fy)
    principal_point: tuple   # (cx, cy)
    skew: float = 0.0

    def calibrate(self, points):
        """CameraModel::calibrate (cv-pinhole/src/lib.rs:108-116): [N, 2] pixel coordinates -> [N, 3] unit bearings."""
        p = np.asarray(points, np.float64).reshape(-1, 2)
        y = (p[:, 1] - self.principal_point[1]) / self.focals[1]
        x = (p[:, 0] - self.principal_point[0] - self.skew * y) / self.focals[0]
        n = np.sqrt(x * x + y * y + 1.0)
        return np.stack([x / n, y / n, 1.0 / n], 1)

    def uncalibrate(self, bearings):
        """CameraModel::uncalibrate (cv-pinhole/src/lib.rs:134-141): unit bearings -> pixel coordinates
        (NaN where the reference returns None: z not sign-positive)."""
        b = np.asarray(bearings, np.float64).reshape(-1, 3)
        with np.errstate(divide="ignore", invalid="ignore"):
            x, y = b[:, 0] / b[:, 2], b[:, 1] / b[:, 2]
            px = x * self.focals[0] + self.skew * y + self.principal_point[0]
            py = y * self.focals[1] + self.principal_point[1]
        out = np.stack([px, py], 1)
        out[np.signbit(b[:, 2])] = np.nan
        return out

    def calibrate_keypoints(self, kps):
        """akaze::KeyPoint implements ImagePoint via (point.0 as f64, point.1 as f64) (akaze/src/lib.rs:95-99)."""
        return self.calibrate(np.stack([kps["x"].astype(np.float64), kps["y"].astype(np.float64)], 1))


@dataclass
class CameraIntrinsicsK1Distortion:
    """cv_pinhole::CameraIntrinsicsK1Distortion (cv-pinhole/src/lib.rs:150-240): simple intrinsics plus one radial coefficient."""
    simple_intrinsics: CameraIntrinsics
    k1: float

    def calibrate(self, points):
        """CameraModel::calibrate (cv-pinhole/src/lib.rs:191-202): [N, 2] pixel coordinates -> [N, 3] unit bearings; the distorted
        point is divided by 1 + k1 r^2 before normalising."""
        s = self.simple_intrinsics
        p = np.asarray(points, np.float64).reshape(-1, 2)
        y = (p[:, 1] - s.principal_point[1]) / s.focals[1]
        x = (p[:, 0] - s.principal_point[0] - s.skew * y) / s.focals[0]
        d = 1.0 + self.k1 * (x * x + y * y)
        x, y = x / d, y / d
        n = np.sqrt(x * x + y * y + 1.0)
        return np.stack([x / n, y / n, 1.0 / n], 1)

    def uncalibrate(self, bearings):
        """CameraModel::uncalibrate (cv-pinhole/src/lib.rs:224-239): unit bearings -> pixel coordinates.  NaN rows where the reference
        returns None (z not sign-positive); its quadratic form is kept, so NaN also where k1 * |u|^2 == 0 (k1 = 0, or the principal
        point) and where 4 k1 |u|^2 > 1."""
        s, k1 = self.simple_intrinsics, self.k1
        b = np.asarray(bearings, np.float64).reshape(-1, 3)
        with np.errstate(divide="ignore", invalid="ignore"):
            ux, uy = b[:, 0] / b[:, 2], b[:, 1] / b[:, 2]
            u2 = ux * ux + uy * uy
            r2_mul_k1 = -(2.0 * k1 * u2 + np.sqrt(1.0 - 4.0 * k1 * u2) - 1.0) / (2.0 * k1 * u2)
            dx, dy = ux * (1.0 + r2_mul_k1), uy * (1.0 + r2_mul_k1)
            px = dx * s.focals[0] + s.skew * dy + s.principal_point[0]
            py = dy * s.focals[1] + s.principal_point[1]
        out = np.stack([px, py], 1)
        out[np.signbit(b[:, 2])] = np.nan
        return out

    def calibrate_keypoints(self, kps):
        """akaze::KeyPoint implements ImagePoint via (point.0 as f64, point.1 as f64) (akaze/src/lib.rs:95-99)."""
        return self.calibrate(np.stack([kps["x"].astype(np.float64), kps["y"].astype(np.float64)], 1))


# ---- include/cvb200_pinhole.h ----------------------------------------------------------------------------------------------------
def _lib(ctx):
    ctx = ctx or default_context(0)
    L = load_pinhole_library()
    if not getattr(L, "_pinhole_bound", False):
        vp, u32, f64, T = C.c_void_p, C.c_uint32, C.c_double, C.POINTER(TriangulatorCfg)
        L.cvb_pose_reprojection_error.argtypes = [vp, T, vp, u32, vp, vp, u32, vp, vp, vp]
        L.cvb_pose_reprojection_error_dev.argtypes = [vp, T, vp, u32, vp, vp, vp, u32, vp, vp, vp, vp]
        L.cvb_eight_point_essential_batch.argtypes = [vp, f64, u32, vp, vp, u32, vp, u32, vp, vp]
        L.cvb_residuals_essential.argtypes = [vp, vp, u32, vp, vp, u32, vp]
        L.cvb_essential_recondition.argtypes = [vp, vp, u32, f64, u32, vp, vp]
        L.cvb_essential_decompose.argtypes = [vp, vp, u32, f64, u32, vp, vp, vp, vp]
        L._pinhole_bound = True
    return ctx, L


def _reprojection(poses, a, b, triangulator, ctx):
    ctx, L = _lib(ctx)
    if isinstance(poses, tuple) and len(poses) == 2 and np.asarray(poses[0]).shape == (3, 3):
        poses = [poses]
    p = _poses_in(poses); a = _f64(a, 3); b = _f64(b, 3)
    _same_len(a, b)
    n = len(a)
    if len(p) not in (1, n):
        raise ValueError(f"expected 1 or {n} poses, got {len(p)}")
    err = np.zeros((n, 4), np.float64); avg = np.zeros(n, np.float64); ok = np.zeros(n, np.uint8)
    ctx.check(L.cvb_pose_reprojection_error(ctx.handle, C.byref(triangulator.cfg), p.ctypes.data, len(p), a.ctypes.data, b.ctypes.data, n,
                                            err.ctypes.data, avg.ctypes.data, ok.ctypes.data))
    return err.reshape(n, 2, 2), avg, ok.astype(bool)


def pose_reprojection_error_batch(poses, a, b, triangulator, ctx=None):
    """pose_reprojection_error for n FeatureMatches (a, b [n, 3] bearings) with one CameraToCamera pose (R, t) for all or one per match
    -> (errors[n, 2, 2]: [a_norm - reproject_a, b_norm - reproject_b], ok[n] bool).  triangulator: any of cv_b200's six."""
    err, _, ok = _reprojection(poses, a, b, triangulator, ctx)
    return err, ok


def average_pose_reprojection_error_batch(poses, a, b, triangulator, ctx=None):
    """average_pose_reprojection_error for n FeatureMatches -> (average[n], ok[n] bool)"""
    _, avg, ok = _reprojection(poses, a, b, triangulator, ctx)
    return avg, ok


def pose_reprojection_error(pose, a, b, triangulator, ctx=None):
    """cv_pinhole::pose_reprojection_error(pose, FeatureMatch(a, b), triangulator) -> [2, 2] array or None"""
    err, ok = pose_reprojection_error_batch([pose], np.reshape(a, (1, 3)), np.reshape(b, (1, 3)), triangulator, ctx)
    return err[0] if ok[0] else None


def average_pose_reprojection_error(pose, a, b, triangulator, ctx=None):
    """cv_pinhole::average_pose_reprojection_error(pose, FeatureMatch(a, b), triangulator) -> float or None"""
    avg, ok = average_pose_reprojection_error_batch([pose], np.reshape(a, (1, 3)), np.reshape(b, (1, 3)), triangulator, ctx)
    return float(avg[0]) if ok[0] else None


def pose_reprojection_error_dev(poses_dev, npose, a_dev, b_dev, n_dev, n_max, found_dev, err_dev, avg_dev, ok_dev, triangulator, ctx=None):
    """cvb_pose_reprojection_error_dev on device pointers (ints, e.g. torch's data_ptr(); found_dev and avg_dev may be 0), enqueued on
    ctx's stream without a synchronisation: the outputs of cvb_arrsac_eight_point_dev and cvb_pair_bearings(_k1)_dev in, err (n_max x 4),
    avg (n_max) and ok (n_max) out; rows at or past *n_dev are left untouched."""
    ctx, L = _lib(ctx)
    ctx.check(L.cvb_pose_reprojection_error_dev(ctx.handle, C.byref(triangulator.cfg), poses_dev, npose, a_dev, b_dev, n_dev, n_max,
                                                found_dev or None, err_dev, avg_dev or None, ok_dev))


def _mats(E):
    E = np.ascontiguousarray(E, np.float64)
    if E.shape[-2:] != (3, 3):
        raise ValueError("expected [m, 3, 3] matrices")
    return E.reshape(-1, 9)


def residuals_essential(Es, a, b, ctx=None):
    """EssentialMatrix::residual of every (E, FeatureMatch): Es [m, 3, 3], a, b [n, 3] -> [m, n]"""
    ctx, L = _lib(ctx)
    E = _mats(Es); a = _f64(a, 3); b = _f64(b, 3)
    _same_len(a, b)
    out = np.zeros((len(E), len(a)), np.float64)
    ctx.check(L.cvb_residuals_essential(ctx.handle, E.ctypes.data, len(E), a.ctypes.data, b.ctypes.data, len(a), out.ctypes.data))
    return out


def essential_recondition_batch(Es, epsilon, max_iterations, ctx=None):
    """EssentialMatrix::recondition of m matrices -> (E[m, 3, 3], ok[m] bool)"""
    ctx, L = _lib(ctx)
    E = _mats(Es)
    out = np.zeros((len(E), 9), np.float64); ok = np.zeros(len(E), np.uint8)
    ctx.check(L.cvb_essential_recondition(ctx.handle, E.ctypes.data, len(E), epsilon, int(max_iterations), out.ctypes.data, ok.ctypes.data))
    return out.reshape(-1, 3, 3), ok.astype(bool)


def essential_decompose_batch(Es, epsilon, max_iterations, ctx=None):
    """EssentialMatrix::possible_rotations_unscaled_translation of m matrices -> (rot_a[m, 3, 3], rot_b[m, 3, 3], t[m, 3], ok[m] bool)"""
    ctx, L = _lib(ctx)
    E = _mats(Es)
    m = len(E)
    ra = np.zeros((m, 9), np.float64); rb = np.zeros((m, 9), np.float64); t = np.zeros((m, 3), np.float64); ok = np.zeros(m, np.uint8)
    ctx.check(L.cvb_essential_decompose(ctx.handle, E.ctypes.data, m, epsilon, int(max_iterations), ra.ctypes.data, rb.ctypes.data,
                                        t.ctypes.data, ok.ctypes.data))
    return ra.reshape(-1, 3, 3), rb.reshape(-1, 3, 3), t, ok.astype(bool)


def eight_point_essential_batch(a, b, samples, epsilon=1e-12, iterations=1000, ctx=None):
    """EightPoint { epsilon, iterations }::from_matches for H samples of 8 match indices -> (E[H, 3, 3], ok[H] bool)"""
    ctx, L = _lib(ctx)
    a, b = _f64(a, 3), _f64(b, 3)
    _same_len(a, b)
    s = np.ascontiguousarray(samples, np.uint32).reshape(-1, 8)
    E = np.zeros((len(s), 9), np.float64); ok = np.zeros(len(s), np.uint8)
    ctx.check(L.cvb_eight_point_essential_batch(ctx.handle, epsilon, int(iterations), a.ctypes.data, b.ctypes.data, len(a), s.ctypes.data,
                                                len(s), E.ctypes.data, ok.ctypes.data))
    return E.reshape(-1, 3, 3), ok.astype(bool)


def _cross_matrix(t):
    return np.array([[0.0, -t[2], t[1]], [t[2], 0.0, -t[0]], [-t[1], t[0], 0.0]])


class EssentialMatrix:
    """cv_pinhole::EssentialMatrix (essential.rs:56-275): `mat` is the 3 x 3 matrix.  Methods return None where the reference does."""

    def __init__(self, mat):
        self.mat = np.array(mat, np.float64).reshape(3, 3)

    def __repr__(self):
        return f"EssentialMatrix({self.mat.tolist()!r})"

    @classmethod
    def from_pose(cls, pose):
        """From<CameraToCamera> (essential.rs:249-253): [t]x R, host numpy.  pose: (R, t)."""
        R, t = pose
        return cls(_cross_matrix(np.asarray(t, np.float64).reshape(3)) @ np.asarray(R, np.float64).reshape(3, 3))

    def residuals(self, a, b, ctx=None):
        """Model<FeatureMatch>::residual for n matches -> [n]"""
        return residuals_essential(self.mat[None], a, b, ctx)[0]

    def recondition(self, epsilon, max_iterations, ctx=None):
        E, ok = essential_recondition_batch(self.mat[None], epsilon, max_iterations, ctx)
        return EssentialMatrix(E[0]) if ok[0] else None

    def possible_rotations_unscaled_translation(self, epsilon, max_iterations, ctx=None):
        """-> (rot_a, rot_b, t) or None"""
        ra, rb, t, ok = essential_decompose_batch(self.mat[None], epsilon, max_iterations, ctx)
        return (ra[0], rb[0], t[0]) if ok[0] else None

    def possible_rotations(self, epsilon, max_iterations, ctx=None):
        """-> [rot_a, rot_b] or None"""
        r = self.possible_rotations_unscaled_translation(epsilon, max_iterations, ctx)
        return None if r is None else [r[0], r[1]]

    def possible_unscaled_poses(self, epsilon, max_iterations, ctx=None):
        """-> [(rot_a, t), (rot_b, t), (rot_a, -t), (rot_b, -t)] CameraToCamera poses or None"""
        r = self.possible_rotations_unscaled_translation(epsilon, max_iterations, ctx)
        return None if r is None else [(r[0], r[2]), (r[1], r[2]), (r[0], -r[2]), (r[1], -r[2])]

    def possible_unscaled_poses_bearing(self, epsilon, max_iterations, ctx=None):
        """-> [(rot_a, t), (rot_b, t)] or None"""
        r = self.possible_rotations_unscaled_translation(epsilon, max_iterations, ctx)
        return None if r is None else [(r[0], r[2]), (r[1], r[2])]
