"""cv_pinhole::CameraIntrinsics (no distortion) and CameraIntrinsicsK1Distortion: pixel <-> unit bearing (cv-pinhole/src/lib.rs:32-240).

Scalar per-keypoint host work in the reference (SURVEY.md section 8a row C1, "negligible; keep on host"); it is
vectorised here over all keypoints in f64 with the reference's operation order.
"""
from dataclasses import dataclass

import numpy as np


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
