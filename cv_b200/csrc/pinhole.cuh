// cv_b200/csrc/pinhole.cuh -- pixel -> unit bearing on the device, shared by the pair bearings (geom.cu) and frame ingestion (frame.cu).
#pragma once
#include "common.cuh"

// CameraIntrinsicsK1Distortion::calibrate (cv-pinhole/src/lib.rs:191-202) in f64 with the reference's operation order: centre, divide
// by the focals, remove skew, divide both components by 1 + k1 r^2 (a true division, as nalgebra's Vector2 / f64), then
// UnitVector3::new_normalize of (x, y, 1).  With k1 = 0 the divisor is exactly 1.0 and x / 1.0 == x, so this is bit for bit
// CameraIntrinsics::calibrate (:108-116) and serves both cameras.  Requires -fmad=false (no contraction of x * x + y * y).
__device__ __forceinline__ void calibrate_k1(const cvb_intrinsics_k1 &K, double px, double py, double *o) {
    const double y0 = (py - K.cy) / K.fy;
    const double x0 = (px - K.cx - K.skew * y0) / K.fx;
    const double d = 1.0 + K.k1 * (x0 * x0 + y0 * y0);
    const double x = x0 / d, y = y0 / d;
    const double n = sqrt(x * x + y * y + 1.0);
    o[0] = x / n; o[1] = y / n; o[2] = 1.0 / n;
}

static inline cvb_intrinsics_k1 intrinsics_k1(const cvb_intrinsics &K) { return cvb_intrinsics_k1{K.fx, K.fy, K.cx, K.cy, K.skew, 0.0}; }
