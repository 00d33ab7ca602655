// cv_b200/csrc/c2c_filter.cuh -- floating-point filter for the consensus predicate
//     CameraToCamera::residual(pose, FeatureMatch(a, b)) < inlier_threshold        (cv-core/src/pose.rs:249-296)
//
// ARRSAC consumes only that one bit per (hypothesis, datum).  The reference obtains it from a full 4x4 symmetric
// eigen-decomposition (residual_c2c in geom.cu restates it with cyclic Jacobi: ~6 k FP64 instructions).  This filter
// decides the same bit with ~25-40 instructions for most outliers (epipolar and cheirality pre-tests) and ~0.8 k instructions otherwise, whenever the decision is provably insensitive to rounding, and
// returns "undecided" otherwise; the caller then runs the exact routine.  It is an exact-predicate filter in the
// computational-geometry sense, not an approximation of the result:
//
//   D = A_a + A_b (the 4x4 two-view design matrix of pose.rs:256-277), eigenvalues 0 <= l1 <= l2 <= l3 <= l4.
//   (1) residual >= l1 / (4 (1 + |t|^2))     [for the minimiser X: l1 = |X_xyz|^2 sin^2(alpha) + |P X|^2 sin^2(beta),
//        |X_xyz| <= 1, |P X|^2 <= 1 + |t|^2, residual = sin^2(alpha/2) + sin^2(beta/2) >= (sin^2 alpha + sin^2 beta)/4]
//       => with s_lo = 8 (1 + |t|^2) thr:  l1 >= s_lo  implies  residual >= 2 thr: certain outlier.
//   (2) the number of negative pivots of an LDL^T factorisation of D - s I equals the number of eigenvalues below s
//       (Sylvester's law of inertia).  Exactly one negative pivot at s_lo and exactly one at s_hi = min(1024 s_lo, 0.01)
//       (>= 16 s_lo, else the filter declines) gives l1 < s_lo < s_hi < l2: inverse iteration with shift s_lo then contracts
//       the error by <= s_lo / (s_hi - s_lo) <= 1/15 per step (1e-3 at the production threshold 1e-7), and a final step that
//       turns the vector by < 1e-11 certifies the eigenvector to ~1e-12 (error after the step <= turn * c / (1 - c) at contraction c).
//       When the count at s_hi is not 1 (small gap l2: low parallax), lower upper shifts s_hi / 8, s_hi / 64, ... down to 16 s_lo
//       are tried: exactly one negative pivot at any of them gives l1 < s_lo < s < l2 and a contraction <= 1/15, which is the case the
//       certificate above is sized for, so the same turn tolerance and residual band apply; only more checked steps may be needed.
//   (3) the residual of that eigenvector is computed with the reference's formula; if it is further from the threshold
//       than 1e-11 + 1e-4 thr (orders of magnitude above the rounding of either evaluation) the comparison is decided.
//   Anything else (tiny pivots, l2 < 16 s_lo, non-finite values, slow convergence, residual inside the band, thresholds so
//   large that s_hi is not small) returns -1.
//
// Compiles for the device (nvcc) and for the host (g++; only the CPU tests do that, to compare every decision with the exact CPU evaluation).
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define C2C_HD __host__ __device__ __forceinline__
#else
#define C2C_HD static inline
#endif
// The filter certifies its decisions by margins, not by bit-equality with anything, so the device build may contract a * b + c
// into one DFMA (the library is compiled -fmad=false for the bit-exact kernels); the host build used by the CPU tests keeps
// separate roundings.  Both are valid evaluations of the same bounds.
#if defined(__CUDA_ARCH__)
#define C2C_FMA(a, b, c) fma((a), (b), (c))
#define C2C_RSQRT(a) rsqrt(a)
#else
#define C2C_FMA(a, b, c) ((a) * (b) + (c))
#define C2C_RSQRT(a) (1.0 / sqrt(a))
#endif

// LDL^T of the symmetric 4x4 matrix m (full storage, row-major) minus s*I.  d[] = pivots, l[] = the six multipliers
// (l10 l20 l30 l21 l31 l32), inv[0..2] = reciprocals of the first three pivots.  Returns the number of negative pivots, or -1 when a
// pivot is too small to trust its sign.
C2C_HD int c2c_ldl4(const double *m, double s, double *d, double *l, double *inv) {
    const double tiny = 1e-11;
    const double m00 = m[0] - s, m11 = m[5] - s, m22 = m[10] - s, m33 = m[15] - s;
    const double m10 = m[4], m20 = m[8], m30 = m[12], m21 = m[9], m31 = m[13], m32 = m[14];
    int neg = 0;
    d[0] = m00;
    if (!(fabs(d[0]) > tiny)) return -1;
    neg += d[0] < 0.0;
    const double i0 = 1.0 / d[0];
    inv[0] = i0;
    l[0] = m10 * i0; l[1] = m20 * i0; l[2] = m30 * i0;
    d[1] = C2C_FMA(-l[0], m10, m11);
    if (!(fabs(d[1]) > tiny)) return -1;
    neg += d[1] < 0.0;
    const double i1 = 1.0 / d[1];
    inv[1] = i1;
    const double u21 = C2C_FMA(-l[1], m10, m21), u31 = C2C_FMA(-l[2], m10, m31);
    l[3] = u21 * i1; l[4] = u31 * i1;
    d[2] = C2C_FMA(-l[3], u21, C2C_FMA(-l[1], m20, m22));
    if (!(fabs(d[2]) > tiny)) return -1;
    neg += d[2] < 0.0;
    const double i2 = 1.0 / d[2];
    inv[2] = i2;
    const double u32 = C2C_FMA(-l[4], u21, C2C_FMA(-l[2], m20, m32));
    l[5] = u32 * i2;
    d[3] = C2C_FMA(-l[5], u32, C2C_FMA(-l[4], u31, C2C_FMA(-l[2], m30, m33)));
    if (!(fabs(d[3]) > 0.0)) return -1;      // the last pivot may be arbitrarily small (l1 close to s): its sign is not used by callers that see 0 or 1 above
    neg += d[3] < 0.0;
    return neg;
}

// x <- (L D L^T)^-1 x
C2C_HD void c2c_ldl4_solve(const double *id, const double *l, double *x) {
    x[1] = C2C_FMA(-l[0], x[0], x[1]);
    x[2] = C2C_FMA(-l[3], x[1], C2C_FMA(-l[1], x[0], x[2]));
    x[3] = C2C_FMA(-l[5], x[2], C2C_FMA(-l[4], x[1], C2C_FMA(-l[2], x[0], x[3])));
    x[0] *= id[0]; x[1] *= id[1]; x[2] *= id[2]; x[3] *= id[3];
    x[2] = C2C_FMA(-l[5], x[3], x[2]);
    x[1] = C2C_FMA(-l[4], x[3], C2C_FMA(-l[3], x[2], x[1]));
    x[0] = C2C_FMA(-l[2], x[3], C2C_FMA(-l[1], x[2], C2C_FMA(-l[0], x[1], x[0])));
}

C2C_HD double c2c_dot4(const double *x, const double *y) {
    return C2C_FMA(x[3], y[3], C2C_FMA(x[2], y[2], C2C_FMA(x[1], y[1], x[0] * y[0])));
}

C2C_HD void c2c_normalise4(double *x) {
    const double in = C2C_RSQRT(c2c_dot4(x, x));
    x[0] *= in; x[1] *= in; x[2] *= in; x[3] *= in;
}

// R row-major 3x3, t[3]: the CameraToCamera pose; a, b: unit bearings of the match.
// Returns 1 (residual < thr), 0 (residual >= thr) or -1 (undecided: evaluate exactly).
C2C_HD int c2c_inlier_filter(const double *R, const double *t, const double *a, const double *b, double thr) {
    const double tt = 1.0 + (t[0] * t[0] + t[1] * t[1] + t[2] * t[2]);
    const double s_lo = 8.0 * tt * thr, s_hi = fmin(1024.0 * s_lo, 0.01);
    if (!(s_hi >= 16.0 * s_lo) || !(thr > 0.0)) return -1;      // contraction <= 1/15 per step, or no filter
    // (0) epipolar pre-test (~25 instructions; decides the bulk of the predicates of a wrong hypothesis).  Whatever point X the
    //     reference triangulates, its bearings a' (first camera) and b' (second camera) are coplanar with the baseline:
    //     b'^T [t]x R a' = 0.  The residual is sin^2(alpha/2) + sin^2(beta/2) with alpha = angle(a, a'), beta = angle(b, b'), and
    //     |a - a'| = 2 sin(alpha/2), |b - b'| = 2 sin(beta/2), ||[t]x R|| = |t|, so
    //       |b^T [t]x R a| = |b^T E a - b'^T E a'| <= |t| (|a - a'| + |b - b'|) <= 2 sqrt(2) |t| sqrt(residual),
    //     i.e. residual >= e^2 / (8 |t|^2).  With a 6 % margin (rounding of e is ~1e-16 |t|): certain outlier.
    {
        const double ra0 = C2C_FMA(R[2], a[2], C2C_FMA(R[1], a[1], R[0] * a[0])), ra1 = C2C_FMA(R[5], a[2], C2C_FMA(R[4], a[1], R[3] * a[0])),
                     ra2 = C2C_FMA(R[8], a[2], C2C_FMA(R[7], a[1], R[6] * a[0]));
        const double c0 = C2C_FMA(t[1], ra2, -(t[2] * ra1)), c1 = C2C_FMA(t[2], ra0, -(t[0] * ra2)), c2 = C2C_FMA(t[0], ra1, -(t[1] * ra0));
        const double e = C2C_FMA(b[2], c2, C2C_FMA(b[1], c1, b[0] * c0));
        if (e * e > 8.5 * (tt - 1.0) * thr + 1e-28) return 0;
        // (0b) cheirality pre-test (~12 more instructions).  An essential matrix yields four poses with the SAME epipolar error; three of
        //     them put the point behind a camera, and the reference finds that out only through the full evaluation (its residual
        //     is then ~1).  Whatever X it triangulates: p = from_homogeneous(X) has unit xyz p^ and w >= 0, q = R p^ + w t, q^ = q / |q|,
        //     residual = ((1 - a.p^) + (1 - b.q^)) / 2.  residual < thr forces |a - p^|^2 + |b - q^|^2 < 4 thr.  With u' = R p^, b' = q^:
        //       u' + w t = |q| b'   =>   w (u' x t) = |q| (u' x b')  and  (u' x b') = w (b' x t)          (cross with u', with b')
        //     hence  (u' x t).(u' x b') = t.b' - (u'.b')(t.u') >= 0   and   (u' x b').(b' x t) = (u'.b')(t.b') - t.u' >= 0.
        //     Replacing u', b' by u = R a, b moves either expression by at most 2 |t| (|a - p^| + |b - q^|) <= 5.66 |t| sqrt(thr);
        //     a value below -10 |t| sqrt(thr) therefore excludes an inlier.  (Only for small thresholds: the bound is linearised.)
        if (thr <= 1e-4) {
            const double tb = C2C_FMA(t[2], b[2], C2C_FMA(t[1], b[1], t[0] * b[0])), ub = C2C_FMA(ra2, b[2], C2C_FMA(ra1, b[1], ra0 * b[0])),
                         tu = C2C_FMA(t[2], ra2, C2C_FMA(t[1], ra1, t[0] * ra0));
            const double c1 = C2C_FMA(-ub, tu, tb), c2 = C2C_FMA(ub, tb, -tu);
            const double lim2 = 100.0 * (tt - 1.0) * thr;
            if ((c1 < 0.0 && c1 * c1 > lim2) || (c2 < 0.0 && c2 * c2 > lim2)) return 0;
        }
    }
    // D = sum over the two views of (M - b b^T M)^T (M - b b^T M), M = [I | 0] resp. [R | t]   (pose.rs:256-277)
    double D[16];
    {
        // view a: columns c = 0..2 are e_c - a a_c, column 3 is zero
        double Ta[3][3];
        for (int c = 0; c < 3; c++)
            for (int r = 0; r < 3; r++) Ta[r][c] = C2C_FMA(-a[r], a[c], r == c ? 1.0 : 0.0);
        double Tb[3][4];
        for (int c = 0; c < 4; c++) {
            const double m0 = c < 3 ? R[c] : t[0], m1 = c < 3 ? R[3 + c] : t[1], m2 = c < 3 ? R[6 + c] : t[2];
            const double btm = C2C_FMA(b[2], m2, C2C_FMA(b[1], m1, b[0] * m0));
            Tb[0][c] = C2C_FMA(-b[0], btm, m0); Tb[1][c] = C2C_FMA(-b[1], btm, m1); Tb[2][c] = C2C_FMA(-b[2], btm, m2);
        }
        for (int i = 0; i < 4; i++)
            for (int j = 0; j <= i; j++) {
                double v = C2C_FMA(Tb[2][i], Tb[2][j], C2C_FMA(Tb[1][i], Tb[1][j], Tb[0][i] * Tb[0][j]));
                if (i < 3) v = C2C_FMA(Ta[2][i], Ta[2][j], C2C_FMA(Ta[1][i], Ta[1][j], C2C_FMA(Ta[0][i], Ta[0][j], v)));
                D[i * 4 + j] = v; D[j * 4 + i] = v;
            }
    }
    double d[4], l[6], id[4], dh[4], lh[6], ih[4];
    const int c_lo = c2c_ldl4(D, s_lo, d, l, id);
    if (c_lo == 0) return 0;                       // l1 > s_lo: residual >= 2 thr
    if (c_lo != 1) return -1;
    // need l2 > s for the contraction bound: s = s_hi, then a ladder of lower shifts down to 16 s_lo (small spectral gap, low
    // parallax).  Every rung keeps the contraction <= s_lo / (s - s_lo) <= 1/15, the worst case the certificate below is sized for.
    for (double s = s_hi; c2c_ldl4(D, s, dh, lh, ih) != 1;) {
        s *= 0.125;
        if (!(s >= 16.0 * s_lo)) return -1;
    }
    id[3] = 1.0 / d[3];
    // inverse iteration with shift s_lo.  Four solves without normalisation (growth <= 1 / |l1 - s_lo| per solve, harmless in
    // f64; error <= 1e-12 at the production threshold), one normalisation, then a checked step y = (D - s_lo I)^-1 x: the
    // direction must not turn by more than 1e-11, measured without a square root or a division as
    //   sin^2(angle(x, y)) = |y - (x.y) x|^2 / |y|^2 <= 1e-22        (|x| = 1).
    // Everything behind this point is independent of the scale of the eigenvector (from_homogeneous divides by |xyz|), so the
    // accepted iterate is used as it is; only a rejected one is normalised for the next turn.  Non-finite values fail the test.
    double x[4] = {0.5, 0.5, 0.5, 0.5};
    c2c_ldl4_solve(id, l, x);
    c2c_ldl4_solve(id, l, x);
    c2c_ldl4_solve(id, l, x);
    c2c_ldl4_solve(id, l, x);
    c2c_normalise4(x);
    double y[4], yy = 0.0;
    int certified = 0;
    for (int it = 0; it < 12; it++) {            // at contraction 1/15: 4 blind + 12 checked steps take an error of 10^7 below 1e-11
        y[0] = x[0]; y[1] = x[1]; y[2] = x[2]; y[3] = x[3];
        c2c_ldl4_solve(id, l, y);
        const double xy = c2c_dot4(x, y);
        yy = c2c_dot4(y, y);
        double r2 = 0.0;
        for (int k = 0; k < 4; k++) { const double r = C2C_FMA(-xy, x[k], y[k]); r2 = C2C_FMA(r, r, r2); }
        if (r2 <= 1e-22 * yy) { certified = 1; break; }
        const double in = C2C_RSQRT(yy);
        for (int k = 0; k < 4; k++) x[k] = y[k] * in;
    }
    if (!certified) return -1;
    // pose.rs:284-295: from_homogeneous (sign of w, unit xyz), transform, cosine distances
    double p[4] = {y[0], y[1], y[2], y[3]};
    if (signbit(p[3])) { p[0] = -p[0]; p[1] = -p[1]; p[2] = -p[2]; p[3] = -p[3]; }
    const double pp = p[0] * p[0] + p[1] * p[1] + p[2] * p[2];
    if (!(pp > 1e-18 * yy)) return -1;
    const double ipn = C2C_RSQRT(pp);
    p[0] *= ipn; p[1] *= ipn; p[2] *= ipn; p[3] *= ipn;
    double q[3];
    for (int r = 0; r < 3; r++) q[r] = R[3 * r] * p[0] + R[3 * r + 1] * p[1] + R[3 * r + 2] * p[2] + t[r] * p[3];
    const double qq = q[0] * q[0] + q[1] * q[1] + q[2] * q[2];
    if (!(qq > 1e-18)) return -1;
    const double res = 0.5 * (1.0 - (a[0] * p[0] + a[1] * p[1] + a[2] * p[2]) + 1.0 - (b[0] * q[0] + b[1] * q[1] + b[2] * q[2]) * C2C_RSQRT(qq));
    if (!isfinite(res)) return -1;
    if (fabs(res - thr) <= 1e-11 + 1e-4 * thr) return -1;
    return res < thr ? 1 : 0;
}
