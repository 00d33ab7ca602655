// cv_b200/csrc/geom.cu -- batched geometric verification on sm_90a (f64).
//
// Every model hypothesis (eight-point / P3P minimal solve) and every (hypothesis, datum) residual runs on
// the GPU, one thread per hypothesis resp. per (hypothesis, datum) pair; ARRSAC's inherently sequential
// bookkeeping (likelihood-ratio test over hypotheses, sort / truncate, RNG draws) stays on the host and
// consumes bit-packed inlier masks.  Reference lines are cited per function (paths relative to the reference checkout).
// The linear algebra that lives in nalgebra upstream (symmetric eigen, SVD, from_matrix_eps) is implemented
// here as cyclic Jacobi / closed forms; f64 results are held to 1e-6 relative (BASELINE north_star) in the parity tests.
#include <float.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <vector>
#include <cooperative_groups.h>
#include "common.cuh"
#include "../../include/cvb200_tri.h"
#include "../../include/cvb200_opt.h"
#include "../../include/cvb200_pinhole.h"
#include "../../include/cvb200_batch.h"
#include "../../include/cvb200_init.h"
#include "../../include/cvb200_constraints.h"
#include "../../include/cvb200_reconstruction.h"
#include "../../include/cvb200_export.h"
#include "../../include/cvb200_register.h"
#include "../../include/cvb200_incorporate.h"
#include "../../include/cvb200_merge.h"
#include "../../include/cvb200_try_init.h"
#include "c2c_filter.cuh"
#include "pinhole.cuh"

namespace {

// ------------------------------------------------------------------------------------------ device math
// One cyclic Jacobi rotation, written with explicit roundings so that the one-thread and the lane-cooperative eigensolvers
// (below) produce the same bits whatever the compiler would contract.
__device__ __forceinline__ void jacobi_cs(double app, double aqq, double apq, double &c, double &s) {
    const double theta = __ddiv_rn(__dsub_rn(aqq, app), __dmul_rn(2.0, apq));
    const double t = __ddiv_rn(theta >= 0.0 ? 1.0 : -1.0, __dadd_rn(fabs(theta), __dsqrt_rn(__dadd_rn(__dmul_rn(theta, theta), 1.0))));
    c = __ddiv_rn(1.0, __dsqrt_rn(__dadd_rn(__dmul_rn(t, t), 1.0)));
    s = __dmul_rn(t, c);
}
__device__ __forceinline__ void jacobi_rot(double &x, double &y, double c, double s) {
    const double a = x, b = y;
    x = __dsub_rn(__dmul_rn(c, a), __dmul_rn(s, b));
    y = __dadd_rn(__dmul_rn(s, a), __dmul_rn(c, b));
}

template <int N>
__device__ bool sym_eigen(const double *Ain, double eps, int max_sweeps, double *d, double *V) {
    double A[N * N];
#pragma unroll
    for (int i = 0; i < N * N; i++) A[i] = Ain[i];
    for (int i = 0; i < N; i++)
        for (int j = 0; j < N; j++) V[i * N + j] = i == j ? 1.0 : 0.0;
    for (int sweep = 0; sweep < max_sweeps; sweep++) {
        double off = 0.0, diag = 0.0;
        for (int i = 0; i < N; i++) {
            diag = __dadd_rn(diag, __dmul_rn(A[i * N + i], A[i * N + i]));
            for (int j = i + 1; j < N; j++) off = __dadd_rn(off, __dmul_rn(A[i * N + j], A[i * N + j]));
        }
        if (off <= eps * eps * diag || off == 0.0) {
            for (int i = 0; i < N; i++) d[i] = A[i * N + i];
            return true;
        }
        for (int p = 0; p < N - 1; p++)
            for (int q = p + 1; q < N; q++) {
                const double apq = A[p * N + q];
                if (apq == 0.0) continue;
                double c, s;
                jacobi_cs(A[p * N + p], A[q * N + q], apq, c, s);
                for (int k = 0; k < N; k++) jacobi_rot(A[k * N + p], A[k * N + q], c, s);
                for (int k = 0; k < N; k++) jacobi_rot(A[p * N + k], A[q * N + k], c, s);
                for (int k = 0; k < N; k++) jacobi_rot(V[k * N + p], V[k * N + q], c, s);
            }
    }
    for (int i = 0; i < N; i++) d[i] = A[i * N + i];
    return false;
}

// The 9x9 eigensolver of the eight-point estimator: Jacobi in round-robin (tournament) order, restated on the checker's side as
// ref_sym_eigen9_rr.  A sweep is nine rounds; round r rotates the four DISJOINT index pairs {(r + k) mod 9, (r - k) mod 9}, k = 1..4:
// the angles come from the matrix in front of the round, then all column rotations (A and V), then all row rotations.  Disjoint pairs
// touch disjoint columns / rows, so JL = 1, 2 or 4 lanes (`mask` = those lanes, `lane` = 0..JL-1; A and V in shared memory, or thread
// local for JL = 1) each take their share of a round's pairs and produce the bits of the sequential order.  A sweep costs nine
// dependent rotation set-ups instead of 36, and the set-up itself is quotient-free: with d = aqq - app, h = 2 apq,
// w = |d| + sqrt(d^2 + h^2), n = sqrt(w^2 + h^2): c = w / n, s = +-|h| / n (two square roots and one level of division on the chain).
__device__ __forceinline__ void jacobi_cs_rr(double app, double aqq, double apq, double &c, double &s) {
    const double d = __dsub_rn(aqq, app), h = __dmul_rn(2.0, apq);
    const double w = __dadd_rn(fabs(d), __dsqrt_rn(__dadd_rn(__dmul_rn(d, d), __dmul_rn(h, h))));
    const double n = __dsqrt_rn(__dadd_rn(__dmul_rn(w, w), __dmul_rn(h, h)));
    const bool pos = d == 0.0 || ((d > 0.0) == (h > 0.0));
    c = __ddiv_rn(w, n);
    s = __ddiv_rn(pos ? fabs(h) : -fabs(h), n);
}
template <int JL>
__device__ bool sym_eigen9_rr(double *A, double *V, int lane, unsigned mask, double eps, int max_sweeps) {
    // JL = 1, 2, 4: a lane owns 4 / JL pairs of a round and all nine rows / columns of their updates;
    // JL = 8, 16: SUB = JL / 4 lanes share a pair (each forms the rotation itself) and split the nine rows / columns
    constexpr int N = 9, SUB = JL > 4 ? JL / 4 : 1, PL = JL >= 4 ? 1 : 4 / JL, PSTEP = JL / SUB;
    const int lp = lane / SUB, sub = lane % SUB;
    for (int e = lane; e < N * N; e += JL) V[e] = (e / N == e % N) ? 1.0 : 0.0;
    if (JL > 1) __syncwarp(mask);
    for (int sweep = 0; sweep < max_sweeps; sweep++) {
        double off = 0.0, diag = 0.0;
        for (int i = 0; i < N; i++) {
            diag = __dadd_rn(diag, __dmul_rn(A[i * N + i], A[i * N + i]));
            for (int j = i + 1; j < N; j++) off = __dadd_rn(off, __dmul_rn(A[i * N + j], A[i * N + j]));
        }
        if (off <= eps * eps * diag || off == 0.0) return true;
        for (int r = 0; r < N; r++) {
            int P[PL], Q[PL];
            bool act[PL];
            double Cc[PL], Ss[PL];
#pragma unroll
            for (int i = 0; i < PL; i++) {
                const int k = 1 + lp + i * PSTEP;
                int a = r + k, b = r + N - k;
                if (a >= N) a -= N;
                if (b >= N) b -= N;
                P[i] = min(a, b); Q[i] = max(a, b);
                const double apq = A[P[i] * N + Q[i]];
                act[i] = apq != 0.0;
                if (act[i]) jacobi_cs_rr(A[P[i] * N + P[i]], A[Q[i] * N + Q[i]], apq, Cc[i], Ss[i]);
            }
            // every lane has read its pivot block before a lane of the same pair rewrites it (lanes of OTHER pairs never touch it:
            // they write their own pairs' columns only)
            if (SUB > 1) __syncwarp(mask);
#pragma unroll
            for (int i = 0; i < PL; i++) {
                if (!act[i]) continue;
                for (int k = sub; k < N; k += SUB) {
                    jacobi_rot(A[k * N + P[i]], A[k * N + Q[i]], Cc[i], Ss[i]);
                    jacobi_rot(V[k * N + P[i]], V[k * N + Q[i]], Cc[i], Ss[i]);
                }
            }
            if (JL > 1) __syncwarp(mask);
#pragma unroll
            for (int i = 0; i < PL; i++) {
                if (!act[i]) continue;
                for (int k = sub; k < N; k += SUB) jacobi_rot(A[P[i] * N + k], A[Q[i] * N + k], Cc[i], Ss[i]);
            }
            if (JL > 1) __syncwarp(mask);
        }
    }
    return false;
}

__device__ __forceinline__ double dot3(const double *a, const double *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
__device__ __forceinline__ double norm3(const double *a) { return sqrt(dot3(a, a)); }
__device__ __forceinline__ void cross3(const double *a, const double *b, double *o) {
    const double r0 = a[1] * b[2] - a[2] * b[1], r1 = a[2] * b[0] - a[0] * b[2], r2 = a[0] * b[1] - a[1] * b[0];
    o[0] = r0; o[1] = r1; o[2] = r2;
}
__device__ void mat3_mul(const double *a, const double *b, double *o) {
    double r[9];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) r[i * 3 + j] = a[i * 3] * b[j] + a[i * 3 + 1] * b[3 + j] + a[i * 3 + 2] * b[6 + j];
    for (int i = 0; i < 9; i++) o[i] = r[i];
}
__device__ __forceinline__ double det3(const double *m) {
    return m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) + m[2] * (m[3] * m[7] - m[4] * m[6]);
}

// sorted SVD of a 3x3 matrix through the eigen-decomposition of MtM; u3 = u1 x u2 (its sign is normalised by
// the det(U) > 0 rule of essential.rs:139-143 anyway).  S (may be null) receives the singular values, descending.
__device__ __noinline__ bool svd3(const double *M, double eps, int iters, double *U, double *Vt, double *S = nullptr) {
    double MtM[9], d[3], V[9];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) MtM[i * 3 + j] = M[i] * M[j] + M[3 + i] * M[3 + j] + M[6 + i] * M[6 + j];
    if (!sym_eigen<3>(MtM, eps, iters, d, V)) return false;
    int ord[3] = {0, 1, 2};
    for (int i = 0; i < 2; i++)
        for (int j = i + 1; j < 3; j++)
            if (d[ord[j]] > d[ord[i]]) { int t = ord[i]; ord[i] = ord[j]; ord[j] = t; }
    double v[3][3], u[3][3], s[3];
    for (int k = 0; k < 3; k++) {
        for (int r = 0; r < 3; r++) v[k][r] = V[r * 3 + ord[k]];
        s[k] = sqrt(d[ord[k]] > 0.0 ? d[ord[k]] : 0.0);
    }
    const double tiny = 1e-12 * (s[0] > 0.0 ? s[0] : 1.0);
    for (int k = 0; k < 2; k++) {
        if (!(s[k] > tiny)) return false;
        for (int r = 0; r < 3; r++) u[k][r] = (M[r * 3] * v[k][0] + M[r * 3 + 1] * v[k][1] + M[r * 3 + 2] * v[k][2]) / s[k];
    }
    cross3(u[0], u[1], u[2]);
    const double nn = norm3(u[2]);
    if (!(nn > 0.0)) return false;
    for (int r = 0; r < 3; r++) u[2][r] /= nn;
    for (int k = 0; k < 3; k++)
        for (int r = 0; r < 3; r++) { U[r * 3 + k] = u[k][r]; Vt[k * 3 + r] = v[k][r]; }
    if (S) for (int k = 0; k < 3; k++) S[k] = s[k];
    return true;
}

// eight-point/src/lib.rs:11-24,43-58 (incl. b / a.z) + cv-pinhole/src/essential.rs:114-162,217-231
__device__ __forceinline__ void eight_point_row(const double *a, const double *b, uint32_t id, double *row /* 9 */) {
    const double *pa = a + 3 * (size_t)id, *pb = b + 3 * (size_t)id;
    const double ap[3] = {pa[0] / pa[2], pa[1] / pa[2], pa[2] / pa[2]};
    const double bp[3] = {pb[0] / pa[2], pb[1] / pa[2], pb[2] / pa[2]};
    for (int j = 0; j < 3; j++)
        for (int k = 0; k < 3; k++) row[3 * j + k] = __dmul_rn(ap[j], bp[k]);
}
__device__ __forceinline__ double eight_point_gram(const double *D /* [8][9] */, int r, int c) {
    double s = 0.0;
    for (int i = 0; i < 8; i++) s = __dadd_rn(s, __dmul_rn(D[i * 9 + r], D[i * 9 + c]));
    return s;
}
// the four poses from the eigenvectors (V column-stacked, d = diagonal after convergence)
__device__ int eight_point_poses(const double *d, const double *V, cvb_pose *out) {
    int best = 0;
    for (int i = 1; i < 9; i++)
        if (d[i] < d[best]) best = i;
    double E[9];
    for (int k = 0; k < 9; k++) E[(k % 3) * 3 + (k / 3)] = V[k * 9 + best];   // Matrix3::from_iterator is column-major
    double U[9], Vt[9];
    if (!svd3(E, 1e-12, 1000, U, Vt)) return 0;
    if (det3(U) < 0.0) for (int r = 0; r < 3; r++) U[r * 3 + 2] *= -1.0;
    if (det3(Vt) < 0.0) for (int c = 0; c < 3; c++) Vt[6 + c] *= -1.0;
    const double W[9] = {0, -1, 0, 1, 0, 0, 0, 0, 1}, Wt[9] = {0, 1, 0, -1, 0, 0, 0, 0, 1};
    double UW[9], Ra[9], Rb[9];
    mat3_mul(U, W, UW); mat3_mul(UW, Vt, Ra);
    mat3_mul(U, Wt, UW); mat3_mul(UW, Vt, Rb);
    const double t[3] = {U[2], U[5], U[8]};
    for (int k = 0; k < 4; k++) {
        for (int i = 0; i < 9; i++) out[k].r[i] = (k & 1) ? Rb[i] : Ra[i];
        for (int r = 0; r < 3; r++) out[k].t[r] = (k & 2) ? -t[r] : t[r];
    }
    return 4;
}
__device__ int eight_point(const double *a, const double *b, const uint32_t *idx, cvb_pose *out) {
    double D[72], EtE[81], d[9], V[81];
    for (int i = 0; i < 8; i++) eight_point_row(a, b, idx[i], D + 9 * i);
    for (int r = 0; r < 9; r++)
        for (int c = 0; c < 9; c++) EtE[r * 9 + c] = eight_point_gram(D, r, c);
    if (!sym_eigen9_rr<1>(EtE, V, 0, 0u, 1e-12, 1000)) return 0;
    for (int i = 0; i < 9; i++) d[i] = EtE[i * 9 + i];
    return eight_point_poses(d, V, out);
}
// JL lanes per hypothesis; sh = 163 doubles of shared memory of this hypothesis (A | V, the design matrix lives in V's place first)
#define EIGHT_SH 163
template <int JL>
__device__ int eight_point_lanes(const double *a, const double *b, const uint32_t *idx, cvb_pose *out, double *sh, int lane, unsigned mask) {
    double *A = sh, *V = sh + 81;
    for (int i = lane; i < 8; i += JL) eight_point_row(a, b, idx[i], V + 9 * i);
    __syncwarp(mask);
    for (int e = lane; e < 81; e += JL) A[e] = eight_point_gram(V, e / 9, e % 9);
    __syncwarp(mask);
    const bool ok = sym_eigen9_rr<JL>(A, V, lane, mask, 1e-12, 1000);
    __syncwarp(mask);
    int n = 0;
    if (ok && lane == 0) {
        double d[9];
        for (int i = 0; i < 9; i++) d[i] = A[i * 9 + i];
        n = eight_point_poses(d, V, out);
    }
    return n;                                                    // valid on lane 0
}

__device__ __forceinline__ void from_homogeneous(double *p) {
    if (signbit(p[3])) { p[0] = -p[0]; p[1] = -p[1]; p[2] = -p[2]; p[3] = -p[3]; }
    const double n = norm3(p);
    p[0] /= n; p[1] /= n; p[2] /= n; p[3] /= n;
}
__device__ __forceinline__ void pose_apply(const cvb_pose &P, const double *x, double *o) {
    for (int r = 0; r < 3; r++) o[r] = dot3(P.r + 3 * r, x) + P.t[r] * x[3];
    o[3] = x[3];
}
__device__ void design_add(const double *R, const double *t, const double *b, double *D) {
    double M[3][4], T[3][4];
    for (int r = 0; r < 3; r++) { M[r][0] = R[3 * r]; M[r][1] = R[3 * r + 1]; M[r][2] = R[3 * r + 2]; M[r][3] = t[r]; }
    for (int c = 0; c < 4; c++) {
        const double btP = b[0] * M[0][c] + b[1] * M[1][c] + b[2] * M[2][c];
        for (int r = 0; r < 3; r++) T[r][c] = M[r][c] - b[r] * btP;
    }
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) D[i * 4 + j] += T[0][i] * T[0][j] + T[1][i] * T[1][j] + T[2][i] * T[2][j];
}

// cv-core/src/pose.rs:249-296: two-view linear-eigen triangulation inside the residual
__device__ double residual_c2c(const cvb_pose &P, const double *a, const double *b) {
    double D[16], d[4], V[16];
    for (int i = 0; i < 16; i++) D[i] = 0.0;
    const double I[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, z[3] = {0, 0, 0};
    design_add(I, z, a, D);
    design_add(P.r, P.t, b, D);
    if (!sym_eigen<4>(D, 1e-12, 1024, d, V)) return 2.0;
    int best = 0;
    for (int i = 1; i < 4; i++)
        if (fabs(d[i]) < fabs(d[best])) best = i;
    double p[4] = {V[best], V[4 + best], V[8 + best], V[12 + best]};
    from_homogeneous(p);
    for (int i = 0; i < 4; i++)
        if (!isfinite(p[i])) return 2.0;
    double q[4];
    pose_apply(P, p, q);
    from_homogeneous(q);
    return 0.5 * (1.0 - dot3(a, p) + 1.0 - dot3(b, q));
}

// cv-core/src/pose.rs:194-202
__device__ double residual_w2c(const cvb_pose &P, const double *bearing, const double *world) {
    double q[4];
    pose_apply(P, world, q);
    from_homogeneous(q);
    return 1.0 - dot3(bearing, q);
}

// ---- lambda twist (lambda-twist/src/lib.rs:110-317, 361-554)
__device__ void root2real(double b, double c, double *r1, double *r2) {
    const double disc = b * b - 4.0 * c;
    if (disc < 0.0) { *r1 = *r2 = 0.5 * b; }
    else if (b < 0.0) { const double y = sqrt(disc); *r1 = 0.5 * (-b + y); *r2 = 0.5 * (-b - y); }
    else { const double y = sqrt(disc); *r1 = 2.0 * c / (-b + y); *r2 = 2.0 * c / (-b - y); }
}
__device__ double cube_root(double b, double c, double d) {
    double r0;
    if (b * b >= 3.0 * c) {
        const double v = sqrt(b * b - 3.0 * c);
        const double t1 = (-b - v) / 3.0;
        double k = ((t1 + b) * t1 + c) * t1 + d;
        if (k > 0.0) r0 = t1 - sqrt(-k / (3.0 * t1 + b));
        else {
            const double t2 = (-b + v) / 3.0;
            k = ((t2 + b) * t2 + c) * t2 + d;
            r0 = t2 + sqrt(-k / (3.0 * t2 + b));
        }
    } else {
        r0 = -b / 3.0;
        if (fabs((3.0 * r0 + 2.0 * b) * r0 + c) < 1e-4) r0 += 1.0;
    }
    for (int i = 0; i < 7; i++) {
        const double fx = ((r0 + b) * r0 + c) * r0 + d, fpx = (3.0 * r0 + 2.0 * b) * r0 + c;
        r0 -= fx / fpx;
    }
    for (int i = 0; i < 43; i++) {
        const double fx = ((r0 + b) * r0 + c) * r0 + d;
        if (fabs(fx) > 1e-13) { const double fpx = (3.0 * r0 + 2.0 * b) * r0 + c; r0 -= fx / fpx; }
        else break;
    }
    return r0;
}
__device__ void eigen_decomposition_singular(const double *x, double *Ev, double *ev) {
    const double m11 = x[0], m12 = x[1], m13 = x[2], m21 = x[3], m22 = x[4], m23 = x[5], m31 = x[6], m32 = x[7], m33 = x[8];
    double v3[3] = {m21 * m32 - m31 * m22, m31 * m12 - m32 * m11, m22 * m11 - m21 * m12};
    const double n = norm3(v3);
    for (int i = 0; i < 3; i++) v3[i] /= n;
    const double x12_sqr = m12 * m12;
    const double b = -m11 - m22 - m33;
    const double c = -x12_sqr - m13 * m13 - m23 * m23 + m11 * (m22 + m33) + m22 * m33;
    double e1, e2;
    root2real(b, c, &e1, &e2);
    if (fabs(e1) < fabs(e2)) { const double t = e1; e1 = e2; e2 = t; }
    ev[0] = e1; ev[1] = e2; ev[2] = 0.0;
    const double mx0011 = -m11 * m22, prec_0 = m12 * m23 - m13 * m22, prec_1 = m12 * m13 - m11 * m23;
    const double es[2] = {e1, e2};
    double v[2][3];
    for (int k = 0; k < 2; k++) {
        const double e = es[k];
        const double tmp = 1.0 / (e * (m11 + m22) + mx0011 - e * e + x12_sqr);
        const double a1 = -(e * m13 + prec_0) * tmp, a2 = -(e * m23 + prec_1) * tmp;
        const double rnorm = 1.0 / sqrt(a1 * a1 + a2 * a2 + 1.0);
        v[k][0] = a1 * rnorm; v[k][1] = a2 * rnorm; v[k][2] = rnorm;
    }
    for (int r = 0; r < 3; r++) { Ev[r * 3] = v[0][r]; Ev[r * 3 + 1] = v[1][r]; Ev[r * 3 + 2] = v3[r]; }
}
__device__ __forceinline__ double l1n(const double *v) { return fabs(v[0]) + fabs(v[1]) + fabs(v[2]); }
__device__ void gn_residual(const double *l, double a12, double a13, double a23, double b12, double b13, double b23, double *r) {
    r[0] = l[0] * l[0] + l[1] * l[1] + b12 * l[0] * l[1] - a12;
    r[1] = l[0] * l[0] + l[2] * l[2] + b13 * l[0] * l[2] - a13;
    r[2] = l[1] * l[1] + l[2] * l[2] + b23 * l[1] * l[2] - a23;
}
__device__ void gauss_newton_refine_lambda(double *l, int iterations, double a12, double a13, double a23, double b12, double b13, double b23) {
    double res[3];
    gn_residual(l, a12, a13, a23, b12, b13, b23, res);
    for (int it = 0; it < iterations; it++) {
        if (l1n(res) < 1e-10) break;
        const double l1 = l[0], l2 = l[1], l3 = l[2];
        const double dr1dl1 = 2.0 * l1 + b12 * l2, dr1dl2 = 2.0 * l2 + b12 * l1, dr2dl1 = 2.0 * l1 + b13 * l3;
        const double dr2dl3 = 2.0 * l3 + b13 * l1, dr3dl2 = 2.0 * l2 + b23 * l3, dr3dl3 = 2.0 * l3 + b23 * l2;
        const double det = 1.0 / (-dr1dl1 * dr2dl3 * dr3dl2 - dr1dl2 * dr2dl1 * dr3dl3);
        const double J[9] = {-dr2dl3 * dr3dl2, -dr1dl2 * dr3dl3, dr1dl2 * dr2dl3,
                             -dr2dl1 * dr3dl3, dr1dl1 * dr3dl3, -dr1dl1 * dr2dl3,
                             dr2dl1 * dr3dl2, -dr1dl1 * dr3dl2, -dr1dl2 * dr2dl1};
        double ln[3], rn[3];
        for (int r = 0; r < 3; r++) ln[r] = l[r] - det * dot3(J + 3 * r, res);
        gn_residual(ln, a12, a13, a23, b12, b13, b23, rn);
        if (l1n(rn) > l1n(res)) break;
        for (int r = 0; r < 3; r++) { l[r] = ln[r]; res[r] = rn[r]; }
    }
}
__device__ bool inv3(const double *m, double *o) {
    const double d = det3(m);
    if (d == 0.0) return false;
    const double id = 1.0 / d;
    o[0] = (m[4] * m[8] - m[5] * m[7]) * id; o[1] = (m[2] * m[7] - m[1] * m[8]) * id; o[2] = (m[1] * m[5] - m[2] * m[4]) * id;
    o[3] = (m[5] * m[6] - m[3] * m[8]) * id; o[4] = (m[0] * m[8] - m[2] * m[6]) * id; o[5] = (m[2] * m[3] - m[0] * m[5]) * id;
    o[6] = (m[3] * m[7] - m[4] * m[6]) * id; o[7] = (m[1] * m[6] - m[0] * m[7]) * id; o[8] = (m[0] * m[4] - m[1] * m[3]) * id;
    return true;
}
// nalgebra Rotation3::from_matrix_eps(m, eps, max_iter, identity)
__device__ void rotation_from_matrix_eps(const double *m, double eps, int max_iter, double *rot) {
    double R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    for (int it = 0; it < max_iter; it++) {
        double axis[3] = {0, 0, 0}, denom = 0.0;
        for (int c = 0; c < 3; c++) {
            const double rc[3] = {R[c], R[3 + c], R[6 + c]}, mc[3] = {m[c], m[3 + c], m[6 + c]};
            double x[3];
            cross3(rc, mc, x);
            for (int k = 0; k < 3; k++) axis[k] += x[k];
            denom += dot3(rc, mc);
        }
        const double sc = fabs(denom) + 2.220446049250313e-16;
        const double aa[3] = {axis[0] / sc, axis[1] / sc, axis[2] / sc};
        const double angle = norm3(aa);
        if (!(angle > eps)) break;
        const double u[3] = {aa[0] / angle, aa[1] / angle, aa[2] / angle};
        const double s = sin(angle), c = cos(angle), omc = 1.0 - c;
        const double Q[9] = {u[0] * u[0] + (1 - u[0] * u[0]) * c, u[0] * u[1] * omc - u[2] * s, u[0] * u[2] * omc + u[1] * s,
                             u[0] * u[1] * omc + u[2] * s, u[1] * u[1] + (1 - u[1] * u[1]) * c, u[1] * u[2] * omc - u[0] * s,
                             u[0] * u[2] * omc - u[1] * s, u[1] * u[2] * omc + u[0] * s, u[2] * u[2] + (1 - u[2] * u[2]) * c};
        mat3_mul(Q, R, R);
    }
    for (int i = 0; i < 9; i++) rot[i] = R[i];
}
__device__ int p3p(const double *bearings, const double *world, const uint32_t *idx, cvb_pose *out) {
    double wp[3][3];
    const double *y[3];
    for (int i = 0; i < 3; i++) {
        const double *w = world + 4 * (size_t)idx[i];
        if (w[3] == 0.0) return 0;
        for (int k = 0; k < 3; k++) wp[i][k] = w[k] / w[3];
        y[i] = bearings + 3 * (size_t)idx[i];
    }
    double d12[3], d13[3], d23[3], d12xd13[3];
    for (int k = 0; k < 3; k++) { d12[k] = wp[0][k] - wp[1][k]; d13[k] = wp[0][k] - wp[2][k]; d23[k] = wp[1][k] - wp[2][k]; }
    cross3(d12, d13, d12xd13);
    const double a12 = dot3(d12, d12), a13 = dot3(d13, d13), a23 = dot3(d23, d23);
    const double c12 = dot3(y[0], y[1]), c23 = dot3(y[1], y[2]), c31 = dot3(y[2], y[0]);
    const double blob = c12 * c23 * c31 - 1.0;
    const double s12_sqr = 1.0 - c12 * c12, s23_sqr = 1.0 - c23 * c23, s31_sqr = 1.0 - c31 * c31;
    const double b12 = -2.0 * c12, b13 = -2.0 * c31, b23 = -2.0 * c23;
    const double p3 = a13 * (a23 * s31_sqr - a13 * s23_sqr);
    const double p2 = 2.0 * blob * a23 * a13 + a13 * (2.0 * a12 + a13) * s23_sqr + a23 * (a23 - a12) * s31_sqr;
    const double p1 = a23 * (a13 - a23) * s12_sqr - a12 * a12 * s23_sqr - 2.0 * a12 * (blob * a23 + a13 * s23_sqr);
    const double p0 = a12 * (a12 * s23_sqr - a23 * s12_sqr);
    const double g = cube_root(p2 / p3, p1 / p3, p0 / p3);
    const double d0_00 = a23 * (1.0 - g), d0_01 = -(a23 * c12), d0_02 = a23 * c31 * g, d0_11 = a23 - a12 + a13 * g;
    const double d0_12 = -c23 * (a13 * g - a12), d0_22 = g * (a13 - a23) - a12;
    const double D0[9] = {d0_00, d0_01, d0_02, d0_01, d0_11, d0_12, d0_02, d0_12, d0_22};
    double Ev[9], ev[3];
    eigen_decomposition_singular(D0, Ev, ev);
    double lambdas[4][3];
    int nl = 0;
    const double eigen_ratio = sqrt(fmax(0.0, -ev[1] / ev[0]));
    for (int sgn = 0; sgn < 2; sgn++) {
        const double ratio = sgn ? -eigen_ratio : eigen_ratio;
        const double w2 = 1.0 / (ratio * Ev[1] - Ev[0]);
        const double w0 = w2 * (Ev[3] - ratio * Ev[4]);
        const double w1 = w2 * (Ev[6] - ratio * Ev[7]);
        const double a = 1.0 / ((a13 - a12) * w1 * w1 - a12 * b13 * w1 - a12);
        const double b = a * (a13 * b12 * w1 - a12 * b13 * w0 - 2.0 * w0 * w1 * (a12 - a13));
        const double c = a * ((a13 - a12) * w0 * w0 + a13 * b12 * w0 + a13);
        if (b * b - 4.0 * c >= 0.0) {
            double tau[2];
            root2real(b, c, &tau[0], &tau[1]);
            for (int k = 0; k < 2; k++) {
                if (tau[k] > 0.0) {
                    const double d = a23 / (tau[k] * (b23 + tau[k]) + 1.0);
                    if (d > 0.0) {
                        const double l2 = sqrt(d), l3 = tau[k] * l2, l1 = w0 * l2 + w1 * l3;
                        if (l1 >= 0.0 && nl < 4) { lambdas[nl][0] = l1; lambdas[nl][1] = l2; lambdas[nl][2] = l3; nl++; }
                    }
                }
            }
        }
    }
    const double X[9] = {d12[0], d13[0], d12xd13[0], d12[1], d13[1], d12xd13[1], d12[2], d13[2], d12xd13[2]};
    double Xi[9];
    if (!inv3(X, Xi)) return 0;
    for (int s = 0; s < nl; s++) {
        double l[3] = {lambdas[s][0], lambdas[s][1], lambdas[s][2]};
        gauss_newton_refine_lambda(l, 5, a12, a13, a23, b12, b13, b23);
        double ry1[3], ry2[3], ry3[3], yd1[3], yd2[3], yx[3];
        for (int k = 0; k < 3; k++) { ry1[k] = l[0] * y[0][k]; ry2[k] = l[1] * y[1][k]; ry3[k] = l[2] * y[2][k]; }
        for (int k = 0; k < 3; k++) { yd1[k] = ry1[k] - ry2[k]; yd2[k] = ry1[k] - ry3[k]; }
        cross3(yd1, yd2, yx);
        const double Y[9] = {yd1[0], yd2[0], yx[0], yd1[1], yd2[1], yx[1], yd1[2], yd2[2], yx[2]};
        double rot[9];
        mat3_mul(Y, Xi, rot);
        for (int k = 0; k < 3; k++) out[s].t[k] = ry1[k] - dot3(rot + 3 * k, wp[0]);
        rotation_from_matrix_eps(rot, 1e-12, 100, out[s].r);
    }
    return nl;
}

// ---- five-point (nister-stewenius/src/lib.rs:50-330).  nalgebra's full_piv_lu / complex_eigenvalues / try_svd are
// implemented as complete-pivoting elimination, Hessenberg + Francis double-shift QR, and one-sided Jacobi.
// `row0`: first eigenvector row used as (x, y, z, 1).  The reference takes rows 5..8 (`fixed_rows::<4>(5)`, lib.rs:229)
// although the monomial basis puts (x, y, z, 1) in rows 6..9, so its essentials violate the cubic constraints; row0 = 5
// reproduces the reference, row0 = 6 is the mathematically correct solver (see DESIGN.md).
constexpr int FPN = 10;
// __noinline__: with every helper inlined into one five-point frame, nvcc 12.9 -O3 produced a wrong complete-pivoting
// elimination on sm_90a (the same text is right stand-alone and on the host); separate frames are bit-identical to the CPU.
__device__ __noinline__ bool lu_full_pivot_solve(const double *Ain, const double *Bin, double *X) {
    double A[FPN][FPN], B[FPN][FPN];
    int colperm[FPN];
    for (int i = 0; i < FPN; i++) for (int j = 0; j < FPN; j++) { A[i][j] = Ain[i * FPN + j]; B[i][j] = Bin[i * FPN + j]; }
    for (int i = 0; i < FPN; i++) colperm[i] = i;
    for (int k = 0; k < FPN; k++) {
        int pr = k, pc = k; double best = -1.0;
        for (int i = k; i < FPN; i++) for (int j = k; j < FPN; j++) if (fabs(A[i][j]) > best) { best = fabs(A[i][j]); pr = i; pc = j; }
        if (best == 0.0) return false;
        if (pr != k) for (int j = 0; j < FPN; j++) { double t = A[k][j]; A[k][j] = A[pr][j]; A[pr][j] = t; t = B[k][j]; B[k][j] = B[pr][j]; B[pr][j] = t; }
        if (pc != k) { for (int i = 0; i < FPN; i++) { double t = A[i][k]; A[i][k] = A[i][pc]; A[i][pc] = t; } int t = colperm[k]; colperm[k] = colperm[pc]; colperm[pc] = t; }
        for (int i = k + 1; i < FPN; i++) {
            const double f = A[i][k] / A[k][k];
            if (f == 0.0) continue;
            for (int j = k; j < FPN; j++) A[i][j] -= f * A[k][j];
            for (int j = 0; j < FPN; j++) B[i][j] -= f * B[k][j];
        }
    }
    double Y[FPN][FPN];
    for (int c = 0; c < FPN; c++)
        for (int i = FPN - 1; i >= 0; i--) {
            double v = B[i][c];
            for (int j = i + 1; j < FPN; j++) v -= A[i][j] * Y[j][c];
            Y[i][c] = v / A[i][i];
        }
    for (int i = 0; i < FPN; i++) for (int c = 0; c < FPN; c++) X[colperm[i] * FPN + c] = Y[i][c];
    return true;
}

__device__ __forceinline__ double fp_sign(double a, double b) { return b >= 0.0 ? fabs(a) : -fabs(a); }
__device__ __noinline__ bool real_eigenvalues10(const double *Ain, double *wr, double *wi) {
    const int n = FPN;
    double a[FPN][FPN];
    for (int i = 0; i < n; i++) for (int j = 0; j < n; j++) a[i][j] = Ain[i * n + j];
    for (int m = 1; m < n - 1; m++) {
        double x = 0.0; int i = m;
        for (int j = m; j < n; j++) if (fabs(a[j][m - 1]) > fabs(x)) { x = a[j][m - 1]; i = j; }
        if (i != m) {
            for (int j = m - 1; j < n; j++) { double t = a[i][j]; a[i][j] = a[m][j]; a[m][j] = t; }
            for (int j = 0; j < n; j++) { double t = a[j][i]; a[j][i] = a[j][m]; a[j][m] = t; }
        }
        if (x != 0.0)
            for (i = m + 1; i < n; i++) {
                double y = a[i][m - 1];
                if (y != 0.0) {
                    y /= x; a[i][m - 1] = y;
                    for (int j = m; j < n; j++) a[i][j] -= y * a[m][j];
                    for (int j = 0; j < n; j++) a[j][m] += y * a[j][i];
                }
            }
    }
    for (int i = 2; i < n; i++) for (int j = 0; j < i - 1; j++) a[i][j] = 0.0;
    int nn = n - 1, l, its;
    double p = 0, q = 0, r = 0, s, t = 0.0, u, v, w, x, y, z, anorm = 0.0;
    for (int i = 0; i < n; i++) for (int j = (i > 0 ? i - 1 : 0); j < n; j++) anorm += fabs(a[i][j]);
    while (nn >= 0) {
        its = 0;
        do {
            for (l = nn; l >= 1; l--) {
                s = fabs(a[l - 1][l - 1]) + fabs(a[l][l]);
                if (s == 0.0) s = anorm;
                if (fabs(a[l][l - 1]) + s == s) { a[l][l - 1] = 0.0; break; }
            }
            x = a[nn][nn];
            if (l == nn) { wr[nn] = x + t; wi[nn--] = 0.0; }
            else {
                y = a[nn - 1][nn - 1]; w = a[nn][nn - 1] * a[nn - 1][nn];
                if (l == nn - 1) {
                    p = 0.5 * (y - x); q = p * p + w; z = sqrt(fabs(q)); x += t;
                    if (q >= 0.0) {
                        z = p + fp_sign(z, p);
                        wr[nn - 1] = wr[nn] = x + z;
                        if (z != 0.0) wr[nn] = x - w / z;
                        wi[nn - 1] = wi[nn] = 0.0;
                    } else { wr[nn - 1] = wr[nn] = x + p; wi[nn] = z; wi[nn - 1] = -z; }
                    nn -= 2;
                } else {
                    if (its == 60) return false;
                    if (its == 10 || its == 20) {
                        t += x;
                        for (int i = 0; i <= nn; i++) a[i][i] -= x;
                        s = fabs(a[nn][nn - 1]) + fabs(a[nn - 1][nn - 2]);
                        y = x = 0.75 * s; w = -0.4375 * s * s;
                    }
                    ++its;
                    int m;
                    for (m = nn - 2; m >= l; m--) {
                        z = a[m][m]; r = x - z; s = y - z;
                        p = (r * s - w) / a[m + 1][m] + a[m][m + 1];
                        q = a[m + 1][m + 1] - z - r - s;
                        r = a[m + 2][m + 1];
                        s = fabs(p) + fabs(q) + fabs(r);
                        p /= s; q /= s; r /= s;
                        if (m == l) break;
                        u = fabs(a[m][m - 1]) * (fabs(q) + fabs(r));
                        v = fabs(p) * (fabs(a[m - 1][m - 1]) + fabs(z) + fabs(a[m + 1][m + 1]));
                        if (u + v == v) break;
                    }
                    for (int i = m + 2; i <= nn; i++) { a[i][i - 2] = 0.0; if (i != m + 2) a[i][i - 3] = 0.0; }
                    for (int k = m; k <= nn - 1; k++) {
                        if (k != m) {
                            p = a[k][k - 1]; q = a[k + 1][k - 1]; r = 0.0;
                            if (k != nn - 1) r = a[k + 2][k - 1];
                            if ((x = fabs(p) + fabs(q) + fabs(r)) != 0.0) { p /= x; q /= x; r /= x; }
                        }
                        if ((s = fp_sign(sqrt(p * p + q * q + r * r), p)) != 0.0) {
                            if (k == m) { if (l != m) a[k][k - 1] = -a[k][k - 1]; }
                            else a[k][k - 1] = -s * x;
                            p += s; x = p / s; y = q / s; z = r / s; q /= p; r /= p;
                            for (int j = k; j <= nn; j++) {
                                p = a[k][j] + q * a[k + 1][j];
                                if (k != nn - 1) { p += r * a[k + 2][j]; a[k + 2][j] -= p * z; }
                                a[k + 1][j] -= p * y; a[k][j] -= p * x;
                            }
                            const int mmin = nn < k + 3 ? nn : k + 3;
                            for (int i = l; i <= mmin; i++) {
                                p = x * a[i][k] + y * a[i][k + 1];
                                if (k != nn - 1) { p += z * a[i][k + 2]; a[i][k + 2] -= p * r; }
                                a[i][k + 1] -= p * q; a[i][k] -= p;
                            }
                        }
                    }
                }
            }
        } while (l < nn - 1);
    }
    return true;
}

// right singular vector of the smallest singular value of an N x N matrix: one-sided Jacobi on the columns (N = 10: the five-point
// solver; N = 4: RelativeDlt's design matrix, which is never squared into DtD)
template <int N>
__device__ __noinline__ bool min_right_singular_vector(const double *Min, double eps, int max_sweeps, double *vec, double *smin) {
    double U[N][N], V[N][N];
    for (int i = 0; i < N; i++) for (int j = 0; j < N; j++) { U[i][j] = Min[i * N + j]; V[i][j] = i == j ? 1.0 : 0.0; }
    bool converged = false;
    for (int sweep = 0; sweep < max_sweeps && !converged; sweep++) {
        converged = true;
        for (int p = 0; p < N - 1; p++)
            for (int q = p + 1; q < N; q++) {
                double alpha = 0, beta = 0, gamma = 0;
                for (int i = 0; i < N; i++) { alpha += U[i][p] * U[i][p]; beta += U[i][q] * U[i][q]; gamma += U[i][p] * U[i][q]; }
                if (gamma == 0.0 || fabs(gamma) <= eps * sqrt(alpha * beta)) continue;
                converged = false;
                const double zeta = (beta - alpha) / (2.0 * gamma);
                const double t = (zeta >= 0.0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
                const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
                for (int i = 0; i < N; i++) {
                    const double up = U[i][p], uq = U[i][q];
                    U[i][p] = c * up - s * uq; U[i][q] = s * up + c * uq;
                    const double vp = V[i][p], vq = V[i][q];
                    V[i][p] = c * vp - s * vq; V[i][q] = s * vp + c * vq;
                }
            }
    }
    if (!converged) return false;
    int best = 0; double bn = -1.0;
    for (int j = 0; j < N; j++) {
        double nn = 0; for (int i = 0; i < N; i++) nn += U[i][j] * U[i][j];
        if (bn < 0.0 || nn < bn) { bn = nn; best = j; }
    }
    *smin = sqrt(bn);
    for (int i = 0; i < N; i++) vec[i] = V[i][best];
    return true;
}

enum { BXXX = 0, BXXY, BXYY, BYYY, BXXZ, BXYZ, BYYZ, BXZZ, BYZZ, BZZZ, BXX, BXY, BYY, BXZ, BYZ, BZZ, BX, BY, BZ, B1 };
__device__ void fp_o1(const double *a, const double *b, double *r) {
    for (int i = 0; i < 20; i++) r[i] = 0.0;
    r[BXX] = a[0] * b[0]; r[BXY] = a[0] * b[1] + a[1] * b[0]; r[BXZ] = a[0] * b[2] + a[2] * b[0];
    r[BYY] = a[1] * b[1]; r[BYZ] = a[1] * b[2] + a[2] * b[1]; r[BZZ] = a[2] * b[2];
    r[BX] = a[0] * b[3] + a[3] * b[0]; r[BY] = a[1] * b[3] + a[3] * b[1]; r[BZ] = a[2] * b[3] + a[3] * b[2]; r[B1] = a[3] * b[3];
}
__device__ void fp_o2(const double *a, const double *b, double *r) {
    r[BXXX] = a[BXX] * b[0];
    r[BXXY] = a[BXX] * b[1] + a[BXY] * b[0];
    r[BXXZ] = a[BXX] * b[2] + a[BXZ] * b[0];
    r[BXYY] = a[BXY] * b[1] + a[BYY] * b[0];
    r[BXYZ] = a[BXY] * b[2] + a[BYZ] * b[0] + a[BXZ] * b[1];
    r[BXZZ] = a[BXZ] * b[2] + a[BZZ] * b[0];
    r[BYYY] = a[BYY] * b[1];
    r[BYYZ] = a[BYY] * b[2] + a[BYZ] * b[1];
    r[BYZZ] = a[BYZ] * b[2] + a[BZZ] * b[1];
    r[BZZZ] = a[BZZ] * b[2];
    r[BXX] = a[BXX] * b[3] + a[BX] * b[0];
    r[BXY] = a[BXY] * b[3] + a[BX] * b[1] + a[BY] * b[0];
    r[BXZ] = a[BXZ] * b[3] + a[BX] * b[2] + a[BZ] * b[0];
    r[BYY] = a[BYY] * b[3] + a[BY] * b[1];
    r[BYZ] = a[BYZ] * b[3] + a[BY] * b[2] + a[BZ] * b[1];
    r[BZZ] = a[BZZ] * b[3] + a[BZ] * b[2];
    r[BX] = a[BX] * b[3] + a[B1] * b[0];
    r[BY] = a[BY] * b[3] + a[B1] * b[1];
    r[BZ] = a[BZ] * b[3] + a[B1] * b[2];
    r[B1] = a[B1] * b[3];
}

// EssentialMatrix::possible_rotations_unscaled_translation (cv-pinhole/src/essential.rs:114-162): Ra = U W Vt, Rb = U Wt Vt and
// t = U's third column, after the det(U), det(Vt) > 0 fix-ups
__device__ __noinline__ bool essential_rotations(const double *E, double eps, int sweeps, double *Ra, double *Rb, double *t) {
    double U[9], Vt[9];
    if (!svd3(E, eps, sweeps, U, Vt)) return false;
    if (det3(U) < 0.0) for (int r = 0; r < 3; r++) U[r * 3 + 2] *= -1.0;
    if (det3(Vt) < 0.0) for (int c = 0; c < 3; c++) Vt[6 + c] *= -1.0;
    const double W[9] = {0, -1, 0, 1, 0, 0, 0, 0, 1}, Wt[9] = {0, 1, 0, -1, 0, 0, 0, 0, 1};
    double UW[9];
    mat3_mul(U, W, UW); mat3_mul(UW, Vt, Ra);
    mat3_mul(U, Wt, UW); mat3_mul(UW, Vt, Rb);
    t[0] = U[2]; t[1] = U[5]; t[2] = U[8];
    return true;
}
// essential matrix -> the four candidate poses (cv-pinhole/src/essential.rs:114-162,217-231) with Estimator::estimate's 1e-12 / 1000
__device__ __noinline__ int essential_poses(const double *E, cvb_pose *out) {
    double Ra[9], Rb[9], t[3];
    if (!essential_rotations(E, 1e-12, 1000, Ra, Rb, t)) return 0;
    for (int k = 0; k < 4; k++) {
        for (int i = 0; i < 9; i++) out[k].r[i] = (k & 1) ? Rb[i] : Ra[i];
        for (int r = 0; r < 3; r++) out[k].t[r] = (k & 2) ? -t[r] : t[r];
    }
    return 4;
}

__device__ int five_point(const double *a, const double *b, const uint32_t *idx, int row0, cvb_pose *out) {
    double A[5][9], EE[81], d[9], V[81];
    for (int i = 0; i < 5; i++) {
        const double *pa = a + 3 * (size_t)idx[i], *pb = b + 3 * (size_t)idx[i];
        for (int j = 0; j < 3; j++)
            for (int k = 0; k < 3; k++) A[i][3 * j + k] = pa[j] * pb[k];
    }
    for (int r = 0; r < 9; r++)
        for (int c = 0; c < 9; c++) { double s = 0; for (int i = 0; i < 5; i++) s += A[i][r] * A[i][c]; EE[r * 9 + c] = s; }
    if (!sym_eigen<9>(EE, 1e-12, 1000, d, V)) return 0;
    int src[9] = {0, 1, 2, 3, 4, 5, 6, 7, 8};
    for (int i = 1; i < 9; i++) { int x = src[i], j = i; while (j > 0 && d[src[j - 1]] > d[x]) { src[j] = src[j - 1]; j--; } src[j] = x; }
    int nullity = -1;
    for (int i = 0; i < 9; i++) if (d[src[i]] > 1e-12) { nullity = i; break; }
    if (nullity != 4) return 0;
    double eb[9][4];
    for (int c = 0; c < 4; c++) for (int r = 0; r < 9; r++) eb[r][c] = V[r * 9 + src[c]];
    double ep[3][3][4];
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) for (int k = 0; k < 4; k++) ep[i][j][k] = eb[3 * i + j][k];
    double M[10][20], t1[20], t2[20], t3[20], acc[20];
    {
        const int ia[3][2] = {{1, 2}, {2, 0}, {0, 1}};
        for (int k = 0; k < 20; k++) acc[k] = 0.0;
        for (int c = 0; c < 3; c++) {
            const int p = ia[c][0], q = ia[c][1];
            fp_o1(ep[0][p], ep[1][q], t1); fp_o1(ep[0][q], ep[1][p], t2);
            for (int k = 0; k < 20; k++) t1[k] -= t2[k];
            fp_o2(t1, ep[2][c], t3);
            for (int k = 0; k < 20; k++) acc[k] += t3[k];
        }
        for (int k = 0; k < 20; k++) M[0][k] = acc[k];
    }
    double eet[3][3][20], L[3][3][20];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            if (i <= j) {
                fp_o1(ep[i][0], ep[j][0], t1); fp_o1(ep[i][1], ep[j][1], t2); fp_o1(ep[i][2], ep[j][2], t3);
                for (int k = 0; k < 20; k++) eet[i][j][k] = t1[k] + t2[k] + t3[k];
            } else for (int k = 0; k < 20; k++) eet[i][j][k] = eet[j][i][k];
        }
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) for (int k = 0; k < 20; k++) L[i][j][k] = eet[i][j][k];
    for (int k = 0; k < 20; k++) {
        const double tr = 0.5 * (eet[0][0][k] + eet[1][1][k] + eet[2][2][k]);
        for (int i = 0; i < 3; i++) L[i][i][k] -= tr;
    }
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            fp_o2(L[i][0], ep[0][j], t1); fp_o2(L[i][1], ep[1][j], t2); fp_o2(L[i][2], ep[2][j], t3);
            for (int k = 0; k < 20; k++) M[1 + i * 3 + j][k] = t1[k] + t2[k] + t3[k];
        }
    double Cl[100], Cr[100], X[100];
    for (int i = 0; i < 10; i++) for (int j = 0; j < 10; j++) { Cl[i * 10 + j] = M[i][j]; Cr[i * 10 + j] = M[i][10 + j]; }
    if (!lu_full_pivot_solve(Cl, Cr, X)) return 0;
    double At[100];
    for (int i = 0; i < 100; i++) At[i] = 0.0;
    for (int j = 0; j < 10; j++) {
        At[0 * 10 + j] = X[0 * 10 + j]; At[1 * 10 + j] = X[1 * 10 + j]; At[2 * 10 + j] = X[2 * 10 + j];
        At[3 * 10 + j] = X[4 * 10 + j]; At[4 * 10 + j] = X[5 * 10 + j]; At[5 * 10 + j] = X[7 * 10 + j];
    }
    At[6 * 10 + 0] = -1.0; At[7 * 10 + 1] = -1.0; At[8 * 10 + 3] = -1.0; At[9 * 10 + 6] = -1.0;
    double wr[10], wi[10];
    if (!real_eigenvalues10(At, wr, wi)) return 0;
    int n = 0;
    for (int i = 0; i < 10; i++) {
        if (wi[i] != 0.0) continue;
        double *Mx = Cl;   // reuse
        double vec[10], smin;
        for (int k = 0; k < 100; k++) Mx[k] = At[k];
        for (int k = 0; k < 10; k++) Mx[k * 10 + k] -= wr[i];
        if (!min_right_singular_vector<FPN>(Mx, 1e-15, 1000, vec, &smin)) continue;
        if (!(smin < 1e-12)) continue;
        double ev[9], E[9];
        for (int r = 0; r < 9; r++) ev[r] = eb[r][0] * vec[row0] + eb[r][1] * vec[row0 + 1] + eb[r][2] * vec[row0 + 2] + eb[r][3] * vec[row0 + 3];
        for (int k = 0; k < 9; k++) E[(k % 3) * 3 + (k / 3)] = ev[k];
        n += essential_poses(E, out + n);
    }
    return n;
}

// ------------------------------------------------------------------------------------------ kernels
template <int KIND>
__global__ void __launch_bounds__(128) k_estimate(const double *__restrict__ a, const double *__restrict__ b,
                                                  const uint32_t *__restrict__ samples, uint32_t H, cvb_pose *poses,
                                                  uint8_t *nposes, int row0) {
    const uint32_t h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= H) return;
    if (KIND == 2) {   // five-point: up to 40 poses per sample, written straight to global memory
        nposes[h] = (uint8_t)five_point(a, b, samples + (size_t)h * 5, row0, poses + (size_t)h * 40);
        return;
    }
    cvb_pose out[4];
    int n;
    if (KIND == 0) n = eight_point(a, b, samples + (size_t)h * 8, out);
    else n = p3p(a, b, samples + (size_t)h * 3, out);
    for (int k = 0; k < n; k++) poses[(size_t)h * 4 + k] = out[k];
    nposes[h] = (uint8_t)n;
}

// one thread per (pose, datum).  MODE 0: write residuals; MODE 1: write bit-packed inlier masks
// (residual < thr) over data [i0, i1): mask word w of pose p at masks[p * words + w].
template <int KIND, int MODE>
__global__ void __launch_bounds__(256) k_residuals(const cvb_pose *__restrict__ poses, uint32_t m,
                                                   const double *__restrict__ a, const double *__restrict__ b,
                                                   uint32_t i0, uint32_t i1, double thr, double *__restrict__ out,
                                                   uint32_t out_stride, uint32_t *__restrict__ masks, uint32_t words) {
    const uint32_t p = blockIdx.y;
    const uint32_t i = i0 + blockIdx.x * blockDim.x + threadIdx.x;
    const bool in = i < i1;
    double r = 3.0;
    if (in) {
        const cvb_pose P = poses[p];
        r = KIND == 0 ? residual_c2c(P, a + 3 * (size_t)i, b + 3 * (size_t)i) : residual_w2c(P, a + 3 * (size_t)i, b + 4 * (size_t)i);
    }
    if (MODE == 0) { if (in) out[(size_t)p * out_stride + i] = r; }
    else {
        const unsigned bits = __ballot_sync(0xffffffffu, in && r < thr);
        // warps behind the data count own no mask word (a row has cdiv(i1 - i0, 32) words, the CTA covers 8)
        if ((threadIdx.x & 31) == 0 && ((i - i0) >> 5) < words) masks[(size_t)p * words + ((i - i0) >> 5)] = bits;
    }
}

// cv-geom/src/triangulation.rs:82-130: n >= 2 observations (WorldToCamera pose, bearing) -> homogeneous world point;
// eps / max_sweeps: the triangulator's epsilon / max_iterations (Default 1e-12 / 1000) handed to try_symmetric_eigen
__device__ bool triangulate_linear_eigen(const cvb_pose *poses, const double *bearings, uint32_t n, double *p, double eps, int max_sweeps) {
    if (n < 2) return false;
    double A[16], d[4], V[16];
    for (int i = 0; i < 16; i++) A[i] = 0.0;
    for (uint32_t i = 0; i < n; i++) design_add(poses[i].r, poses[i].t, bearings + 3 * (size_t)i, A);
    if (!sym_eigen<4>(A, eps, max_sweeps, d, V)) return false;
    int best = 0;
    for (int i = 1; i < 4; i++)
        if (d[i] < d[best]) best = i;
    p[0] = V[best]; p[1] = V[4 + best]; p[2] = V[8 + best]; p[3] = V[12 + best];
    from_homogeneous(p);
    if (!(isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]) && isfinite(p[3]))) return false;
    for (uint32_t i = 0; i < n; i++) {
        const double *bb = bearings + 3 * (size_t)i, *R = poses[i].r;
        const double wb[3] = {R[0] * bb[0] + R[3] * bb[1] + R[6] * bb[2], R[1] * bb[0] + R[4] * bb[1] + R[7] * bb[2],
                              R[2] * bb[0] + R[5] * bb[1] + R[8] * bb[2]};
        if (signbit(dot3(wb, p))) return false;
    }
    return true;
}

// cv-sfm keeps calibrated bearings per feature (CameraModel::calibrate, cv-pinhole/src/lib.rs:108-116, on
// akaze::KeyPoint's ImagePoint, akaze/src/lib.rs:95-99); a FeatureMatch is the bearing pair of a match (cv-sfm/src/lib.rs:1400).
// One thread per match: both bearings in f64 with the reference's operation order (pinhole.cuh; k1 = 0 for CameraIntrinsics).
__global__ void __launch_bounds__(256) k_pair_bearings(const cvb_keypoint *__restrict__ kpa, const cvb_keypoint *__restrict__ kpb,
                                                       const uint32_t *__restrict__ pairs, const uint32_t *__restrict__ npairs,
                                                       uint32_t cap, cvb_intrinsics_k1 K, double *__restrict__ a, double *__restrict__ b) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= min(*npairs, cap)) return;
    const cvb_keypoint ka = kpa[pairs[2 * i]], kb = kpb[pairs[2 * i + 1]];
    calibrate_k1(K, (double)ka.x, (double)ka.y, a + 3 * (size_t)i);
    calibrate_k1(K, (double)kb.x, (double)kb.y, b + 3 * (size_t)i);
}

#include "arrsac_dev.cuh"

// ------------------------------------------------------------------------------------------ post-consensus refinement
// cv-optimize single_view_simple_optimize_l2 / three_view_{simple,adaptive}_optimize_l2 with cv-geom's epipolar gradients,
// and cv-sfm's robustness checks.  One CTA per problem iterates to completion on the device: every iteration the threads
// evaluate the per-landmark tangents, a fixed-shape reduction tree adds them (warp shuffles, then the warps in order; the
// reference adds them in landmark order, so sums agree to rounding, not bit for bit), thread 0 replays the reference's
// bookkeeping (patience counter, pose update) and publishes the pose for the next iteration.
__device__ __forceinline__ void rotv(const double *R, const double *v, double *o) { for (int r = 0; r < 3; r++) o[r] = dot3(R + 3 * r, v); }
__device__ __forceinline__ bool any_nan3(const double *v) { return isnan(v[0]) || isnan(v[1]) || isnan(v[2]); }
__device__ __forceinline__ void normalize3(const double *v, double *o) { const double n = norm3(v); o[0] = v[0] / n; o[1] = v[1] / n; o[2] = v[2] / n; }
// Se3TangentSpace::new (cv-core/src/so3.rs:23-34)
__device__ __forceinline__ void tangent_new(double *t, double *r) {
    if (any_nan3(t)) t[0] = t[1] = t[2] = 0.0;
    if (any_nan3(r)) r[0] = r[1] = r[2] = 0.0;
}
// nalgebra Rotation3::from_scaled_axis
__device__ void rot_from_scaled_axis(const double *v, double *R) {
    const double angle = norm3(v);
    if (angle == 0.0) { for (int i = 0; i < 9; i++) R[i] = (i % 4 == 0) ? 1.0 : 0.0; return; }
    const double ux = v[0] / angle, uy = v[1] / angle, uz = v[2] / angle;
    const double sqx = ux * ux, sqy = uy * uy, sqz = uz * uz, sn = sin(angle), c = cos(angle), omc = 1.0 - c;
    R[0] = sqx + (1.0 - sqx) * c; R[1] = ux * uy * omc - uz * sn; R[2] = ux * uz * omc + uy * sn;
    R[3] = ux * uy * omc + uz * sn; R[4] = sqy + (1.0 - sqy) * c; R[5] = uy * uz * omc - ux * sn;
    R[6] = ux * uz * omc - uy * sn; R[7] = uy * uz * omc + ux * sn; R[8] = sqz + (1.0 - sqz) * c;
}
// pose <- Se3TangentSpace{trans, rot}.isometry() * pose (so3.rs:57-60)
__device__ void apply_delta(const double *trans, const double *rot, cvb_pose *P) {
    double Rd[9], td[3], Rn[9], tn[3];
    rot_from_scaled_axis(rot, Rd);
    rotv(Rd, trans, td);
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) Rn[3 * r + c] = Rd[3 * r] * P->r[c] + Rd[3 * r + 1] * P->r[3 + c] + Rd[3 * r + 2] * P->r[6 + c];
    rotv(Rd, P->t, tn);
    for (int r = 0; r < 3; r++) tn[r] = td[r] + tn[r];
    for (int i = 0; i < 9; i++) P->r[i] = Rn[i];
    for (int i = 0; i < 3; i++) P->t[i] = tn[i];
}
__device__ void pose_inverse(const cvb_pose &P, cvb_pose *o) {
    const double nt[3] = {-P.t[0], -P.t[1], -P.t[2]};
    double R[9];
    for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) R[3 * r + c] = P.r[3 * c + r];
    rotv(R, nt, o->t);
    for (int i = 0; i < 9; i++) o->r[i] = R[i];
}
// cv-geom/src/epipolar.rs:193-198
__device__ void world_pose_gradient(const double *translation, const double *b, double *tg, double *rg) {
    const double d = dot3(translation, b);
    double nt[3];
    for (int i = 0; i < 3; i++) tg[i] = d * b[i] - translation[i];
    normalize3(translation, nt);
    cross3(nt, b, rg);
    tangent_new(tg, rg);
}
// cv-optimize/src/single_view_optimizer.rs:4-14
__device__ bool landmark_delta(const cvb_pose &P, const double *bearing, const double *world, double *tg, double *rg) {
    double q[4];
    pose_apply(P, world, q);
    from_homogeneous(q);
    if (q[3] == 0.0) return false;
    const double p[3] = {q[0] / q[3], q[1] / q[3], q[2] / q[3]};
    world_pose_gradient(p, bearing, tg, rg);
    return true;
}
// epipolar.rs:8-50
__device__ bool sine_l1_point(const double *t, const double *a_in, const double *b_in, double *p) {
    double ca[3], cb[3], na[3], nb[3], a[3], b[3];
    cross3(a_in, t, ca); const double can = norm3(ca); for (int i = 0; i < 3; i++) na[i] = ca[i] / can;
    cross3(b_in, t, cb); const double cbn = norm3(cb); for (int i = 0; i < 3; i++) nb[i] = cb[i] / cbn;
    for (int i = 0; i < 3; i++) { a[i] = a_in[i]; b[i] = b_in[i]; }
    if (can < cbn) { const double d = dot3(a_in, nb); double v[3]; for (int i = 0; i < 3; i++) v[i] = a_in[i] - d * nb[i]; normalize3(v, a); }
    else { const double d = dot3(b_in, na); double v[3]; for (int i = 0; i < 3; i++) v[i] = b_in[i] - d * na[i]; normalize3(v, b); }
    double z[3], tb[3];
    cross3(a, b, z); cross3(t, b, tb);
    double q[4] = {a[0], a[1], a[2], dot3(z, z) / dot3(z, tb)};
    from_homogeneous(q);
    for (int i = 0; i < 4; i++) if (!isfinite(q[i])) return false;
    if (signbit(dot3(q, a)) || signbit(dot3(q, b))) return false;
    if (q[3] == 0.0) return false;
    for (int i = 0; i < 3; i++) p[i] = q[i] / q[3];
    return true;
}
// epipolar.rs:53-71
__device__ void rotation_gradient(const double *t, const double *a, const double *b, double *o) {
    double ca[3], cb[3], na[3], nb[3];
    cross3(a, t, ca); cross3(b, t, cb);
    normalize3(ca, na); normalize3(cb, nb);
    cross3(nb, na, o);
}
// epipolar.rs:85-176: out = [first.t, first.r, second.t, second.r]
__device__ void three_view_gradients(const double *c, const double *f, const double *ftoc, const double *s, const double *stoc, double *out) {
    double stof[3], rcf[3], rcs[3], rfs[3], p[3], q[3], tf[3] = {0, 0, 0}, ts[3] = {0, 0, 0}, tc[3] = {0, 0, 0}, neg[3];
    for (int i = 0; i < 3; i++) stof[i] = stoc[i] - ftoc[i];
    rotation_gradient(ftoc, c, f, rcf); rotation_gradient(stoc, c, s, rcs); rotation_gradient(stof, f, s, rfs);
    double *ft = out, *fr = out + 3, *st = out + 6, *sr = out + 9;
    for (int i = 0; i < 3; i++) {
        fr[i] = rcf[i] * (2.0 / 3.0) + (-rfs[i]) * (1.0 / 3.0);
        sr[i] = rcs[i] * (2.0 / 3.0) + rfs[i] * (1.0 / 3.0);
    }
    for (int i = 0; i < 3; i++) neg[i] = -stoc[i];
    if (sine_l1_point(neg, c, s, p)) { for (int i = 0; i < 3; i++) q[i] = p[i] - ftoc[i]; const double d = dot3(q, f); for (int i = 0; i < 3; i++) tf[i] = q[i] - d * f[i]; }
    for (int i = 0; i < 3; i++) neg[i] = -ftoc[i];
    if (sine_l1_point(neg, c, f, p)) { for (int i = 0; i < 3; i++) q[i] = p[i] - stoc[i]; const double d = dot3(q, s); for (int i = 0; i < 3; i++) ts[i] = q[i] - d * s[i]; }
    for (int i = 0; i < 3; i++) neg[i] = -stof[i];
    if (sine_l1_point(neg, f, s, p)) { for (int i = 0; i < 3; i++) q[i] = p[i] + ftoc[i]; const double d = dot3(q, c); for (int i = 0; i < 3; i++) tc[i] = d * c[i] - q[i]; }
    for (int i = 0; i < 3; i++) {
        ft[i] = tf[i] * (2.0 / 3.0) + tc[i] * (1.0 / 3.0);
        st[i] = ts[i] * (2.0 / 3.0) + tc[i] * (1.0 / 3.0);
    }
    tangent_new(ft, fr); tangent_new(st, sr);
}
// epipolar.rs:200-232
__device__ double epipolar_loss(const double *t, const double *a, const double *b) {
    double ca[3], cb[3];
    cross3(a, t, ca); cross3(b, t, cb);
    const double na2 = dot3(ca, ca), nb2 = dot3(cb, cb);
    double res;
    if (na2 < nb2) { const double sc = 1.0 / sqrt(nb2); const double v[3] = {cb[0] * sc, cb[1] * sc, cb[2] * sc}; res = fabs(dot3(a, v)); }
    else { const double sc = 1.0 / sqrt(na2); const double v[3] = {ca[0] * sc, ca[1] * sc, ca[2] * sc}; res = fabs(dot3(b, v)); }
    if (isnan(res) || signbit(dot3(a, b))) return 1.0;
    return res;
}

constexpr int OPT_NT = 512, OPT_WARPS = OPT_NT / 32;
// sums acc[0..NV) over the CTA into s_out[0..NV) (valid for thread 0 after the call); fixed tree -> run-to-run reproducible
template <int NV>
__device__ __forceinline__ void block_sum(double *acc, double *s_red) {
#pragma unroll
    for (int k = 0; k < NV; k++)
#pragma unroll
        for (int o = 16; o; o >>= 1) acc[k] += __shfl_down_sync(0xffffffffu, acc[k], o);
    const int w = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0)
        for (int k = 0; k < NV; k++) s_red[w * NV + k] = acc[k];
    __syncthreads();
    if (threadIdx.x == 0)
        for (int k = 0; k < NV; k++) {
            double s = s_red[k];
            for (int ww = 1; ww < OPT_WARPS; ww++) s += s_red[ww * NV + k];
            acc[k] = s;
        }
}

// single_view_optimizer.rs:80-135, one CTA per (pose, landmark list)
__global__ void __launch_bounds__(OPT_NT) k_single_view_opt(const cvb_pose *__restrict__ poses_in, const double *__restrict__ bearings,
                                                            const double *__restrict__ world, const uint32_t *__restrict__ offsets,
                                                            double rate, uint32_t iterations, cvb_pose *__restrict__ poses_out,
                                                            uint32_t *__restrict__ updates_out) {
    __shared__ cvb_pose P;
    __shared__ double s_red[OPT_WARPS * 6];
    __shared__ int s_stop;
    const uint32_t b = blockIdx.x, o0 = offsets[b], n = offsets[b + 1] - o0;
    if (threadIdx.x == 0) { P = poses_in[b]; s_stop = 0; }
    __syncthreads();
    double best_t = INFINITY, best_r = INFINITY;
    uint32_t no_improve = 0, updates = 0;
    const double inv_len = 1.0 / (double)n;
    if (n > 0)
        for (uint32_t it = 0; it < iterations; it++) {
            double acc[6] = {0, 0, 0, 0, 0, 0}, tg[3], rg[3];
            const cvb_pose Pl = P;
            for (uint32_t i = threadIdx.x; i < n; i += OPT_NT)
                if (landmark_delta(Pl, bearings + 3 * (size_t)(o0 + i), world + 4 * (size_t)(o0 + i), tg, rg))
                    for (int k = 0; k < 3; k++) { acc[k] += tg[k]; acc[3 + k] += rg[k]; }
            block_sum<6>(acc, s_red);
            if (threadIdx.x == 0) {
                double dt[3], dr[3];
                for (int k = 0; k < 3; k++) { dt[k] = (acc[k] * inv_len) * rate; dr[k] = (acc[3 + k] * inv_len) * rate; }
                no_improve++;
                const double t = norm3(acc), r = norm3(acc + 3);
                if (best_t > t) { best_t = t; no_improve = 0; }
                if (best_r > r) { best_r = r; no_improve = 0; }
                if (no_improve >= 50) s_stop = 1;
                else {
                    apply_delta(dt, dr, &P); updates++;
                    if (it == iterations - 1) s_stop = 1;
                }
            }
            __syncthreads();
            if (s_stop) break;
        }
    if (threadIdx.x == 0) { poses_out[b] = P; updates_out[b] = updates; }
}

// The step of three_view_optimizer.rs:126-272 on the summed gradients acc = [first.t, first.r, second.t, second.r] and, adaptive, their
// norms [first.t, first.r, second.t, second.r]; P: the inverted poses, updated in place.  Returns whether the optimisation stops.
// k_three_view_opt's thread 0 and k_three_view_opt_warp's lane 0 both take it.
__device__ __forceinline__ bool three_view_opt_step(const double *acc, double inv_len, int adaptive, double rate, double (&best)[2][2],
                                                    uint32_t &no_improve, cvb_pose *P, uint32_t &updates, bool last) {
    double d[12];
    if (!adaptive) {
        const double sc = inv_len * rate;
        for (int k = 0; k < 12; k++) d[k] = acc[k] * sc;
        no_improve++;
        for (int v = 0; v < 2; v++) {
            const double t = norm3(acc + 6 * v), r = norm3(acc + 6 * v + 3);
            if (best[v][0] > t) { best[v][0] = t; no_improve = 0; }
            if (best[v][1] > r) { best[v][1] = r; no_improve = 0; }
        }
        if (no_improve >= 50) return true;
    } else {
        for (int v = 0; v < 2; v++) {
            double l2[6];
            for (int k = 0; k < 6; k++) l2[k] = acc[6 * v + k] * inv_len;
            const double tstd = acc[12 + 2 * v] * inv_len, rstd = acc[13 + 2 * v] * inv_len;
            double trate = norm3(l2) / tstd, rrate = norm3(l2 + 3) / rstd;
            if (!isfinite(trate)) trate = 0.0;
            if (!isfinite(rrate)) rrate = 0.0;
            for (int k = 0; k < 3; k++) { d[6 * v + k] = l2[k] * trate; d[6 * v + 3 + k] = l2[3 + k] * rrate; }
        }
    }
    apply_delta(d, d + 3, &P[0]); apply_delta(d + 6, d + 9, &P[1]); updates++;
    return last;
}

// three_view_optimizer.rs:126-272, one CTA per (pose pair, observation triples); obs = [centre, first, second] bearings
__global__ void __launch_bounds__(OPT_NT) k_three_view_opt(const cvb_pose *__restrict__ poses_in, const double *__restrict__ obs,
                                                           const uint32_t *__restrict__ offsets, int adaptive, double rate,
                                                           uint32_t iterations, cvb_pose *__restrict__ poses_out,
                                                           uint32_t *__restrict__ updates_out) {
    __shared__ cvb_pose P[2];
    __shared__ double s_red[OPT_WARPS * 16];
    __shared__ int s_stop;
    const uint32_t b = blockIdx.x, o0 = offsets[b], n = offsets[b + 1] - o0;
    if (threadIdx.x == 0) {
        if (n > 0) { pose_inverse(poses_in[2 * b], &P[0]); pose_inverse(poses_in[2 * b + 1], &P[1]); }
        s_stop = 0;
    }
    __syncthreads();
    double best[2][2] = {{INFINITY, INFINITY}, {INFINITY, INFINITY}};
    uint32_t no_improve = 0, updates = 0;
    const double inv_len = 1.0 / (double)n;
    if (n > 0)
        for (uint32_t it = 0; it < iterations; it++) {
            double acc[16], g[12];
            for (int k = 0; k < 16; k++) acc[k] = 0.0;
            const cvb_pose P0 = P[0], P1 = P[1];
            for (uint32_t i = threadIdx.x; i < n; i += OPT_NT) {
                const double *o = obs + 9 * (size_t)(o0 + i);
                double f[3], s[3];
                rotv(P0.r, o + 3, f); rotv(P1.r, o + 6, s);
                three_view_gradients(o, f, P0.t, s, P1.t, g);
                for (int k = 0; k < 12; k++) acc[k] += g[k];
                if (adaptive) { acc[12] += norm3(g); acc[13] += norm3(g + 3); acc[14] += norm3(g + 6); acc[15] += norm3(g + 9); }
            }
            block_sum<16>(acc, s_red);
            if (threadIdx.x == 0 && three_view_opt_step(acc, inv_len, adaptive, rate, best, no_improve, P, updates, it == iterations - 1))
                s_stop = 1;
            __syncthreads();
            if (s_stop) break;
        }
    if (threadIdx.x == 0) {
        if (n > 0) { pose_inverse(P[0], &poses_out[2 * b]); pose_inverse(P[1], &poses_out[2 * b + 1]); }
        else { poses_out[2 * b] = poses_in[2 * b]; poses_out[2 * b + 1] = poses_in[2 * b + 1]; }
        updates_out[b] = updates;
    }
}

// three_view_optimizer.rs:203-272 (adaptive), one WARP per problem of at most OPT_NT landmarks.  Lane l evaluates landmark 32 r + l of
// row r, each row goes through block_sum's shuffle tree and lane 0 adds the row sums in row order, then +0.0 once for the rows that do not
// exist: exactly k_three_view_opt's sums (a row is one of its warps; its idle threads and warps add +0.0), so the two agree bit for bit.
constexpr int OPTW_NT = 128, OPTW_WARPS = OPTW_NT / 32;
__global__ void __launch_bounds__(OPTW_NT) k_three_view_opt_warp(const cvb_pose *__restrict__ poses_in, const double *__restrict__ obs,
                                                                 const uint32_t *__restrict__ offsets, uint32_t B, uint32_t iterations,
                                                                 cvb_pose *__restrict__ poses_out, uint32_t *__restrict__ updates_out) {
    __shared__ cvb_pose s_P[OPTW_WARPS][2];
    const uint32_t lane = threadIdx.x & 31, w = threadIdx.x >> 5, b = blockIdx.x * OPTW_WARPS + w;
    if (b >= B) return;
    const uint32_t o0 = offsets[b], n = offsets[b + 1] - o0, rows = (n + 31) / 32;
    cvb_pose *P = s_P[w];
    if (lane == 0 && n > 0) { pose_inverse(poses_in[2 * b], &P[0]); pose_inverse(poses_in[2 * b + 1], &P[1]); }
    __syncwarp();
    double best[2][2] = {{INFINITY, INFINITY}, {INFINITY, INFINITY}};
    uint32_t no_improve = 0, updates = 0;
    const double inv_len = 1.0 / (double)n;
    if (n > 0)
        for (uint32_t it = 0; it < iterations; it++) {
            const cvb_pose P0 = P[0], P1 = P[1];
            double tot[16];
            for (uint32_t r = 0; r < rows; r++) {
                double acc[16], g[12];
                for (int k = 0; k < 16; k++) acc[k] = 0.0;
                const uint32_t i = 32 * r + lane;
                if (i < n) {
                    const double *o = obs + 9 * (size_t)(o0 + i);
                    double f[3], s[3];
                    rotv(P0.r, o + 3, f); rotv(P1.r, o + 6, s);
                    three_view_gradients(o, f, P0.t, s, P1.t, g);
                    for (int k = 0; k < 12; k++) acc[k] += g[k];
                    acc[12] += norm3(g); acc[13] += norm3(g + 3); acc[14] += norm3(g + 6); acc[15] += norm3(g + 9);
                }
#pragma unroll
                for (int k = 0; k < 16; k++)
#pragma unroll
                    for (int o = 16; o; o >>= 1) acc[k] += __shfl_down_sync(0xffffffffu, acc[k], o);
                for (int k = 0; k < 16; k++) tot[k] = r == 0 ? acc[k] : tot[k] + acc[k];
            }
            int stop = 0;
            if (lane == 0) {
                if (rows < (uint32_t)OPT_WARPS)
                    for (int k = 0; k < 16; k++) tot[k] = __dadd_rn(tot[k], 0.0);
                stop = three_view_opt_step(tot, inv_len, 1, 0.0, best, no_improve, P, updates, it == iterations - 1);
            }
            stop = __shfl_sync(0xffffffffu, stop, 0);
            __syncwarp();
            if (stop) break;
        }
    if (lane == 0) {
        if (n > 0) { pose_inverse(P[0], &poses_out[2 * b]); pose_inverse(P[1], &poses_out[2 * b + 1]); }
        else { poses_out[2 * b] = poses_in[2 * b]; poses_out[2 * b + 1] = poses_in[2 * b + 1]; }
        updates_out[b] = updates;
    }
}

// cv-optimize's L1 (Weiszfeld) optimizers (include/cvb200_opt.h): the L2 kernels' shape, with per pose the sums of
// g.l1() = Se3TangentSpace::new(t.normalize(), r.normalize()) (so3.rs:23-34,123-125; a zero gradient normalises to NaN and
// becomes zero, but its weights still count) and of the weights 1/(|g.t| + tscale ε), 1/(|g.r| + ε).
// l1 += g.l1(), w[0] += translation weight, w[1] += rotation weight (single_view_optimizer.rs:36-38, three_view_optimizer.rs:53-55)
__device__ __forceinline__ void l1_accumulate(const double *tg, const double *rg, double tse, double eps, double *l1, double *w) {
    double lt[3], lr[3];
    w[0] += 1.0 / (norm3(tg) + tse);
    w[1] += 1.0 / (norm3(rg) + eps);
    normalize3(tg, lt); normalize3(rg, lr);
    tangent_new(lt, lr);
    for (int k = 0; k < 3; k++) { l1[k] += lt[k]; l1[3 + k] += lr[k]; }
}
// l1sum.scale(rate).scale_translation(ts.recip()).scale_rotation(rs.recip()): multiply by rate first, then by the reciprocal
__device__ __forceinline__ void l1_delta(const double *l1, const double *w, double rate, double *d) {
    const double it = 1.0 / w[0], ir = 1.0 / w[1];
    for (int k = 0; k < 3; k++) { d[k] = (l1[k] * rate) * it; d[3 + k] = (l1[3 + k] * rate) * ir; }
}

// single_view_optimizer.rs:16-78, one CTA per (pose, landmark list); acc = [l1sum.t, l1sum.r, ts, rs]
__global__ void __launch_bounds__(OPT_NT) k_single_view_opt_l1(const cvb_pose *__restrict__ poses_in, const double *__restrict__ bearings,
                                                               const double *__restrict__ world, const uint32_t *__restrict__ offsets,
                                                               double eps, double rate, uint32_t iterations, cvb_pose *__restrict__ poses_out,
                                                               uint32_t *__restrict__ updates_out) {
    __shared__ cvb_pose P;
    __shared__ double s_red[OPT_WARPS * 8];
    __shared__ int s_stop;
    const uint32_t b = blockIdx.x, o0 = offsets[b], n = offsets[b + 1] - o0;
    if (threadIdx.x == 0) { P = poses_in[b]; s_stop = 0; }
    __syncthreads();
    double best_t = INFINITY, best_r = INFINITY;
    uint32_t no_improve = 0, updates = 0;
    if (n > 0)
        for (uint32_t it = 0; it < iterations; it++) {
            double acc[8] = {0, 0, 0, 0, 0, 0, 0, 0}, tg[3], rg[3];
            const cvb_pose Pl = P;
            const double tse = norm3(Pl.t) * eps;       // tscale of the current pose (:30)
            for (uint32_t i = threadIdx.x; i < n; i += OPT_NT)
                if (landmark_delta(Pl, bearings + 3 * (size_t)(o0 + i), world + 4 * (size_t)(o0 + i), tg, rg))
                    l1_accumulate(tg, rg, tse, eps, acc, acc + 6);
            block_sum<8>(acc, s_red);
            if (threadIdx.x == 0) {
                double d[6];
                l1_delta(acc, acc + 6, rate, d);
                no_improve++;
                const double t = norm3(acc), r = norm3(acc + 3);   // patience on the unnormalised l1sum (:47-57)
                if (best_t > t) { best_t = t; no_improve = 0; }
                if (best_r > r) { best_r = r; no_improve = 0; }
                if (no_improve >= 50) s_stop = 1;
                else {
                    apply_delta(d, d + 3, &P); updates++;
                    if (it == iterations - 1) s_stop = 1;
                }
            }
            __syncthreads();
            if (s_stop) break;
        }
    if (threadIdx.x == 0) { poses_out[b] = P; updates_out[b] = updates; }
}

// three_view_optimizer.rs:23-124, one CTA per (pose pair, observation triples); acc = [l1sum0 (6), l1sum1 (6), ts0, rs0, ts1, rs1]
__global__ void __launch_bounds__(OPT_NT) k_three_view_opt_l1(const cvb_pose *__restrict__ poses_in, const double *__restrict__ obs,
                                                              const uint32_t *__restrict__ offsets, double eps, double rate,
                                                              uint32_t iterations, cvb_pose *__restrict__ poses_out,
                                                              uint32_t *__restrict__ updates_out) {
    __shared__ cvb_pose P[2];
    __shared__ double s_red[OPT_WARPS * 16];
    __shared__ int s_stop;
    const uint32_t b = blockIdx.x, o0 = offsets[b], n = offsets[b + 1] - o0;
    if (threadIdx.x == 0) {
        if (n > 0) { pose_inverse(poses_in[2 * b], &P[0]); pose_inverse(poses_in[2 * b + 1], &P[1]); }
        s_stop = 0;
    }
    __syncthreads();
    double best[2][2] = {{INFINITY, INFINITY}, {INFINITY, INFINITY}};
    uint32_t no_improve = 0, updates = 0;
    if (n > 0)
        for (uint32_t it = 0; it < iterations; it++) {
            double acc[16], g[12];
            for (int k = 0; k < 16; k++) acc[k] = 0.0;
            const cvb_pose P0 = P[0], P1 = P[1];
            const double tse = (norm3(P0.t) + norm3(P1.t)) * eps;   // tscale of the inverted poses (:45-48)
            for (uint32_t i = threadIdx.x; i < n; i += OPT_NT) {
                const double *o = obs + 9 * (size_t)(o0 + i);
                double f[3], s[3];
                rotv(P0.r, o + 3, f); rotv(P1.r, o + 6, s);
                three_view_gradients(o, f, P0.t, s, P1.t, g);
                l1_accumulate(g, g + 3, tse, eps, acc, acc + 12);
                l1_accumulate(g + 6, g + 9, tse, eps, acc + 6, acc + 14);
            }
            block_sum<16>(acc, s_red);
            if (threadIdx.x == 0) {
                double d[12];
                l1_delta(acc, acc + 12, rate, d);
                l1_delta(acc + 6, acc + 14, rate, d + 6);
                no_improve++;
                for (int v = 0; v < 2; v++) {          // one patience counter over all four norms (:69-81)
                    const double t = norm3(acc + 6 * v), r = norm3(acc + 6 * v + 3);
                    if (best[v][0] > t) { best[v][0] = t; no_improve = 0; }
                    if (best[v][1] > r) { best[v][1] = r; no_improve = 0; }
                }
                if (no_improve >= 50) s_stop = 1;
                else {
                    apply_delta(d, d + 3, &P[0]); apply_delta(d + 6, d + 9, &P[1]); updates++;
                    if (it == iterations - 1) s_stop = 1;
                }
            }
            __syncthreads();
            if (s_stop) break;
        }
    if (threadIdx.x == 0) {
        if (n > 0) { pose_inverse(P[0], &poses_out[2 * b]); pose_inverse(P[1], &poses_out[2 * b + 1]); }
        else { poses_out[2 * b] = poses_in[2 * b]; poses_out[2 * b + 1] = poses_in[2 * b + 1]; }
        updates_out[b] = updates;
    }
}

__device__ void pose_mul(const cvb_pose &A, const cvb_pose &B, cvb_pose *o) {
    for (int i = 0; i < 3; i++)
        for (int c = 0; c < 3; c++) o->r[3 * i + c] = A.r[3 * i] * B.r[c] + A.r[3 * i + 1] * B.r[3 + c] + A.r[3 * i + 2] * B.r[6 + c];
    double sh[3];
    rotv(A.r, B.t, sh);
    for (int i = 0; i < 3; i++) o->t[i] = A.t[i] + sh[i];
}
__device__ double transformed_cosine_distance(const cvb_pose &P, const double *point_h, const double *bearing) {
    double q[4];
    pose_apply(P, point_h, q);
    from_homogeneous(q);
    return 1.0 - dot3(q, bearing);
}
// ---- the triangulators of cv-geom/src/triangulation.rs (include/cvb200_tri.h), each restated on the checker's side as well
// (ref_triangulation.c).  Reference details kept as they are:
//  - Isometry x unit vector applies the rotation only (nalgebra): a world-frame bearing is R^T b, a camera centre R^T (-t).
//  - The cheirality tests use the sign bit (is_sign_positive): a dot product of -0.0 fails.
__device__ __forceinline__ void rotTv(const double *R, const double *v, double *o) {
    for (int c = 0; c < 3; c++) o[c] = R[c] * v[0] + R[3 + c] * v[1] + R[6 + c] * v[2];
}
// camera centre and world-frame bearing of one (WorldToCamera, bearing) observation: pose.inverse().isometry() applied to both
__device__ __forceinline__ void obs_world(const cvb_pose &P, const double *b, double *centre, double *wb) {
    const double nt[3] = {-P.t[0], -P.t[1], -P.t[2]};
    rotTv(P.r, nt, centre);
    rotTv(P.r, b, wb);
}
__device__ __forceinline__ bool finite4(const double *p) { return isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]) && isfinite(p[3]); }
// max_iterations (usize upstream) as the Jacobi sweep bound
__device__ __forceinline__ int tri_sweeps(const cvb_triangulator &T) { return T.max_iterations > 0x7fffffffu ? 0x7fffffff : (int)T.max_iterations; }

// cv-geom/src/triangulation.rs:228-276 SineL1Triangulator.  Kept from the reference:
//  - when LinearEigen's point has w == 0 (point() is None) that point is returned unrefined (:240-244);
//  - scale = optimization_rate / count (:246), and the loop stops when |delta|^2 / |p|^2 < epsilon^2 (:269);
//  - after the refinement there is NO finiteness or cheirality check (:274);
//  - Default is epsilon 1e-12, 1000 iterations, rate 1.0, although the setter's doc comment says 0.01 (:197-199, :218-226).
// W (6 doubles per observation) receives every observation's camera centre and world-frame bearing once, before the loop; the
// reference recomputes them every iteration with the same expressions, so the bits are the same.  The gradients are summed in
// observation order, starting from zero, as the reference's `.sum()` does.
__device__ bool triangulate_sine_l1(const cvb_triangulator &T, const cvb_pose *P, const double *B, uint32_t n, double *W, double *p) {
    if (!triangulate_linear_eigen(P, B, n, p, T.epsilon, tri_sweeps(T))) return false;
    if (p[3] == 0.0) return true;
    double x[3] = {p[0] / p[3], p[1] / p[3], p[2] / p[3]};
    for (uint32_t i = 0; i < n; i++) obs_world(P[i], B + 3 * (size_t)i, W + 6 * (size_t)i, W + 6 * (size_t)i + 3);
    const double scale = T.optimization_rate / (double)n, eps2 = T.epsilon * T.epsilon;
    for (uint32_t it = 0; it < T.max_iterations; it++) {
        double s[3] = {0.0, 0.0, 0.0};
        for (uint32_t i = 0; i < n; i++) {
            const double *c = W + 6 * (size_t)i, *wb = c + 3;
            const double tr[3] = {c[0] - x[0], c[1] - x[1], c[2] - x[2]};
            const double d = dot3(tr, wb);
            for (int k = 0; k < 3; k++) s[k] = s[k] + (tr[k] - d * wb[k]);   // epipolar::point_gradient (epipolar.rs:174-179)
        }
        const double delta[3] = {scale * s[0], scale * s[1], scale * s[2]};
        for (int k = 0; k < 3; k++) x[k] = x[k] + delta[k];
        if (dot3(delta, delta) / dot3(x, x) < eps2) break;
    }
    p[0] = x[0]; p[1] = x[1]; p[2] = x[2]; p[3] = 1.0;
    from_homogeneous(p);   // Projective::from_point
    return true;
}

// cv-geom/src/triangulation.rs:392-442 MeanMeanTriangulator.  For n <= 1 it divides by zero (0 / 0, or a zero projection distance)
// and the finiteness filter returns None, as in the reference; nothing beyond the n observations is read.
__device__ bool triangulate_mean_mean(const cvb_pose *P, const double *B, uint32_t n, double *p) {
    const double total = (double)n;
    double sc[3] = {0.0, 0.0, 0.0}, sb[3] = {0.0, 0.0, 0.0}, c[3], wb[3];
    for (uint32_t i = 0; i < n; i++) {
        obs_world(P[i], B + 3 * (size_t)i, c, wb);
        for (int k = 0; k < 3; k++) { sc[k] = sc[k] + c[k]; sb[k] = sb[k] + wb[k]; }
    }
    const double ac[3] = {sc[0] / total, sc[1] / total, sc[2] / total};
    const double nb = norm3(sb);
    const double ab[3] = {sb[0] / nb, sb[1] / nb, sb[2] / nb};
    double sum = 0.0;
    for (uint32_t i = 0; i < n; i++) {
        obs_world(P[i], B + 3 * (size_t)i, c, wb);
        const double trans[3] = {ac[0] - c[0], ac[1] - c[1], ac[2] - c[2]};
        double q[3], bt[3];
        cross3(ab, wb, q);
        const double r = 1.0 / dot3(q, q);
        const double qs[3] = {q[0] * r, q[1] * r, q[2] * r};
        cross3(wb, trans, bt);
        sum = sum + dot3(qs, bt);
    }
    const double w = 1.0 / (sum / total);
    p[0] = ab[0] + ac[0] * w; p[1] = ab[1] + ac[1] * w; p[2] = ab[2] + ac[2] * w; p[3] = w;
    from_homogeneous(p);
    if (!finite4(p)) return false;
    for (uint32_t i = 0; i < n; i++) {
        obs_world(P[i], B + 3 * (size_t)i, c, wb);
        if (signbit(dot3(wb, p))) return false;
    }
    return true;
}

// TriangulatorObservations (methods 0-2; the host rejects the others).  W: SineL1's scratch, 6 doubles per observation.
__device__ bool triangulate_observations(const cvb_triangulator &T, const cvb_pose *P, const double *B, uint32_t n, double *W, double *p) {
    switch (T.method) {
    case CVB_TRI_SINE_L1: return triangulate_sine_l1(T, P, B, n, W, p);
    case CVB_TRI_MEAN_MEAN: return triangulate_mean_mean(P, B, n, p);
    default: return triangulate_linear_eigen(P, B, n, p, T.epsilon, tri_sweeps(T));
    }
}
// one thread per landmark
__global__ void __launch_bounds__(128) k_triangulate(cvb_triangulator T, const cvb_pose *__restrict__ poses, const double *__restrict__ bearings,
                                                     const uint32_t *__restrict__ offsets, uint32_t L, double *__restrict__ W,
                                                     double *__restrict__ xyzw, uint8_t *__restrict__ ok) {
    const uint32_t l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= L) return;
    const uint32_t o0 = offsets[l], o1 = offsets[l + 1];
    double p[4] = {0, 0, 0, 0};
    const bool good = triangulate_observations(T, poses + o0, bearings + 3 * (size_t)o0, o1 - o0, W ? W + 6 * (size_t)o0 : nullptr, p);
    ok[l] = good ? 1 : 0;
    for (int i = 0; i < 4; i++) xyzw[(size_t)l * 4 + i] = good ? p[i] : 0.0;
}

// TriangulatorRelative of methods 0-2 is the blanket impl (cv-core/src/triangulation.rs:21-35, 52-67): the observations
// [(identity, a), (pose, b)], then CameraPoint::from_homogeneous once more (which can change the last bit)
__device__ bool triangulate_relative_obs(const cvb_triangulator &T, const cvb_pose &P, const double *a, const double *b, double *p) {
    cvb_pose O[2];
    for (int k = 0; k < 9; k++) O[0].r[k] = (k % 4 == 0) ? 1.0 : 0.0;
    O[0].t[0] = O[0].t[1] = O[0].t[2] = 0.0;
    O[1] = P;
    const double B[6] = {a[0], a[1], a[2], b[0], b[1], b[2]};
    double W[12];
    if (!triangulate_observations(T, O, B, 2, W, p)) return false;
    from_homogeneous(p);
    return true;
}
// cv-geom/src/triangulation.rs:322-363 RelativeDltTriangulator.  nalgebra's try_svd (not in the reference checkout) is restated as
// one-sided Jacobi on the 4x4 design matrix itself -- the right singular vector of the smallest singular value -- never as the
// eigenvectors of DtD, which squares the condition number and loses the null vector at low parallax.  epsilon / max_iterations bound
// the Jacobi sweeps as they bound the eigen restatements'.  Default is 1e-12 / 1000 although the doc comments say 1e-9 / 100 (:293-320).
__device__ bool triangulate_relative_dlt(const cvb_triangulator &T, const cvb_pose &P, const double *a, const double *b, double *p) {
    const double D[16] = {-a[2], 0.0, a[0], 0.0,
                          0.0, -a[2], a[1], 0.0,
                          b[0] * P.r[6] - b[2] * P.r[0], b[0] * P.r[7] - b[2] * P.r[1], b[0] * P.r[8] - b[2] * P.r[2], b[0] * P.t[2] - b[2] * P.t[0],
                          b[1] * P.r[6] - b[2] * P.r[3], b[1] * P.r[7] - b[2] * P.r[4], b[1] * P.r[8] - b[2] * P.r[5], b[1] * P.t[2] - b[2] * P.t[1]};
    double smin;
    if (!min_right_singular_vector<4>(D, T.epsilon, tri_sweeps(T), p, &smin)) return false;
    from_homogeneous(p);
    if (!finite4(p)) return false;
    double bw[3];
    rotTv(P.r, b, bw);
    return !signbit(dot3(p, a)) && !signbit(dot3(p, bw));
}
// cv-geom/src/triangulation.rs:472-530 AngularL1Triangulator (linf = false) and :558-606 AngularLInfinityTriangulator (linf = true).
// Both invert the relative pose and swap a and b first (:483-487, :569-573) and build the point on the (corrected) swapped b.
// AngularL1 forms z = b x a; epipolar.rs's sine-L1 point forms a x b, so the two are not shared.
__device__ bool triangulate_angular(bool linf, const cvb_pose &P, const double *a_in, const double *b_in, double *p) {
    const double mt[3] = {-P.t[0], -P.t[1], -P.t[2]};
    // after the swap: b is the old a, a the old b carried by the inverse rotation, t the inverse pose's translation
    double t[3], a[3], b[3] = {a_in[0], a_in[1], a_in[2]};
    rotTv(P.r, mt, t);
    rotTv(P.r, b_in, a);
    const double tn = norm3(t);
    const double nt[3] = {t[0] / tn, t[1] / tn, t[2] / tn};
    if (!linf) {
        double ca[3], cb[3], v[3];
        cross3(a, nt, ca); cross3(b, nt, cb);
        const double can = norm3(ca), cbn = norm3(cb);
        if (can < cbn) {   // algorithm 12: correct a
            const double nb[3] = {cb[0] / cbn, cb[1] / cbn, cb[2] / cbn}, d = dot3(a, nb);
            for (int k = 0; k < 3; k++) v[k] = a[k] - d * nb[k];
            normalize3(v, a);
        } else {           // algorithm 13: correct b
            const double na[3] = {ca[0] / can, ca[1] / can, ca[2] / can}, d = dot3(b, na);
            for (int k = 0; k < 3; k++) v[k] = b[k] - d * na[k];
            normalize3(v, b);
        }
    } else {
        const double sp[3] = {a[0] + b[0], a[1] + b[1], a[2] + b[2]}, sm[3] = {a[0] - b[0], a[1] - b[1], a[2] - b[2]};
        double na[3], nb[3], n[3], va[3], vb[3];
        cross3(sp, nt, na); cross3(sm, nt, nb);
        const double nas = dot3(na, na), nbs = dot3(nb, nb);
        if (nas > nbs) { const double s = sqrt(nas); n[0] = na[0] / s; n[1] = na[1] / s; n[2] = na[2] / s; }
        else { const double s = sqrt(nbs); n[0] = nb[0] / s; n[1] = nb[1] / s; n[2] = nb[2] / s; }
        const double da = dot3(a, n), db = dot3(b, n);
        for (int k = 0; k < 3; k++) { va[k] = a[k] - da * n[k]; vb[k] = b[k] - db * n[k]; }
        normalize3(va, a); normalize3(vb, b);
    }
    double z[3], ta[3];
    cross3(b, a, z); cross3(t, a, ta);
    p[0] = b[0]; p[1] = b[1]; p[2] = b[2]; p[3] = dot3(z, z) / dot3(z, ta);
    from_homogeneous(p);
    if (!finite4(p)) return false;
    return !signbit(dot3(p, a)) && !signbit(dot3(p, b));
}
// TriangulatorRelative::triangulate_relative of all six methods
__device__ __forceinline__ bool triangulate_relative(const cvb_triangulator &T, const cvb_pose &P, const double *a, const double *b, double *p) {
    switch (T.method) {
    case CVB_TRI_RELATIVE_DLT: return triangulate_relative_dlt(T, P, a, b, p);
    case CVB_TRI_ANGULAR_L1: return triangulate_angular(false, P, a, b, p);
    case CVB_TRI_ANGULAR_LINF: return triangulate_angular(true, P, a, b, p);
    default: return triangulate_relative_obs(T, P, a, b, p);
    }
}
// one thread per (relative pose, a, b) triple; npose = 1 shares poses[0]
__global__ void __launch_bounds__(128) k_triangulate_relative(cvb_triangulator T, const cvb_pose *__restrict__ poses, uint32_t npose,
                                                              const double *__restrict__ a, const double *__restrict__ b, uint32_t n,
                                                              double *__restrict__ xyzw, uint8_t *__restrict__ ok) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const cvb_pose P = poses[npose == 1 ? 0 : i];
    const double *ai = a + 3 * (size_t)i, *bi = b + 3 * (size_t)i;
    double p[4] = {0, 0, 0, 0};
    const bool good = triangulate_relative(T, P, ai, bi, p);
    ok[i] = good ? 1 : 0;
    for (int k = 0; k < 4; k++) xyzw[(size_t)i * 4 + k] = good ? p[k] : 0.0;
}

// cv-sfm/src/lib.rs:2570-2620 observation_loss of every observation; one thread per landmark.  The landmarks of three or more
// observations go through the triangulator T (self.triangulator upstream); W: SineL1's scratch, 6 doubles per observation.
__global__ void __launch_bounds__(128) k_observation_losses(cvb_triangulator T, const cvb_pose *__restrict__ poses, const double *__restrict__ bearings,
                                                            const uint32_t *__restrict__ offsets, uint32_t L, double *__restrict__ W,
                                                            double *__restrict__ loss) {
    const uint32_t l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= L) return;
    const uint32_t o0 = offsets[l], n = offsets[l + 1] - o0;
    const cvb_pose *P = poses + o0;
    const double *B = bearings + 3 * (size_t)o0;
    if (n == 0) return;
    if (n == 1) { loss[o0] = 2.0; return; }
    if (n == 2) {
        cvb_pose inv, tot;
        double fb[3];
        pose_inverse(P[0], &inv); pose_mul(P[1], inv, &tot);
        rotv(tot.r, B, fb);
        const double v = 1.0 - cos(asin(epipolar_loss(tot.t, fb, B + 3)));
        loss[o0] = v; loss[o0 + 1] = v;
        return;
    }
    double p[4];
    const bool ok = triangulate_observations(T, P, B, n, W ? W + 6 * (size_t)o0 : nullptr, p);
    for (uint32_t i = 0; i < n; i++) loss[o0 + i] = ok ? transformed_cosine_distance(P[i], p, B + 3 * (size_t)i) : 2.0;
}
// cv-sfm/src/lib.rs:1320-1360 is_tri_landmark_robust with the triangulator T (poses CameraToCamera centre -> first / second);
// B: the centre, first and second bearings, contiguous
__device__ bool tri_landmark_robust(const cvb_triangulator &T, const cvb_pose &first, const cvb_pose &second, const double *B, double max_cos,
                                    double inc_min_cos) {
    const double *c = B, *f = B + 3, *s = B + 6;
    cvb_pose P[3];
    for (int k = 0; k < 9; k++) P[0].r[k] = (k % 4 == 0) ? 1.0 : 0.0;
    P[0].t[0] = P[0].t[1] = P[0].t[2] = 0.0;
    P[1] = first; P[2] = second;
    double p[4], W[18];
    if (!triangulate_observations(T, P, c, 3, W, p)) return false;
    from_homogeneous(p);   // CameraPoint::from_homogeneous(p.0)
    double fc[3], sc[3];
    for (int k = 0; k < 3; k++) {
        fc[k] = first.r[k] * f[0] + first.r[3 + k] * f[1] + first.r[6 + k] * f[2];
        sc[k] = second.r[k] * s[0] + second.r[3 + k] * s[1] + second.r[6 + k] * s[2];
    }
    const bool cosine_ok = 1.0 - dot3(p, c) < max_cos && transformed_cosine_distance(first, p, f) < max_cos
        && transformed_cosine_distance(second, p, s) < max_cos;
    const bool incidence_ok = 1.0 - dot3(c, fc) > inc_min_cos || 1.0 - dot3(c, sc) > inc_min_cos || 1.0 - dot3(fc, sc) > inc_min_cos;
    return cosine_ok && incidence_ok;
}
// one thread per (centre, first, second) observation triple of one pose pair
__global__ void __launch_bounds__(128) k_tri_landmark_robust(cvb_triangulator T, cvb_pose first, cvb_pose second, const double *__restrict__ obs,
                                                             uint32_t n, double max_cos, double inc_min_cos, uint8_t *__restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    out[i] = tri_landmark_robust(T, first, second, obs + 9 * (size_t)i, max_cos, inc_min_cos);
}

#include "init_dev.cuh"
#include "constraints_dev.cuh"
#include "reconstruction_dev.cuh"
#include "export_dev.cuh"
#include "register_dev.cuh"
#include "incorporate_dev.cuh"
#include "merge_dev.cuh"
#include "try_init_dev.cuh"

// ------------------------------------------------------------------------------------------ cv-pinhole (include/cvb200_pinhole.h)
// cv-pinhole/src/lib.rs:314-372 pose_reprojection_error + average_pose_reprojection_error of one FeatureMatch.  Kept from the reference:
//  - a_norm = a.xy / a.z and b_norm = b.xy / b.z come from the INPUT bearings (:320-321);
//  - the triangulated CameraPoint's bearing is its xyz (Projective::bearing, cv-core/src/point.rs:46-49), reprojected only when
//    bearing.z.is_sign_positive() -- a sign-bit test, so +0.0 and +NaN pass and their infinities / NaNs reach the error (:325-328);
//  - point_b = pose.transform(point_a) = from_homogeneous([R xyz + t w; w]) with the same test on its bearing (:329-334);
//  - average = ((0 + |e_a|) + |e_b|) * 0.5 with |v| = sqrt(x x + y y) (:370-371).
// the value of a row the reference returns None for: the quiet NaN of C's NAN and numpy's nan (CUDART_NAN has the sign bit set)
__device__ __forceinline__ double none_nan() { return __longlong_as_double(0x7ff8000000000000ull); }
__device__ bool pose_reprojection(const cvb_triangulator &T, const cvb_pose &P, const double *a, const double *b, double *e, double *avg) {
    const double an[2] = {a[0] / a[2], a[1] / a[2]}, bn[2] = {b[0] / b[2], b[1] / b[2]};
    double p[4] = {0, 0, 0, 0}, q[4];
    if (!triangulate_relative(T, P, a, b, p)) return false;
    if (signbit(p[2])) return false;
    pose_apply(P, p, q);
    from_homogeneous(q);
    if (signbit(q[2])) return false;
    e[0] = an[0] - p[0] / p[2]; e[1] = an[1] - p[1] / p[2];
    e[2] = bn[0] - q[0] / q[2]; e[3] = bn[1] - q[1] / q[2];
    *avg = ((0.0 + sqrt(e[0] * e[0] + e[1] * e[1])) + sqrt(e[2] * e[2] + e[3] * e[3])) * 0.5;
    return true;
}
// one thread per match; rows i < min(*n_dev, n) (n_dev null: n) are written; found (may be null) == 0 marks every row as None
__global__ void __launch_bounds__(128) k_pose_reprojection_error(cvb_triangulator T, const cvb_pose *__restrict__ poses, uint32_t npose,
                                                                 const double *__restrict__ a, const double *__restrict__ b,
                                                                 const uint32_t *__restrict__ n_dev, uint32_t n, const int32_t *__restrict__ found,
                                                                 double *__restrict__ err, double *__restrict__ avg, uint8_t *__restrict__ ok) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (n_dev ? min(*n_dev, n) : n)) return;
    double e[4], m;
    const bool good = (!found || *found != 0) &&
                      pose_reprojection(T, poses[npose == 1 ? 0 : i], a + 3 * (size_t)i, b + 3 * (size_t)i, e, &m);
    ok[i] = good ? 1 : 0;
    for (int k = 0; k < 4; k++) err[(size_t)i * 4 + k] = good ? e[k] : none_nan();
    if (avg) avg[i] = good ? m : none_nan();
}

// EightPoint { epsilon, iterations }::from_matches (eight-point/src/lib.rs:43-58) on one sample of 8 matches: the design rows, Gram
// matrix and round-robin Jacobi of eight_point(), with the caller's epsilon and sweep bound
__global__ void __launch_bounds__(128) k_eight_point_essential(const double *__restrict__ a, const double *__restrict__ b,
                                                               const uint32_t *__restrict__ samples, uint32_t H, double eps, int sweeps,
                                                               double *__restrict__ E_out, uint8_t *__restrict__ ok) {
    const uint32_t h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= H) return;
    double D[72], EtE[81], V[81];
    for (int i = 0; i < 8; i++) eight_point_row(a, b, samples[(size_t)h * 8 + i], D + 9 * i);
    for (int r = 0; r < 9; r++)
        for (int c = 0; c < 9; c++) EtE[r * 9 + c] = eight_point_gram(D, r, c);
    const bool good = sym_eigen9_rr<1>(EtE, V, 0, 0u, eps, sweeps);
    int best = 0;
    for (int i = 1; i < 9; i++)
        if (EtE[i * 9 + i] < EtE[best * 9 + best]) best = i;
    double *E = E_out + (size_t)h * 9;
    for (int k = 0; k < 9; k++) E[(k % 3) * 3 + (k / 3)] = good ? V[k * 9 + best] : none_nan();   // Matrix3::from_iterator: column-major
    ok[h] = good ? 1 : 0;
}

// cv-pinhole/src/essential.rs:266-275 EssentialMatrix::residual as |nb . (E na)|: E na first, then the dot product with nb (nalgebra's
// b^T E a groups (b^T E) a, so the last bit can differ from the reference; the CPU restatement groups it this way too)
__device__ __forceinline__ double residual_essential(const double *E, const double *a, const double *b) {
    const double na[3] = {a[0] / a[2], a[1] / a[2], a[2] / a[2]}, nb[3] = {b[0] / b[2], b[1] / b[2], b[2] / b[2]};
    const double Ea[3] = {dot3(E, na), dot3(E + 3, na), dot3(E + 6, na)};
    return fabs(dot3(nb, Ea));
}
// one thread per (E, datum), the layout of k_residuals
__global__ void __launch_bounds__(256) k_residuals_essential(const double *__restrict__ Es, const double *__restrict__ a,
                                                             const double *__restrict__ b, uint32_t n, double *__restrict__ out) {
    const uint32_t p = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double E[9];
    for (int k = 0; k < 9; k++) E[k] = Es[(size_t)p * 9 + k];
    out[(size_t)p * n + i] = residual_essential(E, a + 3 * (size_t)i, b + 3 * (size_t)i);
}

// cv-pinhole/src/essential.rs:64-77 EssentialMatrix::recondition: SVD::recompose of U diag(s, s, 0) Vt, s = (s0 + s1) / 2 (nalgebra
// scales U's columns, then multiplies by Vt); one thread per matrix
__global__ void __launch_bounds__(128) k_essential_recondition(const double *__restrict__ Es, uint32_t m, double eps, int sweeps,
                                                               double *__restrict__ E_out, uint8_t *__restrict__ ok) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    double E[9], U[9], Vt[9], S[3], R[9];
    for (int k = 0; k < 9; k++) E[k] = Es[(size_t)j * 9 + k];
    const bool good = svd3(E, eps, sweeps, U, Vt, S);
    if (good) {
        const double s = (S[0] + S[1]) / 2.0, d[3] = {s, s, 0.0};
        for (int r = 0; r < 3; r++)
            for (int c = 0; c < 3; c++) U[r * 3 + c] *= d[c];
        mat3_mul(U, Vt, R);
    }
    for (int k = 0; k < 9; k++) E_out[(size_t)j * 9 + k] = good ? R[k] : none_nan();
    ok[j] = good ? 1 : 0;
}

// cv-pinhole/src/essential.rs:114-162 possible_rotations_unscaled_translation; one thread per matrix
__global__ void __launch_bounds__(128) k_essential_decompose(const double *__restrict__ Es, uint32_t m, double eps, int sweeps,
                                                             double *__restrict__ rot_a, double *__restrict__ rot_b, double *__restrict__ t_out,
                                                             uint8_t *__restrict__ ok) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    double E[9], Ra[9], Rb[9], t[3];
    for (int k = 0; k < 9; k++) E[k] = Es[(size_t)j * 9 + k];
    const bool good = essential_rotations(E, eps, sweeps, Ra, Rb, t);
    for (int k = 0; k < 9; k++) { rot_a[(size_t)j * 9 + k] = good ? Ra[k] : none_nan(); rot_b[(size_t)j * 9 + k] = good ? Rb[k] : none_nan(); }
    for (int k = 0; k < 3; k++) t_out[(size_t)j * 3 + k] = good ? t[k] : none_nan();
    ok[j] = good ? 1 : 0;
}

// ------------------------------------------------------------------------------------------ host side
struct DevBuf {
    void *p = nullptr;
    size_t bytes = 0;
    int ensure(cvb_ctx *ctx, size_t need) {
        if (need <= bytes && p) return 0;
        if (p) { cvb_wait(ctx, ctx->stream); cudaFree(p); p = nullptr; bytes = 0; }
        size_t n = std::max<size_t>(need, 256);
        cudaError_t e = cudaMalloc(&p, n);
        if (e != cudaSuccess) return cvb_set_error(ctx, CVB_ENOMEM, "cudaMalloc(%zu): %s", n, cudaGetErrorString(e));
        bytes = n;
        return 0;
    }
};

}  // namespace

// device-resident ARRSAC (arrsac_dev.cuh): buffers + page-locked staging of one context
struct ArsWorkspace {
    DevBuf ctl, raw, samples0, poses0, nposes0, masks0, vm, pass_id, pass_inl, tposes, tinl, tmasks, newposes, nposes_new, newmask,
        nout, pool, samples_new, res, queue;
    DevBuf bdata_a, bdata_b, bcounts;   // the host batch entry's padded rows and counts
    uint32_t *h_raw = nullptr;      // page-locked: B ArrsacCtl headers + batch header, then B raw-draw streams
    size_t h_raw_cap = 0;
    unsigned char *h_res = nullptr; // page-locked result block (B ArrsacCtl)
    size_t h_res_cap = 0;
    cudaEvent_t up_done = nullptr;  // the staging buffer may be rewritten once this has fired
    std::vector<cvb_rng> snaps;     // generator state every ARS_SNAP draws of each problem's staged stream (nsnap per problem)
    uint32_t nraw = 0, nsnap = 0, B = 0;
    bool pending = false;           // a run whose draw count has not been committed to the caller's generator yet
    bool pending_batch = false;     // ... and it came through the batch entry (committed by cvb_arrsac_commit_rng_batch only)
    // CUDA graphs of the whole run (two copies, ~20 + 3 per data block kernels, one copy back), keyed by everything the enqueue
    // depends on; a key is captured the second time it is seen (a one-off call does not pay the instantiation)
    struct GraphKey {
        ArrsacParams P; int kind, row0; const void *a, *b, *n_dev; uint32_t n_host, nmax, cap, nb, B; const void *model, *inl, *ninl, *found;
        const void *ws[22];
    };
    struct GraphEntry { GraphKey key; cudaGraphExec_t exec; uint64_t launches; uint32_t body; };   // body: launches of one WHILE body (0: no WHILE node)
    uint32_t last_body = 0;         // the pending run went through a WHILE-node graph with this many launches per body (counted at commit)
    std::vector<GraphEntry> graphs;
    std::vector<GraphKey> seen;
    int use_graph = -1;             // CVB_NO_GRAPH=1 / CVB_ARS_NO_GRAPH=1 disable
    // the block loop as a WHILE node of the graph (body: score, resolve, book, estimate; k_ars_book clears the condition at the loop's
    // end) instead of one unrolled body per possible data block.  CVB_ARS_WHILE=0 keeps the unrolled graph.
    int use_while = -1;
    cudaStream_t body_stream = nullptr;
};
struct GeomWorkspace {
    DevBuf a, b, samples, poses, nposes, out, masks, offsets, ok;
    DevBuf init;                    // the three-view initialisation's per-call workspace (init_reconstruction_dev)
    DevBuf con, con2;               // the view constraints' snapshot / per-chunk and per-sub-chunk workspaces (view_constraints_dev)
    DevBuf rec;                     // the reconstruction optimisation's workspace (optimize_reconstruction_dev)
    DevBuf exp;                     // the export's workspace (export_dev.cuh's drivers)
    DevBuf reg;                     // frame registration's workspace (register_frame_dev)
    DevBuf inc, incs;               // frame incorporation's snapshot after add_view and the two edits' scratch (incorporate_frame_dev)
    DevBuf mrg, mrgs;               // merging's snapshot after add_view, and the move's snapshots and scratch (merge_dev.cuh's drivers)
    DevBuf tinit, tinits;           // creation's add_reconstruction scratch, and try_init's two-view outputs, init result and lists
    ArsWorkspace *ars = nullptr;
};
void geom_workspace_free(GeomWorkspace *g) {
    if (!g) return;
    DevBuf *bufs[] = {&g->a, &g->b, &g->samples, &g->poses, &g->nposes, &g->out, &g->masks, &g->offsets, &g->ok, &g->init, &g->con,
                      &g->con2, &g->rec, &g->exp, &g->reg, &g->inc, &g->incs, &g->mrg, &g->mrgs,
                      &g->tinit, &g->tinits};
    for (DevBuf *d : bufs) if (d->p) cudaFree(d->p);
    if (g->ars) {
        ArsWorkspace *w = g->ars;
        DevBuf *ab[] = {&w->ctl, &w->raw, &w->samples0, &w->poses0, &w->nposes0, &w->masks0, &w->vm, &w->pass_id, &w->pass_inl, &w->tposes,
                        &w->tinl, &w->tmasks, &w->newposes, &w->nposes_new, &w->newmask, &w->nout, &w->pool, &w->samples_new, &w->res,
                        &w->queue, &w->bdata_a, &w->bdata_b, &w->bcounts};
        for (DevBuf *d : ab) if (d->p) cudaFree(d->p);
        if (w->h_raw) cudaFreeHost(w->h_raw);
        if (w->h_res) cudaFreeHost(w->h_res);
        if (w->up_done) cudaEventDestroy(w->up_done);
        if (w->body_stream) cudaStreamDestroy(w->body_stream);
        for (auto &ge : w->graphs) cudaGraphExecDestroy(ge.exec);
        delete w;
    }
    delete g;
}

namespace {

// estimator kinds: 0 EightPoint, 1 LambdaTwist (P3P), 2 NisterStewenius (five-point)
inline uint32_t kind_K(int kind) { return kind == 0 ? 8u : (kind == 1 ? 3u : 5u); }      // Estimator::MIN_SAMPLES
inline uint32_t kind_M(int kind) { return kind == 2 ? 40u : 4u; }                         // ModelIter capacity
inline int kind_res(int kind) { return kind == 1 ? 1 : 0; }                               // residual: 0 CameraToCamera, 1 WorldToCamera

GeomWorkspace *gws(cvb_ctx *ctx) {
    if (!ctx->geom) ctx->geom = new GeomWorkspace();
    return ctx->geom;
}

int upload(cvb_ctx *ctx, DevBuf &d, const void *src, size_t bytes) {
    int rc = d.ensure(ctx, bytes);
    if (rc) return rc;
    if (bytes) CVB_CUDA(ctx, cudaMemcpyAsync(d.p, src, bytes, cudaMemcpyHostToDevice, ctx->stream));
    return 0;
}

// data stay resident in the workspace (a: n x 3; b: n x 3 or n x 4)
int upload_data(cvb_ctx *ctx, int kind, const double *a, const double *b, uint32_t n) {
    GeomWorkspace *g = gws(ctx);
    int rc = upload(ctx, g->a, a, sizeof(double) * 3 * (size_t)n);
    if (rc) return rc;
    return upload(ctx, g->b, b, sizeof(double) * (kind_res(kind) == 0 ? 3 : 4) * (size_t)n);
}

// estimate H minimal samples (host index lists) -> device poses (H x 4) + host counts
int estimate_dev(cvb_ctx *ctx, int kind, const uint32_t *samples, uint32_t H, std::vector<uint8_t> &nposes, int row0 = 5) {
    GeomWorkspace *g = gws(ctx);
    const uint32_t K = kind_K(kind), M = kind_M(kind);
    int rc = upload(ctx, g->samples, samples, sizeof(uint32_t) * K * (size_t)H);
    if (rc) return rc;
    if ((rc = g->poses.ensure(ctx, sizeof(cvb_pose) * M * (size_t)H))) return rc;
    if ((rc = g->nposes.ensure(ctx, H))) return rc;
    CVB_CUDA(ctx, cudaMemsetAsync(g->poses.p, 0, sizeof(cvb_pose) * M * (size_t)H, ctx->stream));
    {
        CVB_PROF(ctx, kind == 0 ? "k_estimate_eight_point" : (kind == 1 ? "k_estimate_p3p" : "k_estimate_five_point"), 0);
        const double *a = (const double *)g->a.p, *b = (const double *)g->b.p;
        const uint32_t *sp = (const uint32_t *)g->samples.p;
        if (kind == 0) k_estimate<0><<<cdiv(H, 128), 128, 0, ctx->stream>>>(a, b, sp, H, (cvb_pose *)g->poses.p, (uint8_t *)g->nposes.p, row0);
        else if (kind == 1) k_estimate<1><<<cdiv(H, 128), 128, 0, ctx->stream>>>(a, b, sp, H, (cvb_pose *)g->poses.p, (uint8_t *)g->nposes.p, row0);
        else k_estimate<2><<<cdiv(H, 128), 128, 0, ctx->stream>>>(a, b, sp, H, (cvb_pose *)g->poses.p, (uint8_t *)g->nposes.p, row0);
        CVB_LAUNCH_CHECK(ctx);
    }
    nposes.resize(H);
    CVB_CUDA(ctx, cudaMemcpyAsync(nposes.data(), g->nposes.p, H, cudaMemcpyDeviceToHost, ctx->stream));
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    return 0;
}

// inlier masks of m device poses over data [i0, i1) -> host (m x words)
int masks_dev(cvb_ctx *ctx, int kind, const cvb_pose *poses_dev, uint32_t m, uint32_t i0, uint32_t i1, double thr,
              std::vector<uint32_t> &masks, uint32_t *words_out) {
    GeomWorkspace *g = gws(ctx);
    const uint32_t cnt = i1 - i0, words = cdiv(cnt, 32);
    *words_out = words;
    masks.assign((size_t)m * words, 0u);
    if (m == 0 || cnt == 0) return 0;
    int rc = g->masks.ensure(ctx, sizeof(uint32_t) * (size_t)m * words);
    if (rc) return rc;
    for (uint32_t p0 = 0; p0 < m; p0 += 65535) {   // gridDim.y limit
        const uint32_t pm = std::min<uint32_t>(65535, m - p0);
        dim3 grid(cdiv(cnt, 256), pm);
        CVB_PROF(ctx, kind_res(kind) == 0 ? "k_residuals_c2c" : "k_residuals_w2c", (kind_res(kind) == 0 ? 48.0 : 56.0) * pm * cnt);
        if (kind_res(kind) == 0)
            k_residuals<0, 1><<<grid, 256, 0, ctx->stream>>>(poses_dev + p0, pm, (const double *)g->a.p, (const double *)g->b.p, i0, i1, thr, nullptr, 0,
                                                             (uint32_t *)g->masks.p + (size_t)p0 * words, words);
        else
            k_residuals<1, 1><<<grid, 256, 0, ctx->stream>>>(poses_dev + p0, pm, (const double *)g->a.p, (const double *)g->b.p, i0, i1, thr, nullptr, 0,
                                                             (uint32_t *)g->masks.p + (size_t)p0 * words, words);
        CVB_LAUNCH_CHECK(ctx);
    }
    CVB_CUDA(ctx, cudaMemcpyAsync(masks.data(), g->masks.p, sizeof(uint32_t) * (size_t)m * words, cudaMemcpyDeviceToHost, ctx->stream));
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    return 0;
}

inline uint32_t popc_range(const uint32_t *row, uint32_t lo, uint32_t hi) {   // bits [lo, hi)
    uint32_t c = 0;
    for (uint32_t i = lo; i < hi; i++) c += (row[i >> 5] >> (i & 31)) & 1u;
    return c;
}

uint64_t rotl64(uint64_t x, int k) { return (x << k) | (x >> (64 - k)); }

struct Hyp { cvb_pose m; uint32_t inliers; std::vector<uint32_t> mask; };   // mask over ALL n data

void sort_hyps(std::vector<Hyp> &H) {
    std::stable_sort(H.begin(), H.end(), [](const Hyp &x, const Hyp &y) { return x.inliers > y.inliers; });
}

void populate_samples(cvb_rng *rng, uint32_t k, uint32_t len, uint32_t *out) {
    for (uint32_t c = 0; c < k;) {
        uint32_t s = cvb_rng_next_u32(rng) % len;
        bool dup = false;
        for (uint32_t j = 0; j < c; j++) dup |= out[j] == s;
        if (!dup) out[c++] = s;
    }
}

// arrsac::Arrsac::model_inliers, restated (external crate arrsac 0.10.0; see DESIGN.md for what is and is not pinned):
// initialisation with an adaptive SPRT over the first blocks, then block-wise scoring / halving / re-estimation
// from the inliers of the current best.  All residuals come from the GPU as bit masks.
int arrsac_run(cvb_ctx *ctx, const cvb_arrsac_cfg *cfg, int kind, const double *a, const double *b, uint32_t n, cvb_rng *rng,
               cvb_pose *model_out, uint32_t *inliers_out, uint32_t cap, uint32_t *n_inliers, int32_t *found, int row0 = 5) {
    const uint32_t K = kind_K(kind), MM = kind_M(kind);
    *found = 0;
    if (n_inliers) *n_inliers = 0;
    if (n < K) return 0;
    if (cfg->block_size == 0 || cfg->initialization_blocks == 0) return cvb_set_error(ctx, CVB_EINVAL, "block_size / initialization_blocks must be > 0");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    int rc = upload_data(ctx, kind, a, b, n);
    if (rc) return rc;
    GeomWorkspace *g = gws(ctx);
    const double thr = cfg->inlier_threshold;
    const uint32_t nwords = cdiv(n, 32);
    // ---- initialisation: all minimal samples are drawn first (the draws do not depend on any result)
    const uint32_t H0 = cfg->initialization_hypotheses;
    if (H0 == 0) return 0;
    std::vector<uint32_t> samples((size_t)H0 * K);
    for (uint32_t h = 0; h < H0; h++) populate_samples(rng, K, n, samples.data() + (size_t)h * K);
    std::vector<uint8_t> nposes;
    if ((rc = estimate_dev(ctx, kind, samples.data(), H0, nposes, row0))) return rc;
    // inlier masks of every candidate model over the initialisation blocks only (what the SPRT looks at)
    const uint32_t init_n = std::min<uint32_t>(cfg->block_size * cfg->initialization_blocks, n);
    std::vector<uint32_t> masks;
    uint32_t words = 0;
    if ((rc = masks_dev(ctx, kind, (const cvb_pose *)g->poses.p, H0 * MM, 0, init_n, thr, masks, &words))) return rc;
    std::vector<cvb_pose> poses_host((size_t)H0 * MM);
    CVB_CUDA(ctx, cudaMemcpy(poses_host.data(), g->poses.p, sizeof(cvb_pose) * MM * (size_t)H0, cudaMemcpyDeviceToHost));
    float epsilon = cfg->initial_epsilon, delta = cfg->initial_delta;
    uint32_t best_inliers = 0;
    uint64_t rej_inliers = 0, rej_tested = 0;
    std::vector<Hyp> H;
    for (uint32_t h = 0; h < H0; h++)
        for (uint32_t mi = 0; mi < nposes[h]; mi++) {
            const uint32_t *row = masks.data() + ((size_t)h * MM + mi) * words;
            const float pos = delta / epsilon, neg = (1.0f - delta) / (1.0f - epsilon);
            float ratio = 1.0f;
            uint32_t inl = 0, tested = 0;
            bool pass = true;
            for (uint32_t i = 0; i < init_n; i++) {
                tested++;
                if ((row[i >> 5] >> (i & 31)) & 1u) { inl++; ratio *= pos; }
                else ratio *= neg;
                if (ratio > cfg->likelihood_ratio_threshold) { pass = false; break; }
            }
            if (pass) {
                Hyp hy; hy.m = poses_host[(size_t)h * MM + mi]; hy.inliers = inl; hy.mask.assign(nwords, 0u);
                for (uint32_t w = 0; w < words; w++) hy.mask[w] = row[w];
                H.push_back(std::move(hy));
                if (inl > best_inliers) {
                    best_inliers = inl;
                    const float e = (float)inl / (float)init_n;
                    if (e > epsilon && e < 1.0f) epsilon = e; else if (e >= 1.0f) epsilon = 0.999f;
                }
            } else {
                rej_inliers += inl; rej_tested += tested;
                const float d = (float)rej_inliers / (float)rej_tested;
                if (d > 0.0f && d < epsilon) delta = d;
            }
        }
    sort_hyps(H);
    if (H.size() > cfg->max_candidate_hypotheses) H.resize(cfg->max_candidate_hypotheses);
    // the surviving candidates are scored on the remaining data in one launch
    if (init_n < n && !H.empty()) {
        std::vector<cvb_pose> surv(H.size());
        for (size_t i = 0; i < H.size(); i++) surv[i] = H[i].m;
        if ((rc = upload(ctx, g->poses, surv.data(), sizeof(cvb_pose) * surv.size()))) return rc;
        if ((rc = masks_dev(ctx, kind, (const cvb_pose *)g->poses.p, (uint32_t)surv.size(), init_n, n, thr, masks, &words))) return rc;
        for (size_t i = 0; i < H.size(); i++) {
            const uint32_t *row = masks.data() + i * words;
            for (uint32_t j = init_n; j < n; j++)
                if ((row[(j - init_n) >> 5] >> ((j - init_n) & 31)) & 1u) H[i].mask[j >> 5] |= 1u << (j & 31);
        }
    }
    sort_hyps(H);
    if (H.size() > cfg->max_candidate_hypotheses) H.resize(cfg->max_candidate_hypotheses);
    // ---- main loop over further blocks
    std::vector<uint32_t> pool, idx((size_t)std::max<uint32_t>(cfg->estimations_per_block, 1) * K);
    for (uint32_t start = init_n; start < n && H.size() > 1; start += cfg->block_size) {
        const uint32_t end = std::min<uint32_t>(start + cfg->block_size, n);
        for (Hyp &h : H) h.inliers += popc_range(h.mask.data(), start, end);
        sort_hyps(H);
        H.resize(std::max<size_t>(H.size() / 2, 1));
        pool.clear();
        for (uint32_t i = 0; i < end; i++)
            if ((H[0].mask[i >> 5] >> (i & 31)) & 1u) pool.push_back(i);
        if (pool.size() >= K && cfg->estimations_per_block > 0) {
            const uint32_t worst = H.back().inliers;
            const uint32_t G = cfg->estimations_per_block;
            for (uint32_t gi = 0; gi < G; gi++) {
                uint32_t loc[8];
                populate_samples(rng, K, (uint32_t)pool.size(), loc);   // K <= 8
                for (uint32_t k = 0; k < K; k++) idx[(size_t)gi * K + k] = pool[loc[k]];
            }
            if ((rc = estimate_dev(ctx, kind, idx.data(), G, nposes, row0))) return rc;
            if ((rc = masks_dev(ctx, kind, (const cvb_pose *)g->poses.p, G * MM, 0, n, thr, masks, &words))) return rc;
            poses_host.resize((size_t)G * MM);
            CVB_CUDA(ctx, cudaMemcpy(poses_host.data(), g->poses.p, sizeof(cvb_pose) * MM * (size_t)G, cudaMemcpyDeviceToHost));
            for (uint32_t gi = 0; gi < G; gi++)
                for (uint32_t mi = 0; mi < nposes[gi]; mi++) {
                    const uint32_t *row = masks.data() + ((size_t)gi * MM + mi) * words;
                    const uint32_t inl = popc_range(row, 0, end);
                    if (inl > worst) {
                        Hyp hy; hy.m = poses_host[(size_t)gi * MM + mi]; hy.inliers = inl; hy.mask.assign(row, row + words);
                        H.push_back(std::move(hy));
                    }
                }
            sort_hyps(H);
            if (H.size() > cfg->max_candidate_hypotheses) H.resize(cfg->max_candidate_hypotheses);
        }
    }
    if (H.empty()) return 0;
    sort_hyps(H);
    *model_out = H[0].m;
    uint32_t c = 0;
    for (uint32_t i = 0; i < n; i++)
        if ((H[0].mask[i >> 5] >> (i & 31)) & 1u) { if (inliers_out && c < cap) inliers_out[c] = i; c++; }
    if (n_inliers) *n_inliers = c;
    *found = 1;
    (void)nwords;
    if (inliers_out && c > cap) return cvb_set_error(ctx, CVB_ECAP, "inlier capacity %u too small (%u needed)", cap, c);
    return 0;
}


// ---- device-resident ARRSAC driver (kernels: arrsac_dev.cuh).  Enqueues everything on the context stream and returns;
// no host synchronisation between the first kernel and the result.
#define ARS_SNAP 4096u
ArsWorkspace *arsws(cvb_ctx *ctx) {
    GeomWorkspace *g = gws(ctx);
    if (!g->ars) g->ars = new ArsWorkspace();
    return g->ars;
}

// B independent problems in one set of launches (arrsac_dev.cuh: problem pb = blockIdx.x of the one-CTA kernels, blockIdx.y of the
// grids).  Problem pb reads rows [pb * nmax, pb * nmax + min(n, nmax)) of a_dev / b_dev with n = n_dev[pb] (n_host when n_dev is
// NULL), draws from its own generator rngs[pb] and writes model_dev[pb], inl_dev[pb * cap ..], ninl_dev[pb], found_dev[pb].
// `batch` records which commit entry owns the run (B = 1 through the single entry is that entry's run, launch for launch).
int arrsac_run_dev_batch(cvb_ctx *ctx, const cvb_arrsac_cfg *cfg, int kind, const double *a_dev, const double *b_dev, const uint32_t *n_dev,
                         uint32_t n_host, uint32_t nmax, uint32_t B, const cvb_rng *rngs, cvb_pose *model_dev, uint32_t *inl_dev, uint32_t cap,
                         uint32_t *ninl_dev, int32_t *found_dev, int row0, bool batch) {
    if (cfg->block_size == 0 || cfg->initialization_blocks == 0) return cvb_set_error(ctx, CVB_EINVAL, "block_size / initialization_blocks must be > 0");
    ArrsacParams P;
    memset(&P, 0, sizeof(P));
    P.K = kind_K(kind); P.MM = kind_M(kind); P.kind = (uint32_t)kind;
    P.H0 = cfg->initialization_hypotheses; P.ib = cfg->initialization_blocks; P.bs = cfg->block_size;
    P.max_cand = cfg->max_candidate_hypotheses; P.G = cfg->estimations_per_block;
    P.NMAX = std::max<uint32_t>(nmax, 1);
    P.W0 = cdiv(P.bs * P.ib, 32); P.NW = cdiv(P.NMAX, 32);
    P.rows = P.max_cand + P.G * P.MM;
    P.lr_thr = cfg->likelihood_ratio_threshold; P.eps0 = cfg->initial_epsilon; P.delta0 = cfg->initial_delta;
    P.thr = cfg->inlier_threshold; P.row0 = row0;
    // two-stage initial scoring only where a predicate is expensive (CameraToCamera residual); CVB_ARS_EAGER=1 scores everything up front
    { const char *env = getenv("CVB_ARS_EAGER"); const bool eager = (env && env[0] == '1') || kind_res(kind) == 1;
      P.prefix = eager ? P.H0 : std::min<uint32_t>(P.H0, 64); P.cmin = 2;
      if (const char *cm = getenv("CVB_ARS_CMIN")) P.cmin = (uint32_t)std::max(0, atoi(cm)); }
    // early rejection in the block scoring (arrsac_dev.cuh, k_ars_score phase 1); CVB_ARS_EARLY_REJECT=0 scores every word
    { const char *e = getenv("CVB_ARS_EARLY_REJECT"); P.early = (e && e[0] == '0') ? 0u : 1u; }
    if (P.max_cand == 0 || P.rows > ARS_SORT_CAP)
        return cvb_set_error(ctx, CVB_EUNSUPPORTED, "max_candidate_hypotheses + estimations_per_block * %u must be in 1..%u", P.MM, ARS_SORT_CAP);
    if ((uint64_t)P.bs * P.ib + 1 > 2ull * ARS_SORT_CAP) return cvb_set_error(ctx, CVB_EUNSUPPORTED, "block_size * initialization_blocks too large");
    if (P.NMAX >= (1u << 20)) return cvb_set_error(ctx, CVB_EUNSUPPORTED, "more than 2^20 data");
    ArsWorkspace *w = arsws(ctx);
    const uint32_t nb_max = cdiv(P.NMAX, P.bs) + 1;
    const uint32_t nraw = P.H0 * P.K + P.H0 * P.K / 4 + 64 + nb_max * (P.G * P.K + P.G * P.K / 4 + 64);
    P.nraw = nraw; P.qcap = ARS_QCAP / B; P.sdata = nmax;
    const ArsStrides S = ars_strides(P);
    int rc;
    // B slices of every buffer (ars_strides); the queue keeps its size, split between the problems
    if ((rc = w->ctl.ensure(ctx, sizeof(ArrsacCtl) * B + 16))) return rc;
    if ((rc = w->raw.ensure(ctx, sizeof(uint32_t) * (size_t)nraw * B))) return rc;
    if ((rc = w->samples0.ensure(ctx, sizeof(uint32_t) * S.samples0 * B))) return rc;
    if ((rc = w->poses0.ensure(ctx, sizeof(cvb_pose) * S.models0 * B))) return rc;
    if ((rc = w->nposes0.ensure(ctx, S.nposes0 * B))) return rc;
    if ((rc = w->masks0.ensure(ctx, sizeof(uint32_t) * S.models0 * P.W0 * B))) return rc;
    if ((rc = w->vm.ensure(ctx, sizeof(uint32_t) * S.vm * B))) return rc;
    if ((rc = w->pass_id.ensure(ctx, sizeof(uint32_t) * S.models0 * B))) return rc;
    if ((rc = w->pass_inl.ensure(ctx, sizeof(uint32_t) * S.models0 * B))) return rc;
    if ((rc = w->tposes.ensure(ctx, sizeof(cvb_pose) * S.rows2 * B))) return rc;
    if ((rc = w->tinl.ensure(ctx, sizeof(uint32_t) * S.rows2 * B))) return rc;
    if ((rc = w->tmasks.ensure(ctx, sizeof(uint32_t) * S.tmasks * B))) return rc;
    if ((rc = w->newposes.ensure(ctx, sizeof(cvb_pose) * S.nnew * B))) return rc;
    if ((rc = w->nposes_new.ensure(ctx, S.nposes_new * B))) return rc;
    if ((rc = w->newmask.ensure(ctx, sizeof(uint32_t) * S.newmask * B))) return rc;
    if ((rc = w->nout.ensure(ctx, sizeof(uint32_t) * S.nnew * B))) return rc;
    if ((rc = w->pool.ensure(ctx, sizeof(uint32_t) * (size_t)P.NMAX * B))) return rc;
    if ((rc = w->samples_new.ensure(ctx, sizeof(uint32_t) * S.samples_new * B))) return rc;
    if ((rc = w->queue.ensure(ctx, sizeof(uint2) * 2 * (size_t)ARS_QCAP))) return rc;
    // page-locked staging: [B ArrsacCtl headers | batch header (live count) | B raw-draw streams]
    const size_t ctl_bytes = sizeof(ArrsacCtl) * B + 16;
    const size_t hdr = (ctl_bytes + 15) / 16 * 16, stage_bytes = hdr + sizeof(uint32_t) * (size_t)nraw * B;
    if (w->h_raw_cap < stage_bytes) {
        if (w->h_raw) { cvb_wait(ctx, ctx->stream); cudaFreeHost(w->h_raw); w->h_raw = nullptr; w->h_raw_cap = 0; }
        if (cudaHostAlloc((void **)&w->h_raw, stage_bytes, cudaHostAllocDefault) != cudaSuccess) return cvb_set_error(ctx, CVB_ENOMEM, "page-locked staging");
        w->h_raw_cap = stage_bytes;
    }
    const size_t res_bytes = sizeof(ArrsacCtl) * B + sizeof(cvb_pose) + 64;
    if (w->h_res_cap < res_bytes) {
        if (w->h_res) { cvb_wait(ctx, ctx->stream); cudaFreeHost(w->h_res); w->h_res = nullptr; w->h_res_cap = 0; }
        if (cudaHostAlloc((void **)&w->h_res, res_bytes, cudaHostAllocDefault) != cudaSuccess) return cvb_set_error(ctx, CVB_ENOMEM, "page-locked staging");
        w->h_res_cap = res_bytes;
    }
    if (!w->up_done) CVB_CUDA(ctx, cudaEventCreateWithFlags(&w->up_done, cudaEventDisableTiming | cudaEventBlockingSync));
    else CVB_CUDA(ctx, cudaEventSynchronize(w->up_done));       // previous upload has left the staging buffer
    {
        w->nsnap = cdiv(nraw, ARS_SNAP);
        w->snaps.resize((size_t)w->nsnap * B);
        memset(w->h_raw, 0, hdr);
        for (uint32_t pb = 0; pb < B; pb++) {
            cvb_rng g = rngs[pb];
            uint32_t *raw = (uint32_t *)((unsigned char *)w->h_raw + hdr) + (size_t)pb * nraw;
            for (uint32_t i = 0; i < nraw; i++) {
                if (i % ARS_SNAP == 0) w->snaps[(size_t)pb * w->nsnap + i / ARS_SNAP] = g;
                raw[i] = cvb_rng_next_u32(&g);
            }
            ArrsacCtl *h = (ArrsacCtl *)w->h_raw + pb;
            h->nraw = nraw; h->gen = g; h->gen_pos = nraw; h->rng_pos = 0;
        }
        *(uint32_t *)((unsigned char *)w->h_raw + sizeof(ArrsacCtl) * B) = B;     // live problems
        w->nraw = nraw; w->B = B;
    }
    cudaStream_t st = ctx->stream;
    static bool attr_set = false;
    if (!attr_set) {
        cudaFuncSetAttribute(k_ars_book, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ARS_BOOK_SMEM);
        cudaFuncSetAttribute(k_ars_sprt<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024);
        cudaFuncSetAttribute(k_ars_sprt<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024);
        cudaFuncSetAttribute(k_ars_score<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        cudaFuncSetAttribute(k_ars_score<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        attr_set = true;
    }
    bool capturing = false, while_loop = false;
    uint32_t body_launches = 0;
    // everything the stream sees, from the upload of the draw stream to the copy of the control block back
    auto enqueue = [&]() -> int {
        CVB_CUDA(ctx, cudaMemcpyAsync(w->ctl.p, w->h_raw, ctl_bytes, cudaMemcpyHostToDevice, st));
        CVB_CUDA(ctx, cudaMemcpyAsync(w->raw.p, (unsigned char *)w->h_raw + hdr, sizeof(uint32_t) * (size_t)nraw * B, cudaMemcpyHostToDevice, st));
        if (!capturing) CVB_CUDA(ctx, cudaEventRecord(w->up_done, st));      // eager: the staging buffer is free as soon as the two copies are done
        ArrsacCtl *ctl = (ArrsacCtl *)w->ctl.p;
        uint32_t *live = (uint32_t *)((unsigned char *)w->ctl.p + sizeof(ArrsacCtl) * B);
        const uint32_t *raw = (const uint32_t *)w->raw.p;
        const int res = kind_res(kind);
        {
            CVB_PROF(ctx, "k_ars_begin", 0);
            k_ars_begin<<<B, ARS_BOOK_NT, 0, st>>>(ctl, P, n_dev, n_host, raw, (uint32_t *)w->samples0.p);
            CVB_LAUNCH_CHECK(ctx);
        }
        auto estimate = [&](int phase, uint32_t H, const uint32_t *samples, cvb_pose *poses, uint8_t *nposes) -> int {
            if (H == 0) return 0;
            CVB_PROF(ctx, phase == 0 ? "k_ars_estimate_init" : "k_ars_estimate_block", 0);
            // the big initial batch is bound by FP64 issue (4 lanes per hypothesis waste the fewest slots); a block's 64 hypotheses
            // are a latency chain in front of the next scoring (16 lanes: the shortest chain)
            // (8 lanes, or 16 lanes at 64 registers, measured the same 0.137-0.140 ms for the initial batch)
            if (kind == 0 && phase == 0) k_ars_estimate8<4, 5><<<dim3(cdiv(H, 128 / 4), B), 128, 0, st>>>(ctl, phase, H, a_dev, b_dev, samples, poses, nposes, P);
            else if (kind == 0) k_ars_estimate8<16, 5><<<dim3(cdiv(H, 128 / 16), B), 128, 0, st>>>(ctl, phase, H, a_dev, b_dev, samples, poses, nposes, P);
            else if (kind == 1) k_ars_estimate<1><<<dim3(cdiv(H, 128), B), 128, 0, st>>>(ctl, phase, H, a_dev, b_dev, samples, poses, nposes, row0, P);
            else k_ars_estimate<2><<<dim3(cdiv(H, 128), B), 128, 0, st>>>(ctl, phase, H, a_dev, b_dev, samples, poses, nposes, row0, P);
            CVB_LAUNCH_CHECK(ctx);
            return 0;
        };
        // the initial scoring fills the machine (4 CTAs per SM).  A block scores ~200 k predicates on 48 CTAs: a larger grid
    // lowers ONE context's latency, but with 16 pipelined contexts the small grid costs the least SM time (more units per warp, the
    // exact-fallback stragglers amortised), and the step is bound by SM time, not by a pair's latency.  Re-tuned on one H100 80GB
    // HBM3 (700 W) with early rejection in the block scoring: 24 / 32 / 48 / 66 / 132 CTAs gave 1 585 / 1 559-1 598 / 1 583-1 597 /
    // 1 540-1 590 / 1 582-1 589 frames/s in the pipelined bench (two runs each), all inside the run-to-run spread, so 48 stays.
    // CVB_ARS_SGRID overrides.
    const uint32_t sgrid_full = (uint32_t)ctx->num_sms * 4;
        uint32_t sgrid_block = 48;
        if (const char *e = getenv("CVB_ARS_SGRID")) sgrid_block = (uint32_t)std::max(1, atoi(e));
        // CVB_ARS_SCORE_SMEM: unused dynamic shared memory per scoring CTA, a residency limiter.  The kernel needs 128 registers per
        // thread, so two CTAs take an SM's whole register file and nothing of another context can run beside them although they
        // only use the FP64 pipe; > half of the SM's shared memory leaves one CTA per SM and half the registers to other kernels.
        size_t score_smem = 0;
        if (const char *e = getenv("CVB_ARS_SCORE_SMEM")) score_smem = (size_t)std::max(0, atoi(e));
        auto score = [&](int phase) -> int {
            const uint32_t sgrid = phase == 1 ? sgrid_block : sgrid_full;
            CVB_PROF(ctx, phase == 1 ? "k_ars_score_block" : "k_ars_score_init", 0);
            if (res == 0)
                k_ars_score<0><<<dim3(sgrid, B), 256, score_smem, st>>>(ctl, (uint2 *)w->queue.p, P, phase, a_dev, b_dev, (const cvb_pose *)w->poses0.p, (const uint8_t *)w->nposes0.p,
                                                      (uint32_t *)w->masks0.p, (const cvb_pose *)w->tposes.p, (uint32_t *)w->tmasks.p,
                                                      (const cvb_pose *)w->newposes.p, (const uint8_t *)w->nposes_new.p, (uint32_t *)w->newmask.p,
                                                      (uint32_t *)w->nout.p);
            else
                k_ars_score<1><<<dim3(sgrid, B), 256, score_smem, st>>>(ctl, (uint2 *)w->queue.p, P, phase, a_dev, b_dev, (const cvb_pose *)w->poses0.p, (const uint8_t *)w->nposes0.p,
                                                      (uint32_t *)w->masks0.p, (const cvb_pose *)w->tposes.p, (uint32_t *)w->tmasks.p,
                                                      (const cvb_pose *)w->newposes.p, (const uint8_t *)w->nposes_new.p, (uint32_t *)w->newmask.p,
                                                      (uint32_t *)w->nout.p);
            CVB_LAUNCH_CHECK(ctx);
            return 0;
        };
        if ((rc = estimate(0, P.H0, (const uint32_t *)w->samples0.p, (cvb_pose *)w->poses0.p, (uint8_t *)w->nposes0.p))) return rc;
        auto resolve = [&](int stage) -> int {
            CVB_PROF(ctx, "k_ars_resolve", 0);
            k_ars_resolve<<<dim3(sgrid_full, B), 256, 0, st>>>(ctl, (const uint2 *)w->queue.p, stage, P, a_dev, b_dev, (const cvb_pose *)w->poses0.p, (uint32_t *)w->masks0.p);
            CVB_LAUNCH_CHECK(ctx);
            return 0;
        };
        if ((rc = score(0))) return rc;
        if (res == 0 && (rc = resolve(0))) return rc;
        if (P.prefix < P.H0 && P.W0 > 1) {
            if ((rc = score(2))) return rc;
            if (res == 0 && (rc = resolve(1))) return rc;
        }
        {
            CVB_PROF(ctx, "k_ars_sprt", 0);
            if (res == 0)
                k_ars_sprt<0><<<B, ARS_BOOK_NT, 8 * ARS_SORT_CAP, st>>>(ctl, P, a_dev, b_dev, (const cvb_pose *)w->poses0.p, (const uint8_t *)w->nposes0.p, (uint32_t *)w->masks0.p,
                                                        (uint32_t *)w->vm.p, (uint32_t *)w->pass_id.p, (uint32_t *)w->pass_inl.p, (cvb_pose *)w->tposes.p,
                                                        (uint32_t *)w->tinl.p, (uint32_t *)w->tmasks.p);
            else
                k_ars_sprt<1><<<B, ARS_BOOK_NT, 8 * ARS_SORT_CAP, st>>>(ctl, P, a_dev, b_dev, (const cvb_pose *)w->poses0.p, (const uint8_t *)w->nposes0.p, (uint32_t *)w->masks0.p,
                                                        (uint32_t *)w->vm.p, (uint32_t *)w->pass_id.p, (uint32_t *)w->pass_inl.p, (cvb_pose *)w->tposes.p,
                                                        (uint32_t *)w->tinl.p, (uint32_t *)w->tmasks.p);
            CVB_LAUNCH_CHECK(ctx);
        }
        // block loop: the number of launches follows the data count when the host knows it, the capacity otherwise;
        // kernels behind the loop's end return at once (ctl->done)
        const uint32_t n_bound = n_dev ? P.NMAX : std::min(n_host, P.NMAX);
        const uint32_t init_n = std::min(P.bs * P.ib, n_bound);
        const uint32_t nb = n_bound > init_n ? cdiv(n_bound - init_n, P.bs) : 0;
        auto book = [&](unsigned long long cond) -> int {
            CVB_PROF(ctx, "k_ars_book", 0);
            k_ars_book<<<B, ARS_BOOK_NT, ARS_BOOK_SMEM, st>>>(ctl, P, raw, (cvb_pose *)w->tposes.p, (uint32_t *)w->tinl.p, (uint32_t *)w->tmasks.p,
                                                              (const cvb_pose *)w->newposes.p, (const uint8_t *)w->nposes_new.p,
                                                              (const uint32_t *)w->newmask.p, (uint32_t *)w->pool.p, (uint32_t *)w->samples_new.p,
                                                              (uint32_t *)w->nout.p, live, cond);
            CVB_LAUNCH_CHECK(ctx);
            return 0;
        };
        // a block's score, the exact evaluation of the predicates it queued (CameraToCamera only), its bookkeeping
        auto score_block = [&](unsigned long long cond) -> int {
            if ((rc = score(1))) return rc;
            if (res == 0) {
                CVB_PROF(ctx, "k_ars_resolve_block", 0);
                // 64-thread CTAs: a block queues a small fraction of its predicates, spread over as many SMs as possible
                k_ars_resolve_block<<<dim3(sgrid_full, B), 64, 0, st>>>(ctl, (const uint2 *)w->queue.p, P, a_dev, b_dev, (const cvb_pose *)w->tposes.p,
                                                               (uint32_t *)w->tmasks.p, (const cvb_pose *)w->newposes.p, (uint32_t *)w->newmask.p);
                CVB_LAUNCH_CHECK(ctx);
            }
            return book(cond);
        };
        if (capturing && while_loop) {
            // device-side loop: one WHILE node whose body is one block iteration; k_ars_book ends it (block nb at the latest: lo >= n)
            cudaStreamCaptureStatus cs;
            cudaGraph_t g = nullptr;
            const cudaGraphNode_t *deps = nullptr;
            size_t ndeps = 0;
            CVB_CUDA(ctx, cudaStreamGetCaptureInfo(st, &cs, nullptr, &g, &deps, &ndeps));
            cudaGraphConditionalHandle cond;
            CVB_CUDA(ctx, cudaGraphConditionalHandleCreate(&cond, g, 1, cudaGraphCondAssignDefault));
            cudaGraphNodeParams np = {cudaGraphNodeTypeConditional};
            np.conditional.handle = cond;
            np.conditional.type = cudaGraphCondTypeWhile;
            np.conditional.size = 1;
            cudaGraphNode_t node;
            CVB_CUDA(ctx, cudaGraphAddNode(&node, g, deps, ndeps, &np));
            cudaGraph_t body = np.conditional.phGraph_out[0];
            const cudaStream_t outer = st;
            CVB_CUDA(ctx, cudaStreamBeginCaptureToGraph(w->body_stream, body, nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal));
            st = w->body_stream;                     // the launch helpers below capture into the body (restored before any return)
            const uint64_t b0 = ctx->launches;
            rc = score_block(cond);
            if (!rc && nb && P.G) rc = estimate(1, P.G, (const uint32_t *)w->samples_new.p, (cvb_pose *)w->newposes.p, (uint8_t *)w->nposes_new.p);
            body_launches = (uint32_t)(ctx->launches - b0);
            cudaGraph_t same_body = nullptr;
            const cudaError_t be = cudaStreamEndCapture(st, &same_body);
            st = outer;
            if (rc) return rc;
            CVB_CUDA(ctx, be);
            CVB_CUDA(ctx, cudaStreamUpdateCaptureDependencies(st, &node, 1, cudaStreamSetCaptureDependencies));
        } else
        for (uint32_t it = 0; it <= nb; it++) {
            if ((rc = score_block(0))) return rc;
            if (it < nb && P.G)
                if ((rc = estimate(1, P.G, (const uint32_t *)w->samples_new.p, (cvb_pose *)w->newposes.p, (uint8_t *)w->nposes_new.p))) return rc;
        }
        {
            CVB_PROF(ctx, "k_ars_final", 0);
            if (res == 0) k_ars_final<0><<<B, ARS_BOOK_NT, 0, st>>>(ctl, P, a_dev, b_dev, model_dev, inl_dev, cap, ninl_dev, found_dev);
            else k_ars_final<1><<<B, ARS_BOOK_NT, 0, st>>>(ctl, P, a_dev, b_dev, model_dev, inl_dev, cap, ninl_dev, found_dev);
            CVB_LAUNCH_CHECK(ctx);
        }
        CVB_CUDA(ctx, cudaMemcpyAsync(w->h_res, w->ctl.p, sizeof(ArrsacCtl) * B, cudaMemcpyDeviceToHost, st));
        return 0;
    };
    if (w->use_graph < 0) {
        const char *e1 = getenv("CVB_NO_GRAPH"), *e2 = getenv("CVB_ARS_NO_GRAPH");
        w->use_graph = ((e1 && e1[0] == '1') || (e2 && e2[0] == '1')) ? 0 : 1;
    }
    if (!w->use_graph || ctx->prof) {
        if ((rc = enqueue())) return rc;
        w->pending = true; w->pending_batch = batch;
        return 0;
    }
    ArsWorkspace::GraphKey key;
    memset(&key, 0, sizeof(key));
    key.P = P; key.kind = kind; key.row0 = row0; key.a = a_dev; key.b = b_dev; key.n_dev = n_dev; key.n_host = n_host; key.nmax = nmax; key.cap = cap; key.B = B;
    key.model = model_dev; key.inl = inl_dev; key.ninl = ninl_dev; key.found = found_dev;
    {
        const DevBuf *bufs[] = {&w->ctl, &w->raw, &w->samples0, &w->poses0, &w->nposes0, &w->masks0, &w->vm, &w->pass_id, &w->pass_inl, &w->tposes,
                                &w->tinl, &w->tmasks, &w->newposes, &w->nposes_new, &w->newmask, &w->nout, &w->pool, &w->samples_new, &w->queue};
        int i = 0;
        for (const DevBuf *d : bufs) key.ws[i++] = d->p;
        key.ws[i++] = w->h_raw; key.ws[i++] = w->h_res; key.ws[i++] = (const void *)(uintptr_t)nraw;
    }
    auto same = [](const ArsWorkspace::GraphKey &x, const ArsWorkspace::GraphKey &y) { return memcmp(&x, &y, sizeof(x)) == 0; };
    for (auto &ge : w->graphs)
        if (same(ge.key, key)) {
            CVB_CUDA(ctx, cudaGraphLaunch(ge.exec, st));
            CVB_CUDA(ctx, cudaEventRecord(w->up_done, st));       // replay: the staging buffer is free when the run is over
            ctx->launches += ge.launches;
            w->last_body = ge.body;
            w->pending = true; w->pending_batch = batch;
            return 0;
        }
    bool seen = false;
    for (auto &k : w->seen) seen = seen || same(k, key);
    if (!seen) {                                                   // first time: run eagerly, capture if it comes back
        if (w->seen.size() >= 64) w->seen.erase(w->seen.begin());
        w->seen.push_back(key);
        if ((rc = enqueue())) return rc;
        w->pending = true; w->pending_batch = batch;
        return 0;
    }
    const uint64_t l0 = ctx->launches;
    if (w->use_while < 0) {
        const char *e = getenv("CVB_ARS_WHILE");
        w->use_while = (e && e[0] == '0') ? 0 : 1;
    }
    if (w->use_while && !w->body_stream && cudaStreamCreateWithFlags(&w->body_stream, cudaStreamNonBlocking) != cudaSuccess) {
        cudaGetLastError();
        w->use_while = 0;
    }
    cudaGraphExec_t exec = nullptr;
    cudaError_t ce = cudaSuccess;
    for (int attempt = 0; attempt < 2 && !exec; attempt++) {
        ctx->launches = l0;
        capturing = true;
        while_loop = w->use_while != 0;
        CVB_CUDA(ctx, cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
        rc = enqueue();
        cudaGraph_t graph = nullptr;
        ce = cudaStreamEndCapture(st, &graph);
        capturing = false;
        if (!rc && ce == cudaSuccess && graph) ce = cudaGraphInstantiate(&exec, graph, 0);
        if (graph) cudaGraphDestroy(graph);
        if (exec || !while_loop) break;
        cudaGetLastError();                                        // the WHILE node is not available: capture the unrolled loop instead
        w->use_while = 0;
        exec = nullptr;
    }
    if (rc) return rc;
    if (ce != cudaSuccess || !exec) {                              // capture not possible: eager from now on
        cudaGetLastError();
        w->use_graph = 0;
        ctx->launches = l0;
        if ((rc = enqueue())) return rc;
        w->pending = true; w->pending_batch = batch;
        return 0;
    }
    if (w->graphs.size() >= 16) { cudaGraphExecDestroy(w->graphs.front().exec); w->graphs.erase(w->graphs.begin()); }
    w->graphs.push_back({key, exec, ctx->launches - l0, while_loop ? body_launches : 0u});
    w->last_body = while_loop ? body_launches : 0u;
    CVB_CUDA(ctx, cudaGraphLaunch(exec, st));
    CVB_CUDA(ctx, cudaEventRecord(w->up_done, st));
    w->pending = true; w->pending_batch = batch;
    return 0;
}

int arrsac_run_dev(cvb_ctx *ctx, const cvb_arrsac_cfg *cfg, int kind, const double *a_dev, const double *b_dev, const uint32_t *n_dev,
                   uint32_t n_host, uint32_t nmax, const cvb_rng *rng, cvb_pose *model_dev, uint32_t *inl_dev, uint32_t cap,
                   uint32_t *ninl_dev, int32_t *found_dev, int row0) {
    return arrsac_run_dev_batch(ctx, cfg, kind, a_dev, b_dev, n_dev, n_host, nmax, 1, rng, model_dev, inl_dev, cap, ninl_dev, found_dev, row0, false);
}

// after the stream has drained: advance the caller's generator by the draws the run consumed (state in == state the
// reference would hold after model_inliers).  rngs / stats_out: one per problem of the pending run (B of them); `batch` must match
// the entry that started the run, so a run is never committed as the other kind.
int arrsac_commit_rng_batch(cvb_ctx *ctx, cvb_rng *rngs, uint32_t B, ArrsacCtl *stats_out, bool batch) {
    ArsWorkspace *w = arsws(ctx);
    if (!w->pending) return cvb_set_error(ctx, CVB_EINVAL, "no device ARRSAC run to commit");
    if (w->pending_batch != batch)
        return cvb_set_error(ctx, CVB_EINVAL, batch ? "the pending ARRSAC run is a single run: commit it with cvb_arrsac_commit_rng"
                                                    : "the pending ARRSAC run is a batch: commit it with cvb_arrsac_commit_rng_batch");
    if (B != w->B) return cvb_set_error(ctx, CVB_EINVAL, "the pending ARRSAC run has %u problems, not %u", w->B, B);
    const ArrsacCtl *hs = (const ArrsacCtl *)w->h_res;
    if (stats_out) memcpy(stats_out, hs, sizeof(ArrsacCtl) * B);
    if (getenv("CVB_ARS_DEBUG"))
        for (uint32_t pb = 0; pb < B; pb++) {
            const ArrsacCtl *h = hs + pb;
            fprintf(stderr, "[arrsac] n %u models %u pass %u chunks %u turns %u repairs %u lazy %u | sprt us: order %u walk %u commit %u | block iterations %u"
                    " | undecided predicates queued: initial %u block %u | block units: kept %u new %u skipped %u | blocks worst0 %u bar<32 %u not estimated %u\n",
                    h->n, h->Mv, h->npass, h->stat_chunks, h->stat_turns, h->stat_repairs, h->stat_lazy, h->stat_perm_us, h->stat_walk_us,
                    h->stat_commit_us, h->iters, h->q_count + h->q_count2, h->stat_qblk, h->stat_units_kept, h->stat_units_new, h->stat_skip,
                    h->stat_blk_w0, h->stat_blk_lt32, h->stat_blk_bar0);
        }
    // the WHILE body ran (most block iterations of any problem) + 1 times, the capture counted it once
    uint32_t iters = 0;
    for (uint32_t pb = 0; pb < B; pb++) iters = std::max(iters, hs[pb].iters);
    ctx->launches += (uint64_t)w->last_body * iters;
    w->last_body = 0;
    w->pending = false;
    if (!rngs) return 0;
    // every problem is checked before any generator is written: an error leaves all of them where they were
    for (uint32_t pb = 0; pb < B; pb++)
        if (hs[pb].rng_pos >= w->nraw && hs[pb].gen_pos != std::max<uint64_t>(hs[pb].rng_pos, w->nraw))
            return cvb_set_error(ctx, CVB_ECUDA, "generator position mismatch (problem %u)", pb);
    for (uint32_t pb = 0; pb < B; pb++) {
        const uint64_t used = hs[pb].rng_pos;
        if (used >= w->nraw) { rngs[pb] = hs[pb].gen; continue; }
        cvb_rng g = w->snaps[(size_t)pb * w->nsnap + used / ARS_SNAP];
        for (uint64_t i = used / ARS_SNAP * ARS_SNAP; i < used; i++) cvb_rng_next_u32(&g);
        rngs[pb] = g;
    }
    return 0;
}
// the 16 statistics words of cvb_arrsac_commit_rng (13..15 reserved): n, valid initial models, SPRT passes, SPRT commit rounds, block
// iterations, draws, inliers, found, 32-datum units scored in stage 1 / stage 2, predicates resolved exactly from the queues, mask
// words computed by the SPRT itself, SPRT repairs
void arrsac_stats_words(const ArrsacCtl &h, uint32_t *o) {
    o[0] = h.n; o[1] = h.Mv; o[2] = h.npass; o[3] = h.stat_chunks; o[4] = h.iters;
    o[5] = (uint32_t)h.rng_pos; o[6] = h.n_inliers; o[7] = h.found;
    o[8] = h.stat_units0; o[9] = h.stat_units2; o[10] = h.q_count + h.q_count2; o[11] = h.stat_lazy;
    o[12] = h.stat_repairs; o[13] = h.stat_pad /* data walked by the box walks */; o[14] = h.stat_walk_us; o[15] = h.stat_commit_us;
}

int arrsac_commit_rng(cvb_ctx *ctx, cvb_rng *rng, ArrsacCtl *stats_out = nullptr) {
    return arrsac_commit_rng_batch(ctx, rng, 1, stats_out, false);
}

// host-pointer entry: upload, run on the device, one synchronisation at the end
int arrsac_host(cvb_ctx *ctx, const cvb_arrsac_cfg *cfg, int kind, const double *a, const double *b, uint32_t n, cvb_rng *rng,
                cvb_pose *model_out, uint32_t *inliers_out, uint32_t cap, uint32_t *n_inliers, int32_t *found, int row0 = 5) {
    *found = 0;
    if (n_inliers) *n_inliers = 0;
    if (n < kind_K(kind) || cfg->initialization_hypotheses == 0) return 0;
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    int rc = upload_data(ctx, kind, a, b, n);
    if (rc) return rc;
    GeomWorkspace *g = gws(ctx);
    ArsWorkspace *w = arsws(ctx);
    const size_t res_bytes = sizeof(cvb_pose) + 16 + sizeof(uint32_t) * (size_t)n;
    if ((rc = w->res.ensure(ctx, res_bytes))) return rc;
    unsigned char *rd = (unsigned char *)w->res.p;
    cvb_pose *model_dev = (cvb_pose *)rd;
    uint32_t *ninl_dev = (uint32_t *)(rd + sizeof(cvb_pose));
    int32_t *found_dev = (int32_t *)(rd + sizeof(cvb_pose) + 4);
    uint32_t *inl_dev = (uint32_t *)(rd + sizeof(cvb_pose) + 16);
    if ((rc = arrsac_run_dev(ctx, cfg, kind, (const double *)g->a.p, (const double *)g->b.p, nullptr, n, n, rng, model_dev, inl_dev, n, ninl_dev,
                             found_dev, row0))) return rc;
    unsigned char *hs = (unsigned char *)cvb_pinned(ctx, res_bytes);
    if (!hs) return cvb_set_error(ctx, CVB_ENOMEM, "page-locked scratch");
    CVB_CUDA(ctx, cudaMemcpyAsync(hs, rd, res_bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    if ((rc = arrsac_commit_rng(ctx, rng))) return rc;
    const uint32_t c = *(const uint32_t *)(hs + sizeof(cvb_pose));
    *found = *(const int32_t *)(hs + sizeof(cvb_pose) + 4);
    if (!*found) return 0;
    memcpy(model_out, hs, sizeof(cvb_pose));
    if (n_inliers) *n_inliers = c;
    if (inliers_out) memcpy(inliers_out, hs + sizeof(cvb_pose) + 16, sizeof(uint32_t) * std::min(c, cap));
    if (inliers_out && c > cap) return cvb_set_error(ctx, CVB_ECAP, "inlier capacity %u too small (%u needed)", cap, c);
    return 0;
}

bool arrsac_on_host() {     // CVB_ARRSAC_HOST=1: round-1 driver (bookkeeping on the host) kept for A/B tests
    const char *e = getenv("CVB_ARRSAC_HOST");
    return e && e[0] == '1';
}

int residuals_host(cvb_ctx *ctx, int kind, const cvb_pose *poses, uint32_t m, const double *a, const double *b, uint32_t n, double *out) {
    if (!ctx) return CVB_EINVAL;
    if ((m && !poses) || (n && (!a || !b)) || (m && n && !out)) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (m == 0 || n == 0) return 0;
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    int rc = upload_data(ctx, kind, a, b, n);
    if (rc) return rc;
    GeomWorkspace *g = gws(ctx);
    if ((rc = upload(ctx, g->poses, poses, sizeof(cvb_pose) * (size_t)m))) return rc;
    if ((rc = g->out.ensure(ctx, sizeof(double) * (size_t)m * n))) return rc;
    for (uint32_t p0 = 0; p0 < m; p0 += 65535) {
        const uint32_t pm = std::min<uint32_t>(65535, m - p0);
        dim3 grid(cdiv(n, 256), pm);
        CVB_PROF(ctx, kind == 0 ? "k_residuals_c2c" : "k_residuals_w2c", (kind == 0 ? 48.0 : 56.0) * pm * n);
        if (kind == 0)
            k_residuals<0, 0><<<grid, 256, 0, ctx->stream>>>((const cvb_pose *)g->poses.p + p0, pm, (const double *)g->a.p, (const double *)g->b.p, 0, n, 0.0,
                                                             (double *)g->out.p + (size_t)p0 * n, n, nullptr, 0);
        else
            k_residuals<1, 0><<<grid, 256, 0, ctx->stream>>>((const cvb_pose *)g->poses.p + p0, pm, (const double *)g->a.p, (const double *)g->b.p, 0, n, 0.0,
                                                             (double *)g->out.p + (size_t)p0 * n, n, nullptr, 0);
        CVB_LAUNCH_CHECK(ctx);
    }
    CVB_CUDA(ctx, cudaMemcpyAsync(out, g->out.p, sizeof(double) * (size_t)m * n, cudaMemcpyDeviceToHost, ctx->stream));
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    return 0;
}

int estimate_host(cvb_ctx *ctx, int kind, const double *a, const double *b, uint32_t n, const uint32_t *samples, uint32_t H,
                  cvb_pose *poses_out, uint8_t *nposes_out, int row0 = 5) {
    if (!ctx) return CVB_EINVAL;
    if (!a || !b || (H && (!samples || !poses_out || !nposes_out))) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (H == 0) return 0;
    const uint32_t K = kind_K(kind);
    for (size_t i = 0; i < (size_t)H * K; i++)
        if (samples[i] >= n) return cvb_set_error(ctx, CVB_EINVAL, "sample index %u out of range (n = %u)", samples[i], n);
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    int rc = upload_data(ctx, kind, a, b, n);
    if (rc) return rc;
    std::vector<uint8_t> np;
    if ((rc = estimate_dev(ctx, kind, samples, H, np, row0))) return rc;
    memcpy(nposes_out, np.data(), H);
    CVB_CUDA(ctx, cudaMemcpy(poses_out, gws(ctx)->poses.p, sizeof(cvb_pose) * kind_M(kind) * (size_t)H, cudaMemcpyDeviceToHost));
    return 0;
}

// poses (g->out) and per-problem update counts (g->ok) through page-locked scratch to the caller's (possibly pageable) arrays
int download_poses_updates(cvb_ctx *ctx, GeomWorkspace *g, cvb_pose *poses_out, size_t nposes, uint32_t *updates_out, uint32_t B) {
    const size_t pb = sizeof(cvb_pose) * nposes, ub = sizeof(uint32_t) * (size_t)B;
    unsigned char *hs = (unsigned char *)cvb_pinned(ctx, pb + ub);
    if (!hs) return cvb_set_error(ctx, CVB_ENOMEM, "page-locked scratch");
    CVB_CUDA(ctx, cudaMemcpyAsync(hs, g->out.p, pb, cudaMemcpyDeviceToHost, ctx->stream));
    CVB_CUDA(ctx, cudaMemcpyAsync(hs + pb, g->ok.p, ub, cudaMemcpyDeviceToHost, ctx->stream));
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    memcpy(poses_out, hs, pb);
    if (updates_out) memcpy(updates_out, hs + pb, ub);
    return 0;
}

}  // namespace

// ---- batched device ARRSAC (C names in batch_abi.cu, include/cvb200_batch.h) ------------------------------------------------
static int ars_batch_check(cvb_ctx *ctx, const cvb_arrsac_cfg *cfg, int kind, int row0, uint32_t B, const cvb_rng *rngs) {
    if (B > CVB_ARRSAC_BATCH_MAX) return cvb_set_error(ctx, CVB_EUNSUPPORTED, "batch of %u problems: at most %u", B, CVB_ARRSAC_BATCH_MAX);
    if (!cfg || !rngs) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (kind < 0 || kind > 2) return cvb_set_error(ctx, CVB_EINVAL, "kind must be 0 (eight-point), 1 (P3P) or 2 (five-point)");
    if (kind == 2 && row0 != 5 && row0 != 6) return cvb_set_error(ctx, CVB_EINVAL, "eigenvector_row0 must be 5 (reference) or 6 (corrected)");
    return 0;
}

int ars_batch_dev(cvb_ctx *ctx, const cvb_arrsac_cfg *cfg, int kind, int row0, const double *a_dev, const double *b_dev, const uint32_t *n_dev,
                  uint32_t n_max, uint32_t B, const cvb_rng *rngs, cvb_pose *model_out_dev, uint32_t *inliers_out_dev, uint32_t cap,
                  uint32_t *n_inliers_dev, int32_t *found_dev) {
    if (!ctx) return CVB_EINVAL;
    if (B == 0) return 0;
    int rc = ars_batch_check(ctx, cfg, kind, row0, B, rngs);
    if (rc) return rc;
    if (!a_dev || !b_dev || !model_out_dev || !n_inliers_dev || !found_dev) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    return arrsac_run_dev_batch(ctx, cfg, kind, a_dev, b_dev, n_dev, n_max, n_max, B, rngs, model_out_dev, inliers_out_dev, cap, n_inliers_dev,
                                found_dev, kind == 2 ? row0 : 5, true);
}

int ars_commit_rng_batch(cvb_ctx *ctx, cvb_rng *rngs, uint32_t B, uint32_t *stats_out) {
    if (!ctx) return CVB_EINVAL;
    if (!rngs) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    std::vector<ArrsacCtl> h(std::max<uint32_t>(B, 1));
    int rc = arrsac_commit_rng_batch(ctx, rngs, B, h.data(), true);
    if (rc) return rc;
    if (stats_out)
        for (uint32_t pb = 0; pb < B; pb++) arrsac_stats_words(h[pb], stats_out + 16 * (size_t)pb);
    return 0;
}

int ars_batch_host(cvb_ctx *ctx, const cvb_arrsac_cfg *cfg, int kind, int row0, const double *a, const double *b, const uint32_t *offsets,
                   uint32_t B, cvb_rng *rngs, cvb_pose *models_out, uint32_t *inliers_out, uint32_t *n_inliers_out, int32_t *found_out) {
    if (!ctx) return CVB_EINVAL;
    if (B == 0) return 0;
    int rc = ars_batch_check(ctx, cfg, kind, row0, B, rngs);
    if (rc) return rc;
    if (!offsets || !models_out || !n_inliers_out || !found_out) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    uint32_t n_max = 0;
    for (uint32_t pb = 0; pb < B; pb++) {
        if (offsets[pb + 1] < offsets[pb]) return cvb_set_error(ctx, CVB_EINVAL, "offsets must be non-decreasing");
        n_max = std::max(n_max, offsets[pb + 1] - offsets[pb]);
    }
    const uint32_t total = offsets[B] - offsets[0];
    if (total && (!a || !b)) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    for (uint32_t pb = 0; pb < B; pb++) { found_out[pb] = 0; n_inliers_out[pb] = 0; }
    // every problem below MIN_SAMPLES: nothing runs and no generator moves (as in the single entries)
    if (n_max < kind_K(kind) || cfg->initialization_hypotheses == 0) return 0;
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    ArsWorkspace *w = arsws(ctx);
    const uint32_t bc = kind_res(kind) == 0 ? 3 : 4;
    {   // problem pb's rows at pb * n_max (padding rows are never read: the kernels stop at the problem's count)
        std::vector<double> pa((size_t)B * n_max * 3, 0.0), pbv((size_t)B * n_max * bc, 0.0);
        std::vector<uint32_t> cnt(B);
        for (uint32_t pb = 0; pb < B; pb++) {
            cnt[pb] = offsets[pb + 1] - offsets[pb];
            if (!cnt[pb]) continue;
            memcpy(pa.data() + (size_t)pb * n_max * 3, a + 3 * (size_t)offsets[pb], sizeof(double) * 3 * cnt[pb]);
            memcpy(pbv.data() + (size_t)pb * n_max * bc, b + bc * (size_t)offsets[pb], sizeof(double) * bc * cnt[pb]);
        }
        if ((rc = upload(ctx, w->bdata_a, pa.data(), sizeof(double) * pa.size()))) return rc;
        if ((rc = upload(ctx, w->bdata_b, pbv.data(), sizeof(double) * pbv.size()))) return rc;
        if ((rc = upload(ctx, w->bcounts, cnt.data(), sizeof(uint32_t) * B))) return rc;
        CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));       // the pageable sources leave scope
    }
    // result block: B poses | B counts | B found flags | B x n_max inlier indices
    const size_t pose_b = sizeof(cvb_pose) * B, res_bytes = pose_b + 8 * (size_t)B + sizeof(uint32_t) * (size_t)B * n_max;
    if ((rc = w->res.ensure(ctx, res_bytes))) return rc;
    unsigned char *rd = (unsigned char *)w->res.p;
    if ((rc = arrsac_run_dev_batch(ctx, cfg, kind, (const double *)w->bdata_a.p, (const double *)w->bdata_b.p, (const uint32_t *)w->bcounts.p,
                                   n_max, n_max, B, rngs, (cvb_pose *)rd, (uint32_t *)(rd + pose_b + 8 * (size_t)B), n_max,
                                   (uint32_t *)(rd + pose_b), (int32_t *)(rd + pose_b + 4 * (size_t)B), kind == 2 ? row0 : 5, true))) return rc;
    unsigned char *hs = (unsigned char *)cvb_pinned(ctx, res_bytes);
    if (!hs) return cvb_set_error(ctx, CVB_ENOMEM, "page-locked scratch");
    CVB_CUDA(ctx, cudaMemcpyAsync(hs, rd, res_bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    if ((rc = arrsac_commit_rng_batch(ctx, rngs, B, nullptr, true))) return rc;
    const uint32_t *ninl = (const uint32_t *)(hs + pose_b);
    const int32_t *fnd = (const int32_t *)(hs + pose_b + 4 * (size_t)B);
    const uint32_t *inl = (const uint32_t *)(hs + pose_b + 8 * (size_t)B);
    for (uint32_t pb = 0; pb < B; pb++) {
        found_out[pb] = fnd[pb];
        if (!fnd[pb]) continue;
        memcpy(models_out + pb, hs + sizeof(cvb_pose) * pb, sizeof(cvb_pose));
        n_inliers_out[pb] = ninl[pb];
        if (inliers_out) memcpy(inliers_out + offsets[pb] - offsets[0], inl + (size_t)pb * n_max, sizeof(uint32_t) * ninl[pb]);
    }
    return 0;
}

// cv-sfm's init_two_view (cv-sfm/src/lib.rs:1365-1432) of frame `center` against F option frames, on the outputs of
// cvb_frame_features_batch_dev: F symmetric matches, one gather of the matched bearings for all options, one batched ARRSAC.
// Option f's consensus rows: row i = (bearing of center feature pairs[f][i][0], bearing of option feature pairs[f][i][1]).
struct OptionFrames { uint32_t f[CVB_ARRSAC_BATCH_MAX]; };
__global__ void __launch_bounds__(256) k_gather_option_bearings(const double *__restrict__ bear, uint32_t cap, uint32_t center, OptionFrames opt,
                                                                const uint32_t *__restrict__ pairs, const uint32_t *__restrict__ npairs,
                                                                double *__restrict__ a, double *__restrict__ b) {
    const uint32_t f = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= min(npairs[f], cap)) return;
    const uint32_t *p = pairs + ((size_t)f * cap + i) * 2;
    const double *ba = bear + ((size_t)center * cap + p[0]) * 3, *bb = bear + ((size_t)opt.f[f] * cap + p[1]) * 3;
    double *da = a + ((size_t)f * cap + i) * 3, *db = b + ((size_t)f * cap + i) * 3;
    for (int k = 0; k < 3; k++) { da[k] = ba[k]; db[k] = bb[k]; }
}

int two_view_options_dev(cvb_ctx *ctx, const uint8_t *desc_dev, const uint32_t *n_dev, const double *bearings_dev, uint32_t frames, uint32_t cap,
                         uint32_t center, const uint32_t *options, uint32_t F, uint32_t better_by, const cvb_arrsac_cfg *cfg, const cvb_rng *rngs,
                         uint32_t *pairs_out_dev, uint32_t *n_pairs_dev, cvb_pose *model_out_dev, uint32_t *inliers_out_dev,
                         uint32_t *n_inliers_dev, int32_t *found_dev) {
    if (!ctx) return CVB_EINVAL;
    if (F == 0) return 0;
    if (F > CVB_ARRSAC_BATCH_MAX) return cvb_set_error(ctx, CVB_EUNSUPPORTED, "%u options: at most %u", F, CVB_ARRSAC_BATCH_MAX);
    if (!desc_dev || !n_dev || !bearings_dev || !options || !cfg || !rngs || !pairs_out_dev || !n_pairs_dev || !model_out_dev ||
        !n_inliers_dev || !found_dev)
        return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (cap == 0) return cvb_set_error(ctx, CVB_EINVAL, "zero capacity");
    if (center >= frames) return cvb_set_error(ctx, CVB_EINVAL, "center frame %u of %u", center, frames);
    OptionFrames opt;
    memset(&opt, 0, sizeof(opt));
    for (uint32_t f = 0; f < F; f++) {
        if (options[f] >= frames) return cvb_set_error(ctx, CVB_EINVAL, "option %u: frame %u of %u", f, options[f], frames);
        opt.f[f] = options[f];
    }
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    int rc;
    for (uint32_t f = 0; f < F; f++)
        if ((rc = cvb_match_symmetric_pairs_dev(ctx, desc_dev + (size_t)center * cap * 64, n_dev + center, cap, desc_dev + (size_t)opt.f[f] * cap * 64,
                                                n_dev + opt.f[f], cap, better_by, pairs_out_dev + (size_t)f * cap * 2, cap, n_pairs_dev + f)))
            return rc;
    ArsWorkspace *w = arsws(ctx);
    if ((rc = w->bdata_a.ensure(ctx, sizeof(double) * 3 * (size_t)F * cap))) return rc;
    if ((rc = w->bdata_b.ensure(ctx, sizeof(double) * 3 * (size_t)F * cap))) return rc;
    {
        CVB_PROF(ctx, "k_gather_option_bearings", 0);
        k_gather_option_bearings<<<dim3(cdiv(cap, 256), F), 256, 0, ctx->stream>>>(bearings_dev, cap, center, opt, pairs_out_dev, n_pairs_dev,
                                                                                  (double *)w->bdata_a.p, (double *)w->bdata_b.p);
        CVB_LAUNCH_CHECK(ctx);
    }
    return arrsac_run_dev_batch(ctx, cfg, 0, (const double *)w->bdata_a.p, (const double *)w->bdata_b.p, n_pairs_dev, cap, cap, F, rngs,
                                model_out_dev, inliers_out_dev, cap, n_inliers_dev, found_dev, 5, true);
}

// ---- cv-sfm's three-view initialisation (C names in init_abi.cu, include/cvb200_init.h; kernels in init_dev.cuh) -------------
void init_cfg_default(cvb_init_cfg *c) {
    if (!c) return;
    memset(c, 0, sizeof(*c));
    c->robust_observation_incidence_minimum_cosine_distance = 1e-3;
    c->robust_view_bearing_pair_minimum_cosine_distance = 1e-2;
    c->maximum_cosine_distance = 1e-5;
    c->maximum_sine_distance = 1e-1;
    c->two_view_minimum_robust_matches = 1u << 8;
    c->three_view_minimum_relative_scales = 1u << 4;
    c->three_view_optimization_landmarks = 1u << 10;
    c->robust_view_num_robust_bearing_pair = 3;
    c->three_view_filter_loop_iterations = 1u << 3;
    c->three_view_patience = 1u << 16;
    c->three_view_minimum_robust_matches = 32;
}

static size_t init_align(size_t x) { return (x + 255) & ~(size_t)255; }

int init_reconstruction_dev(cvb_ctx *ctx, const cvb_init_cfg *cfg, const cvb_triangulator *tri, const double *bearings_dev, uint32_t frames,
                            uint32_t cap, uint32_t center, const uint32_t *options, uint32_t F, const uint32_t *pairs_dev,
                            const uint32_t *n_pairs_dev, const cvb_pose *model_dev, const uint32_t *inliers_dev, const uint32_t *n_inliers_dev,
                            const int32_t *found_dev, cvb_init_result *result_dev, uint32_t *combined_dev, uint32_t *first_matches_dev,
                            uint32_t *second_matches_dev, cvb_init_pair_stats *stats_dev) {
    if (!ctx) return CVB_EINVAL;
    if (!cfg || !tri || !bearings_dev || !pairs_dev || !n_pairs_dev || !model_dev || !inliers_dev || !n_inliers_dev || !found_dev ||
        !result_dev || !combined_dev || !first_matches_dev || !second_matches_dev || (F && !options))
        return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (F > CVB_ARRSAC_BATCH_MAX) return cvb_set_error(ctx, CVB_EUNSUPPORTED, "%u options: at most %u", F, CVB_ARRSAC_BATCH_MAX);
    if (tri->method < CVB_TRI_LINEAR_EIGEN || tri->method > CVB_TRI_MEAN_MEAN)
        return cvb_set_error(ctx, tri->method >= CVB_TRI_RELATIVE_DLT && tri->method <= CVB_TRI_ANGULAR_LINF ? CVB_EUNSUPPORTED : CVB_EINVAL,
                             "triangulator method %d: init_reconstruction takes a TriangulatorObservations (methods 0-2)", tri->method);
    if (cap == 0) return cvb_set_error(ctx, CVB_EINVAL, "zero capacity");
    if (center >= frames) return cvb_set_error(ctx, CVB_EINVAL, "center frame %u of %u", center, frames);
    InitFrames fr;
    memset(&fr, 0, sizeof(fr));
    fr.center = center;
    for (uint32_t f = 0; f < F; f++) {
        if (options[f] >= frames) return cvb_set_error(ctx, CVB_EINVAL, "option %u: frame %u of %u", f, options[f], frames);
        fr.f[f] = options[f];
    }
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    int W = 0;
    CVB_CUDA(ctx, cudaDeviceGetAttribute(&W, cudaDevAttrMultiProcessorCount, ctx->device));
    const uint32_t Fm = std::max<uint32_t>(F, 1), L = std::max<uint32_t>(std::min(cfg->three_view_optimization_landmarks, cap), 1);
    uint32_t n2 = 1;
    while (n2 < cap) n2 <<= 1;
    // workspace: control | W slots | maps | W x (common triples, 3 flag planes, ratios, sort buffer, optimisation rows) | offsets | poses
    size_t off = 0;
    const size_t o_ctl = off; off += init_align(sizeof(InitCtl));
    const size_t o_slots = off; off += init_align(sizeof(InitSlot) * W);
    const size_t o_map = off; off += init_align(sizeof(uint32_t) * (size_t)Fm * cap);
    const size_t o_common = off; off += init_align(sizeof(uint32_t) * 3 * (size_t)W * cap);
    const size_t o_flags = off; off += init_align((size_t)W * cap);
    const size_t o_ff = off; off += init_align((size_t)W * cap);
    const size_t o_fs = off; off += init_align((size_t)W * cap);
    const size_t o_ratio = off; off += init_align(sizeof(double) * (size_t)W * cap);
    const size_t o_sort = off; off += init_align(sizeof(double) * (size_t)W * n2);
    const size_t o_obs = off; off += init_align(sizeof(double) * 9 * (size_t)W * L);
    const size_t o_offs = off; off += init_align(sizeof(uint32_t) * (W + 1));
    const size_t o_poses = off; off += init_align(sizeof(cvb_pose) * 2 * (size_t)W);
    const size_t o_popt = off; off += init_align(sizeof(cvb_pose) * 2 * (size_t)W);
    const size_t o_upd = off; off += init_align(sizeof(uint32_t) * W);
    GeomWorkspace *g = gws(ctx);
    int rc;
    if ((rc = g->init.ensure(ctx, off))) return rc;
    unsigned char *base = (unsigned char *)g->init.p;
    InitCtl *ctl = (InitCtl *)(base + o_ctl);
    InitSlot *slots = (InitSlot *)(base + o_slots);
    uint32_t *map = (uint32_t *)(base + o_map), *common = (uint32_t *)(base + o_common), *offs = (uint32_t *)(base + o_offs);
    uint8_t *flags = base + o_flags, *ffirst = base + o_ff, *fsecond = base + o_fs;
    double *ratio = (double *)(base + o_ratio), *sortbuf = (double *)(base + o_sort), *obs = (double *)(base + o_obs);
    cvb_pose *poses = (cvb_pose *)(base + o_poses), *popt = (cvb_pose *)(base + o_popt);
    uint32_t *upd = (uint32_t *)(base + o_upd);
    InitParams prm;
    prm.inc = cfg->robust_observation_incidence_minimum_cosine_distance;
    prm.bp_min_cos = cfg->robust_view_bearing_pair_minimum_cosine_distance;
    prm.max_cos = cfg->maximum_cosine_distance;
    prm.max_sine = cfg->maximum_sine_distance;
    prm.min_scales = cfg->three_view_minimum_relative_scales;
    prm.limit = cfg->three_view_optimization_landmarks;
    prm.bp_min = cfg->robust_view_num_robust_bearing_pair;
    prm.min_robust = cfg->three_view_minimum_robust_matches;
    const cvb_triangulator T = *tri;
    const uint32_t npairs_max = F * (F - (F > 0)) / 2;
    cudaStream_t st = ctx->stream;
    {
        CVB_PROF(ctx, "k_init_setup", 0);
        if (stats_dev && npairs_max) CVB_CUDA(ctx, cudaMemsetAsync(stats_dev, 0, sizeof(cvb_init_pair_stats) * npairs_max, st));
        CVB_CUDA(ctx, cudaMemsetAsync(map, 0xff, sizeof(uint32_t) * (size_t)Fm * cap, st));
        k_init_setup<<<1, 32, 0, st>>>(n_inliers_dev, found_dev, F, cfg->two_view_minimum_robust_matches, ctl);
        CVB_LAUNCH_CHECK(ctx);
        if (F) {
            k_init_maps<<<dim3(cdiv(cap, 256), F), 256, 0, st>>>(pairs_dev, inliers_dev, n_inliers_dev, found_dev, cap, map);
            CVB_LAUNCH_CHECK(ctx);
        }
    }
    const dim3 gtri(cdiv(cap, 128), W), gslot(cdiv(W, 128));
    uint32_t *h = (uint32_t *)cvb_pinned(ctx, 4 * sizeof(uint32_t));   // K, P, decided, slot of the control block
    if (!h) return cvb_set_error(ctx, CVB_ENOMEM, "page-locked scratch");
    // the pairs that exist are known on the device only: wave 0 runs whenever F >= 2, and its readback bounds the rest
    uint32_t npairs = npairs_max;
    for (uint32_t wave = 0; wave * (uint32_t)W < npairs; wave++) {
        {
            CVB_PROF(ctx, "k_init_begin", 0);
            k_init_begin<<<gslot, 128, 0, st>>>(ctl, wave * W, W, model_dev, slots, poses);
            CVB_LAUNCH_CHECK(ctx);
        }
        {
            CVB_PROF(ctx, "k_init_common", 0);
            k_init_common<<<W, 256, 0, st>>>(pairs_dev, inliers_dev, n_inliers_dev, map, cap, slots, common);
            CVB_LAUNCH_CHECK(ctx);
        }
        {
            CVB_PROF(ctx, "k_init_flags_scale", 0);
            k_init_flags<0><<<gtri, 128, 0, st>>>(T, bearings_dev, cap, fr, common, poses, prm, 1.0, slots, flags, ratio);
            CVB_LAUNCH_CHECK(ctx);
        }
        {
            CVB_PROF(ctx, "k_init_median", 0);
            k_init_median<<<W, 256, 0, st>>>(cap, n2, prm, flags, ratio, slots, sortbuf, poses);
            CVB_LAUNCH_CHECK(ctx);
        }
        auto opti_set = [&](bool reflag, double max_cos, uint32_t mode) -> int {
            if (reflag) {
                CVB_PROF(ctx, "k_init_flags_opti", 0);
                k_init_flags<1><<<gtri, 128, 0, st>>>(T, bearings_dev, cap, fr, common, poses, prm, max_cos, slots, flags, ratio);
                CVB_LAUNCH_CHECK(ctx);
            }
            {
                CVB_PROF(ctx, "k_init_sizes", 0);
                k_init_sizes<<<1, 32, 0, st>>>(W, mode, prm, slots, offs);
                CVB_LAUNCH_CHECK(ctx);
            }
            {
                CVB_PROF(ctx, "k_init_gather", 0);
                k_init_gather<<<W, 256, 0, st>>>(bearings_dev, cap, fr, common, flags, slots, offs, obs);
                CVB_LAUNCH_CHECK(ctx);
            }
            return 0;
        };
        auto optimise = [&]() -> int {
            {
                CVB_PROF(ctx, "k_three_view_opt", 0);
                k_three_view_opt<<<W, OPT_NT, 0, st>>>(poses, obs, offs, 0, 0.001, cfg->three_view_patience, popt, upd);
                CVB_LAUNCH_CHECK(ctx);
            }
            {
                CVB_PROF(ctx, "k_init_post_opt", 0);
                k_init_post_opt<<<gslot, 128, 0, st>>>(W, popt, upd, slots, poses);
                CVB_LAUNCH_CHECK(ctx);
            }
            return 0;
        };
        // lib.rs:1064-1106: the first set (under the scaled poses) and its robust bearing pairs
        if ((rc = opti_set(true, 1.0, INIT_SZ_RECOUNT | INIT_SZ_FIRST))) return rc;
        {
            CVB_PROF(ctx, "k_init_bearing_pairs", 0);
            k_init_bearing_pairs<<<dim3(cdiv(L, 128), W), 128, 0, st>>>(obs, offs, prm.bp_min_cos, slots);
            CVB_LAUNCH_CHECK(ctx);
        }
        // lib.rs:1112-1187: the filter loop and the final optimisation; the first check reuses the first set
        if ((rc = opti_set(false, 0.0, INIT_SZ_BEARING | INIT_SZ_CHECK))) return rc;
        for (uint32_t it = 0; it < cfg->three_view_filter_loop_iterations; it++) {
            if ((rc = optimise())) return rc;
            if ((rc = opti_set(true, prm.max_cos, INIT_SZ_RECOUNT | INIT_SZ_CHECK))) return rc;
        }
        if ((rc = optimise())) return rc;
        {
            CVB_PROF(ctx, "k_init_final", 0);
            k_init_flags<2><<<gtri, 128, 0, st>>>(T, bearings_dev, cap, fr, common, poses, prm, prm.max_cos, slots, flags, ratio);
            CVB_LAUNCH_CHECK(ctx);
            k_init_bi_flags<<<dim3(cdiv(cap, 128), W, 2), 128, 0, st>>>(bearings_dev, cap, fr, pairs_dev, inliers_dev, n_inliers_dev, map, poses,
                                                                        prm, slots, ffirst, fsecond);
            CVB_LAUNCH_CHECK(ctx);
            k_init_accept<<<gslot, 128, 0, st>>>(W, prm, slots);
            CVB_LAUNCH_CHECK(ctx);
            k_init_decide<<<1, 32, 0, st>>>(W, slots, ctl, stats_dev);
            CVB_LAUNCH_CHECK(ctx);
        }
        CVB_CUDA(ctx, cudaMemcpyAsync(h, ctl, 4 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
        CVB_CUDA(ctx, cvb_wait(ctx, st));
        if ((int32_t)h[2] >= 0) break;
        npairs = h[1];
    }
    {
        CVB_PROF(ctx, "k_init_finish", 0);
        k_init_finish<<<1, 256, 0, st>>>(ctl, slots, cap, pairs_dev, inliers_dev, n_inliers_dev, common, flags, ffirst, fsecond, poses, result_dev,
                                         combined_dev, first_matches_dev, second_matches_dev);
        CVB_LAUNCH_CHECK(ctx);
    }
    return 0;
}

// ---- cv-sfm's three-view constraints (C names in constraints_abi.cu, include/cvb200_constraints.h; kernels in constraints_dev.cuh) ------
void constraints_cfg_default(cvb_constraints_cfg *c) {
    if (!c) return;
    memset(c, 0, sizeof(*c));
    c->robust_observation_incidence_minimum_cosine_distance = 1e-3;
    c->robust_view_bearing_pair_minimum_cosine_distance = 1e-2;
    c->robust_minimum_observations = 3;
    c->robust_view_num_robust_bearing_pair = 3;
    c->optimization_robust_covisibility_minimum_landmarks = 1u << 4;
    c->optimization_minimum_landmarks = 24;
    c->optimization_maximum_landmarks = 64;
    c->optimization_maximum_three_view_constraints = 1u << 6;
    c->optimization_minimum_new_constraints = 4;
    c->constraint_patience = 1u << 12;
}

int three_view_adaptive_optimize_l2_dev(cvb_ctx *ctx, const cvb_pose *poses_dev, uint32_t B, const double *obs_dev, const uint32_t *offsets_dev,
                                        uint32_t iterations, cvb_pose *poses_out_dev, uint32_t *updates_dev) {
    if (!ctx) return CVB_EINVAL;
    if (B == 0) return 0;
    if (!poses_dev || !obs_dev || !offsets_dev || !poses_out_dev || !updates_dev) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    std::vector<uint32_t> off(B + 1);
    CVB_CUDA(ctx, cudaMemcpyAsync(off.data(), offsets_dev, sizeof(uint32_t) * (B + 1), cudaMemcpyDeviceToHost, ctx->stream));
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    for (uint32_t b = 0; b < B; b++) {
        if (off[b + 1] < off[b]) return cvb_set_error(ctx, CVB_EINVAL, "offsets decrease at problem %u", b);
        if (off[b + 1] - off[b] > CVB_CONSTRAINTS_MAX_LANDMARKS)
            return cvb_set_error(ctx, CVB_EUNSUPPORTED, "problem %u: %u landmarks, at most %u", b, off[b + 1] - off[b], CVB_CONSTRAINTS_MAX_LANDMARKS);
    }
    {
        CVB_PROF(ctx, "k_three_view_opt_warp", 0.0);
        k_three_view_opt_warp<<<cdiv(B, OPTW_WARPS), OPTW_NT, 0, ctx->stream>>>(poses_dev, obs_dev, offsets_dev, B, iterations, poses_out_dev,
                                                                              updates_dev);
        CVB_LAUNCH_CHECK(ctx);
    }
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    return 0;
}

static uint32_t con_pow2(uint64_t x) { uint32_t n = 1; while (n < x) n <<= 1; return n; }
static size_t con_align(size_t x) { return (x + 255) & ~(size_t)255; }
// the per-chunk workspace is kept below this; a query that alone exceeds it runs alone
constexpr size_t CON_CHUNK_BYTES = (size_t)256 << 20;

int view_constraints_dev(cvb_ctx *ctx, const cvb_constraints_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses_dev,
                         const uint32_t *view_off_dev, const uint32_t *view_lm_dev, const double *bear_dev, uint32_t n_features, uint32_t L,
                         const uint32_t *lm_off_dev, const uint32_t *obs_dev, uint32_t n_obs, const uint32_t *queries, uint32_t Q,
                         cvb_view_constraint *out_dev, cvb_view_constraints_result *res_dev, cvb_view_constraints_stats *stats_dev) {
    if (!ctx) return CVB_EINVAL;
    if (!cfg || !tri || !poses_dev || !view_off_dev || !lm_off_dev || !res_dev || (Q && !queries) || (n_features && (!view_lm_dev || !bear_dev)) ||
        (n_obs && !obs_dev) || (Q && cfg->optimization_maximum_three_view_constraints && !out_dev))
        return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (tri->method < CVB_TRI_LINEAR_EIGEN || tri->method > CVB_TRI_MEAN_MEAN)
        return cvb_set_error(ctx, tri->method >= CVB_TRI_RELATIVE_DLT && tri->method <= CVB_TRI_ANGULAR_LINF ? CVB_EUNSUPPORTED : CVB_EINVAL,
                             "triangulator method %d: the constraints take a TriangulatorObservations (methods 0-2)", tri->method);
    if (cfg->optimization_maximum_landmarks > CVB_CONSTRAINTS_MAX_LANDMARKS)
        return cvb_set_error(ctx, CVB_EUNSUPPORTED, "optimization_maximum_landmarks %u: at most %u", cfg->optimization_maximum_landmarks,
                             CVB_CONSTRAINTS_MAX_LANDMARKS);
    if (V == 0) return cvb_set_error(ctx, CVB_EINVAL, "no views");
    for (uint32_t i = 0; i < Q; i++)
        if (queries[i] >= V) return cvb_set_error(ctx, CVB_EINVAL, "query %u: view %u of %u", i, queries[i], V);
    if (Q == 0) return 0;
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    int sms = 0;
    CVB_CUDA(ctx, cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, ctx->device));
    cudaStream_t st = ctx->stream;
    std::vector<uint32_t> vo(V + 1);
    CVB_CUDA(ctx, cudaMemcpyAsync(vo.data(), view_off_dev, sizeof(uint32_t) * (V + 1), cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    if (vo[V] != n_features) return cvb_set_error(ctx, CVB_EINVAL, "view_offsets[V] = %u, n_features %u", vo[V], n_features);
    ConParams prm;
    prm.inc = cfg->robust_observation_incidence_minimum_cosine_distance;
    prm.bp_min_cos = cfg->robust_view_bearing_pair_minimum_cosine_distance;
    prm.V = V;
    prm.min_obs = std::min(cfg->robust_minimum_observations, V);
    prm.covis_min = cfg->optimization_robust_covisibility_minimum_landmarks;
    prm.opt_min = cfg->optimization_minimum_landmarks;
    prm.opt_max = cfg->optimization_maximum_landmarks;
    prm.bp_min = cfg->robust_view_num_robust_bearing_pair;
    prm.max_c = cfg->optimization_maximum_three_view_constraints;
    prm.min_new = cfg->optimization_minimum_new_constraints;
    const cvb_triangulator T = *tri;
    const uint32_t maxc = prm.max_c, omax = std::max<uint32_t>(prm.opt_max, 1), vw = (V + 31) / 32;
    // per chunk query: robust list, three V-sized arrays, its ConQuery
    auto bytes_a = [&](uint32_t q) { return sizeof(uint32_t) * ((size_t)(vo[q + 1] - vo[q]) + 3 * (size_t)V) + sizeof(ConQuery); };
    size_t chunk_a = 0, cur = 0;
    for (uint32_t i = 0; i < Q; i++) {
        const size_t b = bytes_a(queries[i]);
        if (cur && cur + b > CON_CHUNK_BYTES) { chunk_a = std::max(chunk_a, cur); cur = 0; }
        cur += b;
    }
    chunk_a = std::max(chunk_a, cur) + 8 * 256;
    // snapshot part: per observation pose, bearing, world bearing (and SineL1's scratch), per landmark the robust flag; then the chunk part
    size_t off = 0;
    const size_t o_pose = off; off += con_align(sizeof(cvb_pose) * (size_t)n_obs);
    const size_t o_bear = off; off += con_align(sizeof(double) * 3 * (size_t)n_obs);
    const size_t o_world = off; off += con_align(sizeof(double) * 3 * (size_t)n_obs);
    const size_t o_W = off; off += tri->method == CVB_TRI_SINE_L1 ? con_align(sizeof(double) * 6 * (size_t)n_obs) : 0;
    const size_t o_rob = off; off += con_align(L);
    const size_t o_chunk = off; off += chunk_a;
    GeomWorkspace *g = gws(ctx);
    int rc;
    if ((rc = g->con.ensure(ctx, off))) return rc;
    unsigned char *base = (unsigned char *)g->con.p;
    cvb_pose *obs_pose = (cvb_pose *)(base + o_pose);
    double *obs_bear = (double *)(base + o_bear), *obs_world = (double *)(base + o_world);
    double *W = tri->method == CVB_TRI_SINE_L1 ? (double *)(base + o_W) : nullptr;
    uint8_t *robust = base + o_rob;
    if (n_obs) {
        CVB_PROF(ctx, "k_con_gather_obs", 0);
        k_con_gather_obs<<<cdiv(n_obs, 256), 256, 0, st>>>(poses_dev, view_off_dev, bear_dev, obs_dev, n_obs, obs_pose, obs_bear, obs_world);
        CVB_LAUNCH_CHECK(ctx);
    }
    if (L) {
        CVB_PROF(ctx, "k_con_robust", 0);
        k_con_robust<<<cdiv(L, 128), 128, 0, st>>>(T, lm_off_dev, L, obs_pose, obs_bear, obs_world, W, prm, robust);
        CVB_LAUNCH_CHECK(ctx);
    }
    std::vector<ConQuery> hq;
    for (uint32_t c0 = 0; c0 < Q;) {
        // chunk [c0, c1): phase A
        uint32_t c1 = c0;
        size_t used = 0, nrl = 0;
        while (c1 < Q && (c1 == c0 || used + bytes_a(queries[c1]) <= CON_CHUNK_BYTES)) { used += bytes_a(queries[c1]); nrl += vo[queries[c1] + 1] - vo[queries[c1]]; c1++; }
        const uint32_t Qc = c1 - c0;
        unsigned char *cb = base + o_chunk;
        size_t co = 0;
        ConQuery *qs = (ConQuery *)(cb + co); co += con_align(sizeof(ConQuery) * Qc);
        uint32_t *cnt = (uint32_t *)(cb + co); co += con_align(sizeof(uint32_t) * (size_t)Qc * V);
        uint32_t *kidx = (uint32_t *)(cb + co); co += con_align(sizeof(uint32_t) * (size_t)Qc * V);
        uint32_t *kview = (uint32_t *)(cb + co); co += con_align(sizeof(uint32_t) * (size_t)Qc * V);
        uint32_t *rlist = (uint32_t *)(cb + co); co += con_align(sizeof(uint32_t) * std::max<size_t>(nrl, 1));
        hq.assign(Qc, ConQuery());
        uint32_t rb = 0;
        for (uint32_t j = 0; j < Qc; j++) {
            memset(&hq[j], 0, sizeof(ConQuery));
            hq[j].q = queries[c0 + j]; hq[j].out = c0 + j; hq[j].rbase = rb;
            rb += vo[hq[j].q + 1] - vo[hq[j].q];
        }
        CVB_CUDA(ctx, cudaMemcpyAsync(qs, hq.data(), sizeof(ConQuery) * Qc, cudaMemcpyHostToDevice, st));
        CVB_CUDA(ctx, cudaMemsetAsync(cnt, 0, sizeof(uint32_t) * (size_t)Qc * V, st));
        {
            CVB_PROF(ctx, "k_con_lists", 0);
            k_con_lists<<<Qc, 256, 0, st>>>(view_off_dev, view_lm_dev, lm_off_dev, obs_dev, robust, prm, qs, rlist, cnt, kidx, kview);
            CVB_LAUNCH_CHECK(ctx);
        }
        CVB_CUDA(ctx, cudaMemcpyAsync(hq.data(), qs, sizeof(ConQuery) * Qc, cudaMemcpyDeviceToHost, st));
        CVB_CUDA(ctx, cvb_wait(ctx, st));
        // phase B over sub-chunks [s0, s1) of the chunk
        auto bytes_b = [&](const ConQuery &q) {
            const uint64_t P = (uint64_t)q.K * (q.K - (q.K > 0)) / 2;
            return sizeof(uint32_t) * ((size_t)q.K * ((q.R + 31) / 32) + 2 * P + vw) + sizeof(unsigned long long) * (con_pow2(P) + con_pow2(q.R)) +
                   (size_t)maxc * (2 * sizeof(double) * 9 * omax + 4 * sizeof(cvb_pose) + sizeof(uint32_t) * 6 + sizeof(double)) + 16 * 256;
        };
        for (uint32_t s0 = 0; s0 < Qc;) {
            uint32_t s1 = s0;
            size_t ub = 0;
            while (s1 < Qc && (s1 == s0 || ub + bytes_b(hq[s1]) <= CON_CHUNK_BYTES)) ub += bytes_b(hq[s1++]);
            const uint32_t Qs = s1 - s0, B = Qs * maxc;
            uint32_t nb = 0, nk = 0, npair = 0, nsort = 0, max_n2 = 1;
            for (uint32_t j = s0; j < s1; j++) {
                ConQuery &q = hq[j];
                const uint64_t P = (uint64_t)q.K * (q.K - (q.K > 0)) / 2;
                if (P >= (1ull << 31)) return cvb_set_error(ctx, CVB_EUNSUPPORTED, "query %u: %u coviews", q.out, q.K);
                q.words = (q.R + 31) / 32; q.bbase = nb; nb += q.K * q.words;
                q.P = (uint32_t)P; q.n2 = con_pow2(P); q.kbase = nk; nk += q.n2; q.obase = npair; npair += q.P;
                q.s2 = con_pow2(q.R); q.sbase = nsort; nsort += q.s2;
                max_n2 = std::max(max_n2, q.n2);
            }
            size_t bo = 0;
            const size_t b_bits = bo; bo += con_align(sizeof(uint32_t) * std::max<uint32_t>(nb, 1));
            const size_t b_keys = bo; bo += con_align(sizeof(unsigned long long) * nk);
            const size_t b_pcnt = bo; bo += con_align(sizeof(uint32_t) * std::max<uint32_t>(npair, 1));
            const size_t b_ord = bo; bo += con_align(sizeof(uint32_t) * std::max<uint32_t>(npair, 1));
            const size_t b_vis = bo; bo += con_align(sizeof(uint32_t) * (size_t)Qs * vw);
            const size_t b_sort = bo; bo += con_align(sizeof(unsigned long long) * nsort);
            const size_t b_rows = bo; bo += con_align(sizeof(double) * 9 * (size_t)std::max<uint32_t>(B, 1) * omax);
            const size_t b_pack = bo; bo += con_align(sizeof(double) * 9 * (size_t)std::max<uint32_t>(B, 1) * omax);
            const size_t b_pin = bo; bo += con_align(sizeof(cvb_pose) * 2 * (size_t)std::max<uint32_t>(B, 1));
            const size_t b_pout = bo; bo += con_align(sizeof(cvb_pose) * 2 * (size_t)std::max<uint32_t>(B, 1));
            const size_t b_pn = bo; bo += con_align(sizeof(uint32_t) * std::max<uint32_t>(B, 1));
            const size_t b_pv = bo; bo += con_align(sizeof(uint32_t) * 3 * (size_t)std::max<uint32_t>(B, 1));
            const size_t b_ps = bo; bo += con_align(sizeof(double) * std::max<uint32_t>(B, 1));
            const size_t b_off = bo; bo += con_align(sizeof(uint32_t) * (B + 1));
            const size_t b_upd = bo; bo += con_align(sizeof(uint32_t) * std::max<uint32_t>(B, 1));
            if ((rc = g->con2.ensure(ctx, bo))) return rc;
            unsigned char *sb = (unsigned char *)g->con2.p;
            uint32_t *bits = (uint32_t *)(sb + b_bits), *pcnt = (uint32_t *)(sb + b_pcnt), *ord = (uint32_t *)(sb + b_ord);
            uint32_t *vis = (uint32_t *)(sb + b_vis), *pn = (uint32_t *)(sb + b_pn), *pv = (uint32_t *)(sb + b_pv);
            uint32_t *poff = (uint32_t *)(sb + b_off), *upd = (uint32_t *)(sb + b_upd);
            unsigned long long *keys = (unsigned long long *)(sb + b_keys), *sortbuf = (unsigned long long *)(sb + b_sort);
            double *rows = (double *)(sb + b_rows), *packed = (double *)(sb + b_pack), *ps = (double *)(sb + b_ps);
            cvb_pose *pin = (cvb_pose *)(sb + b_pin), *pout = (cvb_pose *)(sb + b_pout);
            ConQuery *qsub = qs + s0;
            uint32_t *ki = kidx + (size_t)s0 * V, *kv = kview + (size_t)s0 * V;
            CVB_CUDA(ctx, cudaMemcpyAsync(qsub, hq.data() + s0, sizeof(ConQuery) * Qs, cudaMemcpyHostToDevice, st));
            CVB_CUDA(ctx, cudaMemsetAsync(bits, 0, sizeof(uint32_t) * std::max<uint32_t>(nb, 1), st));
            CVB_CUDA(ctx, cudaMemsetAsync(vis, 0, sizeof(uint32_t) * (size_t)Qs * vw, st));
            {
                CVB_PROF(ctx, "k_con_triples", 0);
                k_con_bits<<<Qs, 256, 0, st>>>(lm_off_dev, obs_dev, prm, qsub, rlist, ki, bits);
                CVB_LAUNCH_CHECK(ctx);
                k_con_pairs<<<dim3(cdiv(max_n2, 8), Qs), 256, 0, st>>>(prm, qsub, bits, keys, pcnt);
                CVB_LAUNCH_CHECK(ctx);
                k_con_order<<<Qs, 1024, 0, st>>>(prm, qsub, kv, keys, vis, ord);
                CVB_LAUNCH_CHECK(ctx);
            }
            {
                CVB_PROF(ctx, "k_con_select", 0);
                k_con_select<<<Qs, 256, 0, st>>>(poses_dev, view_off_dev, bear_dev, lm_off_dev, obs_dev, prm, qsub, rlist, kv, bits, keys, pcnt,
                                                 ord, sortbuf, rows, pin, pn, pv, ps);
                CVB_LAUNCH_CHECK(ctx);
            }
            if (B) {
                {
                    CVB_PROF(ctx, "k_con_pack", 0);
                    k_con_offsets<<<1, 32, 0, st>>>(B, pn, poff);
                    CVB_LAUNCH_CHECK(ctx);
                    k_con_pack<<<B, 256, 0, st>>>(omax, pn, poff, rows, packed);
                    CVB_LAUNCH_CHECK(ctx);
                }
                // The two kernels give the same bits (tests/test_gpu_constraints.py).  A batch that fits one CTA per SM (one query) runs
                // faster on k_three_view_opt's 512 threads per problem; a larger one on k_three_view_opt_warp's eight problems per SM
                // (DESIGN section 4l).
                if (B <= (uint32_t)sms) {
                    CVB_PROF(ctx, "k_three_view_opt", 0);
                    k_three_view_opt<<<B, OPT_NT, 0, st>>>(pin, packed, poff, 1, 0.0, cfg->constraint_patience, pout, upd);
                    CVB_LAUNCH_CHECK(ctx);
                } else {
                    CVB_PROF(ctx, "k_three_view_opt_warp", 0);
                    k_three_view_opt_warp<<<cdiv(B, OPTW_WARPS), OPTW_NT, 0, st>>>(pin, packed, poff, B, cfg->constraint_patience, pout, upd);
                    CVB_LAUNCH_CHECK(ctx);
                }
            }
            {
                CVB_PROF(ctx, "k_con_finish", 0);
                k_con_finish<<<Qs, 64, 0, st>>>(prm, qsub, pout, upd, pn, pv, ps, out_dev, res_dev, stats_dev);
                CVB_LAUNCH_CHECK(ctx);
            }
            s0 = s1;
        }
        c0 = c1;
    }
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    return 0;
}

int view_constraints_check(uint32_t V, const uint32_t *vo, const uint32_t *vl, uint32_t L, const uint32_t *lo, const uint32_t *obs,
                           const uint32_t *queries, uint32_t Q) {
    if (!vo || !lo || (Q && !queries)) return CVB_EINVAL;
    if (V == 0 || vo[0] != 0 || lo[0] != 0) return CVB_EINVAL;
    for (uint32_t v = 0; v < V; v++) if (vo[v + 1] < vo[v]) return CVB_EINVAL;
    for (uint32_t l = 0; l < L; l++) if (lo[l + 1] < lo[l]) return CVB_EINVAL;
    if ((vo[V] && !vl) || (lo[L] && !obs)) return CVB_EINVAL;
    for (uint32_t i = 0; i < Q; i++) if (queries[i] >= V) return CVB_EINVAL;
    for (uint32_t f = 0; f < vo[V]; f++) if (vl[f] >= L) return CVB_EINVAL;
    // every observation names an existing feature of its view, that feature names the landmark back, and no view is observed twice;
    // with as many observations as features, that makes the two CSRs each other's inverse
    if (lo[L] != vo[V]) return CVB_EINVAL;
    std::vector<uint32_t> last(V, 0xffffffffu);
    for (uint32_t l = 0; l < L; l++)
        for (uint32_t o = lo[l]; o < lo[l + 1]; o++) {
            const uint32_t v = obs[2 * (size_t)o], f = obs[2 * (size_t)o + 1];
            if (v >= V || f >= vo[v + 1] - vo[v] || vl[vo[v] + f] != l || last[v] == l) return CVB_EINVAL;
            last[v] = l;
        }
    return 0;
}

int view_constraints(cvb_ctx *ctx, const cvb_constraints_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses,
                     const uint32_t *vo, const uint32_t *vl, const double *bear, uint32_t L, const uint32_t *lo, const uint32_t *obs,
                     const uint32_t *queries, uint32_t Q, cvb_view_constraint *out, cvb_view_constraints_result *res,
                     cvb_view_constraints_stats *stats) {
    if (!ctx) return CVB_EINVAL;
    const uint32_t maxc = cfg ? cfg->optimization_maximum_three_view_constraints : 0;
    if (!cfg || !tri || !poses || !res || (Q && maxc && !out)) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (view_constraints_check(V, vo, vl, L, lo, obs, queries, Q)) return cvb_set_error(ctx, CVB_EINVAL, "malformed snapshot or queries");
    if (vo[V] && !bear) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    const uint32_t nf = vo[V], no = lo[L];
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    size_t off = 0;
    const size_t i_pose = off; off += con_align(sizeof(cvb_pose) * V);
    const size_t i_vo = off; off += con_align(sizeof(uint32_t) * (V + 1));
    const size_t i_vl = off; off += con_align(sizeof(uint32_t) * (size_t)nf);
    const size_t i_bear = off; off += con_align(sizeof(double) * 3 * (size_t)nf);
    const size_t i_lo = off; off += con_align(sizeof(uint32_t) * ((size_t)L + 1));
    const size_t i_obs = off; off += con_align(sizeof(uint32_t) * 2 * (size_t)no);
    const size_t i_out = off; off += con_align(sizeof(cvb_view_constraint) * (size_t)Q * maxc);
    const size_t i_res = off; off += con_align(sizeof(cvb_view_constraints_result) * (size_t)Q);
    const size_t i_st = off; off += con_align(sizeof(cvb_view_constraints_stats) * (size_t)Q);
    GeomWorkspace *g = gws(ctx);
    int rc;
    if ((rc = g->out.ensure(ctx, off))) return rc;
    unsigned char *b = (unsigned char *)g->out.p;
    cudaStream_t st = ctx->stream;
    CVB_CUDA(ctx, cudaMemcpyAsync(b + i_pose, poses, sizeof(cvb_pose) * V, cudaMemcpyHostToDevice, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(b + i_vo, vo, sizeof(uint32_t) * (V + 1), cudaMemcpyHostToDevice, st));
    if (nf) CVB_CUDA(ctx, cudaMemcpyAsync(b + i_vl, vl, sizeof(uint32_t) * (size_t)nf, cudaMemcpyHostToDevice, st));
    if (nf) CVB_CUDA(ctx, cudaMemcpyAsync(b + i_bear, bear, sizeof(double) * 3 * (size_t)nf, cudaMemcpyHostToDevice, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(b + i_lo, lo, sizeof(uint32_t) * ((size_t)L + 1), cudaMemcpyHostToDevice, st));
    if (no) CVB_CUDA(ctx, cudaMemcpyAsync(b + i_obs, obs, sizeof(uint32_t) * 2 * (size_t)no, cudaMemcpyHostToDevice, st));
    if ((rc = view_constraints_dev(ctx, cfg, tri, V, (const cvb_pose *)(b + i_pose), (const uint32_t *)(b + i_vo), (const uint32_t *)(b + i_vl),
                                   (const double *)(b + i_bear), nf, L, (const uint32_t *)(b + i_lo), (const uint32_t *)(b + i_obs), no, queries,
                                   Q, (cvb_view_constraint *)(b + i_out), (cvb_view_constraints_result *)(b + i_res),
                                   stats ? (cvb_view_constraints_stats *)(b + i_st) : nullptr)))
        return rc;
    if (Q && maxc) CVB_CUDA(ctx, cudaMemcpyAsync(out, b + i_out, sizeof(cvb_view_constraint) * (size_t)Q * maxc, cudaMemcpyDeviceToHost, st));
    if (Q) CVB_CUDA(ctx, cudaMemcpyAsync(res, b + i_res, sizeof(cvb_view_constraints_result) * (size_t)Q, cudaMemcpyDeviceToHost, st));
    if (Q && stats) CVB_CUDA(ctx, cudaMemcpyAsync(stats, b + i_st, sizeof(cvb_view_constraints_stats) * (size_t)Q, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    return 0;
}

// ---- cv-sfm's reconstruction optimisation (C names in reconstruction_abi.cu, include/cvb200_reconstruction.h; kernels in
// reconstruction_dev.cuh) -----------------------------------------------------------------------------------------------------------
void recon_cfg_default(cvb_recon_cfg *c) {
    if (!c) return;
    memset(c, 0, sizeof(*c));
    c->graph_optimization_rate = 0.001;
    c->maximum_sine_distance = 0.1;
    c->maximum_cosine_distance = 1e-5;
    c->robust_observation_incidence_minimum_cosine_distance = 1e-3;
    c->optimization_iterations = 1u << 10;
    c->reconstruction_optimization_iterations = 1;
    c->robust_minimum_observations = 3;
    c->minimum_robust_landmarks = 32;
}

int optimize_reconstruction_check(uint32_t V, const uint32_t *vo, const uint32_t *vl, uint32_t L, const uint32_t *lo, const uint32_t *obs,
                                  const cvb_view_constraint *cons, uint32_t C) {
    if (view_constraints_check(V, vo, vl, L, lo, obs, nullptr, 0)) return CVB_EINVAL;
    if (C && !cons) return CVB_EINVAL;
    for (uint32_t c = 0; c < C; c++) {
        const uint32_t *w = cons[c].views;
        if (w[0] >= V || w[1] >= V || w[2] >= V || w[0] == w[1] || w[0] == w[2] || w[1] == w[2]) return CVB_EINVAL;
    }
    return 0;
}

int optimize_reconstruction_dev(cvb_ctx *ctx, const cvb_recon_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses_dev,
                                const uint32_t *view_off_dev, const uint32_t *view_lm_dev, const double *bear_dev, uint32_t n_features,
                                uint32_t L, const uint32_t *lm_off_dev, const uint32_t *obs_dev, uint32_t n_obs,
                                const cvb_view_constraint *cons_dev, uint32_t C, cvb_recon_result *res_dev, cvb_pose *poses_out_dev,
                                uint8_t *view_state_dev, uint8_t *obs_state_dev) {
    if (!ctx) return CVB_EINVAL;
    if (!cfg || !tri || !poses_dev || !view_off_dev || !lm_off_dev || !res_dev || !poses_out_dev || !view_state_dev ||
        (n_features && (!view_lm_dev || !bear_dev)) || (n_obs && (!obs_dev || !obs_state_dev)) || (C && !cons_dev))
        return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (tri->method < CVB_TRI_LINEAR_EIGEN || tri->method > CVB_TRI_MEAN_MEAN)
        return cvb_set_error(ctx, tri->method >= CVB_TRI_RELATIVE_DLT && tri->method <= CVB_TRI_ANGULAR_LINF ? CVB_EUNSUPPORTED : CVB_EINVAL,
                             "triangulator method %d: the filter takes a TriangulatorObservations (methods 0-2)", tri->method);
    if (V == 0) return cvb_set_error(ctx, CVB_EINVAL, "no views");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    uint32_t nf = 0;
    CVB_CUDA(ctx, cudaMemcpyAsync(&nf, view_off_dev + V, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    if (nf != n_features) return cvb_set_error(ctx, CVB_EINVAL, "view_offsets[V] = %u, n_features %u", nf, n_features);
    RecParams prm;
    prm.rate = cfg->graph_optimization_rate;
    prm.max_sin = cfg->maximum_sine_distance;
    prm.max_cos = cfg->maximum_cosine_distance;
    prm.inc = cfg->robust_observation_incidence_minimum_cosine_distance;
    prm.V = V;
    prm.C = C;
    prm.iters = cfg->optimization_iterations;
    prm.min_obs_cfg = cfg->robust_minimum_observations;
    prm.min_robust = cfg->minimum_robust_landmarks;
    const size_t E = 6 * (size_t)C;
    size_t off = 0;
    const size_t o_ctl = off; off += con_align(sizeof(RecCtl));
    const size_t o_pose = off; off += con_align(sizeof(cvb_pose) * 2 * (size_t)V);
    const size_t o_state = off; off += con_align(2 * (size_t)V);
    const size_t o_deg = off; off += con_align(sizeof(uint32_t) * (size_t)V);
    const size_t o_eoff = off; off += con_align(sizeof(uint32_t) * ((size_t)V + 1));
    const size_t o_ev = off; off += con_align(sizeof(uint32_t) * std::max<size_t>(E, 1));
    const size_t o_eo = off; off += con_align(sizeof(uint32_t) * std::max<size_t>(E, 1));
    const size_t o_eT = off; off += con_align(sizeof(cvb_pose) * std::max<size_t>(E, 1));
    const size_t o_se3 = off; off += con_align(sizeof(double) * 6 * std::max<size_t>(E, 1));
    const size_t o_gp = off; off += con_align(sizeof(cvb_pose) * std::max<size_t>(n_obs, 1));
    const size_t o_gb = off; off += con_align(sizeof(double) * 3 * std::max<size_t>(n_obs, 1));
    const size_t o_gw = off; off += con_align(sizeof(double) * 3 * std::max<size_t>(n_obs, 1));
    const size_t o_gi = off; off += con_align(sizeof(uint32_t) * std::max<size_t>(n_obs, 1));
    const size_t o_W = off; off += tri->method == CVB_TRI_SINE_L1 ? con_align(sizeof(double) * 6 * std::max<size_t>(n_obs, 1)) : 0;
    GeomWorkspace *g = gws(ctx);
    int rc;
    if ((rc = g->rec.ensure(ctx, off))) return rc;
    unsigned char *base = (unsigned char *)g->rec.p;
    RecCtl *ctl = (RecCtl *)(base + o_ctl);
    cvb_pose *pbuf = (cvb_pose *)(base + o_pose), *eT = (cvb_pose *)(base + o_eT), *gp = (cvb_pose *)(base + o_gp);
    uint8_t *sbuf = base + o_state;
    uint32_t *deg = (uint32_t *)(base + o_deg), *eoff = (uint32_t *)(base + o_eoff), *ev = (uint32_t *)(base + o_ev);
    uint32_t *eo = (uint32_t *)(base + o_eo), *gi = (uint32_t *)(base + o_gi);
    double *se3 = (double *)(base + o_se3), *gb = (double *)(base + o_gb), *gw = (double *)(base + o_gw);
    double *W = tri->method == CVB_TRI_SINE_L1 ? (double *)(base + o_W) : nullptr;
    int sms = 0, per_sm = 0;
    CVB_CUDA(ctx, cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, ctx->device));
    CVB_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_rec_steps, REC_NT, 0));
    if (per_sm < 1) return cvb_set_error(ctx, CVB_ECUDA, "k_rec_steps cannot be resident");
    // every block must be resident for the grid barrier; more than the larger stage needs would only wait at it
    const size_t need = std::max((E + REC_NT - 1) / REC_NT, ((size_t)V * 32 + REC_NT - 1) / REC_NT);
    const uint32_t grid = (uint32_t)std::max<size_t>(1, std::min<size_t>((size_t)sms * per_sm, need));
    const cvb_triangulator T = *tri;
    {
        CVB_PROF(ctx, "k_rec_init", 0);
        k_rec_init<<<1, 1, 0, st>>>(ctl);
        CVB_LAUNCH_CHECK(ctx);
        CVB_CUDA(ctx, cudaMemcpyAsync(pbuf, poses_dev, sizeof(cvb_pose) * V, cudaMemcpyDeviceToDevice, st));
        CVB_CUDA(ctx, cudaMemsetAsync(sbuf, 0, 2 * (size_t)V, st));
        if (n_obs) CVB_CUDA(ctx, cudaMemsetAsync(obs_state_dev, 0, n_obs, st));
    }
    for (uint32_t r = 0; r < cfg->reconstruction_optimization_iterations; r++) {
        {
            CVB_PROF(ctx, "k_rec_flatten", 0);
            CVB_CUDA(ctx, cudaMemsetAsync(deg, 0, sizeof(uint32_t) * V, st));
            if (C) {
                k_rec_count<<<cdiv(C, 256), 256, 0, st>>>(prm, ctl, cons_dev, sbuf, deg);
                CVB_LAUNCH_CHECK(ctx);
            }
            k_rec_scan<<<1, 32, 0, st>>>(prm, ctl, deg, eoff);
            CVB_LAUNCH_CHECK(ctx);
            if (C) {
                k_rec_place<<<cdiv((size_t)V * 32, 256), 256, 0, st>>>(prm, ctl, cons_dev, sbuf, eoff, ev, eo, eT);
                CVB_LAUNCH_CHECK(ctx);
            }
        }
        if (prm.iters) {
            CVB_PROF(ctx, "k_rec_steps", 0);
            void *args[] = {&prm, &ctl, &eoff, &ev, &eo, &eT, &se3, &pbuf, &sbuf, &r};
            CVB_CUDA(ctx, cudaLaunchCooperativeKernel((const void *)k_rec_steps, dim3(grid), dim3(REC_NT), args, 0, st));
        }
        {
            CVB_PROF(ctx, "k_rec_filter", 0);
            k_rec_present<<<1, 256, 0, st>>>(prm, ctl, sbuf);
            CVB_LAUNCH_CHECK(ctx);
            if (L) {
                k_rec_filter<<<cdiv(L, 128), 128, 0, st>>>(T, prm, ctl, pbuf, sbuf, view_off_dev, bear_dev, lm_off_dev, obs_dev, L, obs_state_dev,
                                                            gp, gb, gw, gi, W);
                CVB_LAUNCH_CHECK(ctx);
            }
            k_rec_judge<<<1, 1, 0, st>>>(prm, ctl, r);
            CVB_LAUNCH_CHECK(ctx);
        }
    }
    {
        CVB_PROF(ctx, "k_rec_finish", 0);
        k_rec_finish<<<1, 256, 0, st>>>(prm, ctl, pbuf, sbuf, cfg->reconstruction_optimization_iterations, res_dev, poses_out_dev, view_state_dev);
        CVB_LAUNCH_CHECK(ctx);
    }
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    return 0;
}

int optimize_reconstruction(cvb_ctx *ctx, const cvb_recon_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses,
                            const uint32_t *vo, const uint32_t *vl, const double *bear, uint32_t L, const uint32_t *lo, const uint32_t *obs,
                            const cvb_view_constraint *cons, uint32_t C, cvb_recon_result *res, cvb_pose *poses_out, uint8_t *view_state,
                            uint8_t *obs_state) {
    if (!ctx) return CVB_EINVAL;
    if (!cfg || !tri || !poses || !res || !poses_out || !view_state) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (optimize_reconstruction_check(V, vo, vl, L, lo, obs, cons, C)) return cvb_set_error(ctx, CVB_EINVAL, "malformed snapshot or constraints");
    const uint32_t nf = vo[V], no = lo[L];
    if ((nf && !bear) || (no && !obs_state)) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    size_t off = 0;
    const size_t i_pose = off; off += con_align(sizeof(cvb_pose) * V);
    const size_t i_vo = off; off += con_align(sizeof(uint32_t) * (V + 1));
    const size_t i_vl = off; off += con_align(sizeof(uint32_t) * (size_t)nf);
    const size_t i_bear = off; off += con_align(sizeof(double) * 3 * (size_t)nf);
    const size_t i_lo = off; off += con_align(sizeof(uint32_t) * ((size_t)L + 1));
    const size_t i_obs = off; off += con_align(sizeof(uint32_t) * 2 * (size_t)no);
    const size_t i_cons = off; off += con_align(sizeof(cvb_view_constraint) * (size_t)C);
    const size_t i_res = off; off += con_align(sizeof(cvb_recon_result));
    const size_t i_pout = off; off += con_align(sizeof(cvb_pose) * V);
    const size_t i_vs = off; off += con_align(V);
    const size_t i_os = off; off += con_align(no);
    GeomWorkspace *g = gws(ctx);
    int rc;
    if ((rc = g->out.ensure(ctx, off))) return rc;
    unsigned char *b = (unsigned char *)g->out.p;
    cudaStream_t st = ctx->stream;
    CVB_CUDA(ctx, cudaMemcpyAsync(b + i_pose, poses, sizeof(cvb_pose) * V, cudaMemcpyHostToDevice, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(b + i_vo, vo, sizeof(uint32_t) * (V + 1), cudaMemcpyHostToDevice, st));
    if (nf) CVB_CUDA(ctx, cudaMemcpyAsync(b + i_vl, vl, sizeof(uint32_t) * (size_t)nf, cudaMemcpyHostToDevice, st));
    if (nf) CVB_CUDA(ctx, cudaMemcpyAsync(b + i_bear, bear, sizeof(double) * 3 * (size_t)nf, cudaMemcpyHostToDevice, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(b + i_lo, lo, sizeof(uint32_t) * ((size_t)L + 1), cudaMemcpyHostToDevice, st));
    if (no) CVB_CUDA(ctx, cudaMemcpyAsync(b + i_obs, obs, sizeof(uint32_t) * 2 * (size_t)no, cudaMemcpyHostToDevice, st));
    if (C) CVB_CUDA(ctx, cudaMemcpyAsync(b + i_cons, cons, sizeof(cvb_view_constraint) * (size_t)C, cudaMemcpyHostToDevice, st));
    if ((rc = optimize_reconstruction_dev(ctx, cfg, tri, V, (const cvb_pose *)(b + i_pose), (const uint32_t *)(b + i_vo),
                                          (const uint32_t *)(b + i_vl), (const double *)(b + i_bear), nf, L, (const uint32_t *)(b + i_lo),
                                          (const uint32_t *)(b + i_obs), no, (const cvb_view_constraint *)(b + i_cons), C,
                                          (cvb_recon_result *)(b + i_res), (cvb_pose *)(b + i_pout), b + i_vs, b + i_os)))
        return rc;
    CVB_CUDA(ctx, cudaMemcpyAsync(res, b + i_res, sizeof(cvb_recon_result), cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(poses_out, b + i_pout, sizeof(cvb_pose) * V, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(view_state, b + i_vs, V, cudaMemcpyDeviceToHost, st));
    if (no) CVB_CUDA(ctx, cudaMemcpyAsync(obs_state, b + i_os, no, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    return 0;
}

// ---- cv-sfm's reconstruction export (C names in export_abi.cu, include/cvb200_export.h; kernels in export_dev.cuh) --------------------
void export_cfg_default(cvb_export_cfg *c) {
    if (!c) return;
    memset(c, 0, sizeof(*c));
    c->robust_observation_incidence_minimum_cosine_distance = 1e-3;
    c->robust_minimum_observations = 3;
}

int export_check(uint32_t V, const uint32_t *vo, const uint32_t *vl, uint32_t L, const uint32_t *lo, const uint32_t *obs,
                 const cvb_view_constraint *cons, uint32_t C, uint32_t first_view) {
    if (optimize_reconstruction_check(V, vo, vl, L, lo, obs, cons, C)) return CVB_EINVAL;
    return first_view < V ? 0 : CVB_EINVAL;
}

namespace {

// the arguments every export entry checks; n_features against view_offsets[V] (read back)
int export_args(cvb_ctx *ctx, const cvb_export_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const uint32_t *view_off_dev,
                uint32_t n_features) {
    if (tri->method < CVB_TRI_LINEAR_EIGEN || tri->method > CVB_TRI_MEAN_MEAN)
        return cvb_set_error(ctx, tri->method >= CVB_TRI_RELATIVE_DLT && tri->method <= CVB_TRI_ANGULAR_LINF ? CVB_EUNSUPPORTED : CVB_EINVAL,
                             "triangulator method %d: the export takes a TriangulatorObservations (methods 0-2)", tri->method);
    if (V == 0) return cvb_set_error(ctx, CVB_EINVAL, "no views");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    uint32_t nf = 0;
    CVB_CUDA(ctx, cudaMemcpyAsync(&nf, view_off_dev + V, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    if (nf != n_features) return cvb_set_error(ctx, CVB_EINVAL, "view_offsets[V] = %u, n_features %u", nf, n_features);
    return 0;
}

// the robust points and states of every landmark (list == nullptr) or of the n landmarks in list, into the workspace; block_cnt (may be
// nullptr) gets the POINT count of every CTA of EXP_NT landmarks
struct ExpRobust { double *points; uint8_t *state; uint32_t *block_cnt, *n_points; };
int export_robust(cvb_ctx *ctx, const cvb_export_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses_dev,
                  const uint32_t *view_off_dev, const double *bear_dev, uint32_t L, const uint32_t *lm_off_dev, const uint32_t *obs_dev,
                  uint32_t n_obs, const uint32_t *list, uint32_t n, bool count, ExpRobust &out) {
    const uint32_t nb = cdiv(std::max<uint32_t>(L, 1), EXP_NT);
    size_t off = 0;
    const size_t o_pose = off; off += con_align(sizeof(cvb_pose) * std::max<size_t>(n_obs, 1));
    const size_t o_bear = off; off += con_align(sizeof(double) * 3 * std::max<size_t>(n_obs, 1));
    const size_t o_world = off; off += con_align(sizeof(double) * 3 * std::max<size_t>(n_obs, 1));
    const size_t o_W = off; off += tri->method == CVB_TRI_SINE_L1 ? con_align(sizeof(double) * 6 * std::max<size_t>(n_obs, 1)) : 0;
    const size_t o_pts = off; off += con_align(sizeof(double) * 4 * std::max<size_t>(L, 1));
    const size_t o_state = off; off += con_align(std::max<size_t>(L, 1));
    const size_t o_cnt = off; off += con_align(sizeof(uint32_t) * ((size_t)nb + 1));
    GeomWorkspace *g = gws(ctx);
    int rc;
    if ((rc = g->exp.ensure(ctx, off))) return rc;
    unsigned char *base = (unsigned char *)g->exp.p;
    cvb_pose *obs_pose = (cvb_pose *)(base + o_pose);
    double *obs_bear = (double *)(base + o_bear), *obs_world = (double *)(base + o_world);
    double *W = tri->method == CVB_TRI_SINE_L1 ? (double *)(base + o_W) : nullptr;
    out.points = (double *)(base + o_pts);
    out.state = base + o_state;
    out.block_cnt = (uint32_t *)(base + o_cnt);
    out.n_points = out.block_cnt + nb;
    cudaStream_t st = ctx->stream;
    if (n_obs) {
        CVB_PROF(ctx, "k_con_gather_obs", 0);
        k_con_gather_obs<<<cdiv(n_obs, 256), 256, 0, st>>>(poses_dev, view_off_dev, bear_dev, obs_dev, n_obs, obs_pose, obs_bear, obs_world);
        CVB_LAUNCH_CHECK(ctx);
    }
    if (n) {
        CVB_PROF(ctx, "k_exp_robust", 0);
        k_exp_robust<<<cdiv(n, EXP_NT), EXP_NT, 0, st>>>(*tri, lm_off_dev, list, n, obs_pose, obs_bear, obs_world, W,
                                                         std::min(cfg->robust_minimum_observations, V),
                                                         cfg->robust_observation_incidence_minimum_cosine_distance, out.points, out.state,
                                                         count ? out.block_cnt : nullptr);
        CVB_LAUNCH_CHECK(ctx);
    }
    return 0;
}

}  // namespace

int robust_landmarks_dev(cvb_ctx *ctx, const cvb_export_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses_dev,
                         const uint32_t *view_off_dev, const uint32_t *view_lm_dev, const double *bear_dev, uint32_t n_features, uint32_t L,
                         const uint32_t *lm_off_dev, const uint32_t *obs_dev, uint32_t n_obs, double *points_dev, uint8_t *state_dev) {
    if (!ctx) return CVB_EINVAL;
    if (!cfg || !tri || !poses_dev || !view_off_dev || !lm_off_dev || (n_features && (!view_lm_dev || !bear_dev)) || (n_obs && !obs_dev) ||
        (L && (!points_dev || !state_dev)))
        return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    int rc;
    if ((rc = export_args(ctx, cfg, tri, V, view_off_dev, n_features))) return rc;
    ExpRobust r;
    if ((rc = export_robust(ctx, cfg, tri, V, poses_dev, view_off_dev, bear_dev, L, lm_off_dev, obs_dev, n_obs, nullptr, L, false, r))) return rc;
    cudaStream_t st = ctx->stream;
    if (L) {
        CVB_CUDA(ctx, cudaMemcpyAsync(points_dev, r.points, sizeof(double) * 4 * (size_t)L, cudaMemcpyDeviceToDevice, st));
        CVB_CUDA(ctx, cudaMemcpyAsync(state_dev, r.state, L, cudaMemcpyDeviceToDevice, st));
    }
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    return 0;
}

int export_reconstruction_dev(cvb_ctx *ctx, const cvb_export_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses_dev,
                              const uint32_t *view_off_dev, const uint32_t *view_lm_dev, const double *bear_dev, const uint8_t *colors_dev,
                              uint32_t n_features, uint32_t L, const uint32_t *lm_off_dev, const uint32_t *obs_dev, uint32_t n_obs,
                              double *points_dev, uint8_t *colors_out_dev, uint32_t *n_points_dev, cvb_export_camera *cameras_dev,
                              double *mean_dev) {
    if (!ctx) return CVB_EINVAL;
    if (!cfg || !tri || !poses_dev || !view_off_dev || !lm_off_dev || !n_points_dev || !cameras_dev ||
        (n_features && (!view_lm_dev || !bear_dev || !colors_dev)) || (n_obs && !obs_dev) || (L && (!points_dev || !colors_out_dev)))
        return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    int rc;
    if ((rc = export_args(ctx, cfg, tri, V, view_off_dev, n_features))) return rc;
    ExpRobust r;
    if ((rc = export_robust(ctx, cfg, tri, V, poses_dev, view_off_dev, bear_dev, L, lm_off_dev, obs_dev, n_obs, nullptr, L, true, r))) return rc;
    cudaStream_t st = ctx->stream;
    const uint32_t nb = cdiv(L, EXP_NT);
    {
        CVB_PROF(ctx, "k_exp_compact", 0);
        k_exp_scan<<<1, 32, 0, st>>>(nb, r.block_cnt, r.n_points);
        CVB_LAUNCH_CHECK(ctx);
        if (L) {
            k_exp_compact<<<nb, EXP_NT, 0, st>>>(L, r.points, r.state, r.block_cnt, view_off_dev, lm_off_dev, obs_dev, colors_dev, points_dev,
                                                 colors_out_dev);
            CVB_LAUNCH_CHECK(ctx);
        }
        CVB_CUDA(ctx, cudaMemcpyAsync(n_points_dev, r.n_points, sizeof(uint32_t), cudaMemcpyDeviceToDevice, st));
    }
    {
        CVB_PROF(ctx, "k_exp_cameras", 0);
        k_exp_cameras<<<cdiv((size_t)V * 32, 256), 256, 0, st>>>(V, poses_dev, view_off_dev, view_lm_dev, r.points, r.state, cameras_dev,
                                                                 mean_dev);
        CVB_LAUNCH_CHECK(ctx);
    }
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    return 0;
}

int normalize_reconstruction_dev(cvb_ctx *ctx, const cvb_export_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses_dev,
                                 const uint32_t *view_off_dev, const uint32_t *view_lm_dev, const double *bear_dev, uint32_t n_features,
                                 uint32_t L, const uint32_t *lm_off_dev, const uint32_t *obs_dev, uint32_t n_obs,
                                 const cvb_view_constraint *cons_dev, uint32_t C, uint32_t first_view, cvb_pose *poses_out_dev,
                                 cvb_view_constraint *cons_out_dev, cvb_normalize_result *res_dev) {
    if (!ctx) return CVB_EINVAL;
    if (!cfg || !tri || !poses_dev || !view_off_dev || !lm_off_dev || !poses_out_dev || !res_dev ||
        (n_features && (!view_lm_dev || !bear_dev)) || (n_obs && !obs_dev) || (C && (!cons_dev || !cons_out_dev)))
        return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (V && first_view >= V) return cvb_set_error(ctx, CVB_EINVAL, "first_view %u of %u views", first_view, V);
    int rc;
    if ((rc = export_args(ctx, cfg, tri, V, view_off_dev, n_features))) return rc;
    cudaStream_t st = ctx->stream;
    // only the first view's landmarks are triangulated: their list is the view's stretch of view_landmarks
    uint32_t f[2];
    CVB_CUDA(ctx, cudaMemcpyAsync(f, view_off_dev + first_view, sizeof(f), cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    ExpRobust r;
    if ((rc = export_robust(ctx, cfg, tri, V, poses_dev, view_off_dev, bear_dev, L, lm_off_dev, obs_dev, n_obs, view_lm_dev + f[0], f[1] - f[0],
                            false, r)))
        return rc;
    {
        CVB_PROF(ctx, "k_exp_normalize", 0);
        k_exp_first_mean<<<1, 32, 0, st>>>(first_view, poses_dev, view_off_dev, view_lm_dev, r.points, r.state, res_dev);
        CVB_LAUNCH_CHECK(ctx);
        k_exp_normalize<<<cdiv(std::max(V, C), 256), 256, 0, st>>>(V, C, first_view, poses_dev, cons_dev, res_dev, poses_out_dev, cons_out_dev);
        CVB_LAUNCH_CHECK(ctx);
    }
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    return 0;
}

namespace {

// the snapshot's host arrays into the context's output workspace; the offsets of what follows them start at `off`
struct ExpUpload { size_t pose, vo, vl, bear, col, lo, obs, cons, end; };
int export_upload(cvb_ctx *ctx, uint32_t V, const cvb_pose *poses, const uint32_t *vo, const uint32_t *vl, const double *bear,
                  const uint8_t *colors, uint32_t L, const uint32_t *lo, const uint32_t *obs, const cvb_view_constraint *cons, uint32_t C,
                  size_t extra, ExpUpload &u, unsigned char *&b) {
    const uint32_t nf = vo[V], no = lo[L];
    size_t off = 0;
    u.pose = off; off += con_align(sizeof(cvb_pose) * V);
    u.vo = off; off += con_align(sizeof(uint32_t) * (V + 1));
    u.vl = off; off += con_align(sizeof(uint32_t) * (size_t)nf);
    u.bear = off; off += con_align(sizeof(double) * 3 * (size_t)nf);
    u.col = off; off += con_align(3 * (size_t)nf);
    u.lo = off; off += con_align(sizeof(uint32_t) * ((size_t)L + 1));
    u.obs = off; off += con_align(sizeof(uint32_t) * 2 * (size_t)no);
    u.cons = off; off += con_align(sizeof(cvb_view_constraint) * (size_t)C);
    u.end = off;
    GeomWorkspace *g = gws(ctx);
    int rc;
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    if ((rc = g->out.ensure(ctx, off + extra))) return rc;
    b = (unsigned char *)g->out.p;
    cudaStream_t st = ctx->stream;
    CVB_CUDA(ctx, cudaMemcpyAsync(b + u.pose, poses, sizeof(cvb_pose) * V, cudaMemcpyHostToDevice, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(b + u.vo, vo, sizeof(uint32_t) * (V + 1), cudaMemcpyHostToDevice, st));
    if (nf) CVB_CUDA(ctx, cudaMemcpyAsync(b + u.vl, vl, sizeof(uint32_t) * (size_t)nf, cudaMemcpyHostToDevice, st));
    if (nf) CVB_CUDA(ctx, cudaMemcpyAsync(b + u.bear, bear, sizeof(double) * 3 * (size_t)nf, cudaMemcpyHostToDevice, st));
    if (nf && colors) CVB_CUDA(ctx, cudaMemcpyAsync(b + u.col, colors, 3 * (size_t)nf, cudaMemcpyHostToDevice, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(b + u.lo, lo, sizeof(uint32_t) * ((size_t)L + 1), cudaMemcpyHostToDevice, st));
    if (no) CVB_CUDA(ctx, cudaMemcpyAsync(b + u.obs, obs, sizeof(uint32_t) * 2 * (size_t)no, cudaMemcpyHostToDevice, st));
    if (C) CVB_CUDA(ctx, cudaMemcpyAsync(b + u.cons, cons, sizeof(cvb_view_constraint) * (size_t)C, cudaMemcpyHostToDevice, st));
    return 0;
}

}  // namespace

int robust_landmarks(cvb_ctx *ctx, const cvb_export_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses,
                     const uint32_t *vo, const uint32_t *vl, const double *bear, uint32_t L, const uint32_t *lo, const uint32_t *obs,
                     double *points, uint8_t *state) {
    if (!ctx) return CVB_EINVAL;
    if (!cfg || !tri || !poses) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (export_check(V, vo, vl, L, lo, obs, nullptr, 0, 0)) return cvb_set_error(ctx, CVB_EINVAL, "malformed snapshot");
    if ((vo[V] && !bear) || (L && (!points || !state))) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    ExpUpload u;
    unsigned char *b;
    const size_t i_pts = con_align(sizeof(double) * 4 * (size_t)L);
    int rc;
    if ((rc = export_upload(ctx, V, poses, vo, vl, bear, nullptr, L, lo, obs, nullptr, 0, i_pts + con_align(L), u, b))) return rc;
    double *pts = (double *)(b + u.end);
    uint8_t *stt = b + u.end + i_pts;
    if ((rc = robust_landmarks_dev(ctx, cfg, tri, V, (const cvb_pose *)(b + u.pose), (const uint32_t *)(b + u.vo), (const uint32_t *)(b + u.vl),
                                   (const double *)(b + u.bear), vo[V], L, (const uint32_t *)(b + u.lo), (const uint32_t *)(b + u.obs), lo[L],
                                   pts, stt)))
        return rc;
    cudaStream_t st = ctx->stream;
    if (L) {
        CVB_CUDA(ctx, cudaMemcpyAsync(points, pts, sizeof(double) * 4 * (size_t)L, cudaMemcpyDeviceToHost, st));
        CVB_CUDA(ctx, cudaMemcpyAsync(state, stt, L, cudaMemcpyDeviceToHost, st));
    }
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    return 0;
}

int export_reconstruction(cvb_ctx *ctx, const cvb_export_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses,
                          const uint32_t *vo, const uint32_t *vl, const double *bear, const uint8_t *colors, uint32_t L, const uint32_t *lo,
                          const uint32_t *obs, double *points, uint8_t *point_colors, uint32_t *n_points, cvb_export_camera *cameras,
                          double *mean) {
    if (!ctx) return CVB_EINVAL;
    if (!cfg || !tri || !poses || !n_points || !cameras) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (export_check(V, vo, vl, L, lo, obs, nullptr, 0, 0)) return cvb_set_error(ctx, CVB_EINVAL, "malformed snapshot");
    if ((vo[V] && (!bear || !colors)) || (L && (!points || !point_colors))) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    size_t x = 0;
    const size_t i_pts = x; x += con_align(sizeof(double) * 3 * (size_t)L);
    const size_t i_col = x; x += con_align(3 * (size_t)L);
    const size_t i_n = x; x += con_align(sizeof(uint32_t));
    const size_t i_cam = x; x += con_align(sizeof(cvb_export_camera) * V);
    const size_t i_mean = x; x += con_align(sizeof(double) * V);
    ExpUpload u;
    unsigned char *b;
    int rc;
    if ((rc = export_upload(ctx, V, poses, vo, vl, bear, colors, L, lo, obs, nullptr, 0, x, u, b))) return rc;
    unsigned char *o = b + u.end;
    if ((rc = export_reconstruction_dev(ctx, cfg, tri, V, (const cvb_pose *)(b + u.pose), (const uint32_t *)(b + u.vo),
                                        (const uint32_t *)(b + u.vl), (const double *)(b + u.bear), b + u.col, vo[V], L,
                                        (const uint32_t *)(b + u.lo), (const uint32_t *)(b + u.obs), lo[L], (double *)(o + i_pts), o + i_col,
                                        (uint32_t *)(o + i_n), (cvb_export_camera *)(o + i_cam), (double *)(o + i_mean))))
        return rc;
    cudaStream_t st = ctx->stream;
    CVB_CUDA(ctx, cudaMemcpyAsync(n_points, o + i_n, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(cameras, o + i_cam, sizeof(cvb_export_camera) * V, cudaMemcpyDeviceToHost, st));
    if (mean) CVB_CUDA(ctx, cudaMemcpyAsync(mean, o + i_mean, sizeof(double) * V, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    if (*n_points) {
        CVB_CUDA(ctx, cudaMemcpyAsync(points, o + i_pts, sizeof(double) * 3 * (size_t)*n_points, cudaMemcpyDeviceToHost, st));
        CVB_CUDA(ctx, cudaMemcpyAsync(point_colors, o + i_col, 3 * (size_t)*n_points, cudaMemcpyDeviceToHost, st));
        CVB_CUDA(ctx, cvb_wait(ctx, st));
    }
    return 0;
}

int normalize_reconstruction(cvb_ctx *ctx, const cvb_export_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses,
                             const uint32_t *vo, const uint32_t *vl, const double *bear, uint32_t L, const uint32_t *lo, const uint32_t *obs,
                             const cvb_view_constraint *cons, uint32_t C, uint32_t first_view, cvb_pose *poses_out,
                             cvb_view_constraint *cons_out, cvb_normalize_result *res) {
    if (!ctx) return CVB_EINVAL;
    if (!cfg || !tri || !poses || !poses_out || !res || (C && !cons_out)) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (export_check(V, vo, vl, L, lo, obs, cons, C, first_view)) return cvb_set_error(ctx, CVB_EINVAL, "malformed snapshot or constraints");
    if (vo[V] && !bear) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    size_t x = 0;
    const size_t i_pout = x; x += con_align(sizeof(cvb_pose) * V);
    const size_t i_cout = x; x += con_align(sizeof(cvb_view_constraint) * (size_t)C);
    const size_t i_res = x; x += con_align(sizeof(cvb_normalize_result));
    ExpUpload u;
    unsigned char *b;
    int rc;
    if ((rc = export_upload(ctx, V, poses, vo, vl, bear, nullptr, L, lo, obs, cons, C, x, u, b))) return rc;
    unsigned char *o = b + u.end;
    if ((rc = normalize_reconstruction_dev(ctx, cfg, tri, V, (const cvb_pose *)(b + u.pose), (const uint32_t *)(b + u.vo),
                                           (const uint32_t *)(b + u.vl), (const double *)(b + u.bear), vo[V], L, (const uint32_t *)(b + u.lo),
                                           (const uint32_t *)(b + u.obs), lo[L], (const cvb_view_constraint *)(b + u.cons), C, first_view,
                                           (cvb_pose *)(o + i_pout), (cvb_view_constraint *)(o + i_cout), (cvb_normalize_result *)(o + i_res))))
        return rc;
    cudaStream_t st = ctx->stream;
    CVB_CUDA(ctx, cudaMemcpyAsync(poses_out, o + i_pout, sizeof(cvb_pose) * V, cudaMemcpyDeviceToHost, st));
    if (C) CVB_CUDA(ctx, cudaMemcpyAsync(cons_out, o + i_cout, sizeof(cvb_view_constraint) * (size_t)C, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(res, o + i_res, sizeof(cvb_normalize_result), cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    return 0;
}

// ---- cv-sfm's frame registration (C names in register_abi.cu, include/cvb200_register.h; kernels in register_dev.cuh) ------------------
void register_cfg_default(cvb_register_cfg *c) {
    if (!c) return;
    memset(c, 0, sizeof(*c));
    c->single_view_optimization_rate = 1e-3;
    c->maximum_sine_distance = 0.1;
    c->maximum_cosine_distance = 1e-5;
    c->robust_observation_incidence_minimum_cosine_distance = 1e-3;
    c->single_view_match_better_by = 24;
    c->single_view_initial_features = 1u << 13;
    c->single_view_minimum_landmarks = 1u << 5;
    c->single_view_optimization_num_matches = 1u << 11;
    c->single_view_filter_loop_iterations = 5;
    c->single_view_patience = 100000;
    c->single_view_minimum_robust_landmarks = 1u << 6;
    c->robust_minimum_observations = 3;
}

int register_check(uint32_t V, const uint32_t *vo, const uint32_t *vl, uint32_t L, const uint32_t *lo, const uint32_t *obs,
                   const uint32_t *view_matches, uint32_t H) {
    return view_constraints_check(V, vo, vl, L, lo, obs, view_matches, H);
}

int register_frame_dev(cvb_ctx *ctx, const cvb_register_cfg *cfg, const cvb_triangulator *tri, const cvb_arrsac_cfg *arrsac, cvb_rng *rng,
                       uint32_t V, const cvb_pose *poses_dev, const uint32_t *view_off_dev, const uint32_t *view_lm_dev, const double *bear_dev,
                       const uint8_t *desc_dev, uint32_t n_features, uint32_t L, const uint32_t *lm_off_dev, const uint32_t *obs_dev,
                       uint32_t n_obs, const uint8_t *new_desc_dev, const double *new_bear_dev, uint32_t N, const uint32_t *view_matches,
                       uint32_t H, cvb_register_result *res_dev, cvb_register_match *matches_dev, uint32_t *inliers_dev,
                       cvb_register_stats *stats_dev) {
    if (!ctx) return CVB_EINVAL;
    if (!cfg || !tri || !arrsac || !rng || !poses_dev || !view_off_dev || !lm_off_dev || !res_dev || (H && !view_matches) ||
        (n_features && (!view_lm_dev || !bear_dev || !desc_dev)) || (n_obs && !obs_dev) ||
        (N && (!new_desc_dev || !new_bear_dev || !matches_dev)))
        return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (tri->method < CVB_TRI_LINEAR_EIGEN || tri->method > CVB_TRI_MEAN_MEAN)
        return cvb_set_error(ctx, tri->method >= CVB_TRI_RELATIVE_DLT && tri->method <= CVB_TRI_ANGULAR_LINF ? CVB_EUNSUPPORTED : CVB_EINVAL,
                             "triangulator method %d: registration takes a TriangulatorObservations (methods 0-2)", tri->method);
    if (V == 0) return cvb_set_error(ctx, CVB_EINVAL, "no views");
    if (N && cfg->single_view_initial_features == 0)   // the reference's subset range would stay empty forever
        return cvb_set_error(ctx, CVB_EINVAL, "single_view_initial_features must be > 0");
    for (uint32_t h = 0; h < H; h++)
        if (view_matches[h] >= V) return cvb_set_error(ctx, CVB_EINVAL, "view match %u of %u views", view_matches[h], V);
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    // the k-NN needs each matched view's stretch of the descriptors: the view offsets, read back once
    std::vector<uint32_t> vo(V + 1);
    CVB_CUDA(ctx, cudaMemcpyAsync(vo.data(), view_off_dev, sizeof(uint32_t) * (V + 1), cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    if (vo[V] != n_features) return cvb_set_error(ctx, CVB_EINVAL, "view_offsets[V] = %u, n_features %u", vo[V], n_features);
    const uint32_t N1 = std::max<uint32_t>(N, 1), H1 = std::max<uint32_t>(H, 1), n2max = con_pow2(N1);
    const size_t S = (size_t)n_obs + N1;   // scratch slots: each landmark is in at most one kept match, plus one slot per match
    const bool sine = tri->method == CVB_TRI_SINE_L1;
    size_t off = 0;
    const size_t o_ctl = off; off += con_align(sizeof(RegCtl));
    const size_t o_idx = off; off += con_align(sizeof(uint32_t) * 3 * (size_t)H1 * N1);
    const size_t o_dist = off; off += con_align(sizeof(uint32_t) * 3 * (size_t)H1 * N1);
    const size_t o_vbase = off; off += con_align(sizeof(uint32_t) * H1);
    const size_t o_dec = off; off += con_align(sizeof(uint2) * N1);
    const size_t o_orig = off; off += con_align(sizeof(RegMatch) * N1);
    const size_t o_cnt = off; off += con_align(sizeof(uint32_t) * std::max<size_t>(L, 1));
    const size_t o_keys = off; off += con_align(sizeof(unsigned long long) * n2max);
    const size_t o_list = off; off += con_align(sizeof(uint32_t) * N1);
    const size_t o_soff = off; off += con_align(sizeof(uint32_t) * N1);
    const size_t o_rob = off; off += con_align(N1);
    const size_t o_cons = off; off += con_align(N1);
    const size_t o_fin = off; off += con_align(N1);
    const size_t o_pt = off; off += con_align(sizeof(double) * 4 * N1);
    const size_t o_sp = off; off += con_align(sizeof(cvb_pose) * S);
    const size_t o_sb = off; off += con_align(sizeof(double) * 3 * S);
    const size_t o_sw = off; off += con_align(sizeof(double) * 3 * S);
    const size_t o_W = off; off += sine ? con_align(sizeof(double) * 6 * S) : 0;
    const size_t o_mb = off; off += con_align(sizeof(double) * 3 * N1);
    const size_t o_mw = off; off += con_align(sizeof(double) * 4 * N1);
    const size_t o_rb = off; off += con_align(sizeof(double) * 3 * N1);
    const size_t o_rw = off; off += con_align(sizeof(double) * 4 * N1);
    const size_t o_inl = off; off += con_align(sizeof(uint32_t) * N1);
    GeomWorkspace *g = gws(ctx);
    int rc;
    if ((rc = g->reg.ensure(ctx, off))) return rc;
    unsigned char *b = (unsigned char *)g->reg.p;
    RegCtl *ctl = (RegCtl *)(b + o_ctl);
    uint32_t *kidx = (uint32_t *)(b + o_idx), *kdist = (uint32_t *)(b + o_dist), *vbase = (uint32_t *)(b + o_vbase);
    uint2 *dec = (uint2 *)(b + o_dec);
    RegMatch *orig = (RegMatch *)(b + o_orig);
    uint32_t *counts = (uint32_t *)(b + o_cnt), *list = (uint32_t *)(b + o_list), *soff = (uint32_t *)(b + o_soff), *inl = (uint32_t *)(b + o_inl);
    unsigned long long *keys = (unsigned long long *)(b + o_keys);
    uint8_t *rob = b + o_rob, *cons = b + o_cons, *fin = b + o_fin;
    double *pt = (double *)(b + o_pt), *sb = (double *)(b + o_sb), *sw = (double *)(b + o_sw), *W = sine ? (double *)(b + o_W) : nullptr;
    double *mb = (double *)(b + o_mb), *mw = (double *)(b + o_mw), *rb = (double *)(b + o_rb), *rw = (double *)(b + o_rw);
    cvb_pose *sp = (cvb_pose *)(b + o_sp);
    std::vector<uint32_t> hbase(H1, 0);
    for (uint32_t h = 0; h < H; h++) hbase[h] = vo[view_matches[h]];
    CVB_CUDA(ctx, cudaMemcpyAsync(vbase, hbase.data(), sizeof(uint32_t) * H1, cudaMemcpyHostToDevice, st));
    CVB_CUDA(ctx, cudaMemsetAsync(ctl, 0, sizeof(RegCtl), st));
    CVB_CUDA(ctx, cudaMemsetAsync(rob, 0, N1, st));
    RegParams prm;
    prm.max_sin = cfg->maximum_sine_distance;
    prm.max_cos = cfg->maximum_cosine_distance;
    prm.inc = cfg->robust_observation_incidence_minimum_cosine_distance;
    prm.better_by = cfg->single_view_match_better_by;
    prm.min_obs = std::min(cfg->robust_minimum_observations, V);
    prm.min_landmarks = cfg->single_view_minimum_landmarks;
    prm.num_matches = cfg->single_view_optimization_num_matches;
    prm.iters = cfg->single_view_filter_loop_iterations;
    prm.min_robust_landmarks = cfg->single_view_minimum_robust_landmarks;
    uint32_t r0 = 0, r1 = std::min(cfg->single_view_initial_features, N), subset = 0;
    for (;;) {
        subset++;
        const uint32_t n = r1 - r0, n2 = con_pow2(std::max<uint32_t>(r1, 1));
        {
            CVB_PROF(ctx, "register_match", 0);
            k_reg_begin<<<1, 1, 0, st>>>(ctl);
            CVB_LAUNCH_CHECK(ctx);
            for (uint32_t hh = 0; hh < H && n; hh++) {
                const uint32_t v = view_matches[hh], m = vo[v + 1] - vo[v];
                uint32_t *ki = kidx + 3 * (size_t)hh * n, *kd = kdist + 3 * (size_t)hh * n;
                if (m == 0) {
                    CVB_CUDA(ctx, cudaMemsetAsync(ki, 0xff, sizeof(uint32_t) * 3 * (size_t)n, st));
                    continue;
                }
                if ((rc = cvb_hamming_knn_dev(ctx, new_desc_dev + 64 * (size_t)r0, n, desc_dev + 64 * (size_t)vo[v], m, 3, ki, kd))) return rc;
            }
            if (n) {
                k_reg_candidates<<<cdiv(n, 128), 128, 0, st>>>(kidx, kdist, n, H, vbase, view_lm_dev, lm_off_dev, obs_dev, prm.better_by, dec, ctl);
                CVB_LAUNCH_CHECK(ctx);
                k_reg_append<<<1, 1024, 0, st>>>(dec, n, r0, orig, ctl);
                CVB_LAUNCH_CHECK(ctx);
            }
            if (L) CVB_CUDA(ctx, cudaMemsetAsync(counts, 0, sizeof(uint32_t) * L, st));
            k_reg_claims<<<cdiv(std::max<uint32_t>(r1, 1), 256), 256, 0, st>>>(orig, ctl, counts);
            CVB_LAUNCH_CHECK(ctx);
            k_reg_keys<<<cdiv(n2, 256), 256, 0, st>>>(orig, counts, lm_off_dev, ctl, n2, keys);
            CVB_LAUNCH_CHECK(ctx);
            k_reg_order<<<1, 1024, 0, st>>>(keys, n2, orig, lm_off_dev, ctl, list, soff);
            CVB_LAUNCH_CHECK(ctx);
            k_reg_gather<<<cdiv(std::max<uint32_t>(r1, 1), 128), 128, 0, st>>>(*tri, prm, ctl, orig, list, soff, poses_dev, view_off_dev, bear_dev,
                                                                                lm_off_dev, obs_dev, sp, sb, sw, W, pt, rob);
            CVB_LAUNCH_CHECK(ctx);
            k_reg_compact<<<1, 1024, 0, st>>>(0, 0, prm, ctl, orig, list, rob, pt, cons, new_bear_dev, mb, mw);
            CVB_LAUNCH_CHECK(ctx);
        }
        {
            CVB_PROF(ctx, "register_consensus", 0);
            if ((rc = cvb_arrsac_p3p_dev(ctx, arrsac, mb, mw, &ctl->cons_n, std::max<uint32_t>(r1, 1), rng, &ctl->model, inl,
                                         std::max<uint32_t>(r1, 1), &ctl->n_inl, &ctl->found)))
                return rc;
            k_reg_take<<<1, 1024, 0, st>>>(prm, ctl, inl, mb, mw, rb, rw);
            CVB_LAUNCH_CHECK(ctx);
        }
        {
            CVB_PROF(ctx, "register_filter", 0);
            for (uint32_t it = 0; it <= prm.iters; it++) {
                k_single_view_opt<<<1, OPT_NT, 0, st>>>(&ctl->pose[it & 1], rb, rw, ctl->opt_off, cfg->single_view_optimization_rate,
                                                        cfg->single_view_patience, &ctl->pose[(it + 1) & 1], &ctl->opt_upd);
                CVB_LAUNCH_CHECK(ctx);
                k_reg_consistent<<<cdiv(std::max<uint32_t>(r1, 1), 128), 128, 0, st>>>(*tri, prm, ctl, (it + 1) & 1, orig, list, soff, lm_off_dev,
                                                                                        new_bear_dev, sp, sb, W, cons);
                CVB_LAUNCH_CHECK(ctx);
                if (it < prm.iters) {
                    k_reg_compact<<<1, 1024, 0, st>>>(1, it + 1, prm, ctl, orig, list, rob, pt, cons, new_bear_dev, rb, rw);
                    CVB_LAUNCH_CHECK(ctx);
                }
            }
            k_reg_final<<<1, 1024, 0, st>>>(prm, ctl, (prm.iters + 1) & 1, subset, orig, list, rob, cons, fin, matches_dev, res_dev, stats_dev);
            CVB_LAUNCH_CHECK(ctx);
            if (inliers_dev && r1) CVB_CUDA(ctx, cudaMemcpyAsync(inliers_dev, inl, sizeof(uint32_t) * r1, cudaMemcpyDeviceToDevice, st));
        }
        RegCtl *h = (RegCtl *)cvb_pinned(ctx, sizeof(RegCtl));
        if (!h) return cvb_set_error(ctx, CVB_ENOMEM, "page-locked scratch");
        CVB_CUDA(ctx, cudaMemcpyAsync(h, ctl, sizeof(RegCtl), cudaMemcpyDeviceToHost, st));
        CVB_CUDA(ctx, cvb_wait(ctx, st));
        const int status = h->status;
        // the consensus ran on the reference's side exactly when the subset got past the robust-landmark count; otherwise the device run
        // (on a count of 0) consumed nothing and is closed without moving the generator, so that no run is left pending
        const bool ran = status != CVB_REGISTER_PANIC && status != CVB_REGISTER_FEW_ROBUST_LANDMARKS;
        if ((rc = cvb_arrsac_commit_rng(ctx, ran ? rng : nullptr, nullptr))) return rc;
        if (status == CVB_REGISTER_OK || status == CVB_REGISTER_PANIC || r1 == N) break;
        r0 = r1;
        r1 = (uint32_t)std::min<uint64_t>(2ull * r1, N);
    }
    return 0;
}

int register_frame(cvb_ctx *ctx, const cvb_register_cfg *cfg, const cvb_triangulator *tri, const cvb_arrsac_cfg *arrsac, cvb_rng *rng,
                   uint32_t V, const cvb_pose *poses, const uint32_t *vo, const uint32_t *vl, const double *bear, const uint8_t *desc, uint32_t L,
                   const uint32_t *lo, const uint32_t *obs, const uint8_t *new_desc, const double *new_bear, uint32_t N,
                   const uint32_t *view_matches, uint32_t H, cvb_register_result *res, cvb_register_match *matches, uint32_t *inliers,
                   cvb_register_stats *stats) {
    if (!ctx) return CVB_EINVAL;
    if (!cfg || !tri || !arrsac || !rng || !poses || !res || (N && (!new_desc || !new_bear || !matches)))
        return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (register_check(V, vo, vl, L, lo, obs, view_matches, H)) return cvb_set_error(ctx, CVB_EINVAL, "malformed snapshot or view matches");
    if (vo[V] && (!bear || !desc)) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    const uint32_t nf = vo[V];
    size_t x = 0;
    const size_t i_desc = x; x += con_align(64 * (size_t)nf);
    const size_t i_nd = x; x += con_align(64 * (size_t)N);
    const size_t i_nb = x; x += con_align(sizeof(double) * 3 * (size_t)N);
    const size_t i_res = x; x += con_align(sizeof(cvb_register_result));
    const size_t i_m = x; x += con_align(sizeof(cvb_register_match) * (size_t)N);
    const size_t i_st = x; x += con_align(sizeof(cvb_register_stats));
    const size_t i_inl = x; x += con_align(sizeof(uint32_t) * (size_t)N);
    ExpUpload u;
    unsigned char *b;
    int rc;
    if ((rc = export_upload(ctx, V, poses, vo, vl, bear, nullptr, L, lo, obs, nullptr, 0, x, u, b))) return rc;
    unsigned char *o = b + u.end;
    cudaStream_t st = ctx->stream;
    if (nf) CVB_CUDA(ctx, cudaMemcpyAsync(o + i_desc, desc, 64 * (size_t)nf, cudaMemcpyHostToDevice, st));
    if (N) CVB_CUDA(ctx, cudaMemcpyAsync(o + i_nd, new_desc, 64 * (size_t)N, cudaMemcpyHostToDevice, st));
    if (N) CVB_CUDA(ctx, cudaMemcpyAsync(o + i_nb, new_bear, sizeof(double) * 3 * (size_t)N, cudaMemcpyHostToDevice, st));
    if ((rc = register_frame_dev(ctx, cfg, tri, arrsac, rng, V, (const cvb_pose *)(b + u.pose), (const uint32_t *)(b + u.vo),
                                 (const uint32_t *)(b + u.vl), (const double *)(b + u.bear), o + i_desc, nf, L, (const uint32_t *)(b + u.lo),
                                 (const uint32_t *)(b + u.obs), lo[L], o + i_nd, (const double *)(o + i_nb), N, view_matches, H,
                                 (cvb_register_result *)(o + i_res), (cvb_register_match *)(o + i_m), inliers ? (uint32_t *)(o + i_inl) : nullptr,
                                 stats ? (cvb_register_stats *)(o + i_st) : nullptr)))
        return rc;
    CVB_CUDA(ctx, cudaMemcpyAsync(res, o + i_res, sizeof(cvb_register_result), cudaMemcpyDeviceToHost, st));
    if (stats) CVB_CUDA(ctx, cudaMemcpyAsync(stats, o + i_st, sizeof(cvb_register_stats), cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    if (res->n_matches) CVB_CUDA(ctx, cudaMemcpyAsync(matches, o + i_m, sizeof(cvb_register_match) * (size_t)res->n_matches, cudaMemcpyDeviceToHost, st));
    if (inliers && res->n_inliers) CVB_CUDA(ctx, cudaMemcpyAsync(inliers, o + i_inl, sizeof(uint32_t) * (size_t)res->n_inliers, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    return 0;
}

// ---- cv-sfm's frame incorporation (C names in incorporate_abi.cu, include/cvb200_incorporate.h; kernels in incorporate_dev.cuh) ---------
int incorporate_check(uint32_t V, const uint32_t *vo, const uint32_t *vl, uint32_t L, const uint32_t *lo, const uint32_t *obs,
                      const cvb_view_constraint *cons, uint32_t C, uint32_t N, const cvb_register_match *matches, uint32_t M,
                      const uint8_t *view_state, uint32_t n_view_state, const uint8_t *obs_state, uint32_t n_obs_state) {
    if (optimize_reconstruction_check(V, vo, vl, L, lo, obs, cons, C)) return CVB_EINVAL;
    if (M && !matches) return CVB_EINVAL;
    if (M) {
        std::vector<uint8_t> used(L, 0);
        for (uint32_t m = 0; m < M; m++) {
            const cvb_register_match &t = matches[m];
            if (t.feature >= N || (m && t.feature <= matches[m - 1].feature)) return CVB_EINVAL;
            if (t.landmark_a >= L || used[t.landmark_a]) return CVB_EINVAL;
            used[t.landmark_a] = 1;
            if (t.landmark_b == CVB_REGISTER_NONE) continue;
            if (t.landmark_b >= L || t.landmark_b == t.landmark_a || used[t.landmark_b]) return CVB_EINVAL;
            used[t.landmark_b] = 1;
            for (uint32_t i = lo[t.landmark_a]; i < lo[t.landmark_a + 1]; i++)   // merge_landmarks' assert!: the two share no view
                for (uint32_t j = lo[t.landmark_b]; j < lo[t.landmark_b + 1]; j++)
                    if (obs[2 * (size_t)i] == obs[2 * (size_t)j]) return CVB_EINVAL;
        }
    }
    if (view_state || obs_state) {
        if (!view_state || n_view_state != V || n_obs_state != lo[L] || (lo[L] && !obs_state)) return CVB_EINVAL;
        for (uint32_t v = 0; v < V; v++)
            if (view_state[v] > CVB_RECON_VIEW_NON_FINITE) return CVB_EINVAL;
        for (uint32_t o = 0; o < lo[L]; o++) {
            if (obs_state[o] > CVB_RECON_OBS_DROPPED) return CVB_EINVAL;
            if ((obs_state[o] == CVB_RECON_OBS_DROPPED) != (view_state[obs[2 * (size_t)o]] != CVB_RECON_VIEW_KEPT)) return CVB_EINVAL;
        }
        for (uint32_t l = 0; l < L; l++) {   // split_observation never splits a landmark's last observation
            uint32_t rest = 0;
            for (uint32_t o = lo[l]; o < lo[l + 1]; o++) rest += obs_state[o] != CVB_RECON_OBS_SPLIT;
            if (lo[l + 1] > lo[l] && rest == 0) return CVB_EINVAL;
        }
    }
    return 0;
}

namespace {

// exclusive scan of n pairs in place, the total into *total; tiles: cdiv(n, INC_TILE) pairs of scratch
int inc_scan(cvb_ctx *ctx, uint32_t n, uint2 *a, uint2 *tiles, uint2 *total) {
    cudaStream_t st = ctx->stream;
    const uint32_t nt = cdiv(n, INC_TILE);
    if (nt) {
        k_inc_tile_sums<<<nt, INC_NT, 0, st>>>(n, a, tiles);
        CVB_LAUNCH_CHECK(ctx);
    }
    k_inc_scan_tiles<<<1, INC_NT, 0, st>>>(nt, tiles, total);
    CVB_LAUNCH_CHECK(ctx);
    if (nt) {
        k_inc_scan_apply<<<nt, INC_NT, 0, st>>>(n, a, tiles);
        CVB_LAUNCH_CHECK(ctx);
    }
    return 0;
}

// the checks every entry makes of the snapshot sizes against the device (one read-back of view_offsets[V] and landmark_offsets[L])
int inc_sizes(cvb_ctx *ctx, uint32_t V, const uint32_t *view_off_dev, uint32_t n_features, uint32_t L, const uint32_t *lm_off_dev,
              uint32_t n_obs) {
    uint32_t *h = (uint32_t *)cvb_pinned(ctx, 2 * sizeof(uint32_t));
    if (!h) return cvb_set_error(ctx, CVB_ENOMEM, "page-locked scratch");
    CVB_CUDA(ctx, cudaMemcpyAsync(h, view_off_dev + V, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CVB_CUDA(ctx, cudaMemcpyAsync(h + 1, lm_off_dev + L, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    if (h[0] != n_features) return cvb_set_error(ctx, CVB_EINVAL, "view_offsets[V] = %u, n_features %u", h[0], n_features);
    if (h[1] != n_obs) return cvb_set_error(ctx, CVB_EINVAL, "landmark_offsets[L] = %u, n_observations %u", h[1], n_obs);
    return 0;
}

// add_view, enqueued on the context's stream (no wait); scratch in the context's incorporate scratch buffer
int add_view_enqueue(cvb_ctx *ctx, uint32_t V, const cvb_pose *poses_dev, const uint32_t *view_off_dev, const uint32_t *view_lm_dev,
                     const double *bear_dev, const uint8_t *desc_dev, const uint8_t *col_dev, uint32_t nf, uint32_t L, const uint32_t *lm_off_dev,
                     const uint32_t *obs_dev, uint32_t n_obs, const cvb_pose *new_pose_dev, const double *new_bear_dev, const uint8_t *new_desc_dev,
                     const uint8_t *new_col_dev, uint32_t N, const cvb_register_match *matches_dev, uint32_t M, cvb_pose *poses_out,
                     uint32_t *view_off_out, uint32_t *view_lm_out, double *bear_out, uint8_t *desc_out, uint8_t *col_out, uint32_t *lm_off_out,
                     uint32_t *obs_out, uint32_t *lmap, cvb_incorporate_counts *counts) {
    const uint32_t n = L + N, nt = cdiv(n, INC_TILE);
    size_t off = 0;
    const size_t o_role = off; off += con_align(sizeof(uint32_t) * std::max<size_t>(L, 1));
    const size_t o_featm = off; off += con_align(sizeof(uint32_t) * std::max<size_t>(N, 1));
    const size_t o_merges = off; off += con_align(sizeof(uint32_t));
    const size_t o_cnt = off; off += con_align(sizeof(uint2) * std::max<size_t>(n, 1));
    const size_t o_tiles = off; off += con_align(sizeof(uint2) * std::max<size_t>(nt, 1));
    const size_t o_total = off; off += con_align(sizeof(uint2));
    GeomWorkspace *g = gws(ctx);
    int rc;
    if ((rc = g->incs.ensure(ctx, off))) return rc;
    unsigned char *b = (unsigned char *)g->incs.p;
    uint32_t *role = (uint32_t *)(b + o_role), *featm = (uint32_t *)(b + o_featm), *merges = (uint32_t *)(b + o_merges);
    uint2 *cnt = (uint2 *)(b + o_cnt), *tiles = (uint2 *)(b + o_tiles), *total = (uint2 *)(b + o_total);
    cudaStream_t st = ctx->stream;
    CVB_PROF(ctx, "k_av", 0);
    CVB_CUDA(ctx, cudaMemsetAsync(b, 0xff, o_merges, st));   // role and featm: INC_NONE
    CVB_CUDA(ctx, cudaMemsetAsync(merges, 0, sizeof(uint32_t), st));
    if (M) {
        k_av_roles<<<cdiv(M, 256), 256, 0, st>>>(M, matches_dev, L, N, role, featm, merges);
        CVB_LAUNCH_CHECK(ctx);
    }
    if (n) {
        k_av_counts<<<cdiv(n, 256), 256, 0, st>>>(L, N, n_obs, lm_off_dev, role, featm, matches_dev, cnt);
        CVB_LAUNCH_CHECK(ctx);
    }
    if ((rc = inc_scan(ctx, n, cnt, tiles, total))) return rc;
    if (n) {
        k_av_place<<<cdiv(n, 256), 256, 0, st>>>(V, L, N, n_obs, lm_off_dev, obs_dev, role, featm, matches_dev, cnt, n, n_obs + N, lm_off_out,
                                                 obs_out, lmap);
        CVB_LAUNCH_CHECK(ctx);
    }
    if (nf + N) {
        k_av_features<<<cdiv(nf + N, 256), 256, 0, st>>>(nf, L, N, view_lm_dev, lmap, featm, matches_dev, cnt, view_lm_out);
        CVB_LAUNCH_CHECK(ctx);
    }
    // the rows that only move: poses, view offsets, bearings, descriptors and colours, the new view's after the old ones
    CVB_CUDA(ctx, cudaMemcpyAsync(poses_out, poses_dev, sizeof(cvb_pose) * V, cudaMemcpyDeviceToDevice, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(poses_out + V, new_pose_dev, sizeof(cvb_pose), cudaMemcpyDeviceToDevice, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(view_off_out, view_off_dev, sizeof(uint32_t) * (V + 1), cudaMemcpyDeviceToDevice, st));
    if (nf) CVB_CUDA(ctx, cudaMemcpyAsync(bear_out, bear_dev, sizeof(double) * 3 * (size_t)nf, cudaMemcpyDeviceToDevice, st));
    if (N) CVB_CUDA(ctx, cudaMemcpyAsync(bear_out + 3 * (size_t)nf, new_bear_dev, sizeof(double) * 3 * (size_t)N, cudaMemcpyDeviceToDevice, st));
    if (desc_out) {
        if (nf) CVB_CUDA(ctx, cudaMemcpyAsync(desc_out, desc_dev, 64 * (size_t)nf, cudaMemcpyDeviceToDevice, st));
        if (N) CVB_CUDA(ctx, cudaMemcpyAsync(desc_out + 64 * (size_t)nf, new_desc_dev, 64 * (size_t)N, cudaMemcpyDeviceToDevice, st));
    }
    if (col_out) {
        if (nf) CVB_CUDA(ctx, cudaMemcpyAsync(col_out, col_dev, 3 * (size_t)nf, cudaMemcpyDeviceToDevice, st));
        if (N) CVB_CUDA(ctx, cudaMemcpyAsync(col_out + 3 * (size_t)nf, new_col_dev, 3 * (size_t)N, cudaMemcpyDeviceToDevice, st));
    }
    k_av_finish<<<1, 1, 0, st>>>(V, nf, N, total, merges, n, view_off_out, lm_off_out, counts);
    CVB_LAUNCH_CHECK(ctx);
    return 0;
}

// apply_optimization, enqueued on the context's stream (no wait); scratch in the context's incorporate scratch buffer
int apply_enqueue(cvb_ctx *ctx, uint32_t V, const cvb_pose *poses_dev, const uint32_t *view_off_dev, const double *bear_dev,
                  const uint8_t *desc_dev, const uint8_t *col_dev, uint32_t nf, uint32_t L, const uint32_t *lm_off_dev, const uint32_t *obs_dev,
                  uint32_t n_obs, const cvb_view_constraint *cons_dev, uint32_t C, const uint8_t *vstate, const uint8_t *ostate,
                  cvb_pose *poses_out, uint32_t *view_off_out, uint32_t *view_lm_out, double *bear_out, uint8_t *desc_out, uint8_t *col_out,
                  uint32_t *lm_off_out, uint32_t *obs_out, cvb_view_constraint *cons_out, uint32_t *vmap, uint32_t *lmap,
                  cvb_incorporate_counts *counts) {
    const uint32_t nmax = std::max(std::max(V, L), std::max(n_obs, C));
    size_t off = 0;
    const size_t o_v = off; off += con_align(sizeof(uint2) * std::max<size_t>(V, 1));
    const size_t o_l = off; off += con_align(sizeof(uint2) * std::max<size_t>(L, 1));
    const size_t o_s = off; off += con_align(sizeof(uint2) * std::max<size_t>(n_obs, 1));
    const size_t o_c = off; off += con_align(sizeof(uint2) * std::max<size_t>(C, 1));
    const size_t o_tiles = off; off += con_align(sizeof(uint2) * std::max<size_t>(cdiv(nmax, INC_TILE), 1));
    const size_t o_tot = off; off += con_align(sizeof(uint2) * 4);
    GeomWorkspace *g = gws(ctx);
    int rc;
    if ((rc = g->incs.ensure(ctx, off))) return rc;
    unsigned char *b = (unsigned char *)g->incs.p;
    uint2 *vcnt = (uint2 *)(b + o_v), *lcnt = (uint2 *)(b + o_l), *scnt = (uint2 *)(b + o_s), *ccnt = (uint2 *)(b + o_c);
    uint2 *tiles = (uint2 *)(b + o_tiles), *tot = (uint2 *)(b + o_tot);
    cudaStream_t st = ctx->stream;
    CVB_PROF(ctx, "k_ap", 0);
    k_ap_view_counts<<<cdiv(V, 256), 256, 0, st>>>(V, nf, view_off_dev, vstate, vcnt);
    CVB_LAUNCH_CHECK(ctx);
    if ((rc = inc_scan(ctx, V, vcnt, tiles, tot + 0))) return rc;
    if (L) {
        k_ap_landmark_counts<<<cdiv(L, 256), 256, 0, st>>>(L, n_obs, lm_off_dev, ostate, lcnt);
        CVB_LAUNCH_CHECK(ctx);
    }
    if ((rc = inc_scan(ctx, L, lcnt, tiles, tot + 1))) return rc;
    if (n_obs) {
        k_ap_split_counts<<<cdiv(n_obs, 256), 256, 0, st>>>(n_obs, ostate, scnt);
        CVB_LAUNCH_CHECK(ctx);
    }
    if ((rc = inc_scan(ctx, n_obs, scnt, tiles, tot + 2))) return rc;
    if (C) {
        k_ap_constraint_counts<<<cdiv(C, 256), 256, 0, st>>>(C, V, cons_dev, vstate, ccnt);
        CVB_LAUNCH_CHECK(ctx);
    }
    if ((rc = inc_scan(ctx, C, ccnt, tiles, tot + 3))) return rc;
    k_ap_views<<<cdiv(V, 256), 256, 0, st>>>(V, poses_dev, vstate, vcnt, poses_out, view_off_out, vmap);
    CVB_LAUNCH_CHECK(ctx);
    k_ap_feature_rows<<<cdiv(V * 32, 256), 256, 0, st>>>(V, nf, view_off_dev, vstate, vcnt, bear_dev, (const uint4 *)desc_dev, col_dev, bear_out,
                                                         (uint4 *)desc_out, col_out);
    CVB_LAUNCH_CHECK(ctx);
    if (L) {
        k_ap_landmarks<<<cdiv(L, 256), 256, 0, st>>>(V, nf, L, n_obs, view_off_dev, vstate, vcnt, lm_off_dev, obs_dev, ostate, lcnt, tot + 1,
                                                     lm_off_out, obs_out, view_lm_out, lmap);
        CVB_LAUNCH_CHECK(ctx);
    }
    if (n_obs) {
        k_ap_splits<<<cdiv(n_obs, 256), 256, 0, st>>>(V, nf, L, n_obs, view_off_dev, vstate, vcnt, obs_dev, ostate, scnt, tot + 1, lm_off_out,
                                                      obs_out, view_lm_out);
        CVB_LAUNCH_CHECK(ctx);
    }
    if (C) {
        k_ap_constraints<<<cdiv(C, 256), 256, 0, st>>>(C, cons_dev, ccnt, tot + 3, vcnt, cons_out);
        CVB_LAUNCH_CHECK(ctx);
    }
    k_ap_finish<<<1, 1, 0, st>>>(tot + 0, tot + 1, tot + 2, tot + 3, L + n_obs, view_off_out, lm_off_out, counts);
    CVB_LAUNCH_CHECK(ctx);
    return 0;
}

}  // namespace

int add_view_dev(cvb_ctx *ctx, uint32_t V, const cvb_pose *poses_dev, const uint32_t *view_off_dev, const uint32_t *view_lm_dev,
                 const double *bear_dev, const uint8_t *desc_dev, const uint8_t *col_dev, uint32_t nf, uint32_t L, const uint32_t *lm_off_dev,
                 const uint32_t *obs_dev, uint32_t n_obs, const cvb_pose *new_pose_dev, const double *new_bear_dev, const uint8_t *new_desc_dev,
                 const uint8_t *new_col_dev, uint32_t N, const cvb_register_match *matches_dev, uint32_t M, cvb_pose *poses_out,
                 uint32_t *view_off_out, uint32_t *view_lm_out, double *bear_out, uint8_t *desc_out, uint8_t *col_out, uint32_t *lm_off_out,
                 uint32_t *obs_out, uint32_t *lmap, cvb_incorporate_counts *counts) {
    if (!ctx) return CVB_EINVAL;
    if (!poses_dev || !view_off_dev || !lm_off_dev || !new_pose_dev || !poses_out || !view_off_out || !lm_off_out || !counts ||
        (nf && (!view_lm_dev || !bear_dev)) || (n_obs && !obs_dev) || (N && !new_bear_dev) || (M && !matches_dev) ||
        (nf + N && (!view_lm_out || !bear_out)) || (n_obs + N && !obs_out) || (L && !lmap))
        return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    // descriptors and colours: the snapshot's, the new frame's and the output all given or all omitted
    if ((nf && (!desc_dev != !desc_out)) || (N && (!new_desc_dev != !desc_out)) || (nf && (!col_dev != !col_out)) ||
        (N && (!new_col_dev != !col_out)))
        return cvb_set_error(ctx, CVB_EINVAL, "descriptors and colours go with the snapshot, the new frame and the output together");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    int rc;
    if ((rc = inc_sizes(ctx, V, view_off_dev, nf, L, lm_off_dev, n_obs))) return rc;
    if ((rc = add_view_enqueue(ctx, V, poses_dev, view_off_dev, view_lm_dev, bear_dev, desc_dev, col_dev, nf, L, lm_off_dev, obs_dev, n_obs,
                               new_pose_dev, new_bear_dev, new_desc_dev, new_col_dev, N, matches_dev, M, poses_out, view_off_out, view_lm_out,
                               bear_out, desc_out, col_out, lm_off_out, obs_out, lmap, counts)))
        return rc;
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    return 0;
}

int apply_optimization_dev(cvb_ctx *ctx, uint32_t V, const cvb_pose *poses_dev, const uint32_t *view_off_dev, const uint32_t *view_lm_dev,
                           const double *bear_dev, const uint8_t *desc_dev, const uint8_t *col_dev, uint32_t nf, uint32_t L,
                           const uint32_t *lm_off_dev, const uint32_t *obs_dev, uint32_t n_obs, const cvb_view_constraint *cons_dev, uint32_t C,
                           const uint8_t *vstate, const uint8_t *ostate, cvb_pose *poses_out, uint32_t *view_off_out, uint32_t *view_lm_out,
                           double *bear_out, uint8_t *desc_out, uint8_t *col_out, uint32_t *lm_off_out, uint32_t *obs_out,
                           cvb_view_constraint *cons_out, uint32_t *vmap, uint32_t *lmap, cvb_incorporate_counts *counts) {
    if (!ctx) return CVB_EINVAL;
    if (!poses_dev || !view_off_dev || !lm_off_dev || !poses_out || !view_off_out || !lm_off_out || !counts ||
        (nf && (!view_lm_dev || !bear_dev || !view_lm_out || !bear_out)) || (n_obs && (!obs_dev || !ostate || !obs_out)) ||
        (C && (!cons_dev || !cons_out)) || (V && (!vstate || !vmap)) || (L && !lmap))
        return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (nf && ((!desc_dev != !desc_out) || (!col_dev != !col_out)))
        return cvb_set_error(ctx, CVB_EINVAL, "descriptors and colours go with the snapshot and the output together");
    if (V == 0) return cvb_set_error(ctx, CVB_EINVAL, "no views");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    int rc;
    if ((rc = inc_sizes(ctx, V, view_off_dev, nf, L, lm_off_dev, n_obs))) return rc;
    if ((rc = apply_enqueue(ctx, V, poses_dev, view_off_dev, bear_dev, desc_dev, col_dev, nf, L, lm_off_dev, obs_dev, n_obs, cons_dev, C, vstate,
                            ostate, poses_out, view_off_out, view_lm_out, bear_out, desc_out, col_out, lm_off_out, obs_out, cons_out, vmap, lmap,
                            counts)))
        return rc;
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    return 0;
}

namespace {

// device rows of one snapshot with the given capacities, carved out of one buffer
struct IncSnap {
    cvb_pose *poses; uint32_t *vo, *vl; double *bear; uint8_t *desc, *col; uint32_t *lo, *obs; cvb_view_constraint *cons;
};
size_t inc_snap_layout(size_t base, uint32_t V, uint32_t nf, uint32_t L, uint32_t n_obs, uint32_t C, bool desc, bool col, size_t *o) {
    size_t off = base;
    o[0] = off; off += con_align(sizeof(cvb_pose) * std::max<size_t>(V, 1));
    o[1] = off; off += con_align(sizeof(uint32_t) * ((size_t)V + 1));
    o[2] = off; off += con_align(sizeof(uint32_t) * std::max<size_t>(nf, 1));
    o[3] = off; off += con_align(sizeof(double) * 3 * std::max<size_t>(nf, 1));
    o[4] = off; off += desc ? con_align(64 * std::max<size_t>(nf, 1)) : 0;
    o[5] = off; off += col ? con_align(3 * std::max<size_t>(nf, 1)) : 0;
    o[6] = off; off += con_align(sizeof(uint32_t) * ((size_t)L + 1));
    o[7] = off; off += con_align(sizeof(uint32_t) * 2 * std::max<size_t>(n_obs, 1));
    o[8] = off; off += con_align(sizeof(cvb_view_constraint) * std::max<size_t>(C, 1));
    return off;
}
IncSnap inc_snap_at(unsigned char *b, const size_t *o, bool desc, bool col) {
    IncSnap s;
    s.poses = (cvb_pose *)(b + o[0]);
    s.vo = (uint32_t *)(b + o[1]);
    s.vl = (uint32_t *)(b + o[2]);
    s.bear = (double *)(b + o[3]);
    s.desc = desc ? b + o[4] : nullptr;
    s.col = col ? b + o[5] : nullptr;
    s.lo = (uint32_t *)(b + o[6]);
    s.obs = (uint32_t *)(b + o[7]);
    s.cons = (cvb_view_constraint *)(b + o[8]);
    return s;
}

}  // namespace

int incorporate_frame_dev(cvb_ctx *ctx, const cvb_register_cfg *rcfg, const cvb_constraints_cfg *ccfg, const cvb_recon_cfg *ocfg,
                          const cvb_triangulator *tri, const cvb_arrsac_cfg *arrsac, cvb_rng *rng, uint32_t V, const cvb_pose *poses_dev,
                          const uint32_t *view_off_dev, const uint32_t *view_lm_dev, const double *bear_dev, const uint8_t *desc_dev,
                          const uint8_t *col_dev, uint32_t nf, uint32_t L, const uint32_t *lm_off_dev, const uint32_t *obs_dev, uint32_t n_obs,
                          const cvb_view_constraint *cons_dev, uint32_t C, const uint8_t *new_desc_dev, const double *new_bear_dev,
                          const uint8_t *new_col_dev, uint32_t N, const uint32_t *view_matches, uint32_t H, cvb_pose *poses_out,
                          uint32_t *view_off_out, uint32_t *view_lm_out, double *bear_out, uint8_t *desc_out, uint8_t *col_out,
                          uint32_t *lm_off_out, uint32_t *obs_out, cvb_view_constraint *cons_out, uint32_t *vmap, uint32_t *lmap,
                          cvb_register_match *matches_out, cvb_incorporate_result *res_dev) {
    if (!ctx) return CVB_EINVAL;
    if (!rcfg || !ccfg || !ocfg || !tri || !arrsac || !rng || !poses_dev || !view_off_dev || !lm_off_dev || !res_dev || !poses_out ||
        !view_off_out || !lm_off_out || (H && !view_matches) || (nf && (!view_lm_dev || !bear_dev || !desc_dev)) || (n_obs && !obs_dev) ||
        (C && !cons_dev) || (N && (!new_desc_dev || !new_bear_dev)) || (nf + N && (!view_lm_out || !bear_out || !desc_out)) ||
        (n_obs + N && !obs_out) || (V && !vmap) || (L && !lmap) || !cons_out)
        return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if ((nf && (!col_dev != !col_out)) || (N && (!new_col_dev != !col_out)))
        return cvb_set_error(ctx, CVB_EINVAL, "colours go with the snapshot, the new frame and the output together");
    if (tri->method < CVB_TRI_LINEAR_EIGEN || tri->method > CVB_TRI_MEAN_MEAN)
        return cvb_set_error(ctx, tri->method >= CVB_TRI_RELATIVE_DLT && tri->method <= CVB_TRI_ANGULAR_LINF ? CVB_EUNSUPPORTED : CVB_EINVAL,
                             "triangulator method %d: incorporation takes a TriangulatorObservations (methods 0-2)", tri->method);
    if (ccfg->optimization_maximum_landmarks > CVB_CONSTRAINTS_MAX_LANDMARKS)
        return cvb_set_error(ctx, CVB_EUNSUPPORTED, "optimization_maximum_landmarks %u > %u", ccfg->optimization_maximum_landmarks,
                             CVB_CONSTRAINTS_MAX_LANDMARKS);
    if (V == 0) return cvb_set_error(ctx, CVB_EINVAL, "no views");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    int rc;
    if ((rc = inc_sizes(ctx, V, view_off_dev, nf, L, lm_off_dev, n_obs))) return rc;
    cudaStream_t st = ctx->stream;
    const bool col = col_out != nullptr;
    const uint32_t maxc = ccfg->optimization_maximum_three_view_constraints;
    const uint32_t V1 = V + 1, nf1 = nf + N, L1 = L + N, no1 = n_obs + N, C1 = C + maxc;
    // the workspace: register's outputs, the snapshot after add_view (with room for the new constraints after the old ones), the
    // optimisation's outputs and the maps of the two edits
    size_t o[9], off = 0;
    const size_t o_rres = off; off += con_align(sizeof(cvb_register_result));
    const size_t o_rst = off; off += con_align(sizeof(cvb_register_stats));
    const size_t o_m = off; off += con_align(sizeof(cvb_register_match) * std::max<size_t>(N, 1));
    const size_t o_cres = off; off += con_align(sizeof(cvb_view_constraints_result));
    const size_t o_ores = off; off += con_align(sizeof(cvb_recon_result));
    const size_t o_cnt = off; off += con_align(sizeof(cvb_incorporate_counts) * 2);
    const size_t o_pout = off; off += con_align(sizeof(cvb_pose) * V1);
    const size_t o_vs = off; off += con_align(V1);
    const size_t o_os = off; off += con_align(std::max<size_t>(no1, 1));
    const size_t o_amap = off; off += con_align(sizeof(uint32_t) * std::max<size_t>(L, 1));
    const size_t o_vmap = off; off += con_align(sizeof(uint32_t) * V1);
    const size_t o_lmap = off; off += con_align(sizeof(uint32_t) * std::max<size_t>(L1, 1));
    off = inc_snap_layout(off, V1, nf1, L1, no1, C1, true, col, o);
    GeomWorkspace *g = gws(ctx);
    if ((rc = g->inc.ensure(ctx, off))) return rc;
    unsigned char *b = (unsigned char *)g->inc.p;
    cvb_register_result *rres = (cvb_register_result *)(b + o_rres);
    cvb_register_stats *rst = (cvb_register_stats *)(b + o_rst);
    cvb_register_match *mt = (cvb_register_match *)(b + o_m);
    cvb_view_constraints_result *cres = (cvb_view_constraints_result *)(b + o_cres);
    cvb_recon_result *ores = (cvb_recon_result *)(b + o_ores);
    cvb_incorporate_counts *cnt = (cvb_incorporate_counts *)(b + o_cnt);
    cvb_pose *pout = (cvb_pose *)(b + o_pout);
    uint8_t *vs = b + o_vs, *os = b + o_os;
    uint32_t *amap = (uint32_t *)(b + o_amap), *avmap = (uint32_t *)(b + o_vmap), *almap = (uint32_t *)(b + o_lmap);
    IncSnap a = inc_snap_at(b, o, true, col);
    cvb_incorporate_result R;
    memset(&R, 0, sizeof(R));
    R.new_view = CVB_INCORPORATE_NONE;
    // 1. register_frame
    if ((rc = register_frame_dev(ctx, rcfg, tri, arrsac, rng, V, poses_dev, view_off_dev, view_lm_dev, bear_dev, desc_dev, nf, L, lm_off_dev,
                                 obs_dev, n_obs, new_desc_dev, new_bear_dev, N, view_matches, H, rres, mt, nullptr, rst)))
        return rc;
    std::vector<cvb_register_match> hm;
    {
        CVB_CUDA(ctx, cudaMemcpyAsync(&R.reg, rres, sizeof(cvb_register_result), cudaMemcpyDeviceToHost, st));
        CVB_CUDA(ctx, cudaMemcpyAsync(&R.reg_stats, rst, sizeof(cvb_register_stats), cudaMemcpyDeviceToHost, st));
        CVB_CUDA(ctx, cvb_wait(ctx, st));
    }
    const uint32_t M = R.reg.status == CVB_REGISTER_OK ? R.reg.n_matches : 0;
    if (matches_out && M) CVB_CUDA(ctx, cudaMemcpyAsync(matches_out, mt, sizeof(cvb_register_match) * M, cudaMemcpyDeviceToDevice, st));
    bool have = false;            // an output snapshot exists
    bool edited = false;          // ... and it came through the apply step (maps composed from add_view's and apply's)
    if (R.reg.status == CVB_REGISTER_PANIC) {
        R.status = CVB_INCORPORATE_REGISTER_PANIC;
    } else if (R.reg.status != CVB_REGISTER_OK) {
        // the input, unchanged
        R.status = CVB_INCORPORATE_NOT_REGISTERED;
        CVB_CUDA(ctx, cudaMemcpyAsync(poses_out, poses_dev, sizeof(cvb_pose) * V, cudaMemcpyDeviceToDevice, st));
        CVB_CUDA(ctx, cudaMemcpyAsync(view_off_out, view_off_dev, sizeof(uint32_t) * (V + 1), cudaMemcpyDeviceToDevice, st));
        if (nf) {
            CVB_CUDA(ctx, cudaMemcpyAsync(view_lm_out, view_lm_dev, sizeof(uint32_t) * nf, cudaMemcpyDeviceToDevice, st));
            CVB_CUDA(ctx, cudaMemcpyAsync(bear_out, bear_dev, sizeof(double) * 3 * (size_t)nf, cudaMemcpyDeviceToDevice, st));
            CVB_CUDA(ctx, cudaMemcpyAsync(desc_out, desc_dev, 64 * (size_t)nf, cudaMemcpyDeviceToDevice, st));
            if (col) CVB_CUDA(ctx, cudaMemcpyAsync(col_out, col_dev, 3 * (size_t)nf, cudaMemcpyDeviceToDevice, st));
        }
        CVB_CUDA(ctx, cudaMemcpyAsync(lm_off_out, lm_off_dev, sizeof(uint32_t) * ((size_t)L + 1), cudaMemcpyDeviceToDevice, st));
        if (n_obs) CVB_CUDA(ctx, cudaMemcpyAsync(obs_out, obs_dev, sizeof(uint32_t) * 2 * (size_t)n_obs, cudaMemcpyDeviceToDevice, st));
        if (C) CVB_CUDA(ctx, cudaMemcpyAsync(cons_out, cons_dev, sizeof(cvb_view_constraint) * C, cudaMemcpyDeviceToDevice, st));
        R.counts.V = V; R.counts.n_features = nf; R.counts.L = L; R.counts.n_observations = n_obs; R.counts.C = C;
        have = true;
    } else {
        // 2. add_view.  Its landmark count follows from the matches without a wait: L - merges + (N - matches)
        uint32_t merges = 0;
        {
            hm.resize(M);
            if (M) CVB_CUDA(ctx, cudaMemcpyAsync(hm.data(), mt, sizeof(cvb_register_match) * M, cudaMemcpyDeviceToHost, st));
            CVB_CUDA(ctx, cvb_wait(ctx, st));
            for (const cvb_register_match &m : hm) merges += m.landmark_b != CVB_REGISTER_NONE;
        }
        const uint32_t La = L - merges + (N - M);
        if ((rc = add_view_enqueue(ctx, V, poses_dev, view_off_dev, view_lm_dev, bear_dev, desc_dev, col_dev, nf, L, lm_off_dev, obs_dev, n_obs,
                                   &rres->pose, new_bear_dev, new_desc_dev, new_col_dev, N, mt, M, a.poses, a.vo, a.vl, a.bear, a.desc, a.col, a.lo,
                                   a.obs, amap, cnt)))
            return rc;
        if (C) CVB_CUDA(ctx, cudaMemcpyAsync(a.cons, cons_dev, sizeof(cvb_view_constraint) * C, cudaMemcpyDeviceToDevice, st));
        // 3. the new view's constraints and record_view_constraints' acceptance
        const uint32_t q = V;
        if ((rc = view_constraints_dev(ctx, ccfg, tri, V1, a.poses, a.vo, a.vl, a.bear, nf1, La, a.lo, a.obs, no1, &q, 1, a.cons + C, cres, nullptr)))
            return rc;
        CVB_CUDA(ctx, cudaMemcpyAsync(&R.con, cres, sizeof(cvb_view_constraints_result), cudaMemcpyDeviceToHost, st));
        CVB_CUDA(ctx, cvb_wait(ctx, st));
        const uint32_t Ca = C + R.con.n_constraints;
        if (!R.con.accepted) {
            // remove_view of the new view: the merges stay
            R.status = CVB_INCORPORATE_REJECTED;
            CVB_CUDA(ctx, cudaMemsetAsync(vs, CVB_RECON_VIEW_KEPT, V, st));
            CVB_CUDA(ctx, cudaMemsetAsync(vs + V, CVB_RECON_VIEW_NO_EDGES, 1, st));
            if (no1) {
                k_inc_reject_states<<<cdiv(no1, 256), 256, 0, st>>>(no1, V, a.obs, os);
                CVB_LAUNCH_CHECK(ctx);
            }
            if ((rc = apply_enqueue(ctx, V1, a.poses, a.vo, a.bear, a.desc, a.col, nf1, La, a.lo, a.obs, no1, a.cons, C, vs, os, poses_out,
                                    view_off_out, view_lm_out, bear_out, desc_out, col_out, lm_off_out, obs_out, cons_out, avmap, almap,
                                    cnt + 1)))
                return rc;
            have = edited = true;
        } else {
            // 4. optimize_reconstruction over the old constraints and the new ones, then its edits
            if ((rc = optimize_reconstruction_dev(ctx, ocfg, tri, V1, a.poses, a.vo, a.vl, a.bear, nf1, La, a.lo, a.obs, no1, a.cons, Ca, ores,
                                                  pout, vs, os)))
                return rc;
            CVB_CUDA(ctx, cudaMemcpyAsync(&R.recon, ores, sizeof(cvb_recon_result), cudaMemcpyDeviceToHost, st));
            CVB_CUDA(ctx, cvb_wait(ctx, st));
            if (R.recon.status == CVB_RECON_KEPT) {
                R.status = CVB_INCORPORATE_KEPT;
                if ((rc = apply_enqueue(ctx, V1, pout, a.vo, a.bear, a.desc, a.col, nf1, La, a.lo, a.obs, no1, a.cons, Ca, vs, os, poses_out,
                                        view_off_out, view_lm_out, bear_out, desc_out, col_out, lm_off_out, obs_out, cons_out, avmap, almap,
                                        cnt + 1)))
                    return rc;
                have = edited = true;
            } else {
                R.status = R.recon.status == CVB_RECON_REMOVED_CONSTRAINTS ? CVB_INCORPORATE_REMOVED_CONSTRAINTS
                         : R.recon.status == CVB_RECON_REMOVED_FILTER      ? CVB_INCORPORATE_REMOVED_FILTER
                                                                           : CVB_INCORPORATE_RECON_PANIC;
            }
        }
    }
    // the maps from the input to the output
    if (!have) {
        if (V) CVB_CUDA(ctx, cudaMemsetAsync(vmap, 0xff, sizeof(uint32_t) * V, st));
        if (L) CVB_CUDA(ctx, cudaMemsetAsync(lmap, 0xff, sizeof(uint32_t) * L, st));
    } else {
        k_inc_compose<<<cdiv(V, 256), 256, 0, st>>>(V, nullptr, V1, edited ? avmap : nullptr, vmap);
        CVB_LAUNCH_CHECK(ctx);
        if (L) {
            k_inc_compose<<<cdiv(L, 256), 256, 0, st>>>(L, edited ? amap : nullptr, L1, edited ? almap : nullptr, lmap);
            CVB_LAUNCH_CHECK(ctx);
        }
    }
    if (edited) {
        uint32_t nv = CVB_INCORPORATE_NONE;
        CVB_CUDA(ctx, cudaMemcpyAsync(&R.counts, cnt + 1, sizeof(cvb_incorporate_counts), cudaMemcpyDeviceToHost, st));
        CVB_CUDA(ctx, cudaMemcpyAsync(&nv, avmap + V, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
        CVB_CUDA(ctx, cvb_wait(ctx, st));
        R.new_view = nv;
    }
    CVB_CUDA(ctx, cudaMemcpyAsync(res_dev, &R, sizeof(R), cudaMemcpyHostToDevice, st));
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    return 0;
}

namespace {

// the host snapshot into the context's output workspace (as export_upload, with descriptors and colours), `extra` bytes after it
int inc_upload(cvb_ctx *ctx, uint32_t V, const cvb_pose *poses, const uint32_t *vo, const uint32_t *vl, const double *bear, const uint8_t *desc,
               const uint8_t *col, uint32_t L, const uint32_t *lo, const uint32_t *obs, const cvb_view_constraint *cons, uint32_t C, size_t extra,
               IncSnap &s, unsigned char *&b, size_t &end) {
    const uint32_t nf = vo[V], no = lo[L];
    size_t o[9];
    end = inc_snap_layout(0, V, nf, L, no, C, desc != nullptr, col != nullptr, o);
    GeomWorkspace *g = gws(ctx);
    int rc;
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    if ((rc = g->out.ensure(ctx, end + extra))) return rc;
    b = (unsigned char *)g->out.p;
    s = inc_snap_at(b, o, desc != nullptr, col != nullptr);
    cudaStream_t st = ctx->stream;
    CVB_CUDA(ctx, cudaMemcpyAsync(s.poses, poses, sizeof(cvb_pose) * V, cudaMemcpyHostToDevice, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(s.vo, vo, sizeof(uint32_t) * ((size_t)V + 1), cudaMemcpyHostToDevice, st));
    if (nf) {
        CVB_CUDA(ctx, cudaMemcpyAsync(s.vl, vl, sizeof(uint32_t) * (size_t)nf, cudaMemcpyHostToDevice, st));
        CVB_CUDA(ctx, cudaMemcpyAsync(s.bear, bear, sizeof(double) * 3 * (size_t)nf, cudaMemcpyHostToDevice, st));
        if (desc) CVB_CUDA(ctx, cudaMemcpyAsync(s.desc, desc, 64 * (size_t)nf, cudaMemcpyHostToDevice, st));
        if (col) CVB_CUDA(ctx, cudaMemcpyAsync(s.col, col, 3 * (size_t)nf, cudaMemcpyHostToDevice, st));
    }
    CVB_CUDA(ctx, cudaMemcpyAsync(s.lo, lo, sizeof(uint32_t) * ((size_t)L + 1), cudaMemcpyHostToDevice, st));
    if (no) CVB_CUDA(ctx, cudaMemcpyAsync(s.obs, obs, sizeof(uint32_t) * 2 * (size_t)no, cudaMemcpyHostToDevice, st));
    if (C) CVB_CUDA(ctx, cudaMemcpyAsync(s.cons, cons, sizeof(cvb_view_constraint) * (size_t)C, cudaMemcpyHostToDevice, st));
    return 0;
}

// an output snapshot of the given counts back to the host
int inc_download(cvb_ctx *ctx, const IncSnap &s, const cvb_incorporate_counts &c, bool desc, bool col, cvb_pose *poses, uint32_t *vo,
                 uint32_t *vl, double *bear, uint8_t *d, uint8_t *co, uint32_t *lo, uint32_t *obs, cvb_view_constraint *cons) {
    cudaStream_t st = ctx->stream;
    if (c.V) CVB_CUDA(ctx, cudaMemcpyAsync(poses, s.poses, sizeof(cvb_pose) * c.V, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(vo, s.vo, sizeof(uint32_t) * ((size_t)c.V + 1), cudaMemcpyDeviceToHost, st));
    if (c.n_features) {
        CVB_CUDA(ctx, cudaMemcpyAsync(vl, s.vl, sizeof(uint32_t) * (size_t)c.n_features, cudaMemcpyDeviceToHost, st));
        CVB_CUDA(ctx, cudaMemcpyAsync(bear, s.bear, sizeof(double) * 3 * (size_t)c.n_features, cudaMemcpyDeviceToHost, st));
        if (desc) CVB_CUDA(ctx, cudaMemcpyAsync(d, s.desc, 64 * (size_t)c.n_features, cudaMemcpyDeviceToHost, st));
        if (col) CVB_CUDA(ctx, cudaMemcpyAsync(co, s.col, 3 * (size_t)c.n_features, cudaMemcpyDeviceToHost, st));
    }
    CVB_CUDA(ctx, cudaMemcpyAsync(lo, s.lo, sizeof(uint32_t) * ((size_t)c.L + 1), cudaMemcpyDeviceToHost, st));
    if (c.n_observations) CVB_CUDA(ctx, cudaMemcpyAsync(obs, s.obs, sizeof(uint32_t) * 2 * (size_t)c.n_observations, cudaMemcpyDeviceToHost, st));
    if (c.C && cons) CVB_CUDA(ctx, cudaMemcpyAsync(cons, s.cons, sizeof(cvb_view_constraint) * (size_t)c.C, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    return 0;
}

}  // namespace

int add_view(cvb_ctx *ctx, uint32_t V, const cvb_pose *poses, const uint32_t *vo, const uint32_t *vl, const double *bear, const uint8_t *desc,
             const uint8_t *col, uint32_t L, const uint32_t *lo, const uint32_t *obs, const cvb_pose *new_pose, const double *new_bear,
             const uint8_t *new_desc, const uint8_t *new_col, uint32_t N, const cvb_register_match *matches, uint32_t M, cvb_pose *poses_out,
             uint32_t *vo_out, uint32_t *vl_out, double *bear_out, uint8_t *desc_out, uint8_t *col_out, uint32_t *lo_out, uint32_t *obs_out,
             uint32_t *lmap, cvb_incorporate_counts *counts) {
    if (!ctx) return CVB_EINVAL;
    if (!poses || !new_pose || !poses_out || !vo_out || !lo_out || !counts) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (incorporate_check(V, vo, vl, L, lo, obs, nullptr, 0, N, matches, M, nullptr, 0, nullptr, 0))
        return cvb_set_error(ctx, CVB_EINVAL, "malformed snapshot or matches");
    const uint32_t nf = vo[V], no = lo[L];
    if ((nf && !bear) || (N && !new_bear) || (nf + N && (!vl_out || !bear_out)) || (no + N && !obs_out) || (L && !lmap))
        return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if ((nf && (!desc != !desc_out)) || (N && (!new_desc != !desc_out)) || (nf && (!col != !col_out)) || (N && (!new_col != !col_out)))
        return cvb_set_error(ctx, CVB_EINVAL, "descriptors and colours go with the snapshot, the new frame and the output together");
    const bool hd = desc_out != nullptr, hc = col_out != nullptr;
    size_t x = 0, o[9];
    const size_t i_np = x; x += con_align(sizeof(cvb_pose));
    const size_t i_nb = x; x += con_align(sizeof(double) * 3 * std::max<size_t>(N, 1));
    const size_t i_nd = x; x += con_align(64 * std::max<size_t>(N, 1));
    const size_t i_nc = x; x += con_align(3 * std::max<size_t>(N, 1));
    const size_t i_m = x; x += con_align(sizeof(cvb_register_match) * std::max<size_t>(M, 1));
    const size_t i_map = x; x += con_align(sizeof(uint32_t) * std::max<size_t>(L, 1));
    const size_t i_cnt = x; x += con_align(sizeof(cvb_incorporate_counts));
    x = inc_snap_layout(x, V + 1, nf + N, L + N, no + N, 0, hd, hc, o);
    IncSnap s;
    unsigned char *b;
    size_t end;
    int rc;
    if ((rc = inc_upload(ctx, V, poses, vo, vl, bear, hd ? desc : nullptr, hc ? col : nullptr, L, lo, obs, nullptr, 0, x, s, b, end))) return rc;
    unsigned char *e = b + end;
    cudaStream_t st = ctx->stream;
    CVB_CUDA(ctx, cudaMemcpyAsync(e + i_np, new_pose, sizeof(cvb_pose), cudaMemcpyHostToDevice, st));
    if (N) {
        CVB_CUDA(ctx, cudaMemcpyAsync(e + i_nb, new_bear, sizeof(double) * 3 * (size_t)N, cudaMemcpyHostToDevice, st));
        if (hd) CVB_CUDA(ctx, cudaMemcpyAsync(e + i_nd, new_desc, 64 * (size_t)N, cudaMemcpyHostToDevice, st));
        if (hc) CVB_CUDA(ctx, cudaMemcpyAsync(e + i_nc, new_col, 3 * (size_t)N, cudaMemcpyHostToDevice, st));
    }
    if (M) CVB_CUDA(ctx, cudaMemcpyAsync(e + i_m, matches, sizeof(cvb_register_match) * M, cudaMemcpyHostToDevice, st));
    IncSnap out = inc_snap_at(e, o, hd, hc);
    if ((rc = add_view_dev(ctx, V, s.poses, s.vo, s.vl, s.bear, s.desc, s.col, nf, L, s.lo, s.obs, no, (const cvb_pose *)(e + i_np),
                           (const double *)(e + i_nb), hd ? e + i_nd : nullptr, hc ? e + i_nc : nullptr, N, (const cvb_register_match *)(e + i_m), M,
                           out.poses, out.vo, out.vl, out.bear, out.desc, out.col, out.lo, out.obs, (uint32_t *)(e + i_map),
                           (cvb_incorporate_counts *)(e + i_cnt))))
        return rc;
    CVB_CUDA(ctx, cudaMemcpyAsync(counts, e + i_cnt, sizeof(cvb_incorporate_counts), cudaMemcpyDeviceToHost, st));
    if (L) CVB_CUDA(ctx, cudaMemcpyAsync(lmap, e + i_map, sizeof(uint32_t) * L, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    return inc_download(ctx, out, *counts, hd, hc, poses_out, vo_out, vl_out, bear_out, desc_out, col_out, lo_out, obs_out, nullptr);
}

int apply_optimization(cvb_ctx *ctx, uint32_t V, const cvb_pose *poses, const uint32_t *vo, const uint32_t *vl, const double *bear,
                       const uint8_t *desc, const uint8_t *col, uint32_t L, const uint32_t *lo, const uint32_t *obs, const cvb_view_constraint *cons,
                       uint32_t C, const uint8_t *vstate, const uint8_t *ostate, cvb_pose *poses_out, uint32_t *vo_out, uint32_t *vl_out,
                       double *bear_out, uint8_t *desc_out, uint8_t *col_out, uint32_t *lo_out, uint32_t *obs_out, cvb_view_constraint *cons_out,
                       uint32_t *vmap, uint32_t *lmap, cvb_incorporate_counts *counts) {
    if (!ctx) return CVB_EINVAL;
    if (!poses || !vstate || !poses_out || !vo_out || !lo_out || !counts || (V && !vmap) || (L && !lmap) || (C && !cons_out))
        return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (incorporate_check(V, vo, vl, L, lo, obs, cons, C, 0, nullptr, 0, vstate, V, ostate, lo ? lo[L] : 0))
        return cvb_set_error(ctx, CVB_EINVAL, "malformed snapshot, constraints or states");
    const uint32_t nf = vo[V], no = lo[L];
    if ((nf && (!bear || !vl_out || !bear_out)) || (no && !obs_out)) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (nf && ((!desc != !desc_out) || (!col != !col_out)))
        return cvb_set_error(ctx, CVB_EINVAL, "descriptors and colours go with the snapshot and the output together");
    const bool hd = desc_out != nullptr, hc = col_out != nullptr;
    size_t x = 0, o[9];
    const size_t i_vs = x; x += con_align(std::max<size_t>(V, 1));
    const size_t i_os = x; x += con_align(std::max<size_t>(no, 1));
    const size_t i_vmap = x; x += con_align(sizeof(uint32_t) * std::max<size_t>(V, 1));
    const size_t i_lmap = x; x += con_align(sizeof(uint32_t) * std::max<size_t>(L, 1));
    const size_t i_cnt = x; x += con_align(sizeof(cvb_incorporate_counts));
    x = inc_snap_layout(x, V, nf, L + no, no, C, hd, hc, o);
    IncSnap s;
    unsigned char *b;
    size_t end;
    int rc;
    if ((rc = inc_upload(ctx, V, poses, vo, vl, bear, hd ? desc : nullptr, hc ? col : nullptr, L, lo, obs, cons, C, x, s, b, end))) return rc;
    unsigned char *e = b + end;
    cudaStream_t st = ctx->stream;
    if (V) CVB_CUDA(ctx, cudaMemcpyAsync(e + i_vs, vstate, V, cudaMemcpyHostToDevice, st));
    if (no) CVB_CUDA(ctx, cudaMemcpyAsync(e + i_os, ostate, no, cudaMemcpyHostToDevice, st));
    IncSnap out = inc_snap_at(e, o, hd, hc);
    if ((rc = apply_optimization_dev(ctx, V, s.poses, s.vo, s.vl, s.bear, s.desc, s.col, nf, L, s.lo, s.obs, no, s.cons, C, e + i_vs, e + i_os,
                                     out.poses, out.vo, out.vl, out.bear, out.desc, out.col, out.lo, out.obs, out.cons, (uint32_t *)(e + i_vmap),
                                     (uint32_t *)(e + i_lmap), (cvb_incorporate_counts *)(e + i_cnt))))
        return rc;
    CVB_CUDA(ctx, cudaMemcpyAsync(counts, e + i_cnt, sizeof(cvb_incorporate_counts), cudaMemcpyDeviceToHost, st));
    if (V) CVB_CUDA(ctx, cudaMemcpyAsync(vmap, e + i_vmap, sizeof(uint32_t) * V, cudaMemcpyDeviceToHost, st));
    if (L) CVB_CUDA(ctx, cudaMemcpyAsync(lmap, e + i_lmap, sizeof(uint32_t) * L, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    return inc_download(ctx, out, *counts, hd, hc, poses_out, vo_out, vl_out, bear_out, desc_out, col_out, lo_out, obs_out, cons_out);
}

int incorporate_frame(cvb_ctx *ctx, const cvb_register_cfg *rcfg, const cvb_constraints_cfg *ccfg, const cvb_recon_cfg *ocfg,
                      const cvb_triangulator *tri, const cvb_arrsac_cfg *arrsac, cvb_rng *rng, uint32_t V, const cvb_pose *poses, const uint32_t *vo,
                      const uint32_t *vl, const double *bear, const uint8_t *desc, const uint8_t *col, uint32_t L, const uint32_t *lo,
                      const uint32_t *obs, const cvb_view_constraint *cons, uint32_t C, const uint8_t *new_desc, const double *new_bear,
                      const uint8_t *new_col, uint32_t N, const uint32_t *view_matches, uint32_t H, cvb_pose *poses_out, uint32_t *vo_out,
                      uint32_t *vl_out, double *bear_out, uint8_t *desc_out, uint8_t *col_out, uint32_t *lo_out, uint32_t *obs_out,
                      cvb_view_constraint *cons_out, uint32_t *vmap, uint32_t *lmap, cvb_register_match *matches, cvb_incorporate_result *res) {
    if (!ctx) return CVB_EINVAL;
    if (!rcfg || !ccfg || !ocfg || !tri || !arrsac || !rng || !poses || !res || !poses_out || !vo_out || !lo_out || !cons_out ||
        (V && !vmap) || (L && !lmap) || (N && (!new_desc || !new_bear)))
        return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (incorporate_check(V, vo, vl, L, lo, obs, cons, C, 0, nullptr, 0, nullptr, 0, nullptr, 0) ||
        register_check(V, vo, vl, L, lo, obs, view_matches, H))
        return cvb_set_error(ctx, CVB_EINVAL, "malformed snapshot, constraints or view matches");
    const uint32_t nf = vo[V], no = lo[L];
    if ((nf && (!bear || !desc)) || (nf + N && (!vl_out || !bear_out || !desc_out)) || (no + N && !obs_out))
        return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if ((nf && (!col != !col_out)) || (N && (!new_col != !col_out)))
        return cvb_set_error(ctx, CVB_EINVAL, "colours go with the snapshot, the new frame and the output together");
    const bool hc = col_out != nullptr;
    const uint32_t maxc = ccfg->optimization_maximum_three_view_constraints;
    size_t x = 0, o[9];
    const size_t i_nd = x; x += con_align(64 * std::max<size_t>(N, 1));
    const size_t i_nb = x; x += con_align(sizeof(double) * 3 * std::max<size_t>(N, 1));
    const size_t i_nc = x; x += con_align(3 * std::max<size_t>(N, 1));
    const size_t i_m = x; x += con_align(sizeof(cvb_register_match) * std::max<size_t>(N, 1));
    const size_t i_vmap = x; x += con_align(sizeof(uint32_t) * std::max<size_t>(V, 1));
    const size_t i_lmap = x; x += con_align(sizeof(uint32_t) * std::max<size_t>(L, 1));
    const size_t i_res = x; x += con_align(sizeof(cvb_incorporate_result));
    x = inc_snap_layout(x, V + 1, nf + N, L + N + no + N, no + N, C + maxc, true, hc, o);
    IncSnap s;
    unsigned char *b;
    size_t end;
    int rc;
    if ((rc = inc_upload(ctx, V, poses, vo, vl, bear, desc, hc ? col : nullptr, L, lo, obs, cons, C, x, s, b, end))) return rc;
    unsigned char *e = b + end;
    cudaStream_t st = ctx->stream;
    if (N) {
        CVB_CUDA(ctx, cudaMemcpyAsync(e + i_nd, new_desc, 64 * (size_t)N, cudaMemcpyHostToDevice, st));
        CVB_CUDA(ctx, cudaMemcpyAsync(e + i_nb, new_bear, sizeof(double) * 3 * (size_t)N, cudaMemcpyHostToDevice, st));
        if (hc) CVB_CUDA(ctx, cudaMemcpyAsync(e + i_nc, new_col, 3 * (size_t)N, cudaMemcpyHostToDevice, st));
    }
    IncSnap out = inc_snap_at(e, o, true, hc);
    cvb_incorporate_result *rd = (cvb_incorporate_result *)(e + i_res);
    if ((rc = incorporate_frame_dev(ctx, rcfg, ccfg, ocfg, tri, arrsac, rng, V, s.poses, s.vo, s.vl, s.bear, s.desc, s.col, nf, L, s.lo, s.obs, no,
                                    s.cons, C, e + i_nd, (const double *)(e + i_nb), hc ? e + i_nc : nullptr, N, view_matches, H, out.poses, out.vo,
                                    out.vl, out.bear, out.desc, out.col, out.lo, out.obs, out.cons, (uint32_t *)(e + i_vmap), (uint32_t *)(e + i_lmap),
                                    (cvb_register_match *)(e + i_m), rd)))
        return rc;
    CVB_CUDA(ctx, cudaMemcpyAsync(res, rd, sizeof(cvb_incorporate_result), cudaMemcpyDeviceToHost, st));
    if (V) CVB_CUDA(ctx, cudaMemcpyAsync(vmap, e + i_vmap, sizeof(uint32_t) * V, cudaMemcpyDeviceToHost, st));
    if (L) CVB_CUDA(ctx, cudaMemcpyAsync(lmap, e + i_lmap, sizeof(uint32_t) * L, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    const uint32_t M = res->reg.status == CVB_REGISTER_OK ? res->reg.n_matches : 0;
    if (matches && M) CVB_CUDA(ctx, cudaMemcpyAsync(matches, e + i_m, sizeof(cvb_register_match) * M, cudaMemcpyDeviceToHost, st));
    const bool have = res->status == CVB_INCORPORATE_KEPT || res->status == CVB_INCORPORATE_REJECTED || res->status == CVB_INCORPORATE_NOT_REGISTERED;
    if (!have) {
        CVB_CUDA(ctx, cvb_wait(ctx, st));
        return 0;
    }
    return inc_download(ctx, out, res->counts, true, hc, poses_out, vo_out, vl_out, bear_out, desc_out, col_out, lo_out, obs_out, cons_out);
}

// ---- cv-sfm's reconstruction merging (C names in merge_abi.cu, include/cvb200_merge.h; kernels in merge_dev.cuh) ------------------------
int merge_check(uint32_t V, const uint32_t *vo, const uint32_t *vl, uint32_t L, const uint32_t *lo, const uint32_t *obs,
                const cvb_view_constraint *cons, uint32_t C, uint32_t VS, const uint32_t *vo_s, const uint32_t *vl_s, uint32_t LS,
                const uint32_t *lo_s, const uint32_t *obs_s, uint32_t view_s, const uint32_t *lmap, int has_col, int has_col_s) {
    if (incorporate_check(V, vo, vl, L, lo, obs, cons, C, 0, nullptr, 0, nullptr, 0, nullptr, 0)) return CVB_EINVAL;
    if (incorporate_check(VS, vo_s, vl_s, LS, lo_s, obs_s, nullptr, 0, 0, nullptr, 0, nullptr, 0, nullptr, 0)) return CVB_EINVAL;
    if (!has_col != !has_col_s) return CVB_EINVAL;
    if (view_s >= VS && !(view_s == CVB_MERGE_NONE && lmap)) return CVB_EINVAL;
    if (lmap) {
        std::vector<uint8_t> used(L, 0);
        for (uint32_t l = 0; l < LS; l++) {
            if (lmap[l] == CVB_MERGE_NONE) continue;
            if (lmap[l] >= L || used[lmap[l]]) return CVB_EINVAL;   // HashMap::insert would overwrite an observation of one view
            used[lmap[l]] = 1;
        }
    }
    return 0;
}

namespace {

// the move edit and the speculative constraint loop of incorporate_reconstruction on device arrays (D: V views, C constraints; S's view
// CSR and landmark CSR).  Leaves the final snapshot in the context's merge scratch (*fin, counts in R.counts), the source landmark map
// (device, LS entries) in *tgt_fin, and on the host the source view map and each moved view's constraint result.
int move_and_constrain(cvb_ctx *ctx, const cvb_constraints_cfg *ccfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses,
                       const uint32_t *vo, const uint32_t *vl, const double *bear, const uint8_t *desc, const uint8_t *col, uint32_t nf, uint32_t L,
                       const uint32_t *lo, const uint32_t *obs, uint32_t n_obs, const cvb_view_constraint *cons, uint32_t C, uint32_t VS,
                       const cvb_pose *poses_s, const uint32_t *vo_s, const uint32_t *vl_s, const double *bear_s, const uint8_t *desc_s,
                       const uint8_t *col_s, uint32_t nf_s, uint32_t LS, const uint32_t *lo_s, const uint32_t *obs_s, uint32_t n_obs_s,
                       uint32_t skip, uint32_t nf_skip, const cvb_pose *wt, const uint32_t *lmap_in, IncSnap &fin, const uint32_t *&tgt_fin,
                       std::vector<uint32_t> &svmap, std::vector<cvb_view_constraints_result> &cres, cvb_move_result &R) {
    cudaStream_t st = ctx->stream;
    const bool hd = desc != nullptr, hc = col != nullptr;
    const uint32_t Q = VS - (skip < VS ? 1u : 0u), maxc = ccfg->optimization_maximum_three_view_constraints;
    const uint32_t VA = V + Q, nfA = nf + nf_s, LA = L + nf_s, noA = n_obs + nf_s, CA = C + Q * maxc, n = L + nf_s;
    size_t oa[9], ob[9], off = 0;
    off = inc_snap_layout(off, VA, nfA, LA, noA, CA, hd, hc, oa);
    off = inc_snap_layout(off, VA, nfA, LA, noA, CA, hd, hc, ob);
    const size_t o_conq = off; off += con_align(sizeof(cvb_view_constraint) * std::max<size_t>((size_t)Q * maxc, 1));
    const size_t o_resq = off; off += con_align(sizeof(cvb_view_constraints_result) * std::max<size_t>(Q, 1));
    const size_t o_cnt = off; off += con_align(sizeof(uint2) * std::max<size_t>(n, 1));
    const size_t o_tiles = off; off += con_align(sizeof(uint2) * std::max<size_t>(cdiv(n, INC_TILE), 1));
    const size_t o_tot = off; off += con_align(sizeof(uint2));
    const size_t o_app = off; off += con_align(sizeof(uint32_t) * std::max<size_t>(L, 1));
    const size_t o_first = off; off += con_align(sizeof(uint32_t) * std::max<size_t>(LS, 1));
    const size_t o_tgt0 = off; off += con_align(sizeof(uint32_t) * std::max<size_t>(LS, 1));
    const size_t o_tgt1 = off; off += con_align(sizeof(uint32_t) * std::max<size_t>(LS, 1));
    const size_t o_vmap = off; off += con_align(sizeof(uint32_t) * std::max<size_t>(VA, 1));
    const size_t o_lmap = off; off += con_align(sizeof(uint32_t) * std::max<size_t>(LA, 1));
    const size_t o_vs = off; off += con_align(std::max<size_t>(VA, 1));
    const size_t o_os = off; off += con_align(std::max<size_t>(noA, 1));
    const size_t o_counts = off; off += con_align(sizeof(cvb_incorporate_counts));
    GeomWorkspace *g = gws(ctx);
    int rc;
    if ((rc = g->mrgs.ensure(ctx, off))) return rc;
    unsigned char *b = (unsigned char *)g->mrgs.p;
    IncSnap A = inc_snap_at(b, oa, hd, hc), B = inc_snap_at(b, ob, hd, hc);
    cvb_view_constraint *conq = (cvb_view_constraint *)(b + o_conq);
    cvb_view_constraints_result *resq = (cvb_view_constraints_result *)(b + o_resq);
    uint2 *cnt = (uint2 *)(b + o_cnt), *tiles = (uint2 *)(b + o_tiles), *total = (uint2 *)(b + o_tot);
    uint32_t *app = (uint32_t *)(b + o_app), *first = (uint32_t *)(b + o_first), *tgt[2] = {(uint32_t *)(b + o_tgt0), (uint32_t *)(b + o_tgt1)};
    uint32_t *vmap_ap = (uint32_t *)(b + o_vmap), *lmap_ap = (uint32_t *)(b + o_lmap);
    uint8_t *vs = b + o_vs, *os = b + o_os;
    cvb_incorporate_counts *dcnt = (cvb_incorporate_counts *)(b + o_counts);
    // 1. the move
    CVB_PROF(ctx, "k_mg", 0);
    CVB_CUDA(ctx, cudaMemsetAsync(cnt, 0, sizeof(uint2) * std::max<size_t>(n, 1), st));
    if (L) CVB_CUDA(ctx, cudaMemsetAsync(app, 0, sizeof(uint32_t) * L, st));
    if (LS) {
        k_mg_landmark_counts<<<cdiv(LS, 256), 256, 0, st>>>(LS, n_obs_s, VS, nf_s, skip, L, lo_s, obs_s, vo_s, lmap_in, app, cnt, first);
        CVB_LAUNCH_CHECK(ctx);
    }
    if (L) {
        k_mg_dest_counts<<<cdiv(L, 256), 256, 0, st>>>(L, n_obs, lo, app, cnt);
        CVB_LAUNCH_CHECK(ctx);
    }
    if ((rc = inc_scan(ctx, n, cnt, tiles, total))) return rc;
    if (L) {
        k_mg_dest_place<<<cdiv(L, 256), 256, 0, st>>>(L, n_obs, lo, obs, cnt, noA, A.lo, A.obs);
        CVB_LAUNCH_CHECK(ctx);
    }
    if (LS) {
        k_mg_landmark_place<<<cdiv(LS, 256), 256, 0, st>>>(LS, n_obs_s, VS, nf_s, skip, V, L, n_obs, lo_s, obs_s, vo_s, lmap_in, lo, cnt, first, LA,
                                                           noA, A.lo, A.obs, tgt[0]);
        CVB_LAUNCH_CHECK(ctx);
    }
    CVB_CUDA(ctx, cudaMemcpyAsync(A.poses, poses, sizeof(cvb_pose) * V, cudaMemcpyDeviceToDevice, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(A.vo, vo, sizeof(uint32_t) * ((size_t)V + 1), cudaMemcpyDeviceToDevice, st));
    if (nf) {
        CVB_CUDA(ctx, cudaMemcpyAsync(A.vl, vl, sizeof(uint32_t) * nf, cudaMemcpyDeviceToDevice, st));
        CVB_CUDA(ctx, cudaMemcpyAsync(A.bear, bear, sizeof(double) * 3 * (size_t)nf, cudaMemcpyDeviceToDevice, st));
        if (hd) CVB_CUDA(ctx, cudaMemcpyAsync(A.desc, desc, 64 * (size_t)nf, cudaMemcpyDeviceToDevice, st));
        if (hc) CVB_CUDA(ctx, cudaMemcpyAsync(A.col, col, 3 * (size_t)nf, cudaMemcpyDeviceToDevice, st));
    }
    if (C) CVB_CUDA(ctx, cudaMemcpyAsync(A.cons, cons, sizeof(cvb_view_constraint) * C, cudaMemcpyDeviceToDevice, st));
    if (VS) {
        k_mg_views<<<cdiv(VS, 128), 128, 0, st>>>(VS, skip, V, nf, nf_s, poses_s, vo_s, wt, A.poses, A.vo);
        CVB_LAUNCH_CHECK(ctx);
        k_mg_feature_rows<<<cdiv(VS * 32, 256), 256, 0, st>>>(VS, skip, nf, nf_s, LS, vo_s, vl_s, bear_s, (const uint4 *)desc_s, col_s, tgt[0], nfA,
                                                              A.vl, A.bear, (uint4 *)A.desc, A.col);
        CVB_LAUNCH_CHECK(ctx);
    }
    const uint32_t nf_moved = nf_s >= nf_skip ? nf_s - nf_skip : 0;
    k_mg_finish<<<1, 1, 0, st>>>(V, Q, nf + nf_moved, total, LA, noA, A.vo, A.lo, dcnt);
    CVB_LAUNCH_CHECK(ctx);
    cvb_incorporate_counts c;
    CVB_CUDA(ctx, cudaMemcpyAsync(&c, dcnt, sizeof(c), cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    memset(&R, 0, sizeof(R));
    R.moved_views = Q;
    R.created_landmarks = c.L - std::min(c.L, L);
    // 2. the constraint loop: one call over every undecided moved view; the results up to the first refusal are final
    std::vector<uint32_t> cur(Q), sv(Q);   // each moved view's current index and its S view
    for (uint32_t v = 0, q = 0; v < VS; v++)
        if (v != skip) { sv[q] = v; cur[q] = V + q; q++; }
    cres.assign(VS, cvb_view_constraints_result{0, 0});
    std::vector<uint8_t> refused(Q, 0);
    std::vector<cvb_view_constraints_result> hres(std::max<uint32_t>(Q, 1));
    std::vector<uint32_t> queries;
    uint32_t Cc = C, start = 0, t = 0;
    IncSnap *curS = &A, *nxtS = &B;
    while (start < Q) {
        queries.assign(cur.begin() + start, cur.end());
        const uint32_t nq = Q - start;
        if ((rc = view_constraints_dev(ctx, ccfg, tri, c.V, curS->poses, curS->vo, curS->vl, curS->bear, c.n_features, c.L, curS->lo, curS->obs,
                                       c.n_observations, queries.data(), nq, conq, resq, nullptr)))
            return rc;
        R.constraint_calls++;
        CVB_CUDA(ctx, cudaMemcpyAsync(hres.data(), resq, sizeof(cvb_view_constraints_result) * nq, cudaMemcpyDeviceToHost, st));
        CVB_CUDA(ctx, cvb_wait(ctx, st));
        uint32_t j = start;
        for (; j < Q; j++) {
            const cvb_view_constraints_result &r = hres[j - start];
            cres[sv[j]] = r;
            if (!r.accepted) break;
            const uint32_t k = std::min(r.n_constraints, maxc);
            if (k) CVB_CUDA(ctx, cudaMemcpyAsync(curS->cons + Cc, conq + (size_t)(j - start) * maxc, sizeof(cvb_view_constraint) * k,
                                                 cudaMemcpyDeviceToDevice, st));
            Cc += k;
        }
        if (j == Q) break;
        // remove_view of the refused view j: its observations DROPPED, every other KEPT
        refused[j] = 1;
        R.refused_views++;
        CVB_CUDA(ctx, cudaMemsetAsync(vs, CVB_RECON_VIEW_KEPT, c.V, st));
        CVB_CUDA(ctx, cudaMemsetAsync(vs + cur[j], CVB_RECON_VIEW_NO_EDGES, 1, st));
        if (c.n_observations) {
            k_inc_reject_states<<<cdiv(c.n_observations, 256), 256, 0, st>>>(c.n_observations, cur[j], curS->obs, os);
            CVB_LAUNCH_CHECK(ctx);
        }
        if ((rc = apply_enqueue(ctx, c.V, curS->poses, curS->vo, curS->bear, curS->desc, curS->col, c.n_features, c.L, curS->lo, curS->obs,
                                c.n_observations, curS->cons, Cc, vs, os, nxtS->poses, nxtS->vo, nxtS->vl, nxtS->bear, nxtS->desc, nxtS->col,
                                nxtS->lo, nxtS->obs, nxtS->cons, vmap_ap, lmap_ap, dcnt)))
            return rc;
        if (LS) {
            k_inc_compose<<<cdiv(LS, 256), 256, 0, st>>>(LS, tgt[t], c.L, lmap_ap, tgt[t ^ 1]);
            CVB_LAUNCH_CHECK(ctx);
        }
        t ^= 1;
        CVB_CUDA(ctx, cudaMemcpyAsync(&c, dcnt, sizeof(c), cudaMemcpyDeviceToHost, st));
        CVB_CUDA(ctx, cvb_wait(ctx, st));
        Cc = c.C;
        for (uint32_t k = j + 1; k < Q; k++) cur[k]--;
        std::swap(curS, nxtS);
        start = j + 1;
    }
    c.C = Cc;
    c.merges = 0;
    R.counts = c;
    svmap.assign(VS, CVB_MERGE_NONE);
    for (uint32_t q = 0; q < Q; q++)
        if (!refused[q]) svmap[sv[q]] = cur[q];
    fin = *curS;
    tgt_fin = tgt[t];
    return 0;
}

// a snapshot of the given counts copied between device arrays
int inc_copy(cvb_ctx *ctx, const IncSnap &s, const cvb_incorporate_counts &c, cvb_pose *poses, uint32_t *vo, uint32_t *vl, double *bear,
             uint8_t *d, uint8_t *co, uint32_t *lo, uint32_t *obs, cvb_view_constraint *cons) {
    cudaStream_t st = ctx->stream;
    const cudaMemcpyKind k = cudaMemcpyDeviceToDevice;
    if (c.V) CVB_CUDA(ctx, cudaMemcpyAsync(poses, s.poses, sizeof(cvb_pose) * c.V, k, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(vo, s.vo, sizeof(uint32_t) * ((size_t)c.V + 1), k, st));
    if (c.n_features) {
        CVB_CUDA(ctx, cudaMemcpyAsync(vl, s.vl, sizeof(uint32_t) * (size_t)c.n_features, k, st));
        CVB_CUDA(ctx, cudaMemcpyAsync(bear, s.bear, sizeof(double) * 3 * (size_t)c.n_features, k, st));
        if (d && s.desc) CVB_CUDA(ctx, cudaMemcpyAsync(d, s.desc, 64 * (size_t)c.n_features, k, st));
        if (co && s.col) CVB_CUDA(ctx, cudaMemcpyAsync(co, s.col, 3 * (size_t)c.n_features, k, st));
    }
    CVB_CUDA(ctx, cudaMemcpyAsync(lo, s.lo, sizeof(uint32_t) * ((size_t)c.L + 1), k, st));
    if (c.n_observations) CVB_CUDA(ctx, cudaMemcpyAsync(obs, s.obs, sizeof(uint32_t) * 2 * (size_t)c.n_observations, k, st));
    if (c.C) CVB_CUDA(ctx, cudaMemcpyAsync(cons, s.cons, sizeof(cvb_view_constraint) * (size_t)c.C, k, st));
    return 0;
}

// two entries of a device offset array, read back
int mg_row(cvb_ctx *ctx, const uint32_t *off_dev, uint32_t i, uint32_t n, uint32_t &r0, uint32_t &r1) {
    uint32_t *h = (uint32_t *)cvb_pinned(ctx, 2 * sizeof(uint32_t));
    if (!h) return cvb_set_error(ctx, CVB_ENOMEM, "page-locked scratch");
    CVB_CUDA(ctx, cudaMemcpyAsync(h, off_dev + i, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    r0 = std::min(h[0], n);
    r1 = std::min(std::max(h[1], r0), n);
    return 0;
}

// the refusals every device entry shares
int mg_args(cvb_ctx *ctx, const cvb_constraints_cfg *ccfg, const cvb_triangulator *tri, uint32_t V) {
    if (tri->method < CVB_TRI_LINEAR_EIGEN || tri->method > CVB_TRI_MEAN_MEAN)
        return cvb_set_error(ctx, tri->method >= CVB_TRI_RELATIVE_DLT && tri->method <= CVB_TRI_ANGULAR_LINF ? CVB_EUNSUPPORTED : CVB_EINVAL,
                             "triangulator method %d: merging takes a TriangulatorObservations (methods 0-2)", tri->method);
    if (ccfg->optimization_maximum_landmarks > CVB_CONSTRAINTS_MAX_LANDMARKS)
        return cvb_set_error(ctx, CVB_EUNSUPPORTED, "optimization_maximum_landmarks %u > %u", ccfg->optimization_maximum_landmarks,
                             CVB_CONSTRAINTS_MAX_LANDMARKS);
    if (V == 0) return cvb_set_error(ctx, CVB_EINVAL, "no views");
    return 0;
}

}  // namespace

int incorporate_reconstruction_dev(cvb_ctx *ctx, const cvb_constraints_cfg *ccfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses,
                                   const uint32_t *vo, const uint32_t *vl, const double *bear, const uint8_t *desc, const uint8_t *col, uint32_t nf,
                                   uint32_t L, const uint32_t *lo, const uint32_t *obs, uint32_t n_obs, const cvb_view_constraint *cons, uint32_t C,
                                   uint32_t VS, const cvb_pose *poses_s, const uint32_t *vo_s, const uint32_t *vl_s, const double *bear_s,
                                   const uint8_t *desc_s, const uint8_t *col_s, uint32_t nf_s, uint32_t LS, const uint32_t *lo_s,
                                   const uint32_t *obs_s, uint32_t n_obs_s, uint32_t skip, const cvb_pose *wt, const uint32_t *lmap_in,
                                   cvb_pose *poses_out, uint32_t *vo_out, uint32_t *vl_out, double *bear_out, uint8_t *desc_out, uint8_t *col_out,
                                   uint32_t *lo_out, uint32_t *obs_out, cvb_view_constraint *cons_out, uint32_t *svmap_dev, uint32_t *slmap_dev,
                                   cvb_view_constraints_result *cres_dev, cvb_move_result *res_dev) {
    if (!ctx) return CVB_EINVAL;
    if (!ccfg || !tri || !poses || !vo || !lo || !poses_s || !vo_s || !lo_s || !wt || !poses_out || !vo_out || !lo_out || !res_dev ||
        (nf && (!vl || !bear)) || (n_obs && !obs) || (C && !cons) || (nf_s && (!vl_s || !bear_s)) || (n_obs_s && !obs_s) ||
        (LS && (!lmap_in || !slmap_dev)) || (VS && (!svmap_dev || !cres_dev)) || (nf + nf_s && (!vl_out || !bear_out)) ||
        (n_obs + nf_s && !obs_out) || !cons_out)
        return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if ((nf && (!desc != !desc_out)) || (nf_s && (!desc_s != !desc_out)) || (nf && (!col != !col_out)) || (nf_s && (!col_s != !col_out)))
        return cvb_set_error(ctx, CVB_EINVAL, "descriptors and colours go with both snapshots and the output together");
    if (skip != CVB_MERGE_NONE && skip >= VS) return cvb_set_error(ctx, CVB_EINVAL, "skip_view %u >= V_S %u", skip, VS);
    int rc;
    if ((rc = mg_args(ctx, ccfg, tri, V))) return rc;
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    if ((rc = inc_sizes(ctx, V, vo, nf, L, lo, n_obs))) return rc;
    if ((rc = inc_sizes(ctx, VS, vo_s, nf_s, LS, lo_s, n_obs_s))) return rc;
    uint32_t r0 = 0, r1 = 0;
    if (skip < VS && (rc = mg_row(ctx, vo_s, skip, nf_s, r0, r1))) return rc;
    IncSnap fin;
    const uint32_t *tgt;
    std::vector<uint32_t> svmap;
    std::vector<cvb_view_constraints_result> cres;
    cvb_move_result R;
    if ((rc = move_and_constrain(ctx, ccfg, tri, V, poses, vo, vl, bear, desc_out ? desc : nullptr, col_out ? col : nullptr, nf, L, lo, obs, n_obs,
                                 cons, C, VS, poses_s, vo_s, vl_s, bear_s, desc_out ? desc_s : nullptr, col_out ? col_s : nullptr, nf_s, LS, lo_s,
                                 obs_s, n_obs_s, skip, r1 - r0, wt, lmap_in, fin, tgt, svmap, cres, R)))
        return rc;
    cudaStream_t st = ctx->stream;
    if ((rc = inc_copy(ctx, fin, R.counts, poses_out, vo_out, vl_out, bear_out, desc_out, col_out, lo_out, obs_out, cons_out))) return rc;
    if (VS) {
        CVB_CUDA(ctx, cudaMemcpyAsync(svmap_dev, svmap.data(), sizeof(uint32_t) * VS, cudaMemcpyHostToDevice, st));
        CVB_CUDA(ctx, cudaMemcpyAsync(cres_dev, cres.data(), sizeof(cvb_view_constraints_result) * VS, cudaMemcpyHostToDevice, st));
    }
    if (LS) CVB_CUDA(ctx, cudaMemcpyAsync(slmap_dev, tgt, sizeof(uint32_t) * LS, cudaMemcpyDeviceToDevice, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(res_dev, &R, sizeof(R), cudaMemcpyHostToDevice, st));
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    return 0;
}

int merge_reconstructions_dev(cvb_ctx *ctx, const cvb_register_cfg *rcfg, const cvb_constraints_cfg *ccfg, const cvb_recon_cfg *ocfg,
                              const cvb_triangulator *tri, const cvb_arrsac_cfg *arrsac, cvb_rng *rng, uint32_t V, const cvb_pose *poses,
                              const uint32_t *vo, const uint32_t *vl, const double *bear, const uint8_t *desc, const uint8_t *col, uint32_t nf,
                              uint32_t L, const uint32_t *lo, const uint32_t *obs, uint32_t n_obs, const cvb_view_constraint *cons, uint32_t C,
                              uint32_t VS, const cvb_pose *poses_s, const uint32_t *vo_s, const uint32_t *vl_s, const double *bear_s,
                              const uint8_t *desc_s, const uint8_t *col_s, uint32_t nf_s, uint32_t LS, const uint32_t *lo_s, const uint32_t *obs_s,
                              uint32_t n_obs_s, uint32_t s_view, const uint32_t *view_matches, uint32_t H, cvb_pose *poses_out, uint32_t *vo_out,
                              uint32_t *vl_out, double *bear_out, uint8_t *desc_out, uint8_t *col_out, uint32_t *lo_out, uint32_t *obs_out,
                              cvb_view_constraint *cons_out, uint32_t *dvmap, uint32_t *dlmap, uint32_t *svmap_dev, uint32_t *slmap_dev,
                              cvb_view_constraints_result *cres_dev, cvb_merge_result *res_dev) {
    if (!ctx) return CVB_EINVAL;
    if (!rcfg || !ccfg || !ocfg || !tri || !arrsac || !rng || !poses || !vo || !lo || !poses_s || !vo_s || !lo_s || !poses_out || !vo_out ||
        !lo_out || !res_dev || !cons_out || (H && !view_matches) || (nf && (!vl || !bear || !desc)) || (n_obs && !obs) || (C && !cons) ||
        (nf_s && (!vl_s || !bear_s || !desc_s)) || (n_obs_s && !obs_s) || (nf + nf_s && (!vl_out || !bear_out || !desc_out)) ||
        (n_obs + nf_s && !obs_out) || !dvmap || (L && !dlmap) || (VS && (!svmap_dev || !cres_dev)) || (LS && !slmap_dev))
        return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if ((nf && (!col != !col_out)) || (nf_s && (!col_s != !col_out)))
        return cvb_set_error(ctx, CVB_EINVAL, "colours go with both snapshots and the output together");
    if (s_view >= VS) return cvb_set_error(ctx, CVB_EINVAL, "s_view %u >= V_S %u", s_view, VS);
    int rc;
    if ((rc = mg_args(ctx, ccfg, tri, V))) return rc;
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    if ((rc = inc_sizes(ctx, V, vo, nf, L, lo, n_obs))) return rc;
    if ((rc = inc_sizes(ctx, VS, vo_s, nf_s, LS, lo_s, n_obs_s))) return rc;
    uint32_t r0, r1;
    if ((rc = mg_row(ctx, vo_s, s_view, nf_s, r0, r1))) return rc;
    const uint32_t N = r1 - r0;
    cudaStream_t st = ctx->stream;
    const bool hc = col_out != nullptr;
    const uint32_t maxc = ccfg->optimization_maximum_three_view_constraints;
    const uint32_t V1 = V + 1, nf1 = nf + N, L1 = L + N, no1 = n_obs + N, C1 = C + maxc;
    const uint32_t VF = V + VS, LF = L + N + nf_s;   // the largest merged snapshot: views, landmarks
    size_t o[9], off = 0;
    const size_t o_rres = off; off += con_align(sizeof(cvb_register_result));
    const size_t o_rst = off; off += con_align(sizeof(cvb_register_stats));
    const size_t o_m = off; off += con_align(sizeof(cvb_register_match) * std::max<size_t>(N, 1));
    const size_t o_cres = off; off += con_align(sizeof(cvb_view_constraints_result));
    const size_t o_ores = off; off += con_align(sizeof(cvb_recon_result));
    const size_t o_cnt = off; off += con_align(sizeof(cvb_incorporate_counts));
    const size_t o_wt = off; off += con_align(sizeof(cvb_pose));
    const size_t o_pout = off; off += con_align(sizeof(cvb_pose) * VF);
    const size_t o_vs = off; off += con_align(VF);
    const size_t o_os = off; off += con_align(std::max<size_t>((size_t)n_obs + N + nf_s, 1));
    const size_t o_amap = off; off += con_align(sizeof(uint32_t) * std::max<size_t>(L, 1));
    const size_t o_ltl = off; off += con_align(sizeof(uint32_t) * std::max<size_t>(LS, 1));
    const size_t o_svm = off; off += con_align(sizeof(uint32_t) * std::max<size_t>(VS, 1));
    const size_t o_vmap = off; off += con_align(sizeof(uint32_t) * VF);
    const size_t o_lmap = off; off += con_align(sizeof(uint32_t) * std::max<size_t>(LF, 1));
    off = inc_snap_layout(off, V1, nf1, L1, no1, C1, true, hc, o);
    GeomWorkspace *g = gws(ctx);
    if ((rc = g->mrg.ensure(ctx, off))) return rc;
    unsigned char *b = (unsigned char *)g->mrg.p;
    cvb_register_result *rres = (cvb_register_result *)(b + o_rres);
    cvb_register_stats *rst = (cvb_register_stats *)(b + o_rst);
    cvb_register_match *mt = (cvb_register_match *)(b + o_m);
    cvb_view_constraints_result *dcres = (cvb_view_constraints_result *)(b + o_cres);
    cvb_recon_result *ores = (cvb_recon_result *)(b + o_ores);
    cvb_incorporate_counts *cnt = (cvb_incorporate_counts *)(b + o_cnt);
    cvb_pose *wt = (cvb_pose *)(b + o_wt), *pout = (cvb_pose *)(b + o_pout);
    uint8_t *vs = b + o_vs, *os = b + o_os;
    uint32_t *amap = (uint32_t *)(b + o_amap), *ltl = (uint32_t *)(b + o_ltl), *svm = (uint32_t *)(b + o_svm);
    uint32_t *avmap = (uint32_t *)(b + o_vmap), *almap = (uint32_t *)(b + o_lmap);
    IncSnap a = inc_snap_at(b, o, true, hc);
    cvb_merge_result R;
    memset(&R, 0, sizeof(R));
    R.dest_view = CVB_MERGE_NONE;
    std::vector<cvb_view_constraints_result> cres(VS, cvb_view_constraints_result{0, 0});
    // 1. register_frame of s_view's frame against D
    if ((rc = register_frame_dev(ctx, rcfg, tri, arrsac, rng, V, poses, vo, vl, bear, desc, nf, L, lo, obs, n_obs, desc_s + 64 * (size_t)r0,
                                 bear_s + 3 * (size_t)r0, N, view_matches, H, rres, mt, nullptr, rst)))
        return rc;
    CVB_CUDA(ctx, cudaMemcpyAsync(&R.reg, rres, sizeof(cvb_register_result), cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(&R.reg_stats, rst, sizeof(cvb_register_stats), cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    const uint32_t M = R.reg.status == CVB_REGISTER_OK ? R.reg.n_matches : 0;
    // the maps: dest from D, src from S; NONE unless set below
    if (L) CVB_CUDA(ctx, cudaMemsetAsync(dlmap, 0xff, sizeof(uint32_t) * L, st));
    CVB_CUDA(ctx, cudaMemsetAsync(dvmap, 0xff, sizeof(uint32_t) * V, st));
    if (LS) CVB_CUDA(ctx, cudaMemsetAsync(slmap_dev, 0xff, sizeof(uint32_t) * LS, st));
    if (VS) CVB_CUDA(ctx, cudaMemsetAsync(svmap_dev, 0xff, sizeof(uint32_t) * VS, st));
    if (R.reg.status == CVB_REGISTER_PANIC) {
        R.status = CVB_MERGE_REGISTER_PANIC;
    } else if (R.reg.status != CVB_REGISTER_OK) {
        R.status = CVB_MERGE_NOT_REGISTERED;   // D unchanged
        IncSnap d{(cvb_pose *)poses, (uint32_t *)vo, (uint32_t *)vl, (double *)bear, (uint8_t *)desc, (uint8_t *)col, (uint32_t *)lo,
                  (uint32_t *)obs, (cvb_view_constraint *)cons};
        R.counts.V = V; R.counts.n_features = nf; R.counts.L = L; R.counts.n_observations = n_obs; R.counts.C = C;
        if ((rc = inc_copy(ctx, d, R.counts, poses_out, vo_out, vl_out, bear_out, desc_out, col_out, lo_out, obs_out, cons_out))) return rc;
        k_inc_compose<<<cdiv(V, 256), 256, 0, st>>>(V, nullptr, V, nullptr, dvmap);
        CVB_LAUNCH_CHECK(ctx);
        if (L) {
            k_inc_compose<<<cdiv(L, 256), 256, 0, st>>>(L, nullptr, L, nullptr, dlmap);
            CVB_LAUNCH_CHECK(ctx);
        }
    } else {
        // 2. add_view of the frame; its landmark count follows from the matches: L - merges + (N - matches)
        std::vector<cvb_register_match> hm(M);
        if (M) CVB_CUDA(ctx, cudaMemcpyAsync(hm.data(), mt, sizeof(cvb_register_match) * M, cudaMemcpyDeviceToHost, st));
        CVB_CUDA(ctx, cvb_wait(ctx, st));
        uint32_t merges = 0;
        for (const cvb_register_match &m : hm) merges += m.landmark_b != CVB_REGISTER_NONE;
        const uint32_t La = L - merges + (N - M);
        if ((rc = add_view_enqueue(ctx, V, poses, vo, vl, bear, desc, col_out ? col : nullptr, nf, L, lo, obs, n_obs, &rres->pose, bear_s + 3 * (size_t)r0,
                                   desc_s + 64 * (size_t)r0, col_out ? col_s + 3 * (size_t)r0 : nullptr, N, mt, M, a.poses, a.vo, a.vl, a.bear, a.desc,
                                   a.col, a.lo, a.obs, amap, cnt)))
            return rc;
        if (C) CVB_CUDA(ctx, cudaMemcpyAsync(a.cons, cons, sizeof(cvb_view_constraint) * C, cudaMemcpyDeviceToDevice, st));
        // 3. the dest view's constraints
        const uint32_t q = V;
        if ((rc = view_constraints_dev(ctx, ccfg, tri, V1, a.poses, a.vo, a.vl, a.bear, nf1, La, a.lo, a.obs, no1, &q, 1, a.cons + C, dcres, nullptr)))
            return rc;
        CVB_CUDA(ctx, cudaMemcpyAsync(&R.con, dcres, sizeof(cvb_view_constraints_result), cudaMemcpyDeviceToHost, st));
        CVB_CUDA(ctx, cvb_wait(ctx, st));
        const uint32_t Ca = C + R.con.n_constraints;
        if (!R.con.accepted) {
            // remove_view of the dest view: the merges stay, S is untouched
            R.status = CVB_MERGE_REJECTED;
            CVB_CUDA(ctx, cudaMemsetAsync(vs, CVB_RECON_VIEW_KEPT, V, st));
            CVB_CUDA(ctx, cudaMemsetAsync(vs + V, CVB_RECON_VIEW_NO_EDGES, 1, st));
            if (no1) {
                k_inc_reject_states<<<cdiv(no1, 256), 256, 0, st>>>(no1, V, a.obs, os);
                CVB_LAUNCH_CHECK(ctx);
            }
            if ((rc = apply_enqueue(ctx, V1, a.poses, a.vo, a.bear, a.desc, a.col, nf1, La, a.lo, a.obs, no1, a.cons, C, vs, os, poses_out, vo_out,
                                    vl_out, bear_out, desc_out, col_out, lo_out, obs_out, cons_out, avmap, almap, cnt)))
                return rc;
            k_inc_compose<<<cdiv(V, 256), 256, 0, st>>>(V, nullptr, V1, avmap, dvmap);
            CVB_LAUNCH_CHECK(ctx);
            if (L) {
                k_inc_compose<<<cdiv(L, 256), 256, 0, st>>>(L, amap, La, almap, dlmap);
                CVB_LAUNCH_CHECK(ctx);
            }
            CVB_CUDA(ctx, cudaMemcpyAsync(&R.counts, cnt, sizeof(cvb_incorporate_counts), cudaMemcpyDeviceToHost, st));
            CVB_CUDA(ctx, cvb_wait(ctx, st));
        } else {
            // 4. landmark_to_landmark and the world transform
            if (LS) CVB_CUDA(ctx, cudaMemsetAsync(ltl, 0xff, sizeof(uint32_t) * LS, st));
            if (M) {
                k_mg_ltl<<<cdiv(M, 256), 256, 0, st>>>(M, mt, N, vl_s + r0, LS, L, amap, ltl);
                CVB_LAUNCH_CHECK(ctx);
            }
            k_mg_world<<<1, 1, 0, st>>>(&rres->pose, poses_s + s_view, wt);
            CVB_LAUNCH_CHECK(ctx);
            // 5. incorporate_reconstruction with s_view skipped
            IncSnap fin;
            const uint32_t *tgt;
            std::vector<uint32_t> svmap;
            if ((rc = move_and_constrain(ctx, ccfg, tri, V1, a.poses, a.vo, a.vl, a.bear, a.desc, a.col, nf1, La, a.lo, a.obs, no1, a.cons, Ca, VS,
                                         poses_s, vo_s, vl_s, bear_s, desc_s, col_out ? col_s : nullptr, nf_s, LS, lo_s, obs_s, n_obs_s, s_view, N, wt,
                                         ltl, fin, tgt, svmap, cres, R.move)))
                return rc;
            svmap[s_view] = V;
            const cvb_incorporate_counts &f = R.move.counts;
            // 6. optimize_reconstruction and its edits
            if ((rc = optimize_reconstruction_dev(ctx, ocfg, tri, f.V, fin.poses, fin.vo, fin.vl, fin.bear, f.n_features, f.L, fin.lo, fin.obs,
                                                  f.n_observations, fin.cons, f.C, ores, pout, vs, os)))
                return rc;
            CVB_CUDA(ctx, cudaMemcpyAsync(&R.recon, ores, sizeof(cvb_recon_result), cudaMemcpyDeviceToHost, st));
            CVB_CUDA(ctx, cvb_wait(ctx, st));
            if (R.recon.status == CVB_RECON_KEPT) {
                R.status = CVB_MERGE_MERGED;
                if ((rc = apply_enqueue(ctx, f.V, pout, fin.vo, fin.bear, fin.desc, fin.col, f.n_features, f.L, fin.lo, fin.obs, f.n_observations,
                                        fin.cons, f.C, vs, os, poses_out, vo_out, vl_out, bear_out, desc_out, col_out, lo_out, obs_out, cons_out, avmap,
                                        almap, cnt)))
                    return rc;
                // D's views and landmarks kept their indices through the move: add_view's maps, then the optimisation's
                k_inc_compose<<<cdiv(V, 256), 256, 0, st>>>(V, nullptr, f.V, avmap, dvmap);
                CVB_LAUNCH_CHECK(ctx);
                if (L) {
                    k_inc_compose<<<cdiv(L, 256), 256, 0, st>>>(L, amap, f.L, almap, dlmap);
                    CVB_LAUNCH_CHECK(ctx);
                }
                CVB_CUDA(ctx, cudaMemcpyAsync(svm, svmap.data(), sizeof(uint32_t) * VS, cudaMemcpyHostToDevice, st));
                k_inc_compose<<<cdiv(VS, 256), 256, 0, st>>>(VS, svm, f.V, avmap, svmap_dev);
                CVB_LAUNCH_CHECK(ctx);
                if (LS) {
                    k_inc_compose<<<cdiv(LS, 256), 256, 0, st>>>(LS, tgt, f.L, almap, slmap_dev);
                    CVB_LAUNCH_CHECK(ctx);
                }
                uint32_t dv = CVB_MERGE_NONE;
                CVB_CUDA(ctx, cudaMemcpyAsync(&R.counts, cnt, sizeof(cvb_incorporate_counts), cudaMemcpyDeviceToHost, st));
                CVB_CUDA(ctx, cudaMemcpyAsync(&dv, avmap + V, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
                CVB_CUDA(ctx, cvb_wait(ctx, st));
                R.dest_view = dv;
            } else {
                R.status = R.recon.status == CVB_RECON_REMOVED_CONSTRAINTS ? CVB_MERGE_REMOVED_CONSTRAINTS
                         : R.recon.status == CVB_RECON_REMOVED_FILTER      ? CVB_MERGE_REMOVED_FILTER
                                                                           : CVB_MERGE_RECON_PANIC;
            }
        }
    }
    if (VS) CVB_CUDA(ctx, cudaMemcpyAsync(cres_dev, cres.data(), sizeof(cvb_view_constraints_result) * VS, cudaMemcpyHostToDevice, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(res_dev, &R, sizeof(R), cudaMemcpyHostToDevice, st));
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    return 0;
}

namespace {

// S's snapshot (no constraints) into device rows laid out by inc_snap_layout
int mg_upload(cvb_ctx *ctx, const IncSnap &s, uint32_t VS, const cvb_pose *poses, const uint32_t *vo, const uint32_t *vl, const double *bear,
              const uint8_t *desc, const uint8_t *col, uint32_t LS, const uint32_t *lo, const uint32_t *obs) {
    cudaStream_t st = ctx->stream;
    const uint32_t nf = vo[VS], no = lo[LS];
    const cudaMemcpyKind k = cudaMemcpyHostToDevice;
    if (VS) CVB_CUDA(ctx, cudaMemcpyAsync(s.poses, poses, sizeof(cvb_pose) * VS, k, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(s.vo, vo, sizeof(uint32_t) * ((size_t)VS + 1), k, st));
    if (nf) {
        CVB_CUDA(ctx, cudaMemcpyAsync(s.vl, vl, sizeof(uint32_t) * (size_t)nf, k, st));
        CVB_CUDA(ctx, cudaMemcpyAsync(s.bear, bear, sizeof(double) * 3 * (size_t)nf, k, st));
        if (desc && s.desc) CVB_CUDA(ctx, cudaMemcpyAsync(s.desc, desc, 64 * (size_t)nf, k, st));
        if (col && s.col) CVB_CUDA(ctx, cudaMemcpyAsync(s.col, col, 3 * (size_t)nf, k, st));
    }
    CVB_CUDA(ctx, cudaMemcpyAsync(s.lo, lo, sizeof(uint32_t) * ((size_t)LS + 1), k, st));
    if (no) CVB_CUDA(ctx, cudaMemcpyAsync(s.obs, obs, sizeof(uint32_t) * 2 * (size_t)no, k, st));
    return 0;
}

}  // namespace

int incorporate_reconstruction(cvb_ctx *ctx, const cvb_constraints_cfg *ccfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses,
                               const uint32_t *vo, const uint32_t *vl, const double *bear, const uint8_t *desc, const uint8_t *col, uint32_t L,
                               const uint32_t *lo, const uint32_t *obs, const cvb_view_constraint *cons, uint32_t C, uint32_t VS,
                               const cvb_pose *poses_s, const uint32_t *vo_s, const uint32_t *vl_s, const double *bear_s, const uint8_t *desc_s,
                               const uint8_t *col_s, uint32_t LS, const uint32_t *lo_s, const uint32_t *obs_s, uint32_t skip, const cvb_pose *wt,
                               const uint32_t *lmap, cvb_pose *poses_out, uint32_t *vo_out, uint32_t *vl_out, double *bear_out, uint8_t *desc_out,
                               uint8_t *col_out, uint32_t *lo_out, uint32_t *obs_out, cvb_view_constraint *cons_out, uint32_t *svmap,
                               uint32_t *slmap, cvb_view_constraints_result *cres, cvb_move_result *res) {
    if (!ctx) return CVB_EINVAL;
    if (!ccfg || !tri || !poses || !poses_s || !wt || !poses_out || !vo_out || !lo_out || !cons_out || !res || (LS && (!lmap || !slmap)) ||
        (VS && (!svmap || !cres)))
        return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    static const uint32_t no_entries = 0;   // a map of L_S = 0 entries
    if (merge_check(V, vo, vl, L, lo, obs, cons, C, VS, vo_s, vl_s, LS, lo_s, obs_s, skip, lmap ? lmap : &no_entries, col != nullptr,
                    col_s != nullptr))
        return cvb_set_error(ctx, CVB_EINVAL, "malformed snapshots, skip_view or landmark map");
    const uint32_t nf = vo[V], no = lo[L], nf_s = vo_s[VS], no_s = lo_s[LS];
    if ((nf && (!bear || !vl_out || !bear_out)) || (nf_s && (!bear_s || !vl_out || !bear_out)) || (no + nf_s && !obs_out))
        return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if ((nf && (!desc != !desc_out)) || (nf_s && (!desc_s != !desc_out)) || (nf && (!col != !col_out)) || (nf_s && (!col_s != !col_out)))
        return cvb_set_error(ctx, CVB_EINVAL, "descriptors and colours go with both snapshots and the output together");
    const bool hd = desc_out != nullptr, hc = col_out != nullptr;
    const uint32_t maxc = ccfg->optimization_maximum_three_view_constraints;
    size_t x = 0, os_[9], o[9];
    const size_t i_wt = x; x += con_align(sizeof(cvb_pose));
    const size_t i_lm = x; x += con_align(sizeof(uint32_t) * std::max<size_t>(LS, 1));
    const size_t i_svm = x; x += con_align(sizeof(uint32_t) * std::max<size_t>(VS, 1));
    const size_t i_slm = x; x += con_align(sizeof(uint32_t) * std::max<size_t>(LS, 1));
    const size_t i_cr = x; x += con_align(sizeof(cvb_view_constraints_result) * std::max<size_t>(VS, 1));
    const size_t i_res = x; x += con_align(sizeof(cvb_move_result));
    x = inc_snap_layout(x, VS, nf_s, LS, no_s, 0, hd, hc, os_);
    x = inc_snap_layout(x, V + VS, nf + nf_s, L + nf_s, no + nf_s, C + VS * maxc, hd, hc, o);
    IncSnap s;
    unsigned char *b;
    size_t end;
    int rc;
    if ((rc = inc_upload(ctx, V, poses, vo, vl, bear, hd ? desc : nullptr, hc ? col : nullptr, L, lo, obs, cons, C, x, s, b, end))) return rc;
    unsigned char *e = b + end;
    cudaStream_t st = ctx->stream;
    IncSnap ss = inc_snap_at(e, os_, hd, hc), out = inc_snap_at(e, o, hd, hc);
    if ((rc = mg_upload(ctx, ss, VS, poses_s, vo_s, vl_s, bear_s, desc_s, col_s, LS, lo_s, obs_s))) return rc;
    CVB_CUDA(ctx, cudaMemcpyAsync(e + i_wt, wt, sizeof(cvb_pose), cudaMemcpyHostToDevice, st));
    if (LS) CVB_CUDA(ctx, cudaMemcpyAsync(e + i_lm, lmap, sizeof(uint32_t) * LS, cudaMemcpyHostToDevice, st));
    if ((rc = incorporate_reconstruction_dev(ctx, ccfg, tri, V, s.poses, s.vo, s.vl, s.bear, s.desc, s.col, nf, L, s.lo, s.obs, no, s.cons, C, VS,
                                             ss.poses, ss.vo, ss.vl, ss.bear, ss.desc, ss.col, nf_s, LS, ss.lo, ss.obs, no_s, skip,
                                             (const cvb_pose *)(e + i_wt), (const uint32_t *)(e + i_lm), out.poses, out.vo, out.vl, out.bear,
                                             out.desc, out.col, out.lo, out.obs, out.cons, (uint32_t *)(e + i_svm), (uint32_t *)(e + i_slm),
                                             (cvb_view_constraints_result *)(e + i_cr), (cvb_move_result *)(e + i_res))))
        return rc;
    CVB_CUDA(ctx, cudaMemcpyAsync(res, e + i_res, sizeof(cvb_move_result), cudaMemcpyDeviceToHost, st));
    if (VS) {
        CVB_CUDA(ctx, cudaMemcpyAsync(svmap, e + i_svm, sizeof(uint32_t) * VS, cudaMemcpyDeviceToHost, st));
        CVB_CUDA(ctx, cudaMemcpyAsync(cres, e + i_cr, sizeof(cvb_view_constraints_result) * VS, cudaMemcpyDeviceToHost, st));
    }
    if (LS) CVB_CUDA(ctx, cudaMemcpyAsync(slmap, e + i_slm, sizeof(uint32_t) * LS, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    return inc_download(ctx, out, res->counts, hd, hc, poses_out, vo_out, vl_out, bear_out, desc_out, col_out, lo_out, obs_out, cons_out);
}

int merge_reconstructions(cvb_ctx *ctx, const cvb_register_cfg *rcfg, const cvb_constraints_cfg *ccfg, const cvb_recon_cfg *ocfg,
                          const cvb_triangulator *tri, const cvb_arrsac_cfg *arrsac, cvb_rng *rng, uint32_t V, const cvb_pose *poses,
                          const uint32_t *vo, const uint32_t *vl, const double *bear, const uint8_t *desc, const uint8_t *col, uint32_t L,
                          const uint32_t *lo, const uint32_t *obs, const cvb_view_constraint *cons, uint32_t C, uint32_t VS, const cvb_pose *poses_s,
                          const uint32_t *vo_s, const uint32_t *vl_s, const double *bear_s, const uint8_t *desc_s, const uint8_t *col_s, uint32_t LS,
                          const uint32_t *lo_s, const uint32_t *obs_s, uint32_t s_view, const uint32_t *view_matches, uint32_t H,
                          cvb_pose *poses_out, uint32_t *vo_out, uint32_t *vl_out, double *bear_out, uint8_t *desc_out, uint8_t *col_out,
                          uint32_t *lo_out, uint32_t *obs_out, cvb_view_constraint *cons_out, uint32_t *dvmap, uint32_t *dlmap, uint32_t *svmap,
                          uint32_t *slmap, cvb_view_constraints_result *cres, cvb_merge_result *res) {
    if (!ctx) return CVB_EINVAL;
    if (!rcfg || !ccfg || !ocfg || !tri || !arrsac || !rng || !poses || !poses_s || !res || !poses_out || !vo_out || !lo_out || !cons_out ||
        !dvmap || (L && !dlmap) || (VS && (!svmap || !cres)) || (LS && !slmap))
        return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (merge_check(V, vo, vl, L, lo, obs, cons, C, VS, vo_s, vl_s, LS, lo_s, obs_s, s_view, nullptr, col != nullptr, col_s != nullptr) ||
        register_check(V, vo, vl, L, lo, obs, view_matches, H))
        return cvb_set_error(ctx, CVB_EINVAL, "malformed snapshots, s_view or view matches");
    const uint32_t nf = vo[V], no = lo[L], nf_s = vo_s[VS], no_s = lo_s[LS];
    if ((nf && (!bear || !desc)) || (nf_s && (!bear_s || !desc_s)) || (nf + nf_s && (!vl_out || !bear_out || !desc_out)) || (no + nf_s && !obs_out))
        return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if ((nf && (!col != !col_out)) || (nf_s && (!col_s != !col_out)))
        return cvb_set_error(ctx, CVB_EINVAL, "colours go with both snapshots and the output together");
    const bool hc = col_out != nullptr;
    const uint32_t maxc = ccfg->optimization_maximum_three_view_constraints;
    size_t x = 0, os_[9], o[9];
    const size_t i_dvm = x; x += con_align(sizeof(uint32_t) * std::max<size_t>(V, 1));
    const size_t i_dlm = x; x += con_align(sizeof(uint32_t) * std::max<size_t>(L, 1));
    const size_t i_svm = x; x += con_align(sizeof(uint32_t) * std::max<size_t>(VS, 1));
    const size_t i_slm = x; x += con_align(sizeof(uint32_t) * std::max<size_t>(LS, 1));
    const size_t i_cr = x; x += con_align(sizeof(cvb_view_constraints_result) * std::max<size_t>(VS, 1));
    const size_t i_res = x; x += con_align(sizeof(cvb_merge_result));
    x = inc_snap_layout(x, VS, nf_s, LS, no_s, 0, true, hc, os_);
    x = inc_snap_layout(x, V + VS, nf + nf_s, L + no + 4 * nf_s, no + 2 * nf_s, C + (VS + 1) * maxc, true, hc, o);
    IncSnap s;
    unsigned char *b;
    size_t end;
    int rc;
    if ((rc = inc_upload(ctx, V, poses, vo, vl, bear, desc, hc ? col : nullptr, L, lo, obs, cons, C, x, s, b, end))) return rc;
    unsigned char *e = b + end;
    cudaStream_t st = ctx->stream;
    IncSnap ss = inc_snap_at(e, os_, true, hc), out = inc_snap_at(e, o, true, hc);
    if ((rc = mg_upload(ctx, ss, VS, poses_s, vo_s, vl_s, bear_s, desc_s, hc ? col_s : nullptr, LS, lo_s, obs_s))) return rc;
    cvb_merge_result *rd = (cvb_merge_result *)(e + i_res);
    if ((rc = merge_reconstructions_dev(ctx, rcfg, ccfg, ocfg, tri, arrsac, rng, V, s.poses, s.vo, s.vl, s.bear, s.desc, s.col, nf, L, s.lo, s.obs, no,
                                        s.cons, C, VS, ss.poses, ss.vo, ss.vl, ss.bear, ss.desc, ss.col, nf_s, LS, ss.lo, ss.obs, no_s, s_view,
                                        view_matches, H, out.poses, out.vo, out.vl, out.bear, out.desc, out.col, out.lo, out.obs, out.cons,
                                        (uint32_t *)(e + i_dvm), (uint32_t *)(e + i_dlm), (uint32_t *)(e + i_svm), (uint32_t *)(e + i_slm),
                                        (cvb_view_constraints_result *)(e + i_cr), rd)))
        return rc;
    CVB_CUDA(ctx, cudaMemcpyAsync(res, rd, sizeof(cvb_merge_result), cudaMemcpyDeviceToHost, st));
    if (V) CVB_CUDA(ctx, cudaMemcpyAsync(dvmap, e + i_dvm, sizeof(uint32_t) * V, cudaMemcpyDeviceToHost, st));
    if (L) CVB_CUDA(ctx, cudaMemcpyAsync(dlmap, e + i_dlm, sizeof(uint32_t) * L, cudaMemcpyDeviceToHost, st));
    if (VS) {
        CVB_CUDA(ctx, cudaMemcpyAsync(svmap, e + i_svm, sizeof(uint32_t) * VS, cudaMemcpyDeviceToHost, st));
        CVB_CUDA(ctx, cudaMemcpyAsync(cres, e + i_cr, sizeof(cvb_view_constraints_result) * VS, cudaMemcpyDeviceToHost, st));
    }
    if (LS) CVB_CUDA(ctx, cudaMemcpyAsync(slmap, e + i_slm, sizeof(uint32_t) * LS, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    const bool have = res->status == CVB_MERGE_MERGED || res->status == CVB_MERGE_REJECTED || res->status == CVB_MERGE_NOT_REGISTERED;
    if (!have) return 0;
    return inc_download(ctx, out, res->counts, true, hc, poses_out, vo_out, vl_out, bear_out, desc_out, col_out, lo_out, obs_out, cons_out);
}

// ---- cv-sfm's reconstruction creation (C names in try_init_abi.cu, include/cvb200_try_init.h; kernels in try_init_dev.cuh) -------------
int try_init_check(uint32_t nc, uint32_t n1, uint32_t n2, uint32_t center, uint32_t first, uint32_t second, const uint32_t *comb, uint32_t K,
                   const uint32_t *fm, uint32_t K1, const uint32_t *sm, uint32_t K2) {
    if (center == first || center == second || first == second) return CVB_EINVAL;
    if ((K && !comb) || (K1 && !fm) || (K2 && !sm)) return CVB_EINVAL;
    // view col (1 or 2): every entry in range, each of its features and each center feature mapped into it at most once (HashMap::insert
    // would otherwise drop an entry or an observation)
    auto view = [&](uint32_t n, const uint32_t *m, uint32_t M, uint32_t col) {
        std::vector<uint8_t> fu(n, 0), cu(nc, 0);
        auto add = [&](uint32_t c, uint32_t f) {
            if (c >= nc || f >= n || fu[f] || cu[c]) return false;
            fu[f] = cu[c] = 1;
            return true;
        };
        for (uint32_t i = 0; i < M; i++)
            if (!add(m[2 * (size_t)i], m[2 * (size_t)i + 1])) return false;
        for (uint32_t i = 0; i < K; i++)
            if (!add(comb[3 * (size_t)i], comb[3 * (size_t)i + col])) return false;
        return true;
    };
    return view(n1, fm, K1, 1) && view(n2, sm, K2, 2) ? 0 : CVB_EINVAL;
}

namespace {

// the refusals of the frame indices every entry shares
int ti_frames(cvb_ctx *ctx, uint32_t frames, uint32_t cap, uint32_t center, uint32_t first, uint32_t second) {
    if (cap == 0) return cvb_set_error(ctx, CVB_EINVAL, "zero capacity");
    if (center >= frames || first >= frames || second >= frames)
        return cvb_set_error(ctx, CVB_EINVAL, "frames %u, %u, %u of %u", center, first, second, frames);
    if (center == first || center == second || first == second) return cvb_set_error(ctx, CVB_EINVAL, "two equal frames");
    return 0;
}

// a grid of at most 64 CTAs of 256 threads: the rows are few, and every try_init_dev.cuh kernel strides past the grid
uint32_t ti_grid(uint32_t n) { return std::max<uint32_t>(std::min<uint32_t>(cdiv(n, 256), 64), 1); }

// add_reconstruction enqueued on the context's stream (no wait); scratch in the context's creation scratch buffer
int add_reconstruction_enqueue(cvb_ctx *ctx, const uint8_t *desc, const uint32_t *n, const double *bear, const uint8_t *col, uint32_t cap,
                               TiFrames fr, const cvb_init_result *ir, const uint32_t *comb, const uint32_t *fm, const uint32_t *sm,
                               cvb_pose *poses_out, uint32_t *vo_out, uint32_t *vl_out, double *bear_out, uint8_t *desc_out, uint8_t *col_out,
                               uint32_t *lo_out, uint32_t *obs_out, cvb_view_constraint *cons_out, cvb_incorporate_counts *counts) {
    const uint32_t n3 = 3 * cap;
    size_t off = 0;
    const size_t o_maps = off; off += con_align(sizeof(uint32_t) * 4 * (size_t)cap);
    const size_t o_cnt = off; off += con_align(sizeof(uint2) * (size_t)n3);
    const size_t o_tiles = off; off += con_align(sizeof(uint2) * (size_t)cdiv(n3, INC_TILE));
    const size_t o_total = off; off += con_align(sizeof(uint2));
    GeomWorkspace *g = gws(ctx);
    int rc;
    if ((rc = g->tinit.ensure(ctx, off))) return rc;
    unsigned char *b = (unsigned char *)g->tinit.p;
    uint32_t *maps = (uint32_t *)(b + o_maps), *fmap1 = maps, *fmap2 = maps + cap, *cmap1 = maps + 2 * (size_t)cap, *cmap2 = maps + 3 * (size_t)cap;
    uint2 *cnt = (uint2 *)(b + o_cnt), *tiles = (uint2 *)(b + o_tiles), *total = (uint2 *)(b + o_total);
    cudaStream_t st = ctx->stream;
    CVB_PROF(ctx, "k_ti", 0);
    k_ti_clear<<<ti_grid(4 * cap), 256, 0, st>>>(4 * cap, maps);
    CVB_LAUNCH_CHECK(ctx);
    k_ti_map<<<ti_grid(cap), 256, 0, st>>>(cap, fr, n, ir, comb, fm, sm, fmap1, fmap2, cmap1, cmap2);
    CVB_LAUNCH_CHECK(ctx);
    k_ti_counts<<<ti_grid(n3), 256, 0, st>>>(cap, fr, n, fmap1, fmap2, cmap1, cmap2, cnt);
    CVB_LAUNCH_CHECK(ctx);
    if ((rc = inc_scan(ctx, n3, cnt, tiles, total))) return rc;
    k_ti_place<<<ti_grid(n3), 256, 0, st>>>(cap, fr, n, bear, (const uint4 *)desc, col, fmap1, fmap2, cmap1, cmap2, cnt, vl_out, bear_out,
                                            (uint4 *)desc_out, col_out, lo_out, obs_out);
    CVB_LAUNCH_CHECK(ctx);
    k_ti_finish<<<1, 1, 0, st>>>(cap, fr, n, ir, total, poses_out, vo_out, lo_out, cons_out, counts);
    CVB_LAUNCH_CHECK(ctx);
    return 0;
}

}  // namespace

int add_reconstruction_dev(cvb_ctx *ctx, const uint8_t *desc, const uint32_t *n, const double *bear, const uint8_t *col, uint32_t frames,
                           uint32_t cap, uint32_t center, uint32_t first, uint32_t second, const cvb_init_result *ir, const uint32_t *comb,
                           const uint32_t *fm, const uint32_t *sm, cvb_pose *poses_out, uint32_t *vo_out, uint32_t *vl_out, double *bear_out,
                           uint8_t *desc_out, uint8_t *col_out, uint32_t *lo_out, uint32_t *obs_out, cvb_view_constraint *cons_out,
                           cvb_incorporate_counts *counts) {
    if (!ctx) return CVB_EINVAL;
    if (!desc || !n || !bear || !ir || !comb || !fm || !sm || !poses_out || !vo_out || !vl_out || !bear_out || !desc_out || !lo_out || !obs_out ||
        !cons_out || !counts)
        return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (!col != !col_out) return cvb_set_error(ctx, CVB_EINVAL, "colours go with the frame store and the output together");
    int rc;
    if ((rc = ti_frames(ctx, frames, cap, center, first, second))) return rc;
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    if ((rc = add_reconstruction_enqueue(ctx, desc, n, bear, col, cap, TiFrames{{center, first, second}}, ir, comb, fm, sm, poses_out, vo_out,
                                         vl_out, bear_out, desc_out, col_out, lo_out, obs_out, cons_out, counts)))
        return rc;
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    return 0;
}

int try_init_dev(cvb_ctx *ctx, const cvb_init_cfg *icfg, const cvb_triangulator *tri, const cvb_arrsac_cfg *arrsac, cvb_rng *rngs,
                 uint32_t better_by, const uint8_t *desc, const uint32_t *n, const double *bear, const uint8_t *col, uint32_t frames, uint32_t cap,
                 uint32_t center, const uint32_t *options, uint32_t F, cvb_pose *poses_out, uint32_t *vo_out, uint32_t *vl_out, double *bear_out,
                 uint8_t *desc_out, uint8_t *col_out, uint32_t *lo_out, uint32_t *obs_out, cvb_view_constraint *cons_out,
                 cvb_try_init_result *res_dev) {
    if (!ctx) return CVB_EINVAL;
    if (!icfg || !tri || !arrsac || (F && (!rngs || !options)) || !desc || !n || !bear || !poses_out || !vo_out || !vl_out || !bear_out ||
        !desc_out || !lo_out || !obs_out || !cons_out || !res_dev)
        return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (!col != !col_out) return cvb_set_error(ctx, CVB_EINVAL, "colours go with the frame store and the output together");
    if (F > CVB_ARRSAC_BATCH_MAX) return cvb_set_error(ctx, CVB_EUNSUPPORTED, "%u options: at most %u", F, CVB_ARRSAC_BATCH_MAX);
    if (tri->method < CVB_TRI_LINEAR_EIGEN || tri->method > CVB_TRI_MEAN_MEAN)
        return cvb_set_error(ctx, tri->method >= CVB_TRI_RELATIVE_DLT && tri->method <= CVB_TRI_ANGULAR_LINF ? CVB_EUNSUPPORTED : CVB_EINVAL,
                             "triangulator method %d: try_init takes a TriangulatorObservations (methods 0-2)", tri->method);
    if (cap == 0) return cvb_set_error(ctx, CVB_EINVAL, "zero capacity");
    if (center >= frames) return cvb_set_error(ctx, CVB_EINVAL, "center frame %u of %u", center, frames);
    for (uint32_t f = 0; f < F; f++)
        if (options[f] >= frames) return cvb_set_error(ctx, CVB_EINVAL, "option %u: frame %u of %u", f, options[f], frames);
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    // the two-view outputs and the init's result and lists stay in the context's creation buffer
    const uint32_t Fm = std::max<uint32_t>(F, 1);
    size_t off = 0;
    const size_t o_pairs = off; off += con_align(sizeof(uint32_t) * 2 * (size_t)Fm * cap);
    const size_t o_np = off; off += con_align(sizeof(uint32_t) * Fm);
    const size_t o_model = off; off += con_align(sizeof(cvb_pose) * Fm);
    const size_t o_inl = off; off += con_align(sizeof(uint32_t) * (size_t)Fm * cap);
    const size_t o_ninl = off; off += con_align(sizeof(uint32_t) * Fm);
    const size_t o_found = off; off += con_align(sizeof(int32_t) * Fm);
    const size_t o_ir = off; off += con_align(sizeof(cvb_init_result));
    const size_t o_comb = off; off += con_align(sizeof(uint32_t) * 3 * (size_t)cap);
    const size_t o_fm = off; off += con_align(sizeof(uint32_t) * 2 * (size_t)cap);
    const size_t o_sm = off; off += con_align(sizeof(uint32_t) * 2 * (size_t)cap);
    GeomWorkspace *g = gws(ctx);
    int rc;
    if ((rc = g->tinits.ensure(ctx, off))) return rc;
    unsigned char *b = (unsigned char *)g->tinits.p;
    uint32_t *pairs = (uint32_t *)(b + o_pairs), *np = (uint32_t *)(b + o_np), *inl = (uint32_t *)(b + o_inl), *ninl = (uint32_t *)(b + o_ninl);
    cvb_pose *model = (cvb_pose *)(b + o_model);
    int32_t *found = (int32_t *)(b + o_found);
    cvb_init_result *ir = (cvb_init_result *)(b + o_ir);
    uint32_t *comb = (uint32_t *)(b + o_comb), *fm = (uint32_t *)(b + o_fm), *sm = (uint32_t *)(b + o_sm);
    cudaStream_t st = ctx->stream;
    if (F) {
        if ((rc = two_view_options_dev(ctx, desc, n, bear, frames, cap, center, options, F, better_by, arrsac, rngs, pairs, np, model, inl, ninl,
                                       found)))
            return rc;
        if ((rc = ars_commit_rng_batch(ctx, rngs, F, nullptr))) return rc;
    }
    if ((rc = init_reconstruction_dev(ctx, icfg, tri, bear, frames, cap, center, options, F, pairs, np, model, inl, ninl, found, ir, comb, fm, sm,
                                      nullptr)))
        return rc;
    cvb_init_result *h = (cvb_init_result *)cvb_pinned(ctx, sizeof(cvb_init_result));
    if (!h) return cvb_set_error(ctx, CVB_ENOMEM, "page-locked scratch");
    CVB_CUDA(ctx, cudaMemcpyAsync(h, ir, sizeof(cvb_init_result), cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    cvb_try_init_result R;
    memset(&R, 0, sizeof(R));
    R.init = *h;
    R.status = R.init.status == CVB_INIT_ACCEPTED ? CVB_TRY_INIT_CREATED
                                                  : (R.init.status == CVB_INIT_NONE_BEARING_PAIRS ? CVB_TRY_INIT_NONE_BEARING_PAIRS : CVB_TRY_INIT_NONE);
    R.frames[0] = center;
    R.frames[1] = R.frames[2] = CVB_TRY_INIT_NO_FRAME;
    if (R.init.status != CVB_INIT_NONE && R.init.first < F && R.init.second < F) {
        R.frames[1] = options[R.init.first];
        R.frames[2] = options[R.init.second];
    }
    // the record first, then (created) the snapshot, whose counts the placement writes into it
    CVB_CUDA(ctx, cudaMemcpyAsync(res_dev, &R, sizeof(R), cudaMemcpyHostToDevice, st));
    if (R.status == CVB_TRY_INIT_CREATED &&
        (rc = add_reconstruction_enqueue(ctx, desc, n, bear, col, cap, TiFrames{{R.frames[0], R.frames[1], R.frames[2]}}, ir, comb, fm, sm,
                                         poses_out, vo_out, vl_out, bear_out, desc_out, col_out, lo_out, obs_out, cons_out, &res_dev->counts)))
        return rc;
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    return 0;
}

int add_reconstruction(cvb_ctx *ctx, const uint8_t *desc, const uint32_t *n, const double *bear, const uint8_t *col, uint32_t frames, uint32_t cap,
                       uint32_t center, uint32_t first, uint32_t second, const cvb_init_result *ir, const uint32_t *comb, const uint32_t *fm,
                       const uint32_t *sm, cvb_pose *poses_out, uint32_t *vo_out, uint32_t *vl_out, double *bear_out, uint8_t *desc_out,
                       uint8_t *col_out, uint32_t *lo_out, uint32_t *obs_out, cvb_view_constraint *cons_out, cvb_incorporate_counts *counts) {
    if (!ctx) return CVB_EINVAL;
    if (!desc || !n || !bear || !ir || !poses_out || !vo_out || !vl_out || !bear_out || !desc_out || !lo_out || !obs_out || !cons_out || !counts)
        return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (!col != !col_out) return cvb_set_error(ctx, CVB_EINVAL, "colours go with the frame store and the output together");
    int rc;
    if ((rc = ti_frames(ctx, frames, cap, center, first, second))) return rc;
    const uint32_t fr[3] = {center, first, second}, K = ir->n_combined, K1 = ir->n_first_matches, K2 = ir->n_second_matches;
    if (try_init_check(std::min(n[center], cap), std::min(n[first], cap), std::min(n[second], cap), center, first, second, comb, K, fm, K1, sm, K2))
        return cvb_set_error(ctx, CVB_EINVAL, "malformed match lists");
    // the three frames as a store of three, the result and the lists uploaded; the outputs after them
    const bool hc = col != nullptr;
    size_t x = 0, o[9];
    const size_t i_desc = x; x += con_align(64 * 3 * (size_t)cap);
    const size_t i_bear = x; x += con_align(sizeof(double) * 9 * (size_t)cap);
    const size_t i_col = x; x += hc ? con_align(9 * (size_t)cap) : 0;
    const size_t i_n = x; x += con_align(sizeof(uint32_t) * 3);
    const size_t i_ir = x; x += con_align(sizeof(cvb_init_result));
    const size_t i_comb = x; x += con_align(sizeof(uint32_t) * 3 * (size_t)cap);
    const size_t i_fm = x; x += con_align(sizeof(uint32_t) * 2 * (size_t)cap);
    const size_t i_sm = x; x += con_align(sizeof(uint32_t) * 2 * (size_t)cap);
    const size_t i_cnt = x; x += con_align(sizeof(cvb_incorporate_counts));
    x = inc_snap_layout(x, 3, 3 * cap, 3 * cap, 3 * cap, 1, true, hc, o);
    GeomWorkspace *g = gws(ctx);
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    if ((rc = g->out.ensure(ctx, x))) return rc;
    unsigned char *b = (unsigned char *)g->out.p;
    IncSnap out = inc_snap_at(b, o, true, hc);
    cudaStream_t st = ctx->stream;
    const cudaMemcpyKind k = cudaMemcpyHostToDevice;
    uint32_t n3[3];
    for (int v = 0; v < 3; v++) {
        n3[v] = std::min(n[fr[v]], cap);
        const size_t s = (size_t)fr[v] * cap;
        CVB_CUDA(ctx, cudaMemcpyAsync(b + i_desc + 64 * (size_t)v * cap, desc + 64 * s, 64 * (size_t)n3[v], k, st));
        CVB_CUDA(ctx, cudaMemcpyAsync(b + i_bear + sizeof(double) * 3 * (size_t)v * cap, bear + 3 * s, sizeof(double) * 3 * (size_t)n3[v], k, st));
        if (hc) CVB_CUDA(ctx, cudaMemcpyAsync(b + i_col + 3 * (size_t)v * cap, col + 3 * s, 3 * (size_t)n3[v], k, st));
    }
    CVB_CUDA(ctx, cudaMemcpyAsync(b + i_n, n3, sizeof(n3), k, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(b + i_ir, ir, sizeof(cvb_init_result), k, st));
    if (K) CVB_CUDA(ctx, cudaMemcpyAsync(b + i_comb, comb, sizeof(uint32_t) * 3 * (size_t)K, k, st));
    if (K1) CVB_CUDA(ctx, cudaMemcpyAsync(b + i_fm, fm, sizeof(uint32_t) * 2 * (size_t)K1, k, st));
    if (K2) CVB_CUDA(ctx, cudaMemcpyAsync(b + i_sm, sm, sizeof(uint32_t) * 2 * (size_t)K2, k, st));
    if ((rc = add_reconstruction_enqueue(ctx, b + i_desc, (const uint32_t *)(b + i_n), (const double *)(b + i_bear), hc ? b + i_col : nullptr, cap,
                                         TiFrames{{0, 1, 2}}, (const cvb_init_result *)(b + i_ir), (const uint32_t *)(b + i_comb),
                                         (const uint32_t *)(b + i_fm), (const uint32_t *)(b + i_sm), out.poses, out.vo, out.vl, out.bear, out.desc,
                                         out.col, out.lo, out.obs, out.cons, (cvb_incorporate_counts *)(b + i_cnt))))
        return rc;
    CVB_CUDA(ctx, cudaMemcpyAsync(counts, b + i_cnt, sizeof(cvb_incorporate_counts), cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    return inc_download(ctx, out, *counts, true, hc, poses_out, vo_out, vl_out, bear_out, desc_out, col_out, lo_out, obs_out, cons_out);
}

int try_init(cvb_ctx *ctx, const cvb_init_cfg *icfg, const cvb_triangulator *tri, const cvb_arrsac_cfg *arrsac, cvb_rng *rngs, uint32_t better_by,
             const uint8_t *desc, const uint32_t *n, const double *bear, const uint8_t *col, uint32_t frames, uint32_t cap, uint32_t center,
             const uint32_t *options, uint32_t F, cvb_pose *poses_out, uint32_t *vo_out, uint32_t *vl_out, double *bear_out, uint8_t *desc_out,
             uint8_t *col_out, uint32_t *lo_out, uint32_t *obs_out, cvb_view_constraint *cons_out, cvb_try_init_result *res) {
    if (!ctx) return CVB_EINVAL;
    if (!desc || !n || !bear || !res || !poses_out || !vo_out || !vl_out || !bear_out || !desc_out || !lo_out || !obs_out || !cons_out)
        return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (!col != !col_out) return cvb_set_error(ctx, CVB_EINVAL, "colours go with the frame store and the output together");
    const bool hc = col != nullptr;
    const size_t rows = (size_t)frames * cap;
    size_t x = 0, o[9];
    const size_t i_desc = x; x += con_align(64 * std::max<size_t>(rows, 1));
    const size_t i_bear = x; x += con_align(sizeof(double) * 3 * std::max<size_t>(rows, 1));
    const size_t i_col = x; x += hc ? con_align(3 * std::max<size_t>(rows, 1)) : 0;
    const size_t i_n = x; x += con_align(sizeof(uint32_t) * std::max<uint32_t>(frames, 1));
    const size_t i_res = x; x += con_align(sizeof(cvb_try_init_result));
    x = inc_snap_layout(x, 3, 3 * cap, 3 * cap, 3 * cap, 1, true, hc, o);
    GeomWorkspace *g = gws(ctx);
    int rc;
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    if ((rc = g->out.ensure(ctx, x))) return rc;
    unsigned char *b = (unsigned char *)g->out.p;
    IncSnap out = inc_snap_at(b, o, true, hc);
    cudaStream_t st = ctx->stream;
    if (rows) {
        CVB_CUDA(ctx, cudaMemcpyAsync(b + i_desc, desc, 64 * rows, cudaMemcpyHostToDevice, st));
        CVB_CUDA(ctx, cudaMemcpyAsync(b + i_bear, bear, sizeof(double) * 3 * rows, cudaMemcpyHostToDevice, st));
        if (hc) CVB_CUDA(ctx, cudaMemcpyAsync(b + i_col, col, 3 * rows, cudaMemcpyHostToDevice, st));
    }
    if (frames) CVB_CUDA(ctx, cudaMemcpyAsync(b + i_n, n, sizeof(uint32_t) * frames, cudaMemcpyHostToDevice, st));
    cvb_try_init_result *rd = (cvb_try_init_result *)(b + i_res);
    if ((rc = try_init_dev(ctx, icfg, tri, arrsac, rngs, better_by, b + i_desc, (const uint32_t *)(b + i_n), (const double *)(b + i_bear),
                           hc ? b + i_col : nullptr, frames, cap, center, options, F, out.poses, out.vo, out.vl, out.bear, out.desc, out.col, out.lo,
                           out.obs, out.cons, rd)))
        return rc;
    CVB_CUDA(ctx, cudaMemcpyAsync(res, rd, sizeof(cvb_try_init_result), cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    if (res->status != CVB_TRY_INIT_CREATED) return 0;
    return inc_download(ctx, out, res->counts, true, hc, poses_out, vo_out, vl_out, bear_out, desc_out, col_out, lo_out, obs_out, cons_out);
}

extern "C" {

void cvb_arrsac_default_cfg(cvb_arrsac_cfg *c, double inlier_threshold) {
    if (!c) return;
    c->inlier_threshold = inlier_threshold;
    c->initialization_hypotheses = 256; c->initialization_blocks = 4; c->max_candidate_hypotheses = 64;
    c->estimations_per_block = 64; c->block_size = 64;
    c->likelihood_ratio_threshold = 1e3f; c->initial_epsilon = 0.1f; c->initial_delta = 0.05f;
}

void cvb_rng_seed_xoshiro256pp(cvb_rng *r, uint64_t seed) {   // SplitMix64 expansion
    if (!r) return;
    r->kind = 0;
    for (int i = 0; i < 4; i++) {
        seed += 0x9e3779b97f4a7c15ull;
        uint64_t z = seed;
        z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
        z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
        r->s[i] = z ^ (z >> 31);
    }
}

void cvb_rng_seed_pcg64(cvb_rng *r, const uint8_t seed[32]) {   // Lcg128Xsl64::from_seed
    if (!r || !seed) return;
    r->kind = 1;
    uint64_t w[4];
    memcpy(w, seed, 32);
    unsigned __int128 state = (unsigned __int128)w[0] | ((unsigned __int128)w[1] << 64);
    unsigned __int128 incr = ((unsigned __int128)w[2] | ((unsigned __int128)w[3] << 64)) | 1;
    const unsigned __int128 MUL = ((unsigned __int128)0x2360ED051FC65DA4ull << 64) | 0x4385DF649FCCF645ull;
    state = state + incr;
    state = state * MUL + incr;
    r->s[0] = (uint64_t)state; r->s[1] = (uint64_t)(state >> 64); r->s[2] = (uint64_t)incr; r->s[3] = (uint64_t)(incr >> 64);
}

uint32_t cvb_rng_next_u32(cvb_rng *r) {
    if (!r) return 0;
    if (r->kind == 0) {
        uint64_t *s = r->s;
        const uint64_t result = rotl64(s[0] + s[3], 23) + s[0];
        const uint64_t t = s[1] << 17;
        s[2] ^= s[0]; s[3] ^= s[1]; s[1] ^= s[2]; s[0] ^= s[3]; s[2] ^= t; s[3] = rotl64(s[3], 45);
        return (uint32_t)(result >> 32);
    }
    unsigned __int128 state = (unsigned __int128)r->s[0] | ((unsigned __int128)r->s[1] << 64);
    const unsigned __int128 incr = (unsigned __int128)r->s[2] | ((unsigned __int128)r->s[3] << 64);
    const unsigned __int128 MUL = ((unsigned __int128)0x2360ED051FC65DA4ull << 64) | 0x4385DF649FCCF645ull;
    state = state * MUL + incr;
    r->s[0] = (uint64_t)state; r->s[1] = (uint64_t)(state >> 64);
    const uint32_t rot = (uint32_t)(state >> 122);
    const uint64_t xsl = (uint64_t)(state >> 64) ^ (uint64_t)state;
    return (uint32_t)((xsl >> rot) | (xsl << ((64 - rot) & 63)));
}

int cvb_eight_point_batch(cvb_ctx *ctx, const double *a, const double *b, uint32_t n, const uint32_t *samples, uint32_t H,
                          cvb_pose *poses_out, uint8_t *nposes_out) {
    return estimate_host(ctx, 0, a, b, n, samples, H, poses_out, nposes_out);
}
int cvb_p3p_batch(cvb_ctx *ctx, const double *bearings, const double *world, uint32_t n, const uint32_t *samples, uint32_t H,
                  cvb_pose *poses_out, uint8_t *nposes_out) {
    return estimate_host(ctx, 1, bearings, world, n, samples, H, poses_out, nposes_out);
}
int cvb_five_point_batch(cvb_ctx *ctx, const double *a, const double *b, uint32_t n, const uint32_t *samples, uint32_t H,
                         int32_t eigenvector_row0, cvb_pose *poses_out, uint8_t *nposes_out) {
    if (ctx && eigenvector_row0 != 5 && eigenvector_row0 != 6) return cvb_set_error(ctx, CVB_EINVAL, "eigenvector_row0 must be 5 (reference) or 6 (corrected)");
    return estimate_host(ctx, 2, a, b, n, samples, H, poses_out, nposes_out, eigenvector_row0);
}
int cvb_residuals_camera_to_camera(cvb_ctx *ctx, const cvb_pose *poses, uint32_t m, const double *a, const double *b, uint32_t n, double *out) {
    return residuals_host(ctx, 0, poses, m, a, b, n, out);
}
int cvb_residuals_world_to_camera(cvb_ctx *ctx, const cvb_pose *poses, uint32_t m, const double *bearings, const double *world, uint32_t n,
                                  double *out) {
    return residuals_host(ctx, 1, poses, m, bearings, world, n, out);
}

// ---- include/cvb200_tri.h --------------------------------------------------------------------------------------------------
void cvb_triangulator_default(cvb_triangulator *t, int32_t method) {
    if (!t) return;
    memset(t, 0, sizeof(*t));
    t->method = method;
    switch (method) {
    case CVB_TRI_LINEAR_EIGEN: case CVB_TRI_RELATIVE_DLT: t->epsilon = 1e-12; t->max_iterations = 1000; break;
    case CVB_TRI_SINE_L1: t->epsilon = 1e-12; t->max_iterations = 1000; t->optimization_rate = 1.0; break;
    default: break;   // MeanMean, AngularL1, AngularLInfinity have no settings
    }
}

// the triangulator must be one of the six methods, and one of the TriangulatorObservations (0-2) unless `relative`
static int tri_check(cvb_ctx *ctx, const cvb_triangulator *tri, bool relative) {
    if (!tri) return cvb_set_error(ctx, CVB_EINVAL, "null triangulator");
    if (tri->method < CVB_TRI_LINEAR_EIGEN || tri->method > CVB_TRI_ANGULAR_LINF)
        return cvb_set_error(ctx, CVB_EINVAL, "unknown triangulator method %d", tri->method);
    if (!relative && tri->method > CVB_TRI_MEAN_MEAN)
        return cvb_set_error(ctx, CVB_EINVAL, "triangulator method %d is TriangulatorRelative only", tri->method);
    return 0;
}
static int offsets_check(cvb_ctx *ctx, const uint32_t *offsets, uint32_t L) {
    for (uint32_t l = 0; l < L; l++)
        if (offsets[l + 1] < offsets[l]) return cvb_set_error(ctx, CVB_EINVAL, "offsets must be non-decreasing");
    return 0;
}
// SineL1's per-observation scratch (camera centre, world-frame bearing) in the workspace buffer `b`, which the observation entry
// points do not otherwise use; null for the other methods
static int sine_l1_scratch(cvb_ctx *ctx, GeomWorkspace *g, const cvb_triangulator *tri, uint32_t nobs, double **W) {
    *W = nullptr;
    if (tri->method != CVB_TRI_SINE_L1) return 0;
    int rc = g->b.ensure(ctx, sizeof(double) * 6 * (size_t)nobs);
    if (rc) return rc;
    *W = (double *)g->b.p;
    return 0;
}

int cvb_triangulate_observations(cvb_ctx *ctx, const cvb_triangulator *tri, const cvb_pose *poses, const double *bearings,
                                 const uint32_t *offsets, uint32_t L, double *xyzw_out, uint8_t *ok_out) {
    if (!ctx) return CVB_EINVAL;
    int rc;
    if ((rc = tri_check(ctx, tri, false))) return rc;
    if (L == 0) return 0;
    if (!poses || !bearings || !offsets || !xyzw_out || !ok_out) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if ((rc = offsets_check(ctx, offsets, L))) return rc;
    const uint32_t nobs = offsets[L];
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    GeomWorkspace *g = gws(ctx);
    double *W;
    if ((rc = upload(ctx, g->poses, poses, sizeof(cvb_pose) * (size_t)nobs))) return rc;
    if ((rc = upload(ctx, g->a, bearings, sizeof(double) * 3 * (size_t)nobs))) return rc;
    if ((rc = upload(ctx, g->offsets, offsets, sizeof(uint32_t) * ((size_t)L + 1)))) return rc;
    if ((rc = g->out.ensure(ctx, sizeof(double) * 4 * (size_t)L))) return rc;
    if ((rc = g->ok.ensure(ctx, L))) return rc;
    if ((rc = sine_l1_scratch(ctx, g, tri, nobs, &W))) return rc;
    {
        CVB_PROF(ctx, "k_triangulate", 120.0 * nobs);
        k_triangulate<<<cdiv(L, 128), 128, 0, ctx->stream>>>(*tri, (const cvb_pose *)g->poses.p, (const double *)g->a.p, (const uint32_t *)g->offsets.p,
                                                             L, W, (double *)g->out.p, (uint8_t *)g->ok.p);
        CVB_LAUNCH_CHECK(ctx);
    }
    CVB_CUDA(ctx, cudaMemcpyAsync(xyzw_out, g->out.p, sizeof(double) * 4 * (size_t)L, cudaMemcpyDeviceToHost, ctx->stream));
    CVB_CUDA(ctx, cudaMemcpyAsync(ok_out, g->ok.p, L, cudaMemcpyDeviceToHost, ctx->stream));
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    return 0;
}

int cvb_triangulate_relative(cvb_ctx *ctx, const cvb_triangulator *tri, const cvb_pose *poses, uint32_t npose, const double *a,
                             const double *b, uint32_t n, double *xyzw_out, uint8_t *ok_out) {
    if (!ctx) return CVB_EINVAL;
    int rc;
    if ((rc = tri_check(ctx, tri, true))) return rc;
    if (n == 0) return 0;
    if (npose != 1 && npose != n) return cvb_set_error(ctx, CVB_EINVAL, "npose must be 1 or n (%u), not %u", n, npose);
    if (!poses || !a || !b || !xyzw_out || !ok_out) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    GeomWorkspace *g = gws(ctx);
    if ((rc = upload(ctx, g->poses, poses, sizeof(cvb_pose) * (size_t)npose))) return rc;
    if ((rc = upload(ctx, g->a, a, sizeof(double) * 3 * (size_t)n))) return rc;
    if ((rc = upload(ctx, g->b, b, sizeof(double) * 3 * (size_t)n))) return rc;
    if ((rc = g->out.ensure(ctx, sizeof(double) * 4 * (size_t)n))) return rc;
    if ((rc = g->ok.ensure(ctx, n))) return rc;
    {
        CVB_PROF(ctx, "k_triangulate_relative", 56.0 * n + sizeof(cvb_pose) * (double)npose);
        k_triangulate_relative<<<cdiv(n, 128), 128, 0, ctx->stream>>>(*tri, (const cvb_pose *)g->poses.p, npose, (const double *)g->a.p,
                                                                      (const double *)g->b.p, n, (double *)g->out.p, (uint8_t *)g->ok.p);
        CVB_LAUNCH_CHECK(ctx);
    }
    CVB_CUDA(ctx, cudaMemcpyAsync(xyzw_out, g->out.p, sizeof(double) * 4 * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
    CVB_CUDA(ctx, cudaMemcpyAsync(ok_out, g->ok.p, n, cudaMemcpyDeviceToHost, ctx->stream));
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    return 0;
}

// LinearEigenTriangulator::default() through the observations entry point (one kernel for every observations triangulator)
int cvb_triangulate_linear_eigen(cvb_ctx *ctx, const cvb_pose *poses, const double *bearings, const uint32_t *offsets, uint32_t L,
                                 double *xyzw_out, uint8_t *ok_out) {
    cvb_triangulator t;
    cvb_triangulator_default(&t, CVB_TRI_LINEAR_EIGEN);
    return cvb_triangulate_observations(ctx, &t, poses, bearings, offsets, L, xyzw_out, ok_out);
}

int cvb_arrsac_eight_point(cvb_ctx *ctx, const cvb_arrsac_cfg *cfg, const double *a, const double *b, uint32_t n, cvb_rng *rng,
                           cvb_pose *model_out, uint32_t *inliers_out, uint32_t cap, uint32_t *n_inliers, int32_t *found) {
    if (!ctx) return CVB_EINVAL;
    if (!cfg || !rng || !model_out || !found || (n && (!a || !b))) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (arrsac_on_host()) return arrsac_run(ctx, cfg, 0, a, b, n, rng, model_out, inliers_out, cap, n_inliers, found);
    return arrsac_host(ctx, cfg, 0, a, b, n, rng, model_out, inliers_out, cap, n_inliers, found);
}
int cvb_arrsac_five_point(cvb_ctx *ctx, const cvb_arrsac_cfg *cfg, const double *a, const double *b, uint32_t n, cvb_rng *rng,
                          int32_t eigenvector_row0, cvb_pose *model_out, uint32_t *inliers_out, uint32_t cap, uint32_t *n_inliers,
                          int32_t *found) {
    if (!ctx) return CVB_EINVAL;
    if (!cfg || !rng || !model_out || !found || (n && (!a || !b))) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (eigenvector_row0 != 5 && eigenvector_row0 != 6) return cvb_set_error(ctx, CVB_EINVAL, "eigenvector_row0 must be 5 (reference) or 6 (corrected)");
    if (arrsac_on_host()) return arrsac_run(ctx, cfg, 2, a, b, n, rng, model_out, inliers_out, cap, n_inliers, found, eigenvector_row0);
    return arrsac_host(ctx, cfg, 2, a, b, n, rng, model_out, inliers_out, cap, n_inliers, found, eigenvector_row0);
}
int cvb_arrsac_p3p(cvb_ctx *ctx, const cvb_arrsac_cfg *cfg, const double *bearings, const double *world, uint32_t n, cvb_rng *rng,
                   cvb_pose *model_out, uint32_t *inliers_out, uint32_t cap, uint32_t *n_inliers, int32_t *found) {
    if (!ctx) return CVB_EINVAL;
    if (!cfg || !rng || !model_out || !found || (n && (!bearings || !world))) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (arrsac_on_host()) return arrsac_run(ctx, cfg, 1, bearings, world, n, rng, model_out, inliers_out, cap, n_inliers, found);
    return arrsac_host(ctx, cfg, 1, bearings, world, n, rng, model_out, inliers_out, cap, n_inliers, found);
}

// ---- device-resident entry points (asynchronous on the context stream) -----------------------------------------------------
int cvb_pair_bearings_dev(cvb_ctx *ctx, const cvb_keypoint *kp_a_dev, const cvb_keypoint *kp_b_dev, const uint32_t *pairs_dev,
                          const uint32_t *n_pairs_dev, uint32_t cap, const cvb_intrinsics *intrinsics, double *a_out_dev, double *b_out_dev) {
    const cvb_intrinsics_k1 K = intrinsics ? intrinsics_k1(*intrinsics) : cvb_intrinsics_k1{};
    return cvb_pair_bearings_k1_dev(ctx, kp_a_dev, kp_b_dev, pairs_dev, n_pairs_dev, cap, intrinsics ? &K : nullptr, a_out_dev, b_out_dev);
}
int cvb_pair_bearings_k1_dev(cvb_ctx *ctx, const cvb_keypoint *kp_a_dev, const cvb_keypoint *kp_b_dev, const uint32_t *pairs_dev,
                             const uint32_t *n_pairs_dev, uint32_t cap, const cvb_intrinsics_k1 *intrinsics, double *a_out_dev,
                             double *b_out_dev) {
    if (!ctx) return CVB_EINVAL;
    if (!kp_a_dev || !kp_b_dev || !pairs_dev || !n_pairs_dev || !intrinsics || !a_out_dev || !b_out_dev) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (cap == 0) return 0;
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    CVB_PROF(ctx, "k_pair_bearings", 0);
    k_pair_bearings<<<cdiv(cap, 256), 256, 0, ctx->stream>>>(kp_a_dev, kp_b_dev, pairs_dev, n_pairs_dev, cap, *intrinsics, a_out_dev, b_out_dev);
    CVB_LAUNCH_CHECK(ctx);
    return 0;
}

static int arrsac_dev_entry(cvb_ctx *ctx, const cvb_arrsac_cfg *cfg, int kind, const double *a_dev, const double *b_dev, const uint32_t *n_dev,
                            uint32_t n_max, const cvb_rng *rng, cvb_pose *model_out_dev, uint32_t *inliers_out_dev, uint32_t cap,
                            uint32_t *n_inliers_dev, int32_t *found_dev) {
    if (!ctx) return CVB_EINVAL;
    if (!cfg || !rng || !a_dev || !b_dev || !n_dev || !model_out_dev || !n_inliers_dev || !found_dev) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    return arrsac_run_dev(ctx, cfg, kind, a_dev, b_dev, n_dev, 0, n_max, rng, model_out_dev, inliers_out_dev, cap, n_inliers_dev, found_dev, 5);
}
int cvb_arrsac_eight_point_dev(cvb_ctx *ctx, const cvb_arrsac_cfg *cfg, const double *a_dev, const double *b_dev, const uint32_t *n_dev,
                               uint32_t n_max, const cvb_rng *rng, cvb_pose *model_out_dev, uint32_t *inliers_out_dev, uint32_t cap,
                               uint32_t *n_inliers_dev, int32_t *found_dev) {
    return arrsac_dev_entry(ctx, cfg, 0, a_dev, b_dev, n_dev, n_max, rng, model_out_dev, inliers_out_dev, cap, n_inliers_dev, found_dev);
}
int cvb_arrsac_p3p_dev(cvb_ctx *ctx, const cvb_arrsac_cfg *cfg, const double *bearings_dev, const double *world_dev, const uint32_t *n_dev,
                       uint32_t n_max, const cvb_rng *rng, cvb_pose *model_out_dev, uint32_t *inliers_out_dev, uint32_t cap,
                       uint32_t *n_inliers_dev, int32_t *found_dev) {
    return arrsac_dev_entry(ctx, cfg, 1, bearings_dev, world_dev, n_dev, n_max, rng, model_out_dev, inliers_out_dev, cap, n_inliers_dev, found_dev);
}
int cvb_arrsac_commit_rng(cvb_ctx *ctx, cvb_rng *rng, uint32_t *stats_out) {
    if (!ctx) return CVB_EINVAL;
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    ArrsacCtl h;
    int rc = arrsac_commit_rng(ctx, rng, &h);
    if (rc) return rc;
    if (stats_out) arrsac_stats_words(h, stats_out);
    return 0;
}

int cvb_single_view_optimize_l2(cvb_ctx *ctx, const cvb_pose *poses, uint32_t B, double optimization_rate, uint32_t iterations,
                                const double *bearings, const double *world, const uint32_t *offsets, cvb_pose *poses_out,
                                uint32_t *updates_out) {
    if (!ctx) return CVB_EINVAL;
    if (B == 0) return 0;
    if (!poses || !offsets || !poses_out) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    for (uint32_t b = 0; b < B; b++)
        if (offsets[b + 1] < offsets[b]) return cvb_set_error(ctx, CVB_EINVAL, "offsets must be non-decreasing");
    const uint32_t n = offsets[B];
    if (n && (!bearings || !world)) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    GeomWorkspace *g = gws(ctx);
    int rc;
    if ((rc = upload(ctx, g->poses, poses, sizeof(cvb_pose) * (size_t)B))) return rc;
    if ((rc = upload(ctx, g->a, bearings, sizeof(double) * 3 * (size_t)n))) return rc;
    if ((rc = upload(ctx, g->b, world, sizeof(double) * 4 * (size_t)n))) return rc;
    if ((rc = upload(ctx, g->offsets, offsets, sizeof(uint32_t) * ((size_t)B + 1)))) return rc;
    if ((rc = g->out.ensure(ctx, sizeof(cvb_pose) * (size_t)B))) return rc;
    if ((rc = g->ok.ensure(ctx, sizeof(uint32_t) * (size_t)B))) return rc;
    {
        CVB_PROF(ctx, "k_single_view_opt", 0.0);
        k_single_view_opt<<<B, OPT_NT, 0, ctx->stream>>>((const cvb_pose *)g->poses.p, (const double *)g->a.p, (const double *)g->b.p,
                                                         (const uint32_t *)g->offsets.p, optimization_rate, iterations, (cvb_pose *)g->out.p,
                                                         (uint32_t *)g->ok.p);
        CVB_LAUNCH_CHECK(ctx);
    }
    return download_poses_updates(ctx, g, poses_out, (size_t)B, updates_out, B);
}

int cvb_three_view_optimize_l2(cvb_ctx *ctx, const cvb_pose *poses, uint32_t B, int32_t adaptive, double optimization_rate,
                               uint32_t iterations, const double *observations, const uint32_t *offsets, cvb_pose *poses_out,
                               uint32_t *updates_out) {
    if (!ctx) return CVB_EINVAL;
    if (B == 0) return 0;
    if (!poses || !offsets || !poses_out) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    for (uint32_t b = 0; b < B; b++)
        if (offsets[b + 1] < offsets[b]) return cvb_set_error(ctx, CVB_EINVAL, "offsets must be non-decreasing");
    const uint32_t n = offsets[B];
    if (n && !observations) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    GeomWorkspace *g = gws(ctx);
    int rc;
    if ((rc = upload(ctx, g->poses, poses, sizeof(cvb_pose) * 2 * (size_t)B))) return rc;
    if ((rc = upload(ctx, g->a, observations, sizeof(double) * 9 * (size_t)n))) return rc;
    if ((rc = upload(ctx, g->offsets, offsets, sizeof(uint32_t) * ((size_t)B + 1)))) return rc;
    if ((rc = g->out.ensure(ctx, sizeof(cvb_pose) * 2 * (size_t)B))) return rc;
    if ((rc = g->ok.ensure(ctx, sizeof(uint32_t) * (size_t)B))) return rc;
    {
        CVB_PROF(ctx, "k_three_view_opt", 0.0);
        k_three_view_opt<<<B, OPT_NT, 0, ctx->stream>>>((const cvb_pose *)g->poses.p, (const double *)g->a.p, (const uint32_t *)g->offsets.p,
                                                        adaptive ? 1 : 0, optimization_rate, iterations, (cvb_pose *)g->out.p, (uint32_t *)g->ok.p);
        CVB_LAUNCH_CHECK(ctx);
    }
    return download_poses_updates(ctx, g, poses_out, 2 * (size_t)B, updates_out, B);
}

}  // extern "C"

// The entry points of include/cvb200_opt.h are exported by libcvb200_opt.so (cv_b200/csrc/opt.cu), a module over this library, so
// that libcvb200.so keeps exporting exactly the C ABI of cvb200.h, cvb200_sfm.h and cvb200_tri.h.  These are their implementations,
// with C++ linkage like the other functions shared between this library's translation units.
int opt_single_view_l1(cvb_ctx *ctx, const cvb_pose *poses, uint32_t B, double epsilon, double optimization_rate, uint32_t iterations,
                        const double *bearings, const double *world, const uint32_t *offsets,
                                cvb_pose *poses_out, uint32_t *updates_out) {
    if (!ctx) return CVB_EINVAL;
    if (B == 0) return 0;
    if (!poses || !offsets || !poses_out) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    int rc;
    if ((rc = offsets_check(ctx, offsets, B))) return rc;
    const uint32_t n = offsets[B];
    if (n && (!bearings || !world)) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    GeomWorkspace *g = gws(ctx);
    if ((rc = upload(ctx, g->poses, poses, sizeof(cvb_pose) * (size_t)B))) return rc;
    if ((rc = upload(ctx, g->a, bearings, sizeof(double) * 3 * (size_t)n))) return rc;
    if ((rc = upload(ctx, g->b, world, sizeof(double) * 4 * (size_t)n))) return rc;
    if ((rc = upload(ctx, g->offsets, offsets, sizeof(uint32_t) * ((size_t)B + 1)))) return rc;
    if ((rc = g->out.ensure(ctx, sizeof(cvb_pose) * (size_t)B))) return rc;
    if ((rc = g->ok.ensure(ctx, sizeof(uint32_t) * (size_t)B))) return rc;
    {
        CVB_PROF(ctx, "k_single_view_opt_l1", 0.0);
        k_single_view_opt_l1<<<B, OPT_NT, 0, ctx->stream>>>((const cvb_pose *)g->poses.p, (const double *)g->a.p, (const double *)g->b.p,
                                                            (const uint32_t *)g->offsets.p, epsilon, optimization_rate, iterations,
                                                            (cvb_pose *)g->out.p, (uint32_t *)g->ok.p);
        CVB_LAUNCH_CHECK(ctx);
    }
    return download_poses_updates(ctx, g, poses_out, (size_t)B, updates_out, B);
}

int opt_three_view_l1(cvb_ctx *ctx, const cvb_pose *poses, uint32_t B, double epsilon, double optimization_rate, uint32_t iterations,
                       const double *observations, const uint32_t *offsets, cvb_pose *poses_out,
                               uint32_t *updates_out) {
    if (!ctx) return CVB_EINVAL;
    if (B == 0) return 0;
    if (!poses || !offsets || !poses_out) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    int rc;
    if ((rc = offsets_check(ctx, offsets, B))) return rc;
    const uint32_t n = offsets[B];
    if (n && !observations) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    GeomWorkspace *g = gws(ctx);
    if ((rc = upload(ctx, g->poses, poses, sizeof(cvb_pose) * 2 * (size_t)B))) return rc;
    if ((rc = upload(ctx, g->a, observations, sizeof(double) * 9 * (size_t)n))) return rc;
    if ((rc = upload(ctx, g->offsets, offsets, sizeof(uint32_t) * ((size_t)B + 1)))) return rc;
    if ((rc = g->out.ensure(ctx, sizeof(cvb_pose) * 2 * (size_t)B))) return rc;
    if ((rc = g->ok.ensure(ctx, sizeof(uint32_t) * (size_t)B))) return rc;
    {
        CVB_PROF(ctx, "k_three_view_opt_l1", 0.0);
        k_three_view_opt_l1<<<B, OPT_NT, 0, ctx->stream>>>((const cvb_pose *)g->poses.p, (const double *)g->a.p, (const uint32_t *)g->offsets.p,
                                                           epsilon, optimization_rate, iterations, (cvb_pose *)g->out.p, (uint32_t *)g->ok.p);
        CVB_LAUNCH_CHECK(ctx);
    }
    return download_poses_updates(ctx, g, poses_out, 2 * (size_t)B, updates_out, B);
}

// The entry points of include/cvb200_pinhole.h, exported by libcvb200_pinhole.so (cv_b200/csrc/pinhole_abi.cu) for the same reason.
// max_iterations (usize upstream) as the Jacobi sweep bound, as tri_sweeps does for the triangulators
static int pinhole_sweeps(uint32_t max_iterations) { return max_iterations > 0x7fffffffu ? 0x7fffffff : (int)max_iterations; }

int pin_pose_reprojection_error(cvb_ctx *ctx, const cvb_triangulator *tri, const cvb_pose *poses, uint32_t npose, const double *a,
                                const double *b, uint32_t n, double *err_out, double *avg_out, uint8_t *ok_out) {
    if (!ctx) return CVB_EINVAL;
    int rc;
    if ((rc = tri_check(ctx, tri, true))) return rc;
    if (n == 0) return 0;
    if (npose != 1 && npose != n) return cvb_set_error(ctx, CVB_EINVAL, "npose must be 1 or n (%u), not %u", n, npose);
    if (!poses || !a || !b || !err_out || !ok_out) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    GeomWorkspace *g = gws(ctx);
    if ((rc = upload(ctx, g->poses, poses, sizeof(cvb_pose) * (size_t)npose))) return rc;
    if ((rc = upload(ctx, g->a, a, sizeof(double) * 3 * (size_t)n))) return rc;
    if ((rc = upload(ctx, g->b, b, sizeof(double) * 3 * (size_t)n))) return rc;
    if ((rc = g->out.ensure(ctx, sizeof(double) * 5 * (size_t)n))) return rc;   // err (n x 4) | avg (n)
    if ((rc = g->ok.ensure(ctx, n))) return rc;
    double *err = (double *)g->out.p, *avg = err + 4 * (size_t)n;
    {
        CVB_PROF(ctx, "k_pose_reprojection_error", 89.0 * n + sizeof(cvb_pose) * (double)npose);
        k_pose_reprojection_error<<<cdiv(n, 128), 128, 0, ctx->stream>>>(*tri, (const cvb_pose *)g->poses.p, npose, (const double *)g->a.p,
                                                                         (const double *)g->b.p, nullptr, n, nullptr, err, avg, (uint8_t *)g->ok.p);
        CVB_LAUNCH_CHECK(ctx);
    }
    CVB_CUDA(ctx, cudaMemcpyAsync(err_out, err, sizeof(double) * 4 * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
    if (avg_out) CVB_CUDA(ctx, cudaMemcpyAsync(avg_out, avg, sizeof(double) * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
    CVB_CUDA(ctx, cudaMemcpyAsync(ok_out, g->ok.p, n, cudaMemcpyDeviceToHost, ctx->stream));
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    return 0;
}

int pin_pose_reprojection_error_dev(cvb_ctx *ctx, const cvb_triangulator *tri, const cvb_pose *poses_dev, uint32_t npose,
                                    const double *a_dev, const double *b_dev, const uint32_t *n_dev, uint32_t n_max,
                                    const int32_t *found_dev, double *err_out_dev, double *avg_out_dev, uint8_t *ok_out_dev) {
    if (!ctx) return CVB_EINVAL;
    int rc;
    if ((rc = tri_check(ctx, tri, true))) return rc;
    if (npose != 1 && npose != n_max) return cvb_set_error(ctx, CVB_EINVAL, "npose must be 1 or n_max (%u), not %u", n_max, npose);
    if (!poses_dev || !a_dev || !b_dev || !n_dev || !err_out_dev || !ok_out_dev) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (n_max == 0) return 0;
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    CVB_PROF(ctx, "k_pose_reprojection_error", 0);
    k_pose_reprojection_error<<<cdiv(n_max, 128), 128, 0, ctx->stream>>>(*tri, poses_dev, npose, a_dev, b_dev, n_dev, n_max, found_dev,
                                                                         err_out_dev, avg_out_dev, ok_out_dev);
    CVB_LAUNCH_CHECK(ctx);
    return 0;
}

int pin_eight_point_essential_batch(cvb_ctx *ctx, double epsilon, uint32_t iterations, const double *a, const double *b, uint32_t n,
                                    const uint32_t *samples, uint32_t H, double *E_out, uint8_t *ok_out) {
    if (!ctx) return CVB_EINVAL;
    if (H == 0) return 0;
    if (!a || !b || !samples || !E_out || !ok_out) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    for (size_t i = 0; i < (size_t)H * 8; i++)
        if (samples[i] >= n) return cvb_set_error(ctx, CVB_EINVAL, "sample index %u out of range (n = %u)", samples[i], n);
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    GeomWorkspace *g = gws(ctx);
    int rc;
    if ((rc = upload_data(ctx, 0, a, b, n))) return rc;
    if ((rc = upload(ctx, g->samples, samples, sizeof(uint32_t) * 8 * (size_t)H))) return rc;
    if ((rc = g->out.ensure(ctx, sizeof(double) * 9 * (size_t)H))) return rc;
    if ((rc = g->ok.ensure(ctx, H))) return rc;
    {
        CVB_PROF(ctx, "k_eight_point_essential", 0);
        k_eight_point_essential<<<cdiv(H, 128), 128, 0, ctx->stream>>>((const double *)g->a.p, (const double *)g->b.p, (const uint32_t *)g->samples.p,
                                                                       H, epsilon, pinhole_sweeps(iterations), (double *)g->out.p, (uint8_t *)g->ok.p);
        CVB_LAUNCH_CHECK(ctx);
    }
    CVB_CUDA(ctx, cudaMemcpyAsync(E_out, g->out.p, sizeof(double) * 9 * (size_t)H, cudaMemcpyDeviceToHost, ctx->stream));
    CVB_CUDA(ctx, cudaMemcpyAsync(ok_out, g->ok.p, H, cudaMemcpyDeviceToHost, ctx->stream));
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    return 0;
}

int pin_residuals_essential(cvb_ctx *ctx, const double *E, uint32_t m, const double *a, const double *b, uint32_t n, double *out) {
    if (!ctx) return CVB_EINVAL;
    if (m == 0 || n == 0) return 0;
    if (!E || !a || !b || !out) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    GeomWorkspace *g = gws(ctx);
    int rc;
    if ((rc = upload_data(ctx, 0, a, b, n))) return rc;
    if ((rc = upload(ctx, g->poses, E, sizeof(double) * 9 * (size_t)m))) return rc;
    if ((rc = g->out.ensure(ctx, sizeof(double) * (size_t)m * n))) return rc;
    for (uint32_t p0 = 0; p0 < m; p0 += 65535) {   // gridDim.y limit
        const uint32_t pm = std::min<uint32_t>(65535, m - p0);
        CVB_PROF(ctx, "k_residuals_essential", 56.0 * pm * n);
        k_residuals_essential<<<dim3(cdiv(n, 256), pm), 256, 0, ctx->stream>>>((const double *)g->poses.p + (size_t)p0 * 9, (const double *)g->a.p,
                                                                               (const double *)g->b.p, n, (double *)g->out.p + (size_t)p0 * n);
        CVB_LAUNCH_CHECK(ctx);
    }
    CVB_CUDA(ctx, cudaMemcpyAsync(out, g->out.p, sizeof(double) * (size_t)m * n, cudaMemcpyDeviceToHost, ctx->stream));
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    return 0;
}

int pin_essential_recondition(cvb_ctx *ctx, const double *E, uint32_t m, double epsilon, uint32_t max_iterations, double *E_out,
                              uint8_t *ok_out) {
    if (!ctx) return CVB_EINVAL;
    if (m == 0) return 0;
    if (!E || !E_out || !ok_out) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    GeomWorkspace *g = gws(ctx);
    int rc;
    if ((rc = upload(ctx, g->poses, E, sizeof(double) * 9 * (size_t)m))) return rc;
    if ((rc = g->out.ensure(ctx, sizeof(double) * 9 * (size_t)m))) return rc;
    if ((rc = g->ok.ensure(ctx, m))) return rc;
    {
        CVB_PROF(ctx, "k_essential_recondition", 144.0 * m);
        k_essential_recondition<<<cdiv(m, 128), 128, 0, ctx->stream>>>((const double *)g->poses.p, m, epsilon, pinhole_sweeps(max_iterations),
                                                                       (double *)g->out.p, (uint8_t *)g->ok.p);
        CVB_LAUNCH_CHECK(ctx);
    }
    CVB_CUDA(ctx, cudaMemcpyAsync(E_out, g->out.p, sizeof(double) * 9 * (size_t)m, cudaMemcpyDeviceToHost, ctx->stream));
    CVB_CUDA(ctx, cudaMemcpyAsync(ok_out, g->ok.p, m, cudaMemcpyDeviceToHost, ctx->stream));
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    return 0;
}

int pin_essential_decompose(cvb_ctx *ctx, const double *E, uint32_t m, double epsilon, uint32_t max_iterations, double *rot_a_out,
                            double *rot_b_out, double *t_out, uint8_t *ok_out) {
    if (!ctx) return CVB_EINVAL;
    if (m == 0) return 0;
    if (!E || !rot_a_out || !rot_b_out || !t_out || !ok_out) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    GeomWorkspace *g = gws(ctx);
    int rc;
    if ((rc = upload(ctx, g->poses, E, sizeof(double) * 9 * (size_t)m))) return rc;
    if ((rc = g->out.ensure(ctx, sizeof(double) * 21 * (size_t)m))) return rc;   // rot_a (m x 9) | rot_b (m x 9) | t (m x 3)
    if ((rc = g->ok.ensure(ctx, m))) return rc;
    double *ra = (double *)g->out.p, *rb = ra + 9 * (size_t)m, *t = rb + 9 * (size_t)m;
    {
        CVB_PROF(ctx, "k_essential_decompose", 240.0 * m);
        k_essential_decompose<<<cdiv(m, 128), 128, 0, ctx->stream>>>((const double *)g->poses.p, m, epsilon, pinhole_sweeps(max_iterations),
                                                                     ra, rb, t, (uint8_t *)g->ok.p);
        CVB_LAUNCH_CHECK(ctx);
    }
    CVB_CUDA(ctx, cudaMemcpyAsync(rot_a_out, ra, sizeof(double) * 9 * (size_t)m, cudaMemcpyDeviceToHost, ctx->stream));
    CVB_CUDA(ctx, cudaMemcpyAsync(rot_b_out, rb, sizeof(double) * 9 * (size_t)m, cudaMemcpyDeviceToHost, ctx->stream));
    CVB_CUDA(ctx, cudaMemcpyAsync(t_out, t, sizeof(double) * 3 * (size_t)m, cudaMemcpyDeviceToHost, ctx->stream));
    CVB_CUDA(ctx, cudaMemcpyAsync(ok_out, g->ok.p, m, cudaMemcpyDeviceToHost, ctx->stream));
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    return 0;
}

extern "C" {

int cvb_observation_losses_tri(cvb_ctx *ctx, const cvb_triangulator *tri, const cvb_pose *poses, const double *bearings,
                               const uint32_t *offsets, uint32_t L, double *loss_out) {
    if (!ctx) return CVB_EINVAL;
    int rc;
    if ((rc = tri_check(ctx, tri, false))) return rc;
    if (L == 0) return 0;
    if (!poses || !bearings || !offsets || !loss_out) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if ((rc = offsets_check(ctx, offsets, L))) return rc;
    const uint32_t nobs = offsets[L];
    if (nobs == 0) return 0;
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    GeomWorkspace *g = gws(ctx);
    double *W;
    if ((rc = upload(ctx, g->poses, poses, sizeof(cvb_pose) * (size_t)nobs))) return rc;
    if ((rc = upload(ctx, g->a, bearings, sizeof(double) * 3 * (size_t)nobs))) return rc;
    if ((rc = upload(ctx, g->offsets, offsets, sizeof(uint32_t) * ((size_t)L + 1)))) return rc;
    if ((rc = g->out.ensure(ctx, sizeof(double) * (size_t)nobs))) return rc;
    if ((rc = sine_l1_scratch(ctx, g, tri, nobs, &W))) return rc;
    {
        CVB_PROF(ctx, "k_observation_losses", 128.0 * nobs);
        k_observation_losses<<<cdiv(L, 128), 128, 0, ctx->stream>>>(*tri, (const cvb_pose *)g->poses.p, (const double *)g->a.p,
                                                                    (const uint32_t *)g->offsets.p, L, W, (double *)g->out.p);
        CVB_LAUNCH_CHECK(ctx);
    }
    CVB_CUDA(ctx, cudaMemcpyAsync(loss_out, g->out.p, sizeof(double) * (size_t)nobs, cudaMemcpyDeviceToHost, ctx->stream));
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    return 0;
}
int cvb_observation_losses(cvb_ctx *ctx, const cvb_pose *poses, const double *bearings, const uint32_t *offsets, uint32_t L,
                           double *loss_out) {
    cvb_triangulator t;
    cvb_triangulator_default(&t, CVB_TRI_LINEAR_EIGEN);
    return cvb_observation_losses_tri(ctx, &t, poses, bearings, offsets, L, loss_out);
}

int cvb_tri_landmarks_robust_tri(cvb_ctx *ctx, const cvb_triangulator *tri, const cvb_pose *first_pose, const cvb_pose *second_pose,
                                 const double *observations, uint32_t n, double maximum_cosine_distance,
                                 double incidence_minimum_cosine_distance, uint8_t *robust_out) {
    if (!ctx) return CVB_EINVAL;
    int rc;
    if ((rc = tri_check(ctx, tri, false))) return rc;
    if (n == 0) return 0;
    if (!first_pose || !second_pose || !observations || !robust_out) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    GeomWorkspace *g = gws(ctx);
    if ((rc = upload(ctx, g->a, observations, sizeof(double) * 9 * (size_t)n))) return rc;
    if ((rc = g->ok.ensure(ctx, n))) return rc;
    {
        CVB_PROF(ctx, "k_tri_landmark_robust", 72.0 * n);
        k_tri_landmark_robust<<<cdiv(n, 128), 128, 0, ctx->stream>>>(*tri, *first_pose, *second_pose, (const double *)g->a.p, n,
                                                                     maximum_cosine_distance, incidence_minimum_cosine_distance, (uint8_t *)g->ok.p);
        CVB_LAUNCH_CHECK(ctx);
    }
    CVB_CUDA(ctx, cudaMemcpyAsync(robust_out, g->ok.p, n, cudaMemcpyDeviceToHost, ctx->stream));
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    return 0;
}
int cvb_tri_landmarks_robust(cvb_ctx *ctx, const cvb_pose *first_pose, const cvb_pose *second_pose, const double *observations, uint32_t n,
                             double maximum_cosine_distance, double incidence_minimum_cosine_distance, uint8_t *robust_out) {
    cvb_triangulator t;
    cvb_triangulator_default(&t, CVB_TRI_LINEAR_EIGEN);
    return cvb_tri_landmarks_robust_tri(ctx, &t, first_pose, second_pose, observations, n, maximum_cosine_distance,
                                        incidence_minimum_cosine_distance, robust_out);
}

}  // extern "C"
