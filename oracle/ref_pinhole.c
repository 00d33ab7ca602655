/* oracle/ref_pinhole.c -- TEST INFRASTRUCTURE: CPU restatement of cv-pinhole's reprojection error and the EssentialMatrix model that
 * include/cvb200_pinhole.h runs on the device.  Not product code.
 *
 * Follows (paths relative to the reference checkout):
 *   cv-pinhole/src/lib.rs:314-372        pose_reprojection_error, average_pose_reprojection_error
 *   cv-core/src/point.rs:20-25, 46-49    Projective::from_homogeneous, Projective::bearing (the xyz of the homogeneous vector)
 *   cv-core/src/pose.rs:125-133          Pose::transform = from_homogeneous(isometry.to_homogeneous() * point)
 *   cv-pinhole/src/essential.rs:64-77    EssentialMatrix::recondition (nalgebra's SVD::recompose: U's columns scaled, then times Vt)
 * The triangulators are ref_triangulate_relative (ref_triangulation.c); from_matches, the decomposition and the residual are
 * ref_eight_point_essential, ref_essential_poses and ref_essential_residual (ref_geom.c), with the 3x3 SVD ref_svd3.
 * All arithmetic is f64 with -ffp-contract=off (oracle/pinhole.mk). */
#include <math.h>
#include <stdint.h>
#include <string.h>
#include "ref_pinhole.h"

/* Projective::from_homogeneous (cv-core/src/point.rs:20-25) */
static void from_homogeneous(double *p) {
    if (signbit(p[3])) { p[0] = -p[0]; p[1] = -p[1]; p[2] = -p[2]; p[3] = -p[3]; }
    const double n = sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]);
    p[0] /= n; p[1] /= n; p[2] /= n; p[3] /= n;
}

/* lib.rs:314-341: a_norm / b_norm from the input bearings; reproject only when the bearing's z is sign-positive (a sign-bit test:
 * +0.0 and +NaN pass) */
int ref_pose_reprojection_error(const ref_triangulator *t, const ref_pose *P, const double *a, const double *b, double err[4], double *avg) {
    const double an[2] = {a[0] / a[2], a[1] / a[2]}, bn[2] = {b[0] / b[2], b[1] / b[2]};
    double p[4], q[4];
    if (!ref_triangulate_relative(t, P, a, b, p)) return 0;
    if (signbit(p[2])) return 0;
    for (int r = 0; r < 3; r++) q[r] = P->R[3 * r] * p[0] + P->R[3 * r + 1] * p[1] + P->R[3 * r + 2] * p[2] + P->t[r] * p[3];
    q[3] = p[3];
    from_homogeneous(q);
    if (signbit(q[2])) return 0;
    err[0] = an[0] - p[0] / p[2]; err[1] = an[1] - p[1] / p[2];
    err[2] = bn[0] - q[0] / q[2]; err[3] = bn[1] - q[1] / q[2];
    /* lib.rs:370-371: errors.iter().map(|v| v.norm()).sum::<f64>() * 0.5 */
    *avg = ((0.0 + sqrt(err[0] * err[0] + err[1] * err[1])) + sqrt(err[2] * err[2] + err[3] * err[3])) * 0.5;
    return 1;
}

/* essential.rs:64-77 */
int ref_essential_recondition(const double *E, double eps, int iters, double *out) {
    double U[9], s[3], Vt[9];
    if (!ref_svd3(E, eps, iters, U, s, Vt)) return 0;
    const double m = (s[0] + s[1]) / 2.0, d[3] = {m, m, 0.0};
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) U[r * 3 + c] *= d[c];
    double R[9];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) R[i * 3 + j] = U[i * 3] * Vt[j] + U[i * 3 + 1] * Vt[3 + j] + U[i * 3 + 2] * Vt[6 + j];
    memcpy(out, R, sizeof(R));
    return 1;
}

static void fill_nan(double *p, int k) { for (int i = 0; i < k; i++) p[i] = NAN; }

void ref_pose_reprojection_error_batch(const ref_triangulator *t, const ref_pose *poses, uint32_t npose, const double *a, const double *b,
                                       uint32_t n, double *err, double *avg, uint8_t *ok) {
    #pragma omp parallel for schedule(static)
    for (uint32_t i = 0; i < n; i++) {
        double m;
        ok[i] = (uint8_t)ref_pose_reprojection_error(t, poses + (npose == 1 ? 0 : i), a + 3 * (size_t)i, b + 3 * (size_t)i, err + 4 * (size_t)i, &m);
        if (!ok[i]) { fill_nan(err + 4 * (size_t)i, 4); m = NAN; }
        if (avg) avg[i] = m;
    }
}

void ref_eight_point_essential_batch(const double *a, const double *b, const uint32_t *samples, uint32_t H, double eps, int iters,
                                     double *E, uint8_t *ok) {
    #pragma omp parallel for schedule(static)
    for (uint32_t h = 0; h < H; h++) {
        double sa[24], sb[24];
        for (int i = 0; i < 8; i++) { memcpy(sa + 3 * i, a + 3 * (size_t)samples[8 * (size_t)h + i], 24); memcpy(sb + 3 * i, b + 3 * (size_t)samples[8 * (size_t)h + i], 24); }
        ok[h] = (uint8_t)ref_eight_point_essential(sa, sb, eps, iters, E + 9 * (size_t)h);
        if (!ok[h]) fill_nan(E + 9 * (size_t)h, 9);
    }
}

void ref_residuals_essential(const double *E, uint32_t m, const double *a, const double *b, uint32_t n, double *out) {
    #pragma omp parallel for schedule(static)
    for (uint32_t p = 0; p < m; p++)
        for (uint32_t i = 0; i < n; i++) out[(size_t)p * n + i] = ref_essential_residual(E + 9 * (size_t)p, a + 3 * (size_t)i, b + 3 * (size_t)i);
}

void ref_essential_recondition_batch(const double *E, uint32_t m, double eps, int iters, double *out, uint8_t *ok) {
    #pragma omp parallel for schedule(static)
    for (uint32_t j = 0; j < m; j++) {
        ok[j] = (uint8_t)ref_essential_recondition(E + 9 * (size_t)j, eps, iters, out + 9 * (size_t)j);
        if (!ok[j]) fill_nan(out + 9 * (size_t)j, 9);
    }
}

/* possible_rotations_unscaled_translation = poses 0 and 1 of ref_essential_poses: (Ra, t), (Rb, t) */
void ref_essential_decompose_batch(const double *E, uint32_t m, double eps, int iters, double *rot_a, double *rot_b, double *t, uint8_t *ok) {
    #pragma omp parallel for schedule(static)
    for (uint32_t j = 0; j < m; j++) {
        ref_pose P[4];
        ok[j] = ref_essential_poses(E + 9 * (size_t)j, eps, iters, P) == 4;
        if (ok[j]) { memcpy(rot_a + 9 * (size_t)j, P[0].R, 72); memcpy(rot_b + 9 * (size_t)j, P[1].R, 72); memcpy(t + 3 * (size_t)j, P[0].t, 24); }
        else { fill_nan(rot_a + 9 * (size_t)j, 9); fill_nan(rot_b + 9 * (size_t)j, 9); fill_nan(t + 3 * (size_t)j, 3); }
    }
}
