/* oracle/ref_triangulation.c -- TEST INFRASTRUCTURE (CPU oracle), not product code.
 *
 * Plain-C restatement of the triangulators of cv-geom/src/triangulation.rs (include/cvb200_tri.h):
 *   :39-130   LinearEigenTriangulator with its epsilon / max_iterations (ref_geom.c's ref_triangulate_linear_eigen is the same
 *             code with the Default constants; tests/test_oracle_triangulation.py checks the two agree bit for bit)
 *   :163-276  SineL1Triangulator, with epipolar::point_gradient (cv-geom/src/epipolar.rs:174-179)
 *   :279-363  RelativeDltTriangulator
 *   :389-442  MeanMeanTriangulator
 *   :469-530  AngularL1Triangulator
 *   :555-606  AngularLInfinityTriangulator
 *   cv-core/src/triangulation.rs:21-35,52-67  the blanket TriangulatorRelative impl of the observations triangulators
 * and from nalgebra (not in the reference checkout): try_svd, restated as one-sided Jacobi on the 4x4 design matrix
 * (min_right_singular_vector, the algorithm of ref_geom.c's five-point helper for any n), whose sweeps epsilon / max_iterations bound
 * as they bound the eigen restatement's.  RelativeDlt's
 * parity with the crate is pinned only by the doc-tests and the unit test (triangulation.rs:651-680), both in
 * tests/test_oracle_triangulation.py.
 *
 * Reference details reproduced, not fixed (the device code in cv_b200/csrc/geom.cu cites the same):
 *   - SineL1 returns LinearEigen's point unrefined when its w == 0 (point() is None, :240-244); after the refinement it applies NO
 *     finiteness or cheirality check (:274); scale = optimization_rate / count (:246); it stops when |delta|^2 / |p|^2 < epsilon^2
 *     (:269); Default is 1e-12 / 1000 / rate 1.0 although the setter's doc comment says 0.01 (:197-199).
 *   - RelativeDlt's Default is 1e-12 / 1000 although its doc comments say 1e-9 and 100 (:293-320).
 *   - Cheirality uses the sign bit (is_sign_positive): -0.0 fails.
 *   - Isometry x unit vector applies the rotation only.
 *   - MeanMean divides by zero for n <= 1 and returns None through the finiteness filter.
 *   - AngularL1 / AngularL-infinity invert the relative pose and swap a and b first (:483-487, :569-573); AngularL1 builds z = b x a
 *     and the point on b, where epipolar.rs's sine-L1 point builds a x b (ref_optimize.c's sine_l1_point is not reused).
 * cv-sfm's observation_loss / is_tri_landmark_robust (cv-sfm/src/lib.rs:1320-1360, 2570-2620) are restated as in ref_optimize.c with
 * self.triangulator in place of LinearEigen.  Sums run in observation order from zero, as nalgebra's `.sum()` and `fold` do.  Built
 * by oracle/tri.mk with oracle/Makefile's flags (-ffp-contract=off). */
#include "ref_triangulation.h"
#include <math.h>
#include <string.h>

static double dot3(const double *a, const double *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
static double norm3(const double *a) { return sqrt(dot3(a, a)); }
static void cross3(const double *a, const double *b, double *o) {
    const double r0 = a[1] * b[2] - a[2] * b[1], r1 = a[2] * b[0] - a[0] * b[2], r2 = a[0] * b[1] - a[1] * b[0];
    o[0] = r0; o[1] = r1; o[2] = r2;
}
static void normalize3(const double *v, double *o) { double n = norm3(v); o[0] = v[0] / n; o[1] = v[1] / n; o[2] = v[2] / n; }
/* R^T v: Rotation3::inverse() * v (Isometry x vector applies the rotation only) */
static void rotTv(const double *R, const double *v, double *o) {
    for (int c = 0; c < 3; c++) o[c] = R[c] * v[0] + R[3 + c] * v[1] + R[6 + c] * v[2];
}
static int finite4(const double *p) { return isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]) && isfinite(p[3]); }
/* Projective::from_homogeneous (cv-core/src/point.rs:20-25) */
static void from_homogeneous(double *p) {
    if (signbit(p[3])) for (int i = 0; i < 4; i++) p[i] = -p[i];
    double n = norm3(p);
    for (int i = 0; i < 4; i++) p[i] /= n;
}
/* camera centre R^T (-t) and world-frame bearing R^T b of one (WorldToCamera, bearing): pose.inverse().isometry() */
static void obs_world(const ref_pose *P, const double *b, double *centre, double *wb) {
    const double nt[3] = {-P->t[0], -P->t[1], -P->t[2]};
    rotTv(P->R, nt, centre);
    rotTv(P->R, b, wb);
}
static int sweeps(const ref_triangulator *t) { return t->max_iterations > 0x7fffffffu ? 0x7fffffff : (int)t->max_iterations; }

/* accumulate (P - b bt P)t (P - b bt P) for a 3x4 pose matrix (triangulation.rs:92-106) */
static void design_add(const ref_pose *P, const double *b, double *D) {
    double M[3][4], T[3][4];
    for (int r = 0; r < 3; r++) { M[r][0] = P->R[3 * r]; M[r][1] = P->R[3 * r + 1]; M[r][2] = P->R[3 * r + 2]; M[r][3] = P->t[r]; }
    for (int c = 0; c < 4; c++) {
        double btP = b[0] * M[0][c] + b[1] * M[1][c] + b[2] * M[2][c];
        for (int r = 0; r < 3; r++) T[r][c] = M[r][c] - b[r] * btP;
    }
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) D[i * 4 + j] += T[0][i] * T[0][j] + T[1][i] * T[1][j] + T[2][i] * T[2][j];
}
/* :82-130 with try_symmetric_eigen(epsilon, max_iterations) restated as ref_sym_eigen */
static int linear_eigen(const ref_pose *poses, const double *bearings, int n, double eps, int max_sweeps, double *out) {
    if (n < 2) return 0;
    double A[16] = {0}, d[4], V[16];
    for (int i = 0; i < n; i++) design_add(&poses[i], bearings + 3 * i, A);
    if (!ref_sym_eigen(4, A, eps, max_sweeps, d, V)) return 0;
    int best = 0;
    for (int i = 1; i < 4; i++)
        if (d[i] < d[best]) best = i;
    double p[4] = {V[best], V[4 + best], V[8 + best], V[12 + best]};
    from_homogeneous(p);
    if (!finite4(p)) return 0;
    for (int i = 0; i < n; i++) {   /* cheirality: (R^-1 b) . p_bearing must be sign-positive */
        double wb[3];
        rotTv(poses[i].R, bearings + 3 * i, wb);
        if (signbit(dot3(wb, p))) return 0;
    }
    memcpy(out, p, sizeof(p));
    return 1;
}
/* right singular vector of the smallest singular value of an n x n matrix, n <= 4: one-sided Jacobi on the columns.  Returns 0 on
 * non-convergence (try_svd's None) */
static int min_right_singular_vector(int n, const double *Min, double eps, int max_sweeps, double *vec) {
    double U[4][4], V[4][4];
    for (int i = 0; i < n; i++) for (int j = 0; j < n; j++) { U[i][j] = Min[i * n + j]; V[i][j] = i == j ? 1.0 : 0.0; }
    int converged = 0;
    for (int sweep = 0; sweep < max_sweeps && !converged; sweep++) {
        converged = 1;
        for (int p = 0; p < n - 1; p++)
            for (int q = p + 1; q < n; q++) {
                double alpha = 0, beta = 0, gamma = 0;
                for (int i = 0; i < n; i++) { alpha += U[i][p] * U[i][p]; beta += U[i][q] * U[i][q]; gamma += U[i][p] * U[i][q]; }
                if (gamma == 0.0 || fabs(gamma) <= eps * sqrt(alpha * beta)) continue;
                converged = 0;
                double zeta = (beta - alpha) / (2.0 * gamma);
                double t = (zeta >= 0.0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
                double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
                for (int i = 0; i < n; i++) {
                    double up = U[i][p], uq = U[i][q];
                    U[i][p] = c * up - s * uq; U[i][q] = s * up + c * uq;
                    double vp = V[i][p], vq = V[i][q];
                    V[i][p] = c * vp - s * vq; V[i][q] = s * vp + c * vq;
                }
            }
    }
    if (!converged) return 0;
    int best = 0; double bn = -1.0;
    for (int j = 0; j < n; j++) {
        double nn = 0; for (int i = 0; i < n; i++) nn += U[i][j] * U[i][j];
        if (bn < 0.0 || nn < bn) { bn = nn; best = j; }
    }
    for (int i = 0; i < n; i++) vec[i] = V[i][best];
    return 1;
}

void ref_triangulator_default(ref_triangulator *t, int32_t method) {
    memset(t, 0, sizeof(*t));
    t->method = method;
    if (method == REF_TRI_LINEAR_EIGEN || method == REF_TRI_SINE_L1 || method == REF_TRI_RELATIVE_DLT) { t->epsilon = 1e-12; t->max_iterations = 1000; }
    if (method == REF_TRI_SINE_L1) t->optimization_rate = 1.0;
}

/* :228-276 */
static int sine_l1(const ref_triangulator *T, const ref_pose *P, const double *B, int n, double *p, uint32_t *iterations) {
    if (!linear_eigen(P, B, n, T->epsilon, sweeps(T), p)) return 0;
    if (p[3] == 0.0) return 1;                        /* point() is None: LinearEigen's point as it is */
    double x[3] = {p[0] / p[3], p[1] / p[3], p[2] / p[3]};
    const double scale = T->optimization_rate / (double)n, eps2 = T->epsilon * T->epsilon;
    uint32_t it = 0;
    while (it < T->max_iterations) {
        it++;
        double s[3] = {0.0, 0.0, 0.0};
        for (int i = 0; i < n; i++) {                 /* the reference recomputes centre and bearing here every iteration */
            double c[3], wb[3];
            obs_world(&P[i], B + 3 * i, c, wb);
            const double tr[3] = {c[0] - x[0], c[1] - x[1], c[2] - x[2]};
            const double d = dot3(tr, wb);
            for (int k = 0; k < 3; k++) s[k] = s[k] + (tr[k] - d * wb[k]);
        }
        const double delta[3] = {scale * s[0], scale * s[1], scale * s[2]};
        for (int k = 0; k < 3; k++) x[k] = x[k] + delta[k];
        if (dot3(delta, delta) / dot3(x, x) < eps2) break;
    }
    if (iterations) *iterations = it;
    p[0] = x[0]; p[1] = x[1]; p[2] = x[2]; p[3] = 1.0;
    from_homogeneous(p);                              /* Projective::from_point; no filter (:274) */
    return 1;
}

/* :392-442 */
static int mean_mean(const ref_pose *P, const double *B, int n, double *p) {
    const double total = (double)n;
    double sc[3] = {0.0, 0.0, 0.0}, sb[3] = {0.0, 0.0, 0.0}, c[3], wb[3];
    for (int i = 0; i < n; i++) {
        obs_world(&P[i], B + 3 * i, c, wb);
        for (int k = 0; k < 3; k++) { sc[k] = sc[k] + c[k]; sb[k] = sb[k] + wb[k]; }
    }
    const double ac[3] = {sc[0] / total, sc[1] / total, sc[2] / total};
    double ab[3];
    normalize3(sb, ab);
    double sum = 0.0;
    for (int i = 0; i < n; i++) {
        obs_world(&P[i], B + 3 * i, c, wb);
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
    if (!finite4(p)) return 0;
    for (int i = 0; i < n; i++) {
        obs_world(&P[i], B + 3 * i, c, wb);
        if (signbit(dot3(wb, p))) return 0;
    }
    return 1;
}

int ref_triangulate_observations(const ref_triangulator *t, const ref_pose *poses, const double *bearings, int n, double *out,
                                 uint32_t *iterations) {
    double p[4] = {0, 0, 0, 0};
    int ok;
    if (iterations) *iterations = 0;
    switch (t->method) {
    case REF_TRI_LINEAR_EIGEN: ok = linear_eigen(poses, bearings, n, t->epsilon, sweeps(t), p); break;
    case REF_TRI_SINE_L1: ok = sine_l1(t, poses, bearings, n, p, iterations); break;
    case REF_TRI_MEAN_MEAN: ok = mean_mean(poses, bearings, n, p); break;
    default: return 0;
    }
    if (ok) memcpy(out, p, sizeof(p));
    return ok;
}

/* :322-363 */
static int relative_dlt(const ref_triangulator *T, const ref_pose *P, const double *a, const double *b, double *p) {
    const double *R = P->R, *t = P->t;
    const double D[16] = {-a[2], 0.0, a[0], 0.0,
                          0.0, -a[2], a[1], 0.0,
                          b[0] * R[6] - b[2] * R[0], b[0] * R[7] - b[2] * R[1], b[0] * R[8] - b[2] * R[2], b[0] * t[2] - b[2] * t[0],
                          b[1] * R[6] - b[2] * R[3], b[1] * R[7] - b[2] * R[4], b[1] * R[8] - b[2] * R[5], b[1] * t[2] - b[2] * t[1]};
    double bw[3];
    if (!min_right_singular_vector(4, D, T->epsilon, sweeps(T), p)) return 0;
    from_homogeneous(p);
    if (!finite4(p)) return 0;
    rotTv(R, b, bw);
    return !signbit(dot3(p, a)) && !signbit(dot3(p, bw));
}

/* :472-530 (linf = 0) and :558-606 (linf = 1) */
static int angular(int linf, const ref_pose *P, const double *a_in, const double *b_in, double *p) {
    const double mt[3] = {-P->t[0], -P->t[1], -P->t[2]};
    double t[3], a[3], b[3] = {a_in[0], a_in[1], a_in[2]};   /* swapped: b is the old a */
    rotTv(P->R, mt, t);                                      /* relative_pose.inverse() translation */
    rotTv(P->R, b_in, a);                                    /* the old b in the old a's camera */
    double nt[3];
    normalize3(t, nt);
    if (!linf) {
        double ca[3], cb[3], v[3];
        cross3(a, nt, ca); cross3(b, nt, cb);
        const double can = norm3(ca), cbn = norm3(cb);
        if (can < cbn) {
            const double nb[3] = {cb[0] / cbn, cb[1] / cbn, cb[2] / cbn}, d = dot3(a, nb);
            for (int k = 0; k < 3; k++) v[k] = a[k] - d * nb[k];
            normalize3(v, a);
        } else {
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
    if (!finite4(p)) return 0;
    return !signbit(dot3(p, a)) && !signbit(dot3(p, b));
}

int ref_triangulate_relative(const ref_triangulator *t, const ref_pose *P, const double *a, const double *b, double *out) {
    double p[4] = {0, 0, 0, 0};
    int ok;
    switch (t->method) {
    case REF_TRI_RELATIVE_DLT: ok = relative_dlt(t, P, a, b, p); break;
    case REF_TRI_ANGULAR_L1: ok = angular(0, P, a, b, p); break;
    case REF_TRI_ANGULAR_LINF: ok = angular(1, P, a, b, p); break;
    default: {   /* the blanket impl: [(identity, a), (pose, b)], then CameraPoint::from_homogeneous */
        ref_pose O[2];
        memset(&O[0], 0, sizeof(ref_pose));
        O[0].R[0] = O[0].R[4] = O[0].R[8] = 1.0;
        O[1] = *P;
        const double B[6] = {a[0], a[1], a[2], b[0], b[1], b[2]};
        ok = ref_triangulate_observations(t, O, B, 2, p, NULL);
        if (ok) from_homogeneous(p);
    }
    }
    if (ok) memcpy(out, p, sizeof(p));
    return ok;
}

/* batches in the layout of include/cvb200_tri.h (rows of failed items zeroed, ok = 0); iterations (may be NULL): L SineL1 counts */
void ref_triangulate_observations_batch(const ref_triangulator *t, const ref_pose *poses, const double *bearings, const uint32_t *offsets,
                                        uint32_t L, double *xyzw, uint8_t *ok, uint32_t *iterations) {
    for (uint32_t l = 0; l < L; l++) {
        const uint32_t o0 = offsets[l];
        memset(xyzw + 4 * (size_t)l, 0, 4 * sizeof(double));
        ok[l] = (uint8_t)ref_triangulate_observations(t, poses + o0, bearings + 3 * (size_t)o0, (int)(offsets[l + 1] - o0), xyzw + 4 * (size_t)l,
                                                      iterations ? iterations + l : NULL);
    }
}
void ref_triangulate_relative_batch(const ref_triangulator *t, const ref_pose *poses, uint32_t npose, const double *a, const double *b,
                                    uint32_t n, double *xyzw, uint8_t *ok) {
    for (uint32_t i = 0; i < n; i++) {
        memset(xyzw + 4 * (size_t)i, 0, 4 * sizeof(double));
        ok[i] = (uint8_t)ref_triangulate_relative(t, poses + (npose == 1 ? 0 : i), a + 3 * (size_t)i, b + 3 * (size_t)i, xyzw + 4 * (size_t)i);
    }
}

/* ---- cv-sfm's robustness filters with the caller's triangulator (ref_optimize.c has them with LinearEigen) */
static void rotv(const double *R, const double *v, double *o) { for (int r = 0; r < 3; r++) o[r] = dot3(R + 3 * r, v); }
static void pose_inverse(const ref_pose *P, ref_pose *o) {
    double nt[3] = {-P->t[0], -P->t[1], -P->t[2]}, R[9];
    for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) R[3 * r + c] = P->R[3 * c + r];
    rotv(R, nt, o->t); memcpy(o->R, R, 72);
}
static void pose_mul(const ref_pose *A, const ref_pose *B, ref_pose *o) { /* A * B */
    ref_pose r;
    for (int i = 0; i < 3; i++) for (int c = 0; c < 3; c++) r.R[3 * i + c] = A->R[3 * i] * B->R[c] + A->R[3 * i + 1] * B->R[3 + c] + A->R[3 * i + 2] * B->R[6 + c];
    double sh[3]; rotv(A->R, B->t, sh);
    for (int i = 0; i < 3; i++) r.t[i] = A->t[i] + sh[i];
    *o = r;
}
static double transformed_cosine_distance(const ref_pose *P, const double *point_h, const double *bearing) {
    double q[4];
    for (int r = 0; r < 3; r++) q[r] = dot3(P->R + 3 * r, point_h) + P->t[r] * point_h[3];
    q[3] = point_h[3];
    from_homogeneous(q);
    return 1.0 - dot3(q, bearing);
}

/* cv-sfm/src/lib.rs:2570-2620 observation_loss for every observation of one landmark (poses are WorldToCamera) */
void ref_observation_losses_tri(const ref_triangulator *tri, const ref_pose *poses, const double *bearings, uint32_t n, double *loss) {
    if (n == 1) { loss[0] = 2.0; return; }
    if (n == 2) {
        ref_pose inv, tot; double fb[3];
        pose_inverse(&poses[0], &inv); pose_mul(&poses[1], &inv, &tot);
        rotv(tot.R, bearings, fb);
        const double l = 1.0 - cos(asin(ref_epipolar_loss(tot.t, fb, bearings + 3)));
        loss[0] = loss[1] = l;
        return;
    }
    double p[4];
    if (!ref_triangulate_observations(tri, poses, bearings, (int)n, p, NULL)) { for (uint32_t i = 0; i < n; i++) loss[i] = 2.0; return; }
    for (uint32_t i = 0; i < n; i++) loss[i] = transformed_cosine_distance(&poses[i], p, bearings + 3 * (size_t)i);
}

/* cv-sfm/src/lib.rs:1320-1360 (poses are CameraToCamera centre -> first / second) */
int ref_is_tri_landmark_robust_tri(const ref_triangulator *tri, const ref_pose *first, const ref_pose *second, const double *c, const double *f,
                                   const double *s, double maximum_cosine_distance, double incidence_minimum_cosine_distance) {
    ref_pose P[3]; double B[9], p[4];
    memset(&P[0], 0, sizeof(ref_pose)); P[0].R[0] = P[0].R[4] = P[0].R[8] = 1.0;
    P[1] = *first; P[2] = *second;
    memcpy(B, c, 24); memcpy(B + 3, f, 24); memcpy(B + 6, s, 24);
    if (!ref_triangulate_observations(tri, P, B, 3, p, NULL)) return 0;
    from_homogeneous(p);   /* CameraPoint::from_homogeneous(p.0) */
    double fc[3], sc[3];
    rotTv(first->R, f, fc); rotTv(second->R, s, sc);
    const int cosine_ok = 1.0 - dot3(p, c) < maximum_cosine_distance
        && transformed_cosine_distance(first, p, f) < maximum_cosine_distance
        && transformed_cosine_distance(second, p, s) < maximum_cosine_distance;
    const int incidence_ok = 1.0 - dot3(c, fc) > incidence_minimum_cosine_distance || 1.0 - dot3(c, sc) > incidence_minimum_cosine_distance
        || 1.0 - dot3(fc, sc) > incidence_minimum_cosine_distance;
    return cosine_ok && incidence_ok;
}
