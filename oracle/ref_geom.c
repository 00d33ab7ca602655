/* oracle/ref_geom.c -- TEST INFRASTRUCTURE: CPU restatement of the geometric-verification half of the
 * hot path (SURVEY.md section 8a rows R1-R8, T1, C1).  Not product code.
 *
 * Follows (paths relative to the reference checkout):
 *   eight-point/src/lib.rs:11-84            encode_epipolar_equation (incl. the b/a.z quirk), from_matches, estimate
 *   cv-pinhole/src/essential.rs:114-231     possible_rotations_unscaled_translation / possible_unscaled_poses
 *   cv-pinhole/src/essential.rs:266-275     EssentialMatrix::residual
 *   cv-pinhole/src/lib.rs:108-116           CameraIntrinsics::calibrate (no distortion)
 *   cv-core/src/pose.rs:194-202, 249-296    WorldToCamera::residual, CameraToCamera::residual
 *   cv-core/src/point.rs:20-25              Projective::from_homogeneous
 *   lambda-twist/src/lib.rs:110-317,361-554 compute_poses_nordberg and helpers
 *   cv-geom/src/triangulation.rs:82-130     LinearEigenTriangulator
 * and, from crates that are NOT in the reference checkout (restated from their published algorithms):
 *   nalgebra 0.30.1   try_symmetric_eigen / SVD  -> here: cyclic Jacobi (same mathematical result up to the
 *                     sign/order of eigenvectors, which nalgebra does not specify either); Rotation3::from_matrix_eps
 *   arrsac 0.10.0     adaptive real-time RANSAC   -> ref_arrsac_* below: restated from the crate's documented
 *                     parameters and the ARRSAC paper.  PARITY UNPINNED against the real crate (source unavailable;
 *                     SURVEY.md hard part 4): the in-tree tests only pin "all 11 matches are inliers"
 *                     (akaze/tests/estimate_pose.rs:75) and "pose from 5 exact points to 1e-6"
 *                     (lambda-twist/tests/consensus.rs:18-66), both checked in tests/test_oracle_geom.py.
 *   rand_xoshiro 0.6 / rand 0.8 SmallRng (xoshiro256++, SplitMix64 seeding), rand_pcg 0.3 Pcg64 (Lcg128Xsl64).
 * All arithmetic is f64; the comparison bar for f64 results is 1e-6 relative (BASELINE.json north_star).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "ref_geom.h"

/* ------------------------------------------------------------------ small linear algebra */
/* cyclic Jacobi eigen-decomposition of a symmetric n x n matrix (row-major, n <= 9).
 * d: eigenvalues, V: eigenvectors as COLUMNS (row-major n x n).  Returns 1 when converged. */
int ref_sym_eigen(int n, const double *Ain, double eps, int max_sweeps, double *d, double *V) {
    double A[81];
    memcpy(A, Ain, sizeof(double) * (size_t)n * n);
    for (int i = 0; i < n; i++)
        for (int j = 0; j < n; j++) V[i * n + j] = i == j ? 1.0 : 0.0;
    for (int sweep = 0; sweep < max_sweeps; sweep++) {
        double off = 0.0, diag = 0.0;
        for (int i = 0; i < n; i++) {
            diag += A[i * n + i] * A[i * n + i];
            for (int j = i + 1; j < n; j++) off += A[i * n + j] * A[i * n + j];
        }
        if (off <= eps * eps * diag || off == 0.0) {
            for (int i = 0; i < n; i++) d[i] = A[i * n + i];
            return 1;
        }
        for (int p = 0; p < n - 1; p++)
            for (int q = p + 1; q < n; q++) {
                double apq = A[p * n + q];
                if (apq == 0.0) continue;
                double app = A[p * n + p], aqq = A[q * n + q];
                double theta = (aqq - app) / (2.0 * apq);
                double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
                for (int k = 0; k < n; k++) {
                    double akp = A[k * n + p], akq = A[k * n + q];
                    A[k * n + p] = c * akp - s * akq;
                    A[k * n + q] = s * akp + c * akq;
                }
                for (int k = 0; k < n; k++) {
                    double apk = A[p * n + k], aqk = A[q * n + k];
                    A[p * n + k] = c * apk - s * aqk;
                    A[q * n + k] = s * apk + c * aqk;
                }
                for (int k = 0; k < n; k++) {
                    double vkp = V[k * n + p], vkq = V[k * n + q];
                    V[k * n + p] = c * vkp - s * vkq;
                    V[k * n + q] = s * vkp + c * vkq;
                }
            }
    }
    for (int i = 0; i < n; i++) d[i] = A[i * n + i];
    return 0;
}

/* The 9 x 9 eigensolver of the eight-point estimator: Jacobi in ROUND-ROBIN (tournament) order.  A sweep is nine rounds; round r
 * rotates the four disjoint index pairs {(r + k) mod 9, (r - k) mod 9}, k = 1..4 (index r rests; every pair of a sweep occurs exactly
 * once because 2 is invertible mod 9).  The four angles of a round are taken from the matrix in front of the round, then the column
 * rotations of all four pairs are applied (to A and to V), then the row rotations: disjoint pairs touch disjoint columns / rows, so
 * the result does not depend on the order inside a phase -- which is what lets the four rotations of a round run concurrently on the
 * device with identical bits.  The rotation is formed without the quotient theta: with d = aqq - app, h = 2 apq,
 *   w = |d| + sqrt(d^2 + h^2),  n = sqrt(w^2 + h^2),  c = w / n,  s = +-|h| / n   (sign of theta = d / h, + for theta = 0)
 * which is the textbook t = sgn(theta) / (|theta| + sqrt(theta^2 + 1)), c = 1 / sqrt(t^2 + 1), s = t c with two square roots and one
 * level of division on the dependent path instead of two square roots and three divisions.
 * (The reference calls nalgebra's symmetric_eigen, a tridiagonal QR iteration; every Jacobi variant is a restatement whose
 * eigenvectors agree with it to rounding, eigenvector signs being normalised downstream: essential.rs:139-143.) */
int ref_sym_eigen9_rr(const double *Ain, double eps, int max_sweeps, double *d, double *V) {
    enum { n = 9 };
    double A[81];
    memcpy(A, Ain, sizeof(A));
    for (int i = 0; i < n; i++)
        for (int j = 0; j < n; j++) V[i * n + j] = i == j ? 1.0 : 0.0;
    for (int sweep = 0; sweep < max_sweeps; sweep++) {
        double off = 0.0, diag = 0.0;
        for (int i = 0; i < n; i++) {
            diag += A[i * n + i] * A[i * n + i];
            for (int j = i + 1; j < n; j++) off += A[i * n + j] * A[i * n + j];
        }
        if (off <= eps * eps * diag || off == 0.0) {
            for (int i = 0; i < n; i++) d[i] = A[i * n + i];
            return 1;
        }
        for (int r = 0; r < n; r++) {
            int P[4], Q[4], act[4];
            double C[4], S[4];
            for (int k = 1; k <= 4; k++) {
                const int a = (r + k) % n, b = (r + n - k) % n;
                const int p = a < b ? a : b, q = a < b ? b : a;
                P[k - 1] = p; Q[k - 1] = q;
                const double apq = A[p * n + q];
                act[k - 1] = apq != 0.0;
                if (!act[k - 1]) continue;
                const double dd = A[q * n + q] - A[p * n + p], h = 2.0 * apq;
                const double w = fabs(dd) + sqrt(dd * dd + h * h);
                const double nn = sqrt(w * w + h * h);
                const int pos = dd == 0.0 || ((dd > 0.0) == (h > 0.0));
                C[k - 1] = w / nn;
                S[k - 1] = (pos ? fabs(h) : -fabs(h)) / nn;
            }
            for (int i = 0; i < 4; i++) {
                if (!act[i]) continue;
                const int p = P[i], q = Q[i];
                const double c = C[i], s2 = S[i];
                for (int k = 0; k < n; k++) {
                    const double akp = A[k * n + p], akq = A[k * n + q];
                    A[k * n + p] = c * akp - s2 * akq;
                    A[k * n + q] = s2 * akp + c * akq;
                    const double vkp = V[k * n + p], vkq = V[k * n + q];
                    V[k * n + p] = c * vkp - s2 * vkq;
                    V[k * n + q] = s2 * vkp + c * vkq;
                }
            }
            for (int i = 0; i < 4; i++) {
                if (!act[i]) continue;
                const int p = P[i], q = Q[i];
                const double c = C[i], s2 = S[i];
                for (int k = 0; k < n; k++) {
                    const double apk = A[p * n + k], aqk = A[q * n + k];
                    A[p * n + k] = c * apk - s2 * aqk;
                    A[q * n + k] = s2 * apk + c * aqk;
                }
            }
        }
    }
    for (int i = 0; i < n; i++) d[i] = A[i * n + i];
    return 0;
}

static void mat3_mul(const double *a, const double *b, double *o) {
    double r[9];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) r[i * 3 + j] = a[i * 3] * b[j] + a[i * 3 + 1] * b[3 + j] + a[i * 3 + 2] * b[6 + j];
    memcpy(o, r, sizeof(r));
}
static double det3(const double *m) {
    return m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) + m[2] * (m[3] * m[7] - m[4] * m[6]);
}
static void cross3(const double *a, const double *b, double *o) {
    double r[3] = {a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]};
    o[0] = r[0]; o[1] = r[1]; o[2] = r[2];
}
static double dot3(const double *a, const double *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
static double norm3(const double *a) { return sqrt(dot3(a, a)); }

/* sorted (descending) SVD of a 3x3 matrix: M = U diag(s) Vt, via the eigen-decomposition of MtM */
int ref_svd3(const double *M, double eps, int max_iter, double *U, double *s, double *Vt) {
    double MtM[9], d[3], V[9];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) MtM[i * 3 + j] = M[i] * M[j] + M[3 + i] * M[3 + j] + M[6 + i] * M[6 + j];
    if (!ref_sym_eigen(3, MtM, eps, max_iter, d, V)) return 0;
    int ord[3] = {0, 1, 2};
    for (int i = 0; i < 2; i++)
        for (int j = i + 1; j < 3; j++)
            if (d[ord[j]] > d[ord[i]]) { int t = ord[i]; ord[i] = ord[j]; ord[j] = t; }
    double v[3][3], u[3][3];
    for (int k = 0; k < 3; k++) {
        for (int r = 0; r < 3; r++) v[k][r] = V[r * 3 + ord[k]];
        s[k] = sqrt(d[ord[k]] > 0.0 ? d[ord[k]] : 0.0);
    }
    /* u_k = M v_k / s_k for the two leading triplets; the third left vector is fixed up to sign by
     * orthogonality and its sign is normalised by the caller's det(U) > 0 rule (essential.rs:139-143),
     * so u_3 = u_1 x u_2 (robust when s_3 ~ 0, the essential-matrix case). */
    double tiny = 1e-12 * (s[0] > 0.0 ? s[0] : 1.0);
    for (int k = 0; k < 2; k++) {
        if (!(s[k] > tiny)) return 0; /* rank <= 1: no essential-matrix decomposition */
        for (int r = 0; r < 3; r++) u[k][r] = (M[r * 3] * v[k][0] + M[r * 3 + 1] * v[k][1] + M[r * 3 + 2] * v[k][2]) / s[k];
    }
    cross3(u[0], u[1], u[2]);
    {
        double nn = norm3(u[2]);
        if (!(nn > 0.0)) return 0;
        for (int r = 0; r < 3; r++) u[2][r] /= nn;
    }
    for (int k = 0; k < 3; k++)
        for (int r = 0; r < 3; r++) { U[r * 3 + k] = u[k][r]; Vt[k * 3 + r] = v[k][r]; }
    return 1;
}

/* ------------------------------------------------------------------ eight-point */
/* eight-point/src/lib.rs:11-24,43-58: a, b are unit bearings (8 x 3 each). E is row-major. */
int ref_eight_point_essential(const double *a, const double *b, double eps, int iters, double *E) {
    double A[8][9], EtE[81], d[9], V[81];
    for (int i = 0; i < 8; i++) {
        const double *pa = a + 3 * i, *pb = b + 3 * i;
        double ap[3] = {pa[0] / pa[2], pa[1] / pa[2], pa[2] / pa[2]};
        double bp[3] = {pb[0] / pa[2], pb[1] / pa[2], pb[2] / pa[2]}; /* sic: b is divided by a.z (lib.rs:16) */
        for (int j = 0; j < 3; j++)
            for (int k = 0; k < 3; k++) A[i][3 * j + k] = ap[j] * bp[k];
    }
    for (int r = 0; r < 9; r++)
        for (int c = 0; c < 9; c++) {
            double s = 0.0;
            for (int i = 0; i < 8; i++) s += A[i][r] * A[i][c];
            EtE[r * 9 + c] = s;
        }
    if (!ref_sym_eigen9_rr(EtE, eps, iters, d, V)) return 0;
    int best = 0;
    for (int i = 1; i < 9; i++)
        if (d[i] < d[best]) best = i;
    /* Matrix3::from_iterator fills column-major: e[0..3] is column 0 (lib.rs:56) */
    for (int k = 0; k < 9; k++) E[(k % 3) * 3 + (k / 3)] = V[k * 9 + best];
    return 1;
}

/* cv-pinhole/src/essential.rs:114-162,217-231 -> 4 poses (R row-major, t) in the reference's order */
int ref_essential_poses(const double *E, double eps, int iters, ref_pose out[4]) {
    double U[9], s[3], Vt[9];
    if (!ref_svd3(E, eps, iters, U, s, Vt)) return 0;
    if (det3(U) < 0.0) for (int r = 0; r < 3; r++) U[r * 3 + 2] *= -1.0;
    if (det3(Vt) < 0.0) for (int c = 0; c < 3; c++) Vt[6 + c] *= -1.0;
    const double W[9] = {0, -1, 0, 1, 0, 0, 0, 0, 1}, Wt[9] = {0, 1, 0, -1, 0, 0, 0, 0, 1};
    double UW[9], Ra[9], Rb[9];
    mat3_mul(U, W, UW); mat3_mul(UW, Vt, Ra);
    mat3_mul(U, Wt, UW); mat3_mul(UW, Vt, Rb);
    double t[3] = {U[2], U[5], U[8]};
    for (int k = 0; k < 4; k++) {
        memcpy(out[k].R, (k & 1) ? Rb : Ra, sizeof(double) * 9);
        for (int r = 0; r < 3; r++) out[k].t[r] = (k & 2) ? -t[r] : t[r];
    }
    return 4;
}

int ref_eight_point(const double *a, const double *b, ref_pose out[4]) { /* Estimator::estimate, eps 1e-12, 1000 */
    double E[9];
    if (!ref_eight_point_essential(a, b, 1e-12, 1000, E)) return 0;
    return ref_essential_poses(E, 1e-12, 1000, out);
}

/* essential.rs:266-275 */
double ref_essential_residual(const double *E, const double *a, const double *b) {
    double na[3] = {a[0] / a[2], a[1] / a[2], a[2] / a[2]}, nb[3] = {b[0] / b[2], b[1] / b[2], b[2] / b[2]};
    double Ea[3] = {dot3(E, na), dot3(E + 3, na), dot3(E + 6, na)};
    return fabs(dot3(nb, Ea));
}

/* ------------------------------------------------------------------ five-point (nister-stewenius/src/lib.rs) */
/* nalgebra pieces used by the reference and restated here: full_piv_lu().solve (Gaussian elimination with
 * complete pivoting), complex_eigenvalues() (Hessenberg reduction + Francis double-shift QR, EISPACK hqr),
 * try_svd(false, true, ..) (one-sided Jacobi: accurate small singular values + right singular vectors). */
#define FP_N 10
static int lu_full_pivot_solve(const double *Ain, const double *Bin, double *X) { /* A X = B, all 10x10 row-major */
    double A[FP_N][FP_N], B[FP_N][FP_N];
    int colperm[FP_N];
    memcpy(A, Ain, sizeof(A)); memcpy(B, Bin, sizeof(B));
    for (int i = 0; i < FP_N; i++) colperm[i] = i;
    for (int k = 0; k < FP_N; k++) {
        int pr = k, pc = k; double best = -1.0;
        for (int i = k; i < FP_N; i++) for (int j = k; j < FP_N; j++) if (fabs(A[i][j]) > best) { best = fabs(A[i][j]); pr = i; pc = j; }
        if (best == 0.0) return 0; /* singular: nalgebra's solve returns None */
        if (pr != k) for (int j = 0; j < FP_N; j++) { double t = A[k][j]; A[k][j] = A[pr][j]; A[pr][j] = t; t = B[k][j]; B[k][j] = B[pr][j]; B[pr][j] = t; }
        if (pc != k) { for (int i = 0; i < FP_N; i++) { double t = A[i][k]; A[i][k] = A[i][pc]; A[i][pc] = t; } int t = colperm[k]; colperm[k] = colperm[pc]; colperm[pc] = t; }
        for (int i = k + 1; i < FP_N; i++) {
            double f = A[i][k] / A[k][k];
            if (f == 0.0) continue;
            for (int j = k; j < FP_N; j++) A[i][j] -= f * A[k][j];
            for (int j = 0; j < FP_N; j++) B[i][j] -= f * B[k][j];
        }
    }
    double Y[FP_N][FP_N];
    for (int c = 0; c < FP_N; c++)
        for (int i = FP_N - 1; i >= 0; i--) {
            double v = B[i][c];
            for (int j = i + 1; j < FP_N; j++) v -= A[i][j] * Y[j][c];
            Y[i][c] = v / A[i][i];
        }
    for (int i = 0; i < FP_N; i++) for (int c = 0; c < FP_N; c++) X[colperm[i] * FP_N + c] = Y[i][c];
    return 1;
}

#define FP_SIGN(a, b) ((b) >= 0.0 ? fabs(a) : -fabs(a))
/* eigenvalues of a real 10x10 matrix: wr + i wi (wi == 0 exactly for real eigenvalues). returns 0 on non-convergence */
int ref_real_eigenvalues10(const double *Ain, double *wr, double *wi) {
    const int n = FP_N;
    double a[FP_N][FP_N];
    memcpy(a, Ain, sizeof(a));
    /* reduction to upper Hessenberg form by stabilised elementary similarity transformations */
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
    /* Francis double-shift QR on the Hessenberg matrix */
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
                        z = p + FP_SIGN(z, p);
                        wr[nn - 1] = wr[nn] = x + z;
                        if (z != 0.0) wr[nn] = x - w / z;
                        wi[nn - 1] = wi[nn] = 0.0;
                    } else { wr[nn - 1] = wr[nn] = x + p; wi[nn] = z; wi[nn - 1] = -z; }
                    nn -= 2;
                } else {
                    if (its == 60) return 0;
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
                        if ((s = FP_SIGN(sqrt(p * p + q * q + r * r), p)) != 0.0) {
                            if (k == m) { if (l != m) a[k][k - 1] = -a[k][k - 1]; }
                            else a[k][k - 1] = -s * x;
                            p += s; x = p / s; y = q / s; z = r / s; q /= p; r /= p;
                            for (int j = k; j <= nn; j++) {
                                p = a[k][j] + q * a[k + 1][j];
                                if (k != nn - 1) { p += r * a[k + 2][j]; a[k + 2][j] -= p * z; }
                                a[k + 1][j] -= p * y; a[k][j] -= p * x;
                            }
                            int mmin = nn < k + 3 ? nn : k + 3;
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
    return 1;
}

/* right singular vector of the smallest singular value of a 10x10 matrix (one-sided Jacobi on the columns);
 * *smin receives that singular value. returns 0 on non-convergence */
static int min_right_singular_vector10(const double *Min, double eps, int max_sweeps, double *vec, double *smin) {
    double U[FP_N][FP_N], V[FP_N][FP_N];
    memcpy(U, Min, sizeof(U));
    for (int i = 0; i < FP_N; i++) for (int j = 0; j < FP_N; j++) V[i][j] = i == j ? 1.0 : 0.0;
    int converged = 0;
    for (int sweep = 0; sweep < max_sweeps && !converged; sweep++) {
        converged = 1;
        for (int p = 0; p < FP_N - 1; p++)
            for (int q = p + 1; q < FP_N; q++) {
                double alpha = 0, beta = 0, gamma = 0;
                for (int i = 0; i < FP_N; i++) { alpha += U[i][p] * U[i][p]; beta += U[i][q] * U[i][q]; gamma += U[i][p] * U[i][q]; }
                if (gamma == 0.0 || fabs(gamma) <= eps * sqrt(alpha * beta)) continue;
                converged = 0;
                double zeta = (beta - alpha) / (2.0 * gamma);
                double t = (zeta >= 0.0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
                double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
                for (int i = 0; i < FP_N; i++) {
                    double up = U[i][p], uq = U[i][q];
                    U[i][p] = c * up - s * uq; U[i][q] = s * up + c * uq;
                    double vp = V[i][p], vq = V[i][q];
                    V[i][p] = c * vp - s * vq; V[i][q] = s * vp + c * vq;
                }
            }
    }
    if (!converged) return 0;
    int best = 0; double bn = -1.0;
    for (int j = 0; j < FP_N; j++) {
        double nn = 0; for (int i = 0; i < FP_N; i++) nn += U[i][j] * U[i][j];
        if (bn < 0.0 || nn < bn) { bn = nn; best = j; }
    }
    *smin = sqrt(bn);
    for (int i = 0; i < FP_N; i++) vec[i] = V[i][best];
    return 1;
}

#ifndef REF_FIVE_POINT_ROW0
#define REF_FIVE_POINT_ROW0 5
#endif
static int ref_five_point_row0 = REF_FIVE_POINT_ROW0;
double ref_fp_dbg[30];   /* last call: (wr, wi, smin) per eigenvalue, for tests */
void ref_five_point_set_row0(int r0) { ref_five_point_row0 = r0; }   /* 5 = reference behaviour, 6 = corrected */

enum { BXXX = 0, BXXY, BXYY, BYYY, BXXZ, BXYZ, BYYZ, BXZZ, BYZZ, BZZZ, BXX, BXY, BYY, BXZ, BYZ, BZZ, BX, BY, BZ, B1 };
static void fp_o1(const double *a, const double *b, double *r) { /* lib.rs:98-111 */
    for (int i = 0; i < 20; i++) r[i] = 0.0;
    r[BXX] = a[0] * b[0]; r[BXY] = a[0] * b[1] + a[1] * b[0]; r[BXZ] = a[0] * b[2] + a[2] * b[0];
    r[BYY] = a[1] * b[1]; r[BYZ] = a[1] * b[2] + a[2] * b[1]; r[BZZ] = a[2] * b[2];
    r[BX] = a[0] * b[3] + a[3] * b[0]; r[BY] = a[1] * b[3] + a[3] * b[1]; r[BZ] = a[2] * b[3] + a[3] * b[2]; r[B1] = a[3] * b[3];
}
static void fp_o2(const double *a, const double *b, double *r) { /* lib.rs:113-136 */
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

/* nister-stewenius/src/lib.rs:50-96,138-330: five matches (a, b: 5 x 3 unit bearings) -> up to 10 essential matrices
 * (row-major) ; returns the count */
int ref_five_point_essentials(const double *a, const double *b, double *Es) {
    /* step 1: null space of the 5x9 epipolar constraint (lib.rs:50-96) */
    double A[5][9], EE[81], d[9], V[81];
    for (int i = 0; i < 5; i++)
        for (int j = 0; j < 3; j++)
            for (int k = 0; k < 3; k++) A[i][3 * j + k] = a[3 * i + j] * b[3 * i + k];
    for (int r = 0; r < 9; r++)
        for (int c = 0; c < 9; c++) { double s = 0; for (int i = 0; i < 5; i++) s += A[i][r] * A[i][c]; EE[r * 9 + c] = s; }
    if (!ref_sym_eigen(9, EE, 1e-12, 1000, d, V)) return 0;
    int src[9] = {0, 1, 2, 3, 4, 5, 6, 7, 8};
    for (int i = 1; i < 9; i++) { int x = src[i], j = i; while (j > 0 && d[src[j - 1]] > d[x]) { src[j] = src[j - 1]; j--; } src[j] = x; }
    int nullity = -1;
    for (int i = 0; i < 9; i++) if (d[src[i]] > 1e-12) { nullity = i; break; }
    if (nullity != 4) return 0;
    double eb[9][4];
    for (int c = 0; c < 4; c++) for (int r = 0; r < 9; r++) eb[r][c] = V[r * 9 + src[c]];
    /* step 2: polynomial constraints (lib.rs:138-204) */
    double ep[3][3][4];
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) for (int k = 0; k < 4; k++) ep[i][j][k] = eb[3 * i + j][k];
    double M[10][20], t1[20], t2[20], t3[20], acc[20];
    {
        const int ia[3][2] = {{1, 2}, {2, 0}, {0, 1}};
        for (int k = 0; k < 20; k++) acc[k] = 0.0;
        for (int c = 0; c < 3; c++) {   /* det(E): sum_c (e0[p] e1[q] - e0[q] e1[p]) e2[c] with (p, q) = cyclic */
            int p = ia[c][0], q = ia[c][1];
            fp_o1(ep[0][p], ep[1][q], t1); fp_o1(ep[0][q], ep[1][p], t2);
            for (int k = 0; k < 20; k++) t1[k] -= t2[k];
            fp_o2(t1, ep[2][c], t3);
            for (int k = 0; k < 20; k++) acc[k] += t3[k];
        }
        memcpy(M[0], acc, sizeof(acc));
    }
    double eet[3][3][20], L[3][3][20];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            if (i <= j) {
                fp_o1(ep[i][0], ep[j][0], t1); fp_o1(ep[i][1], ep[j][1], t2); fp_o1(ep[i][2], ep[j][2], t3);
                for (int k = 0; k < 20; k++) eet[i][j][k] = t1[k] + t2[k] + t3[k];
            } else memcpy(eet[i][j], eet[j][i], sizeof(t1));
        }
    memcpy(L, eet, sizeof(L));
    for (int k = 0; k < 20; k++) {
        double tr = 0.5 * (eet[0][0][k] + eet[1][1][k] + eet[2][2][k]);
        for (int i = 0; i < 3; i++) L[i][i][k] -= tr;
    }
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            fp_o2(L[i][0], ep[0][j], t1); fp_o2(L[i][1], ep[1][j], t2); fp_o2(L[i][2], ep[2][j], t3);
            for (int k = 0; k < 20; k++) M[1 + i * 3 + j][k] = t1[k] + t2[k] + t3[k];
        }
    /* step 3: Gauss-Jordan through a fully pivoted LU (lib.rs:255-262) */
    double Cl[100], Cr[100], X[100];
    for (int i = 0; i < 10; i++) for (int j = 0; j < 10; j++) { Cl[i * 10 + j] = M[i][j]; Cr[i * 10 + j] = M[i][10 + j]; }
    if (!lu_full_pivot_solve(Cl, Cr, X)) return 0;
    /* action matrix (lib.rs:266-278) */
    double At[100];
    memset(At, 0, sizeof(At));
    for (int j = 0; j < 10; j++) {
        At[0 * 10 + j] = X[0 * 10 + j]; At[1 * 10 + j] = X[1 * 10 + j]; At[2 * 10 + j] = X[2 * 10 + j];
        At[3 * 10 + j] = X[4 * 10 + j]; At[4 * 10 + j] = X[5 * 10 + j]; At[5 * 10 + j] = X[7 * 10 + j];
    }
    At[6 * 10 + 0] = -1.0; At[7 * 10 + 1] = -1.0; At[8 * 10 + 3] = -1.0; At[9 * 10 + 6] = -1.0;
    /* eigenvalues; for the real ones the eigenvector via the smallest right singular vector (lib.rs:206-237) */
    double wr[10], wi[10];
    if (!ref_real_eigenvalues10(At, wr, wi)) return 0;
    int ne = 0;
    for (int i = 0; i < 10; i++) {
        ref_fp_dbg[i * 3] = wr[i]; ref_fp_dbg[i * 3 + 1] = wi[i]; ref_fp_dbg[i * 3 + 2] = -1.0;
        if (wi[i] != 0.0) continue;
        double Mx[100], vec[10], smin;
        memcpy(Mx, At, sizeof(Mx));
        for (int k = 0; k < 10; k++) Mx[k * 10 + k] -= wr[i];
        if (!min_right_singular_vector10(Mx, 1e-15, 1000, vec, &smin)) continue;
        ref_fp_dbg[i * 3 + 2] = smin;
        if (!(smin < 1e-12)) continue;
        double ev[9];
        /* `v.fixed_rows::<4>(5)` (lib.rs:229): rows 5..8 of the eigenvector.  The monomial basis is
         * [xx xy yy xz yz zz x y z 1], so (x, y, z, 1) are rows 6..9 (OpenMVG, from which this solver derives, takes
         * tail<4>()): the reference is off by one and its essentials do not satisfy the cubic constraints -- which is
         * presumably why nister-stewenius/tests/manual.rs is commented out upstream.  The restatement reproduces the
         * reference (REF_FIVE_POINT_ROW0 = 5); building with -DREF_FIVE_POINT_ROW0=6 gives the mathematically correct
         * solver and is used by tests/test_oracle_geom.py to validate every other step of the restatement. */
        const int r0 = ref_five_point_row0;
        for (int r = 0; r < 9; r++) ev[r] = eb[r][0] * vec[r0] + eb[r][1] * vec[r0 + 1] + eb[r][2] * vec[r0 + 2] + eb[r][3] * vec[r0 + 3];
        for (int k = 0; k < 9; k++) Es[ne * 9 + (k % 3) * 3 + (k / 3)] = ev[k]; /* Matrix3::from_iterator: column-major */
        ne++;
    }
    return ne;
}

/* Estimator::estimate (lib.rs:310-329): up to 40 CameraToCamera poses */
int ref_five_point(const double *a, const double *b, ref_pose *out) {
    double Es[90];
    int ne = ref_five_point_essentials(a, b, Es), n = 0;
    for (int i = 0; i < ne; i++) {
        ref_pose p4[4];
        if (ref_essential_poses(Es + 9 * i, 1e-12, 1000, p4) == 4) { memcpy(out + n, p4, sizeof(p4)); n += 4; }
    }
    return n;
}

/* ------------------------------------------------------------------ residuals */
/* point.rs:20-25 Projective::from_homogeneous */
static void from_homogeneous(double *p) {
    if (signbit(p[3])) for (int i = 0; i < 4; i++) p[i] = -p[i];
    double n = norm3(p);
    for (int i = 0; i < 4; i++) p[i] /= n;
}
static void pose_apply(const ref_pose *P, const double *x, double *o) { /* to_homogeneous() * x */
    for (int r = 0; r < 3; r++) o[r] = dot3(P->R + 3 * r, x) + P->t[r] * x[3];
    o[3] = x[3];
}
/* accumulate (P - b bt P)t (P - b bt P) for a 3x4 pose matrix */
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

/* cv-core/src/pose.rs:249-296 */
double ref_residual_c2c(const ref_pose *P, const double *a, const double *b) {
    double D[16] = {0}, d[4], V[16];
    ref_pose I = {{1, 0, 0, 0, 1, 0, 0, 0, 1}, {0, 0, 0}};
    design_add(&I, a, D);
    design_add(P, b, D);
    if (!ref_sym_eigen(4, D, 1e-12, 1024, d, V)) return 2.0;
    int best = 0;
    for (int i = 1; i < 4; i++)
        if (fabs(d[i]) < fabs(d[best])) best = i;
    double p[4] = {V[best], V[4 + best], V[8 + best], V[12 + best]};
    from_homogeneous(p);
    for (int i = 0; i < 4; i++) if (!isfinite(p[i])) return 2.0;
    double q[4];
    pose_apply(P, p, q);
    from_homogeneous(q);
    return 0.5 * (1.0 - dot3(a, p) + 1.0 - dot3(b, q));
}

/* cv-core/src/pose.rs:194-202; world is a homogeneous WorldPoint (xyz unit, w >= 0) */
double ref_residual_w2c(const ref_pose *P, const double *bearing, const double *world) {
    double q[4];
    pose_apply(P, world, q);
    from_homogeneous(q);
    return 1.0 - dot3(bearing, q);
}

/* ------------------------------------------------------------------ lambda twist */
static void root2real(double b, double c, double *r1, double *r2) { /* lib.rs:423-435 */
    double disc = b * b - 4.0 * c;
    if (disc < 0.0) { *r1 = *r2 = 0.5 * b; }
    else if (b < 0.0) { double y = sqrt(disc); *r1 = 0.5 * (-b + y); *r2 = 0.5 * (-b - y); }
    else { double y = sqrt(disc); *r1 = 2.0 * c / (-b + y); *r2 = 2.0 * c / (-b - y); }
}
static double cube_root(double b, double c, double d) { /* lib.rs:458-506 */
    double r0;
    if (b * b >= 3.0 * c) {
        double v = sqrt(b * b - 3.0 * c);
        double t1 = (-b - v) / 3.0;
        double k = ((t1 + b) * t1 + c) * t1 + d;
        if (k > 0.0) r0 = t1 - sqrt(-k / (3.0 * t1 + b));
        else {
            double t2 = (-b + v) / 3.0;
            k = ((t2 + b) * t2 + c) * t2 + d;
            r0 = t2 + sqrt(-k / (3.0 * t2 + b));
        }
    } else {
        r0 = -b / 3.0;
        if (fabs((3.0 * r0 + 2.0 * b) * r0 + c) < 1e-4) r0 += 1.0;
    }
    for (int i = 0; i < 7; i++) {
        double fx = ((r0 + b) * r0 + c) * r0 + d, fpx = (3.0 * r0 + 2.0 * b) * r0 + c;
        r0 -= fx / fpx;
    }
    for (int i = 0; i < 43; i++) {
        double fx = ((r0 + b) * r0 + c) * r0 + d;
        if (fabs(fx) > 1e-13) { double fpx = (3.0 * r0 + 2.0 * b) * r0 + c; r0 -= fx / fpx; }
        else break;
    }
    return r0;
}
/* lib.rs:510-554; x row-major symmetric; Ev columns v1 v2 v3 (row-major), ev[0..2] */
static void eigen_decomposition_singular(const double *x, double *Ev, double *ev) {
    /* nalgebra linear index is column-major: x[1]=m21 x[2]=m31 x[3]=m12 x[4]=m22 x[5]=m32 */
    double m11 = x[0], m12 = x[1], m13 = x[2], m21 = x[3], m22 = x[4], m23 = x[5], m31 = x[6], m32 = x[7], m33 = x[8];
    double v3[3] = {m21 * m32 - m31 * m22, m31 * m12 - m32 * m11, m22 * m11 - m21 * m12};
    double n = norm3(v3);
    for (int i = 0; i < 3; i++) v3[i] /= n;
    double x12_sqr = m12 * m12;
    double b = -m11 - m22 - m33;
    double c = -x12_sqr - m13 * m13 - m23 * m23 + m11 * (m22 + m33) + m22 * m33;
    double e1, e2;
    root2real(b, c, &e1, &e2);
    if (fabs(e1) < fabs(e2)) { double t = e1; e1 = e2; e2 = t; }
    ev[0] = e1; ev[1] = e2; ev[2] = 0.0;
    double mx0011 = -m11 * m22, prec_0 = m12 * m23 - m13 * m22, prec_1 = m12 * m13 - m11 * m23;
    double es[2] = {e1, e2}, v[2][3];
    for (int k = 0; k < 2; k++) {
        double e = es[k];
        double tmp = 1.0 / (e * (m11 + m22) + mx0011 - e * e + x12_sqr);
        double a1 = -(e * m13 + prec_0) * tmp, a2 = -(e * m23 + prec_1) * tmp;
        double rnorm = 1.0 / sqrt(a1 * a1 + a2 * a2 + 1.0);
        v[k][0] = a1 * rnorm; v[k][1] = a2 * rnorm; v[k][2] = rnorm;
    }
    for (int r = 0; r < 3; r++) { Ev[r * 3] = v[0][r]; Ev[r * 3 + 1] = v[1][r]; Ev[r * 3 + 2] = v3[r]; }
}
static double l1n(const double *v) { return fabs(v[0]) + fabs(v[1]) + fabs(v[2]); }
static void gn_residual(const double *l, double a12, double a13, double a23, double b12, double b13, double b23, double *r) {
    r[0] = l[0] * l[0] + l[1] * l[1] + b12 * l[0] * l[1] - a12;
    r[1] = l[0] * l[0] + l[2] * l[2] + b13 * l[0] * l[2] - a13;
    r[2] = l[1] * l[1] + l[2] * l[2] + b23 * l[1] * l[2] - a23;
}
/* lib.rs:361-412 */
static void gauss_newton_refine_lambda(double *l, int iterations, double a12, double a13, double a23, double b12, double b13, double b23) {
    double res[3];
    gn_residual(l, a12, a13, a23, b12, b13, b23, res);
    for (int it = 0; it < iterations; it++) {
        if (l1n(res) < 1e-10) break;
        double l1 = l[0], l2 = l[1], l3 = l[2];
        double dr1dl1 = 2.0 * l1 + b12 * l2, dr1dl2 = 2.0 * l2 + b12 * l1, dr2dl1 = 2.0 * l1 + b13 * l3;
        double dr2dl3 = 2.0 * l3 + b13 * l1, dr3dl2 = 2.0 * l2 + b23 * l3, dr3dl3 = 2.0 * l3 + b23 * l2;
        double det = 1.0 / (-dr1dl1 * dr2dl3 * dr3dl2 - dr1dl2 * dr2dl1 * dr3dl3);
        double J[9] = {-dr2dl3 * dr3dl2, -dr1dl2 * dr3dl3, dr1dl2 * dr2dl3,
                       -dr2dl1 * dr3dl3, dr1dl1 * dr3dl3, -dr1dl1 * dr2dl3,
                       dr2dl1 * dr3dl2, -dr1dl1 * dr3dl2, -dr1dl2 * dr2dl1};
        double ln[3], rn[3];
        for (int r = 0; r < 3; r++) ln[r] = l[r] - det * dot3(J + 3 * r, res);
        gn_residual(ln, a12, a13, a23, b12, b13, b23, rn);
        if (l1n(rn) > l1n(res)) break;
        memcpy(l, ln, sizeof(ln)); memcpy(res, rn, sizeof(rn));
    }
}
static int inv3(const double *m, double *o) {
    double d = det3(m);
    if (d == 0.0) return 0;
    double id = 1.0 / d;
    o[0] = (m[4] * m[8] - m[5] * m[7]) * id; o[1] = (m[2] * m[7] - m[1] * m[8]) * id; o[2] = (m[1] * m[5] - m[2] * m[4]) * id;
    o[3] = (m[5] * m[6] - m[3] * m[8]) * id; o[4] = (m[0] * m[8] - m[2] * m[6]) * id; o[5] = (m[2] * m[3] - m[0] * m[5]) * id;
    o[6] = (m[3] * m[7] - m[4] * m[6]) * id; o[7] = (m[1] * m[6] - m[0] * m[7]) * id; o[8] = (m[0] * m[4] - m[1] * m[3]) * id;
    return 1;
}
/* nalgebra Rotation3::from_matrix_eps(m, eps, max_iter, identity): iterative closest rotation */
static void rotation_from_matrix_eps(const double *m, double eps, int max_iter, double *rot) {
    double R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    for (int it = 0; it < max_iter; it++) {
        double axis[3] = {0, 0, 0}, denom = 0.0;
        for (int c = 0; c < 3; c++) {
            double rc[3] = {R[c], R[3 + c], R[6 + c]}, mc[3] = {m[c], m[3 + c], m[6 + c]}, x[3];
            cross3(rc, mc, x);
            for (int k = 0; k < 3; k++) axis[k] += x[k];
            denom += dot3(rc, mc);
        }
        double sc = fabs(denom) + 2.220446049250313e-16;
        double aa[3] = {axis[0] / sc, axis[1] / sc, axis[2] / sc};
        double angle = norm3(aa);
        if (!(angle > eps)) break;
        double u[3] = {aa[0] / angle, aa[1] / angle, aa[2] / angle};
        double s = sin(angle), c = cos(angle), omc = 1.0 - c;
        double Q[9] = {u[0] * u[0] + (1 - u[0] * u[0]) * c, u[0] * u[1] * omc - u[2] * s, u[0] * u[2] * omc + u[1] * s,
                       u[0] * u[1] * omc + u[2] * s, u[1] * u[1] + (1 - u[1] * u[1]) * c, u[1] * u[2] * omc - u[0] * s,
                       u[0] * u[2] * omc - u[1] * s, u[1] * u[2] * omc + u[0] * s, u[2] * u[2] + (1 - u[2] * u[2]) * c};
        mat3_mul(Q, R, R);
    }
    memcpy(rot, R, sizeof(R));
}

/* lambda-twist/src/lib.rs:110-317: samples = 3 x (bearing xyz, world homogeneous xyzw); out: <= 4 WorldToCamera */
int ref_p3p(const double *bearings, const double *world, ref_pose out[4]) {
    double wp[3][3];
    for (int i = 0; i < 3; i++) {
        const double *w = world + 4 * i;
        if (w[3] == 0.0) return 0; /* Projective::point() -> None */
        for (int k = 0; k < 3; k++) wp[i][k] = w[k] / w[3];
    }
    const double *y1 = bearings, *y2 = bearings + 3, *y3 = bearings + 6;
    double d12[3], d13[3], d23[3], d12xd13[3];
    for (int k = 0; k < 3; k++) { d12[k] = wp[0][k] - wp[1][k]; d13[k] = wp[0][k] - wp[2][k]; d23[k] = wp[1][k] - wp[2][k]; }
    cross3(d12, d13, d12xd13);
    double a12 = dot3(d12, d12), a13 = dot3(d13, d13), a23 = dot3(d23, d23);
    double c12 = dot3(y1, y2), c23 = dot3(y2, y3), c31 = dot3(y3, y1);
    double blob = c12 * c23 * c31 - 1.0;
    double s12_sqr = 1.0 - c12 * c12, s23_sqr = 1.0 - c23 * c23, s31_sqr = 1.0 - c31 * c31;
    double b12 = -2.0 * c12, b13 = -2.0 * c31, b23 = -2.0 * c23;
    double p3 = a13 * (a23 * s31_sqr - a13 * s23_sqr);
    double p2 = 2.0 * blob * a23 * a13 + a13 * (2.0 * a12 + a13) * s23_sqr + a23 * (a23 - a12) * s31_sqr;
    double p1 = a23 * (a13 - a23) * s12_sqr - a12 * a12 * s23_sqr - 2.0 * a12 * (blob * a23 + a13 * s23_sqr);
    double p0 = a12 * (a12 * s23_sqr - a23 * s12_sqr);
    double g = cube_root(p2 / p3, p1 / p3, p0 / p3);
    double d0_00 = a23 * (1.0 - g), d0_01 = -(a23 * c12), d0_02 = a23 * c31 * g, d0_11 = a23 - a12 + a13 * g;
    double d0_12 = -c23 * (a13 * g - a12), d0_22 = g * (a13 - a23) - a12;
    double D0[9] = {d0_00, d0_01, d0_02, d0_01, d0_11, d0_12, d0_02, d0_12, d0_22}, Ev[9], ev[3];
    eigen_decomposition_singular(D0, Ev, ev);
    double lambdas[4][3];
    int nl = 0;
    double eigen_ratio = sqrt(fmax(0.0, -ev[1] / ev[0]));
    for (int sgn = 0; sgn < 2; sgn++) {
        double ratio = sgn ? -eigen_ratio : eigen_ratio;
        /* m11 = Ev[0], m12 = Ev[1], m21 = Ev[3], m22 = Ev[4], m31 = Ev[6], m32 = Ev[7] */
        double w2 = 1.0 / (ratio * Ev[1] - Ev[0]);
        double w0 = w2 * (Ev[3] - ratio * Ev[4]);
        double w1 = w2 * (Ev[6] - ratio * Ev[7]);
        double a = 1.0 / ((a13 - a12) * w1 * w1 - a12 * b13 * w1 - a12);
        double b = a * (a13 * b12 * w1 - a12 * b13 * w0 - 2.0 * w0 * w1 * (a12 - a13));
        double c = a * ((a13 - a12) * w0 * w0 + a13 * b12 * w0 + a13);
        if (b * b - 4.0 * c >= 0.0) {
            double tau[2];
            root2real(b, c, &tau[0], &tau[1]);
            for (int k = 0; k < 2; k++) {
                if (tau[k] > 0.0) {
                    double d = a23 / (tau[k] * (b23 + tau[k]) + 1.0);
                    if (d > 0.0) {
                        double l2 = sqrt(d), l3 = tau[k] * l2, l1 = w0 * l2 + w1 * l3;
                        if (l1 >= 0.0 && nl < 4) { lambdas[nl][0] = l1; lambdas[nl][1] = l2; lambdas[nl][2] = l3; nl++; }
                    }
                }
            }
        }
    }
    double X[9] = {d12[0], d13[0], d12xd13[0], d12[1], d13[1], d12xd13[1], d12[2], d13[2], d12xd13[2]}, Xi[9];
    if (!inv3(X, Xi)) return 0;
    for (int s = 0; s < nl; s++) {
        double l[3] = {lambdas[s][0], lambdas[s][1], lambdas[s][2]};
        gauss_newton_refine_lambda(l, 5, a12, a13, a23, b12, b13, b23);
        double ry1[3], ry2[3], ry3[3], yd1[3], yd2[3], yx[3];
        for (int k = 0; k < 3; k++) { ry1[k] = l[0] * y1[k]; ry2[k] = l[1] * y2[k]; ry3[k] = l[2] * y3[k]; }
        for (int k = 0; k < 3; k++) { yd1[k] = ry1[k] - ry2[k]; yd2[k] = ry1[k] - ry3[k]; }
        cross3(yd1, yd2, yx);
        double Y[9] = {yd1[0], yd2[0], yx[0], yd1[1], yd2[1], yx[1], yd1[2], yd2[2], yx[2]}, rot[9];
        mat3_mul(Y, Xi, rot);
        for (int k = 0; k < 3; k++) out[s].t[k] = ry1[k] - dot3(rot + 3 * k, wp[0]);
        rotation_from_matrix_eps(rot, 1e-12, 100, out[s].R);
    }
    return nl;
}

/* exported for the tests that mirror nister-stewenius/src/lib.rs:368-417 (o1_manual, o2_manual) */
void ref_fp_o1(const double *a, const double *b, double *r) { fp_o1(a, b, r); }
void ref_fp_o2(const double *a, const double *b, double *r) { fp_o2(a, b, r); }

/* ------------------------------------------------------------------ triangulation */
/* cv-geom/src/triangulation.rs:82-130: n (pose, bearing) observations -> homogeneous world point; returns 1 = Some */
int ref_triangulate_linear_eigen(const ref_pose *poses, const double *bearings, int n, double *out) {
    if (n < 2) return 0;
    double A[16] = {0}, d[4], V[16];
    for (int i = 0; i < n; i++) design_add(&poses[i], bearings + 3 * i, A);
    if (!ref_sym_eigen(4, A, 1e-12, 1000, d, V)) return 0;
    int best = 0;
    for (int i = 1; i < 4; i++)
        if (d[i] < d[best]) best = i;
    double p[4] = {V[best], V[4 + best], V[8 + best], V[12 + best]};
    from_homogeneous(p);
    for (int i = 0; i < 4; i++) if (!isfinite(p[i])) return 0;
    for (int i = 0; i < n; i++) { /* cheirality: (R^-1 b) . p_bearing must be sign-positive */
        const double *b = bearings + 3 * i, *R = poses[i].R;
        double wb[3] = {R[0] * b[0] + R[3] * b[1] + R[6] * b[2], R[1] * b[0] + R[4] * b[1] + R[7] * b[2], R[2] * b[0] + R[5] * b[1] + R[8] * b[2]};
        if (signbit(dot3(wb, p))) return 0;
    }
    memcpy(out, p, sizeof(p));
    return 1;
}

/* cv-pinhole/src/lib.rs:108-116 calibrate: pixel -> unit bearing */
void ref_calibrate(double fx, double fy, double cx, double cy, double skew, double px, double py, double *bearing) {
    double y = (py - cy) / fy;
    double x = (px - cx - skew * y) / fx;
    double n = sqrt(x * x + y * y + 1.0);
    bearing[0] = x / n; bearing[1] = y / n; bearing[2] = 1.0 / n;
}

/* ------------------------------------------------------------------ RNGs */
static uint64_t rotl64(uint64_t x, int k) { return (x << k) | (x >> (64 - k)); }
void ref_rng_seed_xoshiro(ref_rng *r, uint64_t seed) { /* rand_xoshiro seed_from_u64: SplitMix64 */
    r->kind = 0;
    for (int i = 0; i < 4; i++) {
        seed += 0x9e3779b97f4a7c15ull;
        uint64_t z = seed;
        z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
        z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
        r->s[i] = z ^ (z >> 31);
    }
}
void ref_rng_seed_pcg64(ref_rng *r, const uint8_t seed[32]) { /* rand_pcg::Pcg64::from_seed */
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
uint32_t ref_rng_next_u32(ref_rng *r) {
    if (r->kind == 0) { /* xoshiro256++ ; next_u32 = upper half of next_u64 */
        uint64_t *s = r->s;
        uint64_t result = rotl64(s[0] + s[3], 23) + s[0];
        uint64_t t = s[1] << 17;
        s[2] ^= s[0]; s[3] ^= s[1]; s[1] ^= s[2]; s[0] ^= s[3]; s[2] ^= t; s[3] = rotl64(s[3], 45);
        return (uint32_t)(result >> 32);
    }
    unsigned __int128 state = (unsigned __int128)r->s[0] | ((unsigned __int128)r->s[1] << 64);
    unsigned __int128 incr = (unsigned __int128)r->s[2] | ((unsigned __int128)r->s[3] << 64);
    const unsigned __int128 MUL = ((unsigned __int128)0x2360ED051FC65DA4ull << 64) | 0x4385DF649FCCF645ull;
    state = state * MUL + incr;
    r->s[0] = (uint64_t)state; r->s[1] = (uint64_t)(state >> 64);
    uint32_t rot = (uint32_t)(state >> 122);
    uint64_t xsl = (uint64_t)(state >> 64) ^ (uint64_t)state;
    uint64_t out = (xsl >> rot) | (xsl << ((64 - rot) & 63));
    return (uint32_t)out;
}

/* ------------------------------------------------------------------ ARRSAC (restated; parity unpinned, see header) */
void ref_arrsac_default_cfg(ref_arrsac_cfg *c, double inlier_threshold) {
    c->inlier_threshold = inlier_threshold;
    c->initialization_hypotheses = 256; c->initialization_blocks = 4; c->max_candidate_hypotheses = 64;
    c->estimations_per_block = 64; c->block_size = 64;
    c->likelihood_ratio_threshold = 1e3f; c->initial_epsilon = 0.1f; c->initial_delta = 0.05f;
}

typedef struct { ref_pose m; uint32_t inliers; } hyp_t;
typedef struct { hyp_t *v; size_t n, cap; } hyp_vec;
static void hv_push(hyp_vec *h, const ref_pose *m, uint32_t inl) {
    if (h->n == h->cap) { h->cap = h->cap ? h->cap * 2 : 256; h->v = (hyp_t *)realloc(h->v, h->cap * sizeof(hyp_t)); }
    h->v[h->n].m = *m; h->v[h->n].inliers = inl; h->n++;
}
/* stable sort by inliers descending */
static void hv_sort(hyp_vec *h) {
    for (size_t i = 1; i < h->n; i++) {
        hyp_t x = h->v[i];
        size_t j = i;
        while (j > 0 && h->v[j - 1].inliers < x.inliers) { h->v[j] = h->v[j - 1]; j--; }
        h->v[j] = x;
    }
}

/* kind: 0 = EightPoint over FeatureMatch (a, b: n x 3 each), 1 = LambdaTwist over FeatureWorldMatch (a = bearings n x 3,
 * b = world n x 4), 2 = NisterStewenius over FeatureMatch */
static double model_residual(int kind, const ref_pose *m, const double *a, const double *b, uint32_t i) {
    return kind != 1 ? ref_residual_c2c(m, a + 3 * (size_t)i, b + 3 * (size_t)i) : ref_residual_w2c(m, a + 3 * (size_t)i, b + 4 * (size_t)i);
}
static int model_estimate(int kind, const double *a, const double *b, const uint32_t *idx, ref_pose *out) {
    if (kind == 2) { /* NisterStewenius over FeatureMatch: 5 samples, up to 40 poses */
        double sa[15], sb[15];
        for (int k = 0; k < 5; k++) { memcpy(sa + 3 * k, a + 3 * (size_t)idx[k], 24); memcpy(sb + 3 * k, b + 3 * (size_t)idx[k], 24); }
        return ref_five_point(sa, sb, out);
    }
    if (kind == 0) {
        double sa[24], sb[24];
        for (int k = 0; k < 8; k++) { memcpy(sa + 3 * k, a + 3 * (size_t)idx[k], 24); memcpy(sb + 3 * k, b + 3 * (size_t)idx[k], 24); }
        return ref_eight_point(sa, sb, out);
    }
    double sa[9], sb[12];
    for (int k = 0; k < 3; k++) { memcpy(sa + 3 * k, a + 3 * (size_t)idx[k], 24); memcpy(sb + 4 * k, b + 4 * (size_t)idx[k], 32); }
    return ref_p3p(sa, sb, out);
}
/* MIN_SAMPLES distinct indices: next_u32() % len with rejection of repeats */
static void populate_samples(ref_rng *rng, uint32_t k, uint32_t len, uint32_t *out) {
    for (uint32_t c = 0; c < k;) {
        uint32_t s = ref_rng_next_u32(rng) % len;
        int dup = 0;
        for (uint32_t j = 0; j < c; j++) dup |= out[j] == s;
        if (!dup) out[c++] = s;
    }
}

int ref_arrsac(const ref_arrsac_cfg *cfg, int kind, const double *a, const double *b, uint32_t n, ref_rng *rng,
               ref_pose *model_out, uint32_t *inliers_out, uint32_t *n_inliers) {
    const uint32_t K = kind == 0 ? 8 : (kind == 1 ? 3 : 5);
    *n_inliers = 0;
    if (n < K) return 0;
    const double thr = cfg->inlier_threshold;
    hyp_vec H = {0};
    /* ---- initialisation: hypotheses from random minimal samples, adaptive SPRT on the first blocks */
    float epsilon = cfg->initial_epsilon, delta = cfg->initial_delta;
    const uint32_t init_n = (uint32_t)(cfg->block_size * cfg->initialization_blocks) < n ? cfg->block_size * cfg->initialization_blocks : n;
    uint32_t best_inliers = 0;
    uint64_t rej_inliers = 0, rej_tested = 0;
    uint32_t idx[8];
    ref_pose models[40];
    for (uint32_t h = 0; h < cfg->initialization_hypotheses; h++) {
        populate_samples(rng, K, n, idx);
        int nm = model_estimate(kind, a, b, idx, models);
        for (int m = 0; m < nm; m++) {
            const float pos = delta / epsilon, neg = (1.0f - delta) / (1.0f - epsilon);
            float ratio = 1.0f;
            uint32_t inl = 0, tested = 0;
            int pass = 1;
            for (uint32_t i = 0; i < init_n; i++) {
                tested++;
                if (model_residual(kind, &models[m], a, b, i) < thr) { inl++; ratio *= pos; }
                else ratio *= neg;
                if (ratio > cfg->likelihood_ratio_threshold) { pass = 0; break; }
            }
            if (pass) {
                hv_push(&H, &models[m], inl);
                if (inl > best_inliers) {
                    best_inliers = inl;
                    float e = (float)inl / (float)init_n;
                    if (e > epsilon && e < 1.0f) epsilon = e; else if (e >= 1.0f) epsilon = 0.999f;
                }
            } else {
                rej_inliers += inl; rej_tested += tested;
                float d = (float)rej_inliers / (float)rej_tested;
                if (d > 0.0f && d < epsilon) delta = d;
            }
        }
    }
    hv_sort(&H);
    if (H.n > cfg->max_candidate_hypotheses) H.n = cfg->max_candidate_hypotheses;
    /* ---- main loop over further blocks of data */
    uint32_t *pool = (uint32_t *)malloc(sizeof(uint32_t) * (size_t)n);
    for (uint32_t start = init_n; start < n && H.n > 1; start += cfg->block_size) {
        uint32_t end = start + cfg->block_size < n ? start + cfg->block_size : n;
        /* (the per-hypothesis counts are independent: OpenMP over hypotheses does not change any result) */
#pragma omp parallel for schedule(dynamic, 4)
        for (size_t h = 0; h < H.n; h++)
            for (uint32_t i = start; i < end; i++)
                if (model_residual(kind, &H.v[h].m, a, b, i) < thr) H.v[h].inliers++;
        hv_sort(&H);
        size_t keep = H.n / 2 > 1 ? H.n / 2 : 1;
        H.n = keep;
        /* new hypotheses from the inliers (so far) of the current best */
        uint32_t np = 0;
        for (uint32_t i = 0; i < end; i++)
            if (model_residual(kind, &H.v[0].m, a, b, i) < thr) pool[np++] = i;
        if (np >= K) {
            const uint32_t worst = H.v[H.n - 1].inliers;   /* bar a new hypothesis has to beat */
            const uint32_t G = cfg->estimations_per_block;
            /* the draws are sequential; estimation and scoring of the G samples are independent of each other */
            uint32_t *gidx = (uint32_t *)malloc(sizeof(uint32_t) * 8 * (size_t)(G ? G : 1));
            ref_pose *gm = (ref_pose *)malloc(sizeof(ref_pose) * 40 * (size_t)(G ? G : 1));
            int *gnm = (int *)malloc(sizeof(int) * (size_t)(G ? G : 1));
            uint32_t *ginl = (uint32_t *)malloc(sizeof(uint32_t) * 40 * (size_t)(G ? G : 1));
            for (uint32_t g = 0; g < G; g++) {
                uint32_t loc[8];
                populate_samples(rng, K, np, loc);
                for (uint32_t k = 0; k < K; k++) gidx[8 * (size_t)g + k] = pool[loc[k]];
            }
#pragma omp parallel for schedule(dynamic, 1)
            for (uint32_t g = 0; g < G; g++) {
                gnm[g] = model_estimate(kind, a, b, gidx + 8 * (size_t)g, gm + 40 * (size_t)g);
                for (int m = 0; m < gnm[g]; m++) {
                    uint32_t inl = 0;
                    for (uint32_t i = 0; i < end; i++)
                        if (model_residual(kind, &gm[40 * (size_t)g + m], a, b, i) < thr) inl++;
                    ginl[40 * (size_t)g + m] = inl;
                }
            }
            for (uint32_t g = 0; g < G; g++)
                for (int m = 0; m < gnm[g]; m++)
                    if (ginl[40 * (size_t)g + m] > worst) hv_push(&H, &gm[40 * (size_t)g + m], ginl[40 * (size_t)g + m]);
            free(gidx); free(gm); free(gnm); free(ginl);
            hv_sort(&H);
            if (H.n > cfg->max_candidate_hypotheses) H.n = cfg->max_candidate_hypotheses;
        }
    }
    free(pool);
    if (H.n == 0) { free(H.v); return 0; }
    hv_sort(&H);
    *model_out = H.v[0].m;
    uint32_t c = 0;
    for (uint32_t i = 0; i < n; i++)
        if (model_residual(kind, model_out, a, b, i) < thr) { if (inliers_out) inliers_out[c] = i; c++; }
    *n_inliers = c;
    free(H.v);
    return 1;
}
