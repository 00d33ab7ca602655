/* Test infrastructure: a plain C translation unit against include/cvb200_pinhole.h that calls EVERY entry point that header declares, so
 * that the prototypes a Rust / cgo / JNI binding transcribes are checked by a C compiler (ctypes never sees the header).
 *   mode 0 (no GPU): context creation reports no device; every entry point rejects a null context.
 *   mode 1 (GPU):    bad arguments are rejected with CVB_EINVAL, empty batches are no-ops, an exact match has no reprojection error,
 *                    the essential matrix of a pose is a fixed point of recondition and decomposes back to the pose's rotation.
 * Build: gcc -std=c11 -Wall -Wextra -Werror abi_smoke_pinhole.c -I../../include -L../../cv_b200 -lcvb200_pinhole -lcvb200 -lm */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "cvb200_pinhole.h"

#define CHECK(cond) do { if (!(cond)) { fprintf(stderr, "abi_smoke_pinhole: %s:%d: %s\n", __FILE__, __LINE__, #cond); return 1; } } while (0)

static int no_gpu_checks(void) {
    cvb_ctx *ctx = NULL;
    const int rc = cvb_ctx_create(0, &ctx);
    if (rc == CVB_OK) { cvb_ctx_destroy(ctx); return -1; }      /* a GPU is present: the caller runs mode 1 */
    CHECK(rc == CVB_ENODEV && ctx == NULL);                     /* no CPU fallback */
    cvb_triangulator tri;
    cvb_triangulator_default(&tri, CVB_TRI_LINEAR_EIGEN);
    cvb_pose pose;
    memset(&pose, 0, sizeof(pose));
    double d[64] = {0};
    uint32_t samples[8] = {0}, n = 1;
    int32_t found = 1;
    uint8_t ok[4];
    CHECK(cvb_pose_reprojection_error(NULL, &tri, &pose, 1, d, d, 1, d, d, ok) == CVB_EINVAL);
    CHECK(cvb_pose_reprojection_error_dev(NULL, &tri, &pose, 1, d, d, &n, 1, &found, d, d, ok) == CVB_EINVAL);
    CHECK(cvb_eight_point_essential_batch(NULL, 1e-12, 1000, d, d, 1, samples, 1, d, ok) == CVB_EINVAL);
    CHECK(cvb_residuals_essential(NULL, d, 1, d, d, 1, d) == CVB_EINVAL);
    CHECK(cvb_essential_recondition(NULL, d, 1, 1e-12, 1000, d, ok) == CVB_EINVAL);
    CHECK(cvb_essential_decompose(NULL, d, 1, 1e-12, 1000, d, d, d, ok) == CVB_EINVAL);
    return 0;
}

static void rot_z(double c, double s, double *R) { double r[9] = {c, -s, 0, s, c, 0, 0, 0, 1}; memcpy(R, r, sizeof(r)); }

static int gpu_workflow(void) {
    cvb_ctx *ctx = NULL;
    CHECK(cvb_ctx_create(0, &ctx) == CVB_OK);
    cvb_triangulator tri;
    cvb_triangulator_default(&tri, CVB_TRI_LINEAR_EIGEN);
    cvb_pose pose;
    rot_z(cos(0.1), sin(0.1), pose.r);
    pose.t[0] = 0.5; pose.t[1] = -0.1; pose.t[2] = 0.05;
    /* cv-pinhole/src/lib.rs:291-313: an exact match has no reprojection error */
    enum { N = 12 };
    double a[3 * N], b[3 * N], err[4 * N], avg[N];
    uint8_t ok[N];
    for (int i = 0; i < N; i++) {
        const double X[3] = {-1.0 + 0.2 * i, 0.4 - 0.07 * i, 3.0 + 0.3 * i};
        double Y[3];
        for (int r = 0; r < 3; r++) Y[r] = pose.r[3 * r] * X[0] + pose.r[3 * r + 1] * X[1] + pose.r[3 * r + 2] * X[2] + pose.t[r];
        const double nx = sqrt(X[0] * X[0] + X[1] * X[1] + X[2] * X[2]), ny = sqrt(Y[0] * Y[0] + Y[1] * Y[1] + Y[2] * Y[2]);
        for (int r = 0; r < 3; r++) { a[3 * i + r] = X[r] / nx; b[3 * i + r] = Y[r] / ny; }
    }
    CHECK(cvb_pose_reprojection_error(ctx, &tri, &pose, 1, a, b, N, err, avg, ok) == CVB_OK);
    for (int i = 0; i < N; i++) CHECK(ok[i] == 1 && avg[i] < 1e-9);
    CHECK(cvb_pose_reprojection_error(ctx, &tri, &pose, 1, a, b, N, err, NULL, ok) == CVB_OK);     /* avg_out may be NULL */
    CHECK(cvb_pose_reprojection_error(ctx, &tri, &pose, 0, a, b, 0, err, avg, ok) == CVB_OK);     /* n == 0 */
    CHECK(cvb_pose_reprojection_error(ctx, &tri, &pose, 2, a, b, N, err, avg, ok) == CVB_EINVAL);  /* npose neither 1 nor n */
    CHECK(strlen(cvb_last_error(ctx)) > 0);
    cvb_triangulator bad = tri;
    bad.method = 9;
    CHECK(cvb_pose_reprojection_error(ctx, &bad, &pose, 1, a, b, N, err, avg, ok) == CVB_EINVAL);
    CHECK(cvb_pose_reprojection_error(ctx, &tri, &pose, 1, NULL, b, N, err, avg, ok) == CVB_EINVAL);
    /* the _dev form rejects host-side argument errors before touching device memory */
    CHECK(cvb_pose_reprojection_error_dev(ctx, &tri, NULL, 1, a, b, NULL, 4, NULL, err, avg, ok) == CVB_EINVAL);
    CHECK(cvb_pose_reprojection_error_dev(ctx, &bad, NULL, 1, NULL, NULL, NULL, 4, NULL, NULL, NULL, NULL) == CVB_EINVAL);
    /* the essential matrix of the pose: [t]x R */
    const double *t = pose.t, tx[9] = {0, -t[2], t[1], t[2], 0, -t[0], -t[1], t[0], 0};
    double E[9], Er[9], ra[9], rb[9], tt[3], res[N];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) E[3 * i + j] = tx[3 * i] * pose.r[j] + tx[3 * i + 1] * pose.r[3 + j] + tx[3 * i + 2] * pose.r[6 + j];
    CHECK(cvb_residuals_essential(ctx, E, 1, a, b, N, res) == CVB_OK);
    for (int i = 0; i < N; i++) CHECK(res[i] < 1e-12);
    CHECK(cvb_essential_recondition(ctx, E, 1, 1e-12, 1000, Er, ok) == CVB_OK && ok[0] == 1);
    for (int k = 0; k < 9; k++) CHECK(fabs(Er[k] - E[k]) < 1e-12);
    CHECK(cvb_essential_decompose(ctx, E, 1, 1e-6, 50, ra, rb, tt, ok) == CVB_OK && ok[0] == 1);
    double da = 0, db = 0;
    for (int k = 0; k < 9; k++) { da += fabs(ra[k] - pose.r[k]); db += fabs(rb[k] - pose.r[k]); }
    CHECK(da < 1e-6 || db < 1e-6);
    const double zero[9] = {0};
    CHECK(cvb_essential_decompose(ctx, zero, 1, 1e-12, 1000, ra, rb, tt, ok) == CVB_OK && ok[0] == 0 && isnan(ra[0]) && isnan(tt[2]));
    CHECK(cvb_essential_recondition(ctx, E, 1, 1e-12, 0, Er, ok) == CVB_OK && ok[0] == 0);      /* no sweep: no result */
    uint32_t samples[8] = {0, 1, 2, 3, 4, 5, 6, 7};
    CHECK(cvb_eight_point_essential_batch(ctx, 1e-12, 1000, a, b, N, samples, 1, Er, ok) == CVB_OK && ok[0] == 1);
    CHECK(cvb_residuals_essential(ctx, Er, 1, a, b, N, res) == CVB_OK);
    for (int i = 0; i < N; i++) CHECK(res[i] < 1e-9);
    samples[3] = N;
    CHECK(cvb_eight_point_essential_batch(ctx, 1e-12, 1000, a, b, N, samples, 1, Er, ok) == CVB_EINVAL);   /* index out of range */
    CHECK(cvb_eight_point_essential_batch(ctx, 1e-12, 1000, a, b, N, samples, 0, Er, ok) == CVB_OK);       /* H == 0 */
    cvb_ctx_destroy(ctx);
    printf("GPU workflow ok\n");
    return 0;
}

int main(int argc, char **argv) {
    const int mode = argc > 1 ? atoi(argv[1]) : 0;
    if (mode == 0) {
        const int r = no_gpu_checks();
        if (r > 0) return 1;
        printf(r < 0 ? "GPU present: mode 0 skipped\n" : "no-GPU checks ok\n");
        return 0;
    }
    return gpu_workflow();
}
