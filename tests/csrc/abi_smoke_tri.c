/* Test infrastructure: a plain C translation unit against include/cvb200_tri.h that calls EVERY entry point that header declares, so
 * that the prototypes a Rust / cgo / JNI binding transcribes are checked by a C compiler (ctypes never sees the header).
 *   mode 0 (no GPU): context creation reports no device; every entry point rejects a null context; the defaults are the reference's.
 *   mode 1 (GPU):    bad arguments are rejected with CVB_EINVAL; every method recovers the doc-tests' point (0.3, 0.1, 2.0).
 * Build: gcc -std=c11 -Wall -Wextra -Werror abi_smoke_tri.c -I../../include -L../../cv_b200 -lcvb200 -lm */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "cvb200_tri.h"

#define CHECK(cond) do { if (!(cond)) { fprintf(stderr, "abi_smoke_tri: %s:%d: %s\n", __FILE__, __LINE__, #cond); return 1; } } while (0)

static int defaults(void) {
    cvb_triangulator t;
    cvb_triangulator_default(&t, CVB_TRI_SINE_L1);
    CHECK(t.method == CVB_TRI_SINE_L1 && t.epsilon == 1e-12 && t.max_iterations == 1000 && t.optimization_rate == 1.0);
    cvb_triangulator_default(&t, CVB_TRI_RELATIVE_DLT);
    CHECK(t.method == CVB_TRI_RELATIVE_DLT && t.epsilon == 1e-12 && t.max_iterations == 1000);
    cvb_triangulator_default(&t, CVB_TRI_LINEAR_EIGEN);
    CHECK(t.method == CVB_TRI_LINEAR_EIGEN && t.epsilon == 1e-12 && t.max_iterations == 1000);
    cvb_triangulator_default(NULL, CVB_TRI_MEAN_MEAN);   /* a null configuration is ignored */
    return 0;
}

static int no_gpu_checks(void) {
    cvb_ctx *ctx = NULL;
    const int rc = cvb_ctx_create(0, &ctx);
    if (rc == CVB_OK) { cvb_ctx_destroy(ctx); return -1; }      /* a GPU is present: the caller runs mode 1 */
    CHECK(rc == CVB_ENODEV && ctx == NULL);                     /* no CPU fallback */
    cvb_triangulator t;
    cvb_triangulator_default(&t, CVB_TRI_SINE_L1);
    cvb_pose pose;
    memset(&pose, 0, sizeof(pose));
    double d[16] = {0};
    uint32_t off[2] = {0, 1};
    uint8_t ok[2];
    CHECK(cvb_triangulate_observations(NULL, &t, &pose, d, off, 1, d, ok) == CVB_EINVAL);
    CHECK(cvb_triangulate_relative(NULL, &t, &pose, 1, d, d, 1, d, ok) == CVB_EINVAL);
    CHECK(cvb_observation_losses_tri(NULL, &t, &pose, d, off, 1, d) == CVB_EINVAL);
    CHECK(cvb_tri_landmarks_robust_tri(NULL, &t, &pose, &pose, d, 1, 1e-5, 1e-3, ok) == CVB_EINVAL);
    return 0;
}

static void rodrigues(const double *v, double *R) {
    const double th = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]), k[3] = {v[0] / th, v[1] / th, v[2] / th};
    const double s = sin(th), c = 1.0 - cos(th);
    const double K[9] = {0, -k[2], k[1], k[2], 0, -k[0], -k[1], k[0], 0};
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            double kk = 0;
            for (int m = 0; m < 3; m++) kk += K[3 * i + m] * K[3 * m + j];
            R[3 * i + j] = (i == j ? 1.0 : 0.0) + s * K[3 * i + j] + c * kk;
        }
}

static int gpu_workflow(void) {
    cvb_ctx *ctx = NULL;
    CHECK(cvb_ctx_create(0, &ctx) == CVB_OK);
    /* the doc-tests' scene (cv-geom/src/triangulation.rs:26-38): camera A at the origin, B = A moved by (0.1, 0.1, 0.1), exp([0.1]^3) */
    cvb_pose rel, obs[2];
    const double v[3] = {0.1, 0.1, 0.1}, X[3] = {0.3, 0.1, 2.0};
    rodrigues(v, rel.r);
    rel.t[0] = rel.t[1] = rel.t[2] = 0.1;
    double a[3], b[3], na = 0, nb = 0, B[6], xyzw[4 * 2];
    for (int i = 0; i < 3; i++) { a[i] = X[i]; b[i] = rel.r[3 * i] * X[0] + rel.r[3 * i + 1] * X[1] + rel.r[3 * i + 2] * X[2] + rel.t[i]; }
    for (int i = 0; i < 3; i++) { na += a[i] * a[i]; nb += b[i] * b[i]; }
    for (int i = 0; i < 3; i++) { a[i] /= sqrt(na); b[i] /= sqrt(nb); B[i] = a[i]; B[3 + i] = b[i]; }
    memset(&obs[0], 0, sizeof(cvb_pose));
    obs[0].r[0] = obs[0].r[4] = obs[0].r[8] = 1.0;
    obs[1] = rel;
    uint8_t ok[2];
    cvb_triangulator t;
    for (int m = CVB_TRI_LINEAR_EIGEN; m <= CVB_TRI_ANGULAR_LINF; m++) {
        cvb_triangulator_default(&t, m);
        CHECK(cvb_triangulate_relative(ctx, &t, &rel, 1, a, b, 1, xyzw, ok) == CVB_OK && ok[0] == 1);
        const double tol = m == CVB_TRI_MEAN_MEAN ? 1e-2 : 1e-6;
        double e = 0;
        for (int i = 0; i < 3; i++) e += (xyzw[i] / xyzw[3] - X[i]) * (xyzw[i] / xyzw[3] - X[i]);
        CHECK(sqrt(e) < tol);
        if (m <= CVB_TRI_MEAN_MEAN) {
            const uint32_t off[3] = {0, 2, 2};
            CHECK(cvb_triangulate_observations(ctx, &t, obs, B, off, 2, xyzw, ok) == CVB_OK && ok[0] == 1 && ok[1] == 0);
            double loss[2];
            CHECK(cvb_observation_losses_tri(ctx, &t, obs, B, off, 1, loss) == CVB_OK);
        }
    }
    /* bad arguments */
    const uint32_t bad_off[3] = {0, 2, 1};
    cvb_triangulator_default(&t, CVB_TRI_ANGULAR_L1);
    CHECK(cvb_triangulate_observations(ctx, &t, obs, B, bad_off, 1, xyzw, ok) == CVB_EINVAL);      /* relative-only method */
    CHECK(strlen(cvb_last_error(ctx)) > 0);
    double obs9[9] = {0};
    CHECK(cvb_tri_landmarks_robust_tri(ctx, &t, &rel, &rel, obs9, 1, 1e-5, 1e-3, ok) == CVB_EINVAL);
    t.method = 6;
    CHECK(cvb_triangulate_relative(ctx, &t, &rel, 1, a, b, 1, xyzw, ok) == CVB_EINVAL);          /* unknown method */
    CHECK(cvb_triangulate_relative(ctx, NULL, &rel, 1, a, b, 1, xyzw, ok) == CVB_EINVAL);        /* null configuration */
    cvb_triangulator_default(&t, CVB_TRI_MEAN_MEAN);
    CHECK(cvb_triangulate_observations(ctx, &t, obs, B, bad_off, 2, xyzw, ok) == CVB_EINVAL);     /* offsets not monotone */
    double a2[6] = {a[0], a[1], a[2], a[0], a[1], a[2]}, b2[6] = {b[0], b[1], b[2], b[0], b[1], b[2]};
    CHECK(cvb_triangulate_relative(ctx, &t, obs, 2, a2, b2, 3, xyzw, ok) == CVB_EINVAL);          /* npose neither 1 nor n */
    CHECK(cvb_triangulate_relative(ctx, &t, obs, 2, a2, b2, 2, xyzw, ok) == CVB_OK);
    cvb_ctx_destroy(ctx);
    printf("GPU workflow ok\n");
    return 0;
}

int main(int argc, char **argv) {
    const int mode = argc > 1 ? atoi(argv[1]) : 0;
    if (defaults()) return 1;
    if (mode == 0) {
        const int r = no_gpu_checks();
        if (r > 0) return 1;
        printf(r < 0 ? "GPU present: mode 0 skipped\n" : "no-GPU checks ok\n");
        return 0;
    }
    return gpu_workflow();
}
