/* Test infrastructure: a plain C translation unit against include/cvb200_opt.h that calls EVERY entry point that header declares, so
 * that the prototypes a Rust / cgo / JNI binding transcribes are checked by a C compiler (ctypes never sees the header).
 *   mode 0 (no GPU): context creation reports no device; every entry point rejects a null context.
 *   mode 1 (GPU):    bad arguments are rejected with CVB_EINVAL, B == 0 is a no-op, an exact pose stays put, an empty problem returns
 *                    its input pose bit for bit.
 * Build: gcc -std=c11 -Wall -Wextra -Werror abi_smoke_opt.c -I../../include -L../../cv_b200 -lcvb200_opt -lcvb200 -lm */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "cvb200_opt.h"

#define CHECK(cond) do { if (!(cond)) { fprintf(stderr, "abi_smoke_opt: %s:%d: %s\n", __FILE__, __LINE__, #cond); return 1; } } while (0)

static int no_gpu_checks(void) {
    cvb_ctx *ctx = NULL;
    const int rc = cvb_ctx_create(0, &ctx);
    if (rc == CVB_OK) { cvb_ctx_destroy(ctx); return -1; }      /* a GPU is present: the caller runs mode 1 */
    CHECK(rc == CVB_ENODEV && ctx == NULL);                     /* no CPU fallback */
    cvb_pose pose[2];
    memset(pose, 0, sizeof(pose));
    double d[16] = {0};
    uint32_t off[2] = {0, 1}, upd[1];
    CHECK(cvb_single_view_optimize_l1(NULL, pose, 1, 1e-12, 0.1, 10, d, d, off, pose, upd) == CVB_EINVAL);
    CHECK(cvb_three_view_optimize_l1(NULL, pose, 1, 1e-12, 0.1, 10, d, off, pose, NULL) == CVB_EINVAL);
    return 0;
}

static int gpu_workflow(void) {
    cvb_ctx *ctx = NULL;
    CHECK(cvb_ctx_create(0, &ctx) == CVB_OK);
    /* pose (I, (0.5, 0, 0)); landmarks exactly on their bearings */
    cvb_pose pose, out[2];
    memset(&pose, 0, sizeof(pose));
    pose.r[0] = pose.r[4] = pose.r[8] = 1.0;
    pose.t[0] = 0.5;
    enum { N = 40 };
    double bearings[3 * N], world[4 * N];
    for (int i = 0; i < N; i++) {
        const double c[3] = {-1.0 + 0.05 * i, 0.5 - 0.025 * i, 2.0 + 0.1 * i}, n = sqrt(c[0] * c[0] + c[1] * c[1] + c[2] * c[2]);
        for (int k = 0; k < 3; k++) { bearings[3 * i + k] = c[k] / n; world[4 * i + k] = c[k] - pose.t[k]; }
        world[4 * i + 3] = 1.0;
    }
    const uint32_t off[3] = {0, N, N};
    uint32_t upd[2];
    cvb_pose in[2] = {pose, pose};
    in[1].t[1] = 0.25;
    CHECK(cvb_single_view_optimize_l1(ctx, in, 2, 1e-12, 1e-3, 20, bearings, world, off, out, upd) == CVB_OK);
    CHECK(upd[0] == 20 && upd[1] == 0);
    for (int k = 0; k < 3; k++) CHECK(fabs(out[0].t[k] - pose.t[k]) < 1e-9);
    CHECK(memcmp(&out[1], &in[1], sizeof(cvb_pose)) == 0);                                       /* no landmarks: untouched */
    CHECK(cvb_single_view_optimize_l1(ctx, in, 1, 1e-12, 1e-3, 20, bearings, world, off, out, NULL) == CVB_OK);
    CHECK(cvb_single_view_optimize_l1(ctx, in, 0, 1e-12, 1e-3, 20, NULL, NULL, NULL, NULL, NULL) == CVB_OK);   /* B == 0 */
    /* bad arguments */
    const uint32_t bad_off[3] = {0, 2, 1};
    CHECK(cvb_single_view_optimize_l1(ctx, in, 2, 1e-12, 1e-3, 20, bearings, world, bad_off, out, upd) == CVB_EINVAL);
    CHECK(strlen(cvb_last_error(ctx)) > 0);
    CHECK(cvb_single_view_optimize_l1(ctx, in, 1, 1e-12, 1e-3, 20, NULL, world, off, out, upd) == CVB_EINVAL);
    CHECK(cvb_single_view_optimize_l1(ctx, NULL, 1, 1e-12, 1e-3, 20, bearings, world, off, out, upd) == CVB_EINVAL);
    double obs[9] = {0, 0, 1, 0, 0, 1, 0, 0, 1};
    cvb_pose pair[2] = {pose, pose};
    const uint32_t off1[2] = {0, 1}, off0[2] = {0, 0}, bad1[2] = {1, 0};
    CHECK(cvb_three_view_optimize_l1(ctx, pair, 1, 1e-12, 0.1, 5, NULL, off1, out, upd) == CVB_EINVAL);
    CHECK(cvb_three_view_optimize_l1(ctx, pair, 1, 1e-12, 0.1, 5, obs, bad1, out, upd) == CVB_EINVAL);
    CHECK(cvb_three_view_optimize_l1(ctx, pair, 1, 1e-12, 0.1, 5, obs, off1, out, upd) == CVB_OK);
    CHECK(cvb_three_view_optimize_l1(ctx, pair, 1, 1e-12, 0.1, 5, NULL, off0, out, upd) == CVB_OK && upd[0] == 0);
    CHECK(memcmp(out, pair, sizeof(pair)) == 0);                                                 /* no double inversion */
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
