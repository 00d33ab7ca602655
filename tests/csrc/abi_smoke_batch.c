/* Test infrastructure: a plain C translation unit against include/cvb200_batch.h that calls EVERY entry point that header declares, so
 * that the prototypes a Rust / cgo / JNI binding transcribes are checked by a C compiler (ctypes never sees the header).
 *   mode 0 (no GPU): context creation reports no device, and every entry point returns CVB_EINVAL for the missing context.
 *   mode 1 (GPU):    a host batch of three noiseless two-view problems finds (nearly) every match an inlier of each; B above the maximum is
 *                    CVB_EUNSUPPORTED, B = 0 a no-op, a NULL generator array CVB_EINVAL, and a batch commit without a pending batch
 *                    CVB_EINVAL.  (tests/test_gpu_arrsac_batch.py holds every result to the oracle and to the single calls.)
 * Build: gcc -std=c11 -Wall -Wextra -Werror abi_smoke_batch.c -I../../include -L../../cv_b200 -lcvb200_batch -lcvb200 -lm */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "cvb200_batch.h"

#define CHECK(cond) do { if (!(cond)) { fprintf(stderr, "abi_smoke_batch: %s:%d: %s\n", __FILE__, __LINE__, #cond); return 1; } } while (0)

enum { B = 3, NPER = 200, N = B * NPER };
static double a[N * 3], b[N * 3];
static uint32_t inl[N];

static void unit3(double *v) { const double n = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]); v[0] /= n; v[1] /= n; v[2] /= n; }

static int no_context(void) {
    cvb_arrsac_cfg cfg;
    cvb_arrsac_default_cfg(&cfg, 1e-6);
    cvb_rng rngs[B];
    cvb_pose models[B];
    uint32_t offs[B + 1] = {0, NPER, 2 * NPER, N}, cnt[B], stats[16 * B];
    int32_t found[B];
    CHECK(cvb_arrsac_batch_dev(NULL, &cfg, 0, 5, a, b, NULL, NPER, B, rngs, models, inl, NPER, cnt, found) == CVB_EINVAL);
    CHECK(cvb_arrsac_batch(NULL, &cfg, 0, 5, a, b, offs, B, rngs, models, inl, cnt, found) == CVB_EINVAL);
    CHECK(cvb_arrsac_commit_rng_batch(NULL, rngs, B, stats) == CVB_EINVAL);
    uint32_t opts[2] = {1, 2}, npairs[2];
    CHECK(cvb_two_view_options_dev(NULL, NULL, NULL, NULL, 3, 8, 0, opts, 2, 24, &cfg, rngs, inl, npairs, models, inl, cnt, found) == CVB_EINVAL);
    return 0;
}

int main(int argc, char **argv) {
    const int gpu = argc > 1 && atoi(argv[1]) == 1;
    /* problem p: points in front of camera 1, camera 2 shifted along x by 0.5 + 0.1 p (pure translation) */
    srand(7);
    for (int p = 0; p < B; p++)
        for (int i = 0; i < NPER; i++) {
            double P[3] = {4.0 * rand() / RAND_MAX - 2.0, 4.0 * rand() / RAND_MAX - 2.0, 3.0 + 5.0 * rand() / RAND_MAX};
            double *pa = a + 3 * (p * NPER + i), *pb = b + 3 * (p * NPER + i);
            memcpy(pa, P, sizeof P); unit3(pa);
            pb[0] = P[0] + 0.5 + 0.1 * p; pb[1] = P[1]; pb[2] = P[2]; unit3(pb);
        }
    if (no_context()) return 1;
    cvb_ctx *ctx = NULL;
    int rc = cvb_ctx_create(0, &ctx);
    if (!gpu) {
        CHECK(rc == CVB_ENODEV && ctx == NULL);
        printf("no-device checks ok\n");
        return 0;
    }
    CHECK(rc == 0 && ctx);
    cvb_arrsac_cfg cfg;
    cvb_arrsac_default_cfg(&cfg, 1e-6);
    cvb_rng rngs[B];
    for (int p = 0; p < B; p++) cvb_rng_seed_xoshiro256pp(&rngs[p], 100 + p);
    cvb_pose models[B];
    uint32_t offs[B + 1] = {0, NPER, 2 * NPER, N}, cnt[B], stats[16 * B];
    int32_t found[B];
    CHECK(cvb_arrsac_batch(ctx, &cfg, 0, 5, a, b, offs, B, rngs, models, inl, cnt, found) == 0);
    for (int p = 0; p < B; p++) {
        CHECK(found[p] == 1 && cnt[p] + 2 >= NPER && cnt[p] <= NPER);
        for (uint32_t i = 1; i < cnt[p]; i++) CHECK(inl[offs[p] + i - 1] < inl[offs[p] + i] && inl[offs[p] + i] < NPER);
    }
    CHECK(cvb_arrsac_batch(ctx, &cfg, 0, 5, a, b, offs, CVB_ARRSAC_BATCH_MAX + 1, rngs, models, inl, cnt, found) == CVB_EUNSUPPORTED);
    CHECK(cvb_arrsac_batch(ctx, &cfg, 0, 5, a, b, offs, 0, rngs, models, inl, cnt, found) == 0);
    CHECK(cvb_arrsac_batch(ctx, &cfg, 0, 5, a, b, offs, B, NULL, models, inl, cnt, found) == CVB_EINVAL);
    CHECK(cvb_arrsac_batch_dev(ctx, &cfg, 0, 5, NULL, b, NULL, NPER, B, rngs, models, inl, NPER, cnt, found) == CVB_EINVAL);
    CHECK(cvb_arrsac_commit_rng_batch(ctx, rngs, B, stats) == CVB_EINVAL);      /* nothing pending */
    uint32_t opts[2] = {1, 5}, npairs[2];
    CHECK(cvb_two_view_options_dev(ctx, (const uint8_t *)a, inl, a, 3, 8, 0, opts, 2, 24, &cfg, rngs, inl, npairs, models, inl, cnt, found)
          == CVB_EINVAL);                                                      /* option frame 5 of 3: refused before any launch */
    cvb_ctx_destroy(ctx);
    printf("GPU workflow ok: %d problems, %u inliers each\n", B, cnt[0]);
    return 0;
}
