/* Test infrastructure: a plain C translation unit against include/cvb200_init.h that calls EVERY entry point that header declares, so
 * that the prototypes a Rust / cgo / JNI binding transcribes are checked by a C compiler (ctypes never sees the header).
 *   mode 0 (no GPU): the defaults are cv-sfm's, context creation reports no device, and the entry returns CVB_EINVAL for the missing
 *                    context.
 *   mode 1 (GPU):    a RelativeDlt triangulator and F above the maximum are CVB_EUNSUPPORTED; cap = 0, a NULL bearing array and an
 *                    option frame out of range are CVB_EINVAL.  (tests/test_gpu_init.py holds every result to the oracle.)
 * Build: gcc -std=c11 -Wall -Wextra -Werror abi_smoke_init.c -I../../include -L../../cv_b200 -lcvb200_init -lcvb200 -lm */
#include <stdio.h>
#include <stdlib.h>
#include "cvb200_init.h"

#define CHECK(cond) do { if (!(cond)) { fprintf(stderr, "abi_smoke_init: %s:%d: %s\n", __FILE__, __LINE__, #cond); return 1; } } while (0)

int main(int argc, char **argv) {
    const int gpu = argc > 1 && atoi(argv[1]) == 1;
    cvb_init_cfg cfg;
    cvb_init_cfg_default(&cfg);
    CHECK(cfg.two_view_minimum_robust_matches == 256 && cfg.three_view_minimum_relative_scales == 16 &&
          cfg.three_view_optimization_landmarks == 1024 && cfg.robust_view_num_robust_bearing_pair == 3 &&
          cfg.three_view_filter_loop_iterations == 8 && cfg.three_view_patience == 65536 && cfg.three_view_minimum_robust_matches == 32);
    CHECK(cfg.robust_observation_incidence_minimum_cosine_distance == 1e-3 && cfg.robust_view_bearing_pair_minimum_cosine_distance == 1e-2 &&
          cfg.maximum_cosine_distance == 1e-5 && cfg.maximum_sine_distance == 1e-1);
    cvb_triangulator tri;
    cvb_triangulator_default(&tri, CVB_TRI_LINEAR_EIGEN);
    uint32_t opts[2] = {1, 2};
    CHECK(cvb_init_reconstruction_dev(NULL, &cfg, &tri, NULL, 3, 8, 0, opts, 2, NULL, NULL, NULL, NULL, NULL, NULL, NULL, NULL, NULL, NULL,
                                      NULL) == CVB_EINVAL);
    cvb_ctx *ctx = NULL;
    int rc = cvb_ctx_create(0, &ctx);
    if (!gpu) {
        CHECK(rc == CVB_ENODEV && ctx == NULL);
        printf("no-device checks ok\n");
        return 0;
    }
    CHECK(rc == 0 && ctx);
    /* argument errors are refused before anything touches the (here host) buffers */
    enum { FR = 3, CAP = 8 };
    static double bear[FR * CAP * 3];
    static uint32_t pairs[2 * CAP * 2], npairs[2], inl[2 * CAP], ninl[2], comb[CAP * 3], fm[CAP * 2], sm[CAP * 2];
    static int32_t found[2];
    static cvb_pose model[2];
    static cvb_init_result res;
    static cvb_init_pair_stats stats[1];
    cvb_triangulator dlt;
    cvb_triangulator_default(&dlt, CVB_TRI_RELATIVE_DLT);
    CHECK(cvb_init_reconstruction_dev(ctx, &cfg, &dlt, bear, FR, CAP, 0, opts, 2, pairs, npairs, model, inl, ninl, found, &res, comb, fm, sm,
                                      stats) == CVB_EUNSUPPORTED);
    CHECK(cvb_init_reconstruction_dev(ctx, &cfg, &tri, bear, FR, 0, 0, opts, 2, pairs, npairs, model, inl, ninl, found, &res, comb, fm, sm,
                                      stats) == CVB_EINVAL);
    CHECK(cvb_init_reconstruction_dev(ctx, &cfg, &tri, bear, FR, CAP, 0, opts, CVB_ARRSAC_BATCH_MAX + 1, pairs, npairs, model, inl, ninl,
                                      found, &res, comb, fm, sm, stats) == CVB_EUNSUPPORTED);
    CHECK(cvb_init_reconstruction_dev(ctx, &cfg, &tri, NULL, FR, CAP, 0, opts, 2, pairs, npairs, model, inl, ninl, found, &res, comb, fm, sm,
                                      stats) == CVB_EINVAL);
    opts[1] = FR;
    CHECK(cvb_init_reconstruction_dev(ctx, &cfg, &tri, bear, FR, CAP, 0, opts, 2, pairs, npairs, model, inl, ninl, found, &res, comb, fm, sm,
                                      stats) == CVB_EINVAL);
    cvb_ctx_destroy(ctx);
    printf("GPU workflow ok: argument errors refused\n");
    return 0;
}
