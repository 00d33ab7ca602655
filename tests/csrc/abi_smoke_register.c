/* Test infrastructure: a plain C translation unit against include/cvb200_register.h that calls EVERY entry point that header declares, so
 * that the prototypes a Rust / cgo / JNI binding transcribes are checked by a C compiler (ctypes never sees the header).
 *   mode 0 (no GPU): the defaults are cv-sfm's, the host validator accepts well-formed inputs and refuses malformed ones, context creation
 *                    reports no device, and the entries return CVB_EINVAL for the missing context.
 *   mode 1 (GPU):    a RelativeDlt triangulator is CVB_EUNSUPPORTED; a view match out of range, a NULL argument and an empty first subset
 *                    are CVB_EINVAL; a tiny
 *                    snapshot whose features cannot reach three candidate landmarks is the reference's panic, and no consensus run is left to commit.
 *                    (tests/test_gpu_register.py holds every result to the oracle.)
 * Build: gcc -std=c11 -Wall -Wextra -Werror abi_smoke_register.c -I../../include -L../../cv_b200 -lcvb200_register -lcvb200 -lm */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "cvb200_register.h"

#define CHECK(cond) do { if (!(cond)) { fprintf(stderr, "abi_smoke_register: %s:%d: %s\n", __FILE__, __LINE__, #cond); return 1; } } while (0)

int main(int argc, char **argv) {
    const int gpu = argc > 1 && atoi(argv[1]) == 1;
    cvb_register_cfg cfg;
    cvb_register_cfg_default(&cfg);
    CHECK(cfg.single_view_match_better_by == 24 && cfg.single_view_initial_features == 8192 && cfg.single_view_minimum_landmarks == 32 &&
          cfg.single_view_optimization_num_matches == 2048 && cfg.single_view_filter_loop_iterations == 5 &&
          cfg.single_view_patience == 100000 && cfg.single_view_optimization_rate == 1e-3 &&
          cfg.single_view_minimum_robust_landmarks == 64 && cfg.maximum_sine_distance == 0.1 && cfg.maximum_cosine_distance == 1e-5 &&
          cfg.robust_minimum_observations == 3 && cfg.robust_observation_incidence_minimum_cosine_distance == 1e-3);
    /* two views of one landmark (feature 0 of each) */
    uint32_t vo[3] = {0, 1, 2}, vl[2] = {0, 0}, lo[2] = {0, 2}, obs[4] = {0, 0, 1, 0}, vm[2] = {0, 1}, bad[1] = {2};
    cvb_pose poses[2] = {{{1, 0, 0, 0, 1, 0, 0, 0, 1}, {0, 0, 0}}, {{1, 0, 0, 0, 1, 0, 0, 0, 1}, {-1, 0, 0}}};
    double bear[6] = {0, 0, 1, 0, 0, 1}, new_bear[3] = {0, 0, 1};
    uint8_t desc[128], new_desc[64];
    memset(desc, 0, sizeof(desc));
    memset(new_desc, 0, sizeof(new_desc));
    CHECK(cvb_register_check(2, vo, vl, 1, lo, obs, vm, 2) == 0);
    CHECK(cvb_register_check(2, vo, vl, 1, lo, obs, bad, 1) == CVB_EINVAL);
    CHECK(cvb_register_check(2, vo, vl, 1, lo, obs, NULL, 1) == CVB_EINVAL);
    vl[1] = 1;
    CHECK(cvb_register_check(2, vo, vl, 1, lo, obs, vm, 2) == CVB_EINVAL);
    vl[1] = 0;
    cvb_triangulator tri;
    cvb_triangulator_default(&tri, CVB_TRI_LINEAR_EIGEN);
    cvb_arrsac_cfg ars;
    cvb_arrsac_default_cfg(&ars, 1e-5);
    cvb_rng rng;
    cvb_rng_seed_xoshiro256pp(&rng, 7);
    cvb_register_result res;
    cvb_register_match matches[1];
    uint32_t inl[1];
    cvb_register_stats stats;
    CHECK(cvb_register_frame(NULL, &cfg, &tri, &ars, &rng, 2, poses, vo, vl, bear, desc, 1, lo, obs, new_desc, new_bear, 1, vm, 2, &res, matches,
                             inl, &stats) == CVB_EINVAL);
    CHECK(cvb_register_frame_dev(NULL, &cfg, &tri, &ars, &rng, 2, poses, vo, vl, bear, desc, 2, 1, lo, obs, 2, new_desc, new_bear, 1, vm, 2,
                                 &res, matches, inl, &stats) == CVB_EINVAL);
    cvb_ctx *ctx = NULL;
    int rc = cvb_ctx_create(0, &ctx);
    if (!gpu) {
        CHECK(rc == CVB_ENODEV && ctx == NULL);
        printf("no-device checks ok\n");
        return 0;
    }
    CHECK(rc == 0 && ctx);
    cvb_triangulator dlt;
    cvb_triangulator_default(&dlt, CVB_TRI_RELATIVE_DLT);
    CHECK(cvb_register_frame(ctx, &cfg, &dlt, &ars, &rng, 2, poses, vo, vl, bear, desc, 1, lo, obs, new_desc, new_bear, 1, vm, 2, &res, matches,
                             NULL, NULL) == CVB_EUNSUPPORTED);
    CHECK(cvb_register_frame(ctx, &cfg, &tri, &ars, &rng, 2, poses, vo, vl, bear, desc, 1, lo, obs, new_desc, new_bear, 1, bad, 1, &res, matches,
                             NULL, NULL) == CVB_EINVAL);
    CHECK(cvb_register_frame(ctx, &cfg, &tri, NULL, &rng, 2, poses, vo, vl, bear, desc, 1, lo, obs, new_desc, new_bear, 1, vm, 2, &res, matches,
                             NULL, NULL) == CVB_EINVAL);
    cfg.single_view_initial_features = 0;   /* the reference's subset loop would never end */
    CHECK(cvb_register_frame(ctx, &cfg, &tri, &ars, &rng, 2, poses, vo, vl, bear, desc, 1, lo, obs, new_desc, new_bear, 1, vm, 2, &res, matches,
                             inl, NULL) == CVB_EINVAL);
    cfg.single_view_initial_features = 8192;
    const cvb_rng before = rng;
    CHECK(cvb_register_frame(ctx, &cfg, &tri, &ars, &rng, 2, poses, vo, vl, bear, desc, 1, lo, obs, new_desc, new_bear, 1, vm, 2, &res, matches,
                             inl, &stats) == 0);
    CHECK(res.status == CVB_REGISTER_PANIC && res.n_matches == 0 && res.n_inliers == 0 && stats.subsets == 1 && memcmp(&before, &rng, sizeof(rng)) == 0);
    CHECK(cvb_arrsac_commit_rng(ctx, &rng, NULL) == CVB_EINVAL);   /* the call left no consensus run pending */
    cvb_ctx_destroy(ctx);
    printf("GPU workflow ok: argument errors refused, a frame without three candidate landmarks is the reference's panic\n");
    return 0;
}
