/* Test infrastructure: a plain C translation unit against include/cvb200_constraints.h that calls EVERY entry point that header declares,
 * so that the prototypes a Rust / cgo / JNI binding transcribes are checked by a C compiler (ctypes never sees the header).
 *   mode 0 (no GPU): the defaults are cv-sfm's, the host validator accepts a well-formed snapshot and refuses a malformed one, context
 *                    creation reports no device, and the entries return CVB_EINVAL for the missing context.
 *   mode 1 (GPU):    a RelativeDlt triangulator and optimization_maximum_landmarks above 512 are CVB_EUNSUPPORTED; a query out of range is
 *                    CVB_EINVAL; a tiny snapshot runs.  (tests/test_gpu_constraints.py holds every result to the oracle.)
 * Build: gcc -std=c11 -Wall -Wextra -Werror abi_smoke_constraints.c -I../../include -L../../cv_b200 -lcvb200_constraints -lcvb200 -lm */
#include <stdio.h>
#include <stdlib.h>
#include "cvb200_constraints.h"

#define CHECK(cond) do { if (!(cond)) { fprintf(stderr, "abi_smoke_constraints: %s:%d: %s\n", __FILE__, __LINE__, #cond); return 1; } } while (0)

int main(int argc, char **argv) {
    const int gpu = argc > 1 && atoi(argv[1]) == 1;
    cvb_constraints_cfg cfg;
    cvb_constraints_cfg_default(&cfg);
    CHECK(cfg.robust_minimum_observations == 3 && cfg.robust_view_num_robust_bearing_pair == 3 &&
          cfg.optimization_robust_covisibility_minimum_landmarks == 16 && cfg.optimization_minimum_landmarks == 24 &&
          cfg.optimization_maximum_landmarks == 64 && cfg.optimization_maximum_three_view_constraints == 64 &&
          cfg.optimization_minimum_new_constraints == 4 && cfg.constraint_patience == 4096);
    CHECK(cfg.robust_observation_incidence_minimum_cosine_distance == 1e-3 && cfg.robust_view_bearing_pair_minimum_cosine_distance == 1e-2);
    /* three views, one landmark seen by all three (feature 0 of each) */
    uint32_t vo[4] = {0, 1, 2, 3}, vl[3] = {0, 0, 0}, lo[2] = {0, 3}, obs[6] = {0, 0, 1, 0, 2, 0}, q[2] = {0, 2};
    CHECK(cvb_view_constraints_check(3, vo, vl, 1, lo, obs, q, 2) == 0);
    obs[3] = 1;   /* feature 1 of view 1 does not exist */
    CHECK(cvb_view_constraints_check(3, vo, vl, 1, lo, obs, q, 2) == CVB_EINVAL);
    obs[3] = 0;
    cvb_triangulator tri;
    cvb_triangulator_default(&tri, CVB_TRI_LINEAR_EIGEN);
    cvb_pose poses[3] = {{{1, 0, 0, 0, 1, 0, 0, 0, 1}, {0, 0, 0}}, {{1, 0, 0, 0, 1, 0, 0, 0, 1}, {-1, 0, 0}}, {{1, 0, 0, 0, 1, 0, 0, 0, 1}, {-2, 0, 0}}};
    double bear[9] = {0, 0, 1, 0, 0, 1, 0, 0, 1};
    static cvb_view_constraint out[2 * 64];
    cvb_view_constraints_result res[2];
    cvb_view_constraints_stats st[2];
    CHECK(cvb_view_constraints(NULL, &cfg, &tri, 3, poses, vo, vl, bear, 1, lo, obs, q, 2, out, res, st) == CVB_EINVAL);
    CHECK(cvb_view_constraints_dev(NULL, &cfg, &tri, 3, poses, vo, vl, bear, 3, 1, lo, obs, 3, q, 2, out, res, st) == CVB_EINVAL);
    CHECK(cvb_three_view_adaptive_optimize_l2_dev(NULL, poses, 1, bear, vo, 1, poses, vo) == CVB_EINVAL);
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
    CHECK(cvb_view_constraints(ctx, &cfg, &dlt, 3, poses, vo, vl, bear, 1, lo, obs, q, 2, out, res, st) == CVB_EUNSUPPORTED);
    cvb_constraints_cfg big = cfg;
    big.optimization_maximum_landmarks = CVB_CONSTRAINTS_MAX_LANDMARKS + 1;
    CHECK(cvb_view_constraints(ctx, &big, &tri, 3, poses, vo, vl, bear, 1, lo, obs, q, 2, out, res, st) == CVB_EUNSUPPORTED);
    q[1] = 3;
    CHECK(cvb_view_constraints(ctx, &cfg, &tri, 3, poses, vo, vl, bear, 1, lo, obs, q, 2, out, res, st) == CVB_EINVAL);
    q[1] = 2;
    CHECK(cvb_view_constraints(ctx, &cfg, &tri, 3, poses, vo, vl, bear, 1, lo, obs, q, 2, out, res, st) == 0);
    CHECK(res[0].n_constraints == 0 && res[0].accepted == 0 && st[0].robust_landmarks == 0);   /* identical bearings: no incidence */
    cvb_ctx_destroy(ctx);
    printf("GPU workflow ok: argument errors refused, a tiny snapshot runs\n");
    return 0;
}
