/* Test infrastructure: a plain C translation unit against include/cvb200_reconstruction.h that calls EVERY entry point that header
 * declares, so that the prototypes a Rust / cgo / JNI binding transcribes are checked by a C compiler (ctypes never sees the header).
 *   mode 0 (no GPU): the defaults are cv-sfm's, the host validator accepts well-formed inputs and refuses malformed ones, context creation
 *                    reports no device, and the entries return CVB_EINVAL for the missing context.
 *   mode 1 (GPU):    a RelativeDlt triangulator is CVB_EUNSUPPORTED; a constraint view out of range is CVB_EINVAL; a tiny reconstruction
 *                    runs.  (tests/test_gpu_reconstruction.py holds every result to the oracle.)
 * Build: gcc -std=c11 -Wall -Wextra -Werror abi_smoke_reconstruction.c -I../../include -L../../cv_b200 -lcvb200_reconstruction -lcvb200 -lm */
#include <stdio.h>
#include <stdlib.h>
#include "cvb200_reconstruction.h"

#define CHECK(cond) do { if (!(cond)) { fprintf(stderr, "abi_smoke_reconstruction: %s:%d: %s\n", __FILE__, __LINE__, #cond); return 1; } } while (0)

int main(int argc, char **argv) {
    const int gpu = argc > 1 && atoi(argv[1]) == 1;
    cvb_recon_cfg cfg;
    cvb_recon_cfg_default(&cfg);
    CHECK(cfg.optimization_iterations == 1024 && cfg.reconstruction_optimization_iterations == 1 && cfg.robust_minimum_observations == 3 &&
          cfg.minimum_robust_landmarks == 32);
    CHECK(cfg.graph_optimization_rate == 0.001 && cfg.maximum_sine_distance == 0.1 && cfg.maximum_cosine_distance == 1e-5 &&
          cfg.robust_observation_incidence_minimum_cosine_distance == 1e-3);
    /* three views, one landmark seen by all three (feature 0 of each), one constraint over them */
    uint32_t vo[4] = {0, 1, 2, 3}, vl[3] = {0, 0, 0}, lo[2] = {0, 3}, obs[6] = {0, 0, 1, 0, 2, 0};
    cvb_pose poses[3] = {{{1, 0, 0, 0, 1, 0, 0, 0, 1}, {0, 0, 0}}, {{1, 0, 0, 0, 1, 0, 0, 0, 1}, {-1, 0, 0}}, {{1, 0, 0, 0, 1, 0, 0, 0, 1}, {-2, 0, 0}}};
    cvb_view_constraint con = {{0, 1, 2}, 0, {poses[1], poses[2]}};
    CHECK(cvb_optimize_reconstruction_check(3, vo, vl, 1, lo, obs, &con, 1) == 0);
    con.views[2] = 3;
    CHECK(cvb_optimize_reconstruction_check(3, vo, vl, 1, lo, obs, &con, 1) == CVB_EINVAL);
    con.views[2] = 1;
    CHECK(cvb_optimize_reconstruction_check(3, vo, vl, 1, lo, obs, &con, 1) == CVB_EINVAL);
    con.views[2] = 2;
    CHECK(cvb_optimize_reconstruction_check(3, vo, vl, 1, lo, obs, NULL, 1) == CVB_EINVAL);
    cvb_triangulator tri;
    cvb_triangulator_default(&tri, CVB_TRI_LINEAR_EIGEN);
    double bear[9] = {0, 0, 1, 0, 0, 1, 0, 0, 1};
    cvb_recon_result res;
    cvb_pose pout[3];
    uint8_t vs[3], os[3];
    CHECK(cvb_optimize_reconstruction(NULL, &cfg, &tri, 3, poses, vo, vl, bear, 1, lo, obs, &con, 1, &res, pout, vs, os) == CVB_EINVAL);
    CHECK(cvb_optimize_reconstruction_dev(NULL, &cfg, &tri, 3, poses, vo, vl, bear, 3, 1, lo, obs, 3, &con, 1, &res, pout, vs, os) == CVB_EINVAL);
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
    CHECK(cvb_optimize_reconstruction(ctx, &cfg, &dlt, 3, poses, vo, vl, bear, 1, lo, obs, &con, 1, &res, pout, vs, os) == CVB_EUNSUPPORTED);
    con.views[0] = 5;
    CHECK(cvb_optimize_reconstruction(ctx, &cfg, &tri, 3, poses, vo, vl, bear, 1, lo, obs, &con, 1, &res, pout, vs, os) == CVB_EINVAL);
    con.views[0] = 0;
    CHECK(cvb_optimize_reconstruction(ctx, &cfg, &tri, 3, poses, vo, vl, bear, 1, lo, obs, &con, 1, &res, pout, vs, os) == 0);
    /* exact constraint at exact poses: a fixed point; identical bearings: no robust landmark, so the filter removes it */
    CHECK(res.status == CVB_RECON_REMOVED_FILTER && res.views_removed == 0 && res.robust_after == 0 && vs[0] == CVB_RECON_VIEW_KEPT);
    cvb_ctx_destroy(ctx);
    printf("GPU workflow ok: argument errors refused, a tiny reconstruction runs\n");
    return 0;
}
