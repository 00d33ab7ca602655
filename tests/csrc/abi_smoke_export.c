/* Test infrastructure: a plain C translation unit against include/cvb200_export.h that calls EVERY entry point that header declares, so
 * that the prototypes a Rust / cgo / JNI binding transcribes are checked by a C compiler (ctypes never sees the header).
 *   mode 0 (no GPU): the defaults are cv-sfm's, the host validator accepts well-formed inputs and refuses malformed ones, context creation
 *                    reports no device, and the entries return CVB_EINVAL for the missing context.
 *   mode 1 (GPU):    a RelativeDlt triangulator is CVB_EUNSUPPORTED; first_view out of range is CVB_EINVAL; a tiny reconstruction is
 *                    triangulated, exported and normalised.  (tests/test_gpu_export.py holds every result to the oracle.)
 * Build: gcc -std=c11 -Wall -Wextra -Werror abi_smoke_export.c -I../../include -L../../cv_b200 -lcvb200_export -lcvb200 -lm */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include "cvb200_export.h"

#define CHECK(cond) do { if (!(cond)) { fprintf(stderr, "abi_smoke_export: %s:%d: %s\n", __FILE__, __LINE__, #cond); return 1; } } while (0)

int main(int argc, char **argv) {
    const int gpu = argc > 1 && atoi(argv[1]) == 1;
    cvb_export_cfg cfg;
    cvb_export_cfg_default(&cfg);
    CHECK(cfg.robust_minimum_observations == 3 && cfg.robust_observation_incidence_minimum_cosine_distance == 1e-3);
    /* three views looking down +z from x = 0, 1, 2; one landmark at (1, 0, 5) seen by all three (feature 0 of each) */
    uint32_t vo[4] = {0, 1, 2, 3}, vl[3] = {0, 0, 0}, lo[2] = {0, 3}, obs[6] = {0, 0, 1, 0, 2, 0};
    cvb_pose poses[3] = {{{1, 0, 0, 0, 1, 0, 0, 0, 1}, {0, 0, 0}}, {{1, 0, 0, 0, 1, 0, 0, 0, 1}, {-1, 0, 0}}, {{1, 0, 0, 0, 1, 0, 0, 0, 1}, {-2, 0, 0}}};
    const double r = sqrt(26.0);
    double bear[9] = {1 / r, 0, 5 / r, 0, 0, 1, -1 / r, 0, 5 / r};
    uint8_t colors[9] = {10, 20, 30, 40, 50, 60, 70, 80, 90};
    cvb_view_constraint con = {{0, 1, 2}, 0, {poses[1], poses[2]}};
    CHECK(cvb_export_check(3, vo, vl, 1, lo, obs, &con, 1, 0) == 0);
    CHECK(cvb_export_check(3, vo, vl, 1, lo, obs, NULL, 0, 2) == 0);
    CHECK(cvb_export_check(3, vo, vl, 1, lo, obs, &con, 1, 3) == CVB_EINVAL);
    con.views[2] = 1;
    CHECK(cvb_export_check(3, vo, vl, 1, lo, obs, &con, 1, 0) == CVB_EINVAL);
    con.views[2] = 2;
    cvb_triangulator tri;
    cvb_triangulator_default(&tri, CVB_TRI_LINEAR_EIGEN);
    double points4[4], points[3], mean[3];
    uint8_t state[1], pcol[3];
    uint32_t n_points = 0;
    cvb_export_camera cams[3];
    cvb_pose pout[3];
    cvb_view_constraint cout[1];
    cvb_normalize_result res;
    CHECK(cvb_robust_landmarks(NULL, &cfg, &tri, 3, poses, vo, vl, bear, 1, lo, obs, points4, state) == CVB_EINVAL);
    CHECK(cvb_robust_landmarks_dev(NULL, &cfg, &tri, 3, poses, vo, vl, bear, 3, 1, lo, obs, 3, points4, state) == CVB_EINVAL);
    CHECK(cvb_export_reconstruction(NULL, &cfg, &tri, 3, poses, vo, vl, bear, colors, 1, lo, obs, points, pcol, &n_points, cams, mean) ==
          CVB_EINVAL);
    CHECK(cvb_export_reconstruction_dev(NULL, &cfg, &tri, 3, poses, vo, vl, bear, colors, 3, 1, lo, obs, 3, points, pcol, &n_points, cams,
                                        mean) == CVB_EINVAL);
    CHECK(cvb_normalize_reconstruction(NULL, &cfg, &tri, 3, poses, vo, vl, bear, 1, lo, obs, &con, 1, 0, pout, cout, &res) == CVB_EINVAL);
    CHECK(cvb_normalize_reconstruction_dev(NULL, &cfg, &tri, 3, poses, vo, vl, bear, 3, 1, lo, obs, 3, &con, 1, 0, pout, cout, &res) ==
          CVB_EINVAL);
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
    CHECK(cvb_robust_landmarks(ctx, &cfg, &dlt, 3, poses, vo, vl, bear, 1, lo, obs, points4, state) == CVB_EUNSUPPORTED);
    CHECK(cvb_normalize_reconstruction(ctx, &cfg, &tri, 3, poses, vo, vl, bear, 1, lo, obs, &con, 1, 3, pout, cout, &res) == CVB_EINVAL);
    CHECK(cvb_robust_landmarks(ctx, &cfg, &tri, 3, poses, vo, vl, bear, 1, lo, obs, points4, state) == 0);
    CHECK(state[0] == CVB_EXPORT_POINT && fabs(points4[0] / points4[3] - 1.0) < 1e-9 && fabs(points4[2] / points4[3] - 5.0) < 1e-9);
    CHECK(cvb_export_reconstruction(ctx, &cfg, &tri, 3, poses, vo, vl, bear, colors, 1, lo, obs, points, pcol, &n_points, cams, mean) == 0);
    CHECK(n_points == 1 && pcol[0] == 10 && fabs(mean[1] - 5.0) < 1e-9 && fabs(cams[2].optical_center[0] - 2.0) < 1e-12);
    CHECK(cvb_normalize_reconstruction(ctx, &cfg, &tri, 3, poses, vo, vl, bear, 1, lo, obs, &con, 1, 1, pout, cout, &res) == 0);
    CHECK(res.normalized == 1 && res.robust_points == 1 && fabs(res.mean_distance - 5.0) < 1e-9 && fabs(pout[0].t[0] - 0.2) < 1e-9);
    cvb_ctx_destroy(ctx);
    printf("GPU workflow ok: argument errors refused, a tiny reconstruction is exported and normalised\n");
    return 0;
}
