/* Test infrastructure: a plain C translation unit against include/cvb200_try_init.h that calls EVERY entry point that header declares, so
 * that the prototypes a Rust / cgo / JNI binding transcribes are checked by a C compiler (ctypes never sees the header).
 *   mode 0 (no GPU): the host validator accepts well-formed lists and refuses broken ones, context creation reports no device, and the
 *                    entries return CVB_EINVAL for the missing context.
 *   mode 1 (GPU):    add_reconstruction of three small frames gives the pinned views, landmarks and observations, and try_init without
 *                    options is None with no snapshot.  (tests/test_gpu_try_init.py holds every result to the oracle.)
 * Build: gcc -std=c11 -Wall -Wextra -Werror abi_smoke_try_init.c -I../../include -L../../cv_b200 -lcvb200_try_init -lcvb200 -lm */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "cvb200_try_init.h"

#define CHECK(cond) do { if (!(cond)) { fprintf(stderr, "abi_smoke_try_init: %s:%d: %s\n", __FILE__, __LINE__, #cond); return 1; } } while (0)
#define CAP 4

int main(int argc, char **argv) {
    const int gpu = argc > 1 && atoi(argv[1]) == 1;
    /* three frames of 3, 2 and 3 features; center 0 is matched to feature 0 of both others, center 1 to feature 1 of the first, center
     * 2 to feature 1 of the second; feature 2 of the second is a new landmark */
    uint32_t counts[3] = {3, 2, 3}, comb[3] = {0, 0, 0}, fm[2] = {1, 1}, sm[2] = {2, 1};
    uint32_t dup_f[2] = {1, 0}, dup_c[2] = {0, 1}, far[2] = {3, 1};
    CHECK(cvb_try_init_check(3, 2, 3, 0, 1, 2, comb, 1, fm, 1, sm, 1) == 0);
    CHECK(cvb_try_init_check(3, 2, 3, 0, 1, 2, NULL, 0, NULL, 0, NULL, 0) == 0);
    CHECK(cvb_try_init_check(3, 2, 3, 0, 1, 2, comb, 1, dup_f, 1, sm, 1) == CVB_EINVAL);   /* first feature 0 twice */
    CHECK(cvb_try_init_check(3, 2, 3, 0, 1, 2, comb, 1, dup_c, 1, sm, 1) == CVB_EINVAL);   /* center 0 twice into the first view */
    CHECK(cvb_try_init_check(3, 2, 3, 0, 1, 2, comb, 1, far, 1, sm, 1) == CVB_EINVAL);     /* center feature out of range */
    CHECK(cvb_try_init_check(3, 2, 3, 0, 1, 1, comb, 1, fm, 1, sm, 1) == CVB_EINVAL);      /* two equal frames */
    double bear[3 * CAP * 3];
    uint8_t desc[3 * CAP * 64];
    for (int i = 0; i < 3 * CAP * 3; i++) bear[i] = (i % 3 == 2) ? 1.0 : 0.0;
    for (int i = 0; i < 3 * CAP * 64; i++) desc[i] = (uint8_t)i;
    cvb_init_result ir;
    memset(&ir, 0, sizeof(ir));
    ir.status = CVB_INIT_ACCEPTED;
    ir.n_combined = ir.n_first_matches = ir.n_second_matches = 1;
    for (int k = 0; k < 9; k++) ir.first_pose.r[k] = ir.second_pose.r[k] = k % 4 == 0;
    ir.first_pose.t[0] = 1.0;
    ir.second_pose.t[0] = 2.0;
    cvb_init_cfg icfg;
    cvb_init_cfg_default(&icfg);
    cvb_triangulator tri;
    cvb_triangulator_default(&tri, CVB_TRI_LINEAR_EIGEN);
    cvb_arrsac_cfg ars;
    cvb_arrsac_default_cfg(&ars, 1e-5);
    cvb_rng rng;
    cvb_rng_seed_xoshiro256pp(&rng, 7);
    uint32_t options[1] = {1};
    /* outputs with the capacities of 3 cap rows */
    cvb_pose p_out[3];
    uint32_t vo_out[4], vl_out[3 * CAP], lo_out[3 * CAP + 1], obs_out[2 * 3 * CAP];
    double bear_out[3 * 3 * CAP];
    uint8_t desc_out[3 * CAP * 64];
    cvb_view_constraint cons_out[1];
    cvb_incorporate_counts cnt;
    cvb_try_init_result res;
    CHECK(cvb_add_reconstruction(NULL, desc, counts, bear, NULL, 3, CAP, 0, 1, 2, &ir, comb, fm, sm, p_out, vo_out, vl_out, bear_out, desc_out, NULL,
                                 lo_out, obs_out, cons_out, &cnt) == CVB_EINVAL);
    CHECK(cvb_add_reconstruction_dev(NULL, desc, counts, bear, NULL, 3, CAP, 0, 1, 2, &ir, comb, fm, sm, p_out, vo_out, vl_out, bear_out, desc_out,
                                     NULL, lo_out, obs_out, cons_out, &cnt) == CVB_EINVAL);
    CHECK(cvb_try_init(NULL, &icfg, &tri, &ars, &rng, 24, desc, counts, bear, NULL, 3, CAP, 0, options, 1, p_out, vo_out, vl_out, bear_out, desc_out,
                       NULL, lo_out, obs_out, cons_out, &res) == CVB_EINVAL);
    CHECK(cvb_try_init_dev(NULL, &icfg, &tri, &ars, &rng, 24, desc, counts, bear, NULL, 3, CAP, 0, options, 1, p_out, vo_out, vl_out, bear_out,
                           desc_out, NULL, lo_out, obs_out, cons_out, &res) == CVB_EINVAL);
    cvb_ctx *ctx = NULL;
    int rc = cvb_ctx_create(0, &ctx);
    if (!gpu) {
        CHECK(rc == CVB_ENODEV && ctx == NULL);
        printf("no-device checks ok\n");
        return 0;
    }
    CHECK(rc == 0 && ctx);
    CHECK(cvb_add_reconstruction(ctx, desc, counts, bear, NULL, 3, CAP, 0, 1, 2, &ir, comb, fm, sm, p_out, vo_out, vl_out, bear_out, desc_out, NULL,
                                 lo_out, obs_out, cons_out, &cnt) == 0);
    const uint32_t vo_want[4] = {0, 3, 5, 8}, vl_want[8] = {0, 1, 2, 0, 1, 0, 2, 3}, lo_want[5] = {0, 3, 5, 7, 8};
    const uint32_t obs_want[16] = {0, 0, 1, 0, 2, 0, 0, 1, 1, 1, 0, 2, 2, 1, 2, 2};
    CHECK(cnt.V == 3 && cnt.n_features == 8 && cnt.L == 4 && cnt.n_observations == 8 && cnt.C == 1 && cnt.merges == 0);
    CHECK(memcmp(vo_out, vo_want, sizeof(vo_want)) == 0 && memcmp(vl_out, vl_want, sizeof(vl_want)) == 0 &&
          memcmp(lo_out, lo_want, sizeof(lo_want)) == 0 && memcmp(obs_out, obs_want, sizeof(obs_want)) == 0);
    CHECK(p_out[0].r[0] == 1.0 && p_out[0].t[0] == 0.0 && p_out[1].t[0] == 1.0 && p_out[2].t[0] == 2.0);
    CHECK(cons_out[0].views[0] == 0 && cons_out[0].views[1] == 1 && cons_out[0].views[2] == 2 && cons_out[0].poses[1].t[0] == 2.0);
    CHECK(memcmp(desc_out + 3 * 64, desc + CAP * 64, 64) == 0 && bear_out[3 * 7 + 2] == 1.0);
    /* no options: init_reconstruction is None, nothing is written */
    CHECK(cvb_try_init(ctx, &icfg, &tri, &ars, &rng, 24, desc, counts, bear, NULL, 3, CAP, 0, NULL, 0, p_out, vo_out, vl_out, bear_out, desc_out,
                       NULL, lo_out, obs_out, cons_out, &res) == 0);
    CHECK(res.status == CVB_TRY_INIT_NONE && res.frames[0] == 0 && res.frames[1] == CVB_TRY_INIT_NO_FRAME && res.counts.V == 0);
    cvb_ctx_destroy(ctx);
    printf("GPU workflow ok: add_reconstruction gives the pinned snapshot, try_init without options is None\n");
    return 0;
}
