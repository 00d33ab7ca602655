/* Test infrastructure: a plain C translation unit against include/cvb200_incorporate.h that calls EVERY entry point that header declares,
 * so that the prototypes a Rust / cgo / JNI binding transcribes are checked by a C compiler (ctypes never sees the header).
 *   mode 0 (no GPU): the host validator accepts a well-formed add_view and apply and refuses broken ones, context creation reports no
 *                    device, and the entries return CVB_EINVAL for the missing context.
 *   mode 1 (GPU):    add_view of one feature matched to a landmark, then the new view removed again, gives the input back; an
 *                    incorporate_frame whose frame cannot reach three candidate landmarks is the register panic, with no snapshot.
 *                    (tests/test_gpu_incorporate.py holds every result to the oracle.)
 * Build: gcc -std=c11 -Wall -Wextra -Werror abi_smoke_incorporate.c -I../../include -L../../cv_b200 -lcvb200_incorporate -lcvb200 -lm */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "cvb200_incorporate.h"

#define CHECK(cond) do { if (!(cond)) { fprintf(stderr, "abi_smoke_incorporate: %s:%d: %s\n", __FILE__, __LINE__, #cond); return 1; } } while (0)

int main(int argc, char **argv) {
    const int gpu = argc > 1 && atoi(argv[1]) == 1;
    /* two views of one landmark (feature 0 of each), and a second landmark seen by view 1 only */
    uint32_t vo[3] = {0, 1, 3}, vl[3] = {0, 0, 1}, lo[3] = {0, 2, 3}, obs[6] = {0, 0, 1, 0, 1, 1}, vm[2] = {0, 1};
    cvb_pose poses[2] = {{{1, 0, 0, 0, 1, 0, 0, 0, 1}, {0, 0, 0}}, {{1, 0, 0, 0, 1, 0, 0, 0, 1}, {-1, 0, 0}}};
    double bear[9] = {0, 0, 1, 0, 0, 1, 0, 0, 1}, new_bear[6] = {0, 0, 1, 0, 0, 1};
    uint8_t desc[3 * 64], new_desc[2 * 64];
    memset(desc, 0, sizeof(desc));
    memset(new_desc, 0, sizeof(new_desc));
    cvb_register_match m[1] = {{1, 0, CVB_REGISTER_NONE}}, bad[1] = {{2, 0, CVB_REGISTER_NONE}}, pair[1] = {{0, 0, 1}};
    uint8_t vs[2] = {0, 0}, os[3] = {0, 0, 0};
    CHECK(cvb_incorporate_check(2, vo, vl, 2, lo, obs, NULL, 0, 2, m, 1, NULL, 0, NULL, 0) == 0);
    CHECK(cvb_incorporate_check(2, vo, vl, 2, lo, obs, NULL, 0, 2, bad, 1, NULL, 0, NULL, 0) == CVB_EINVAL);    /* feature >= N */
    CHECK(cvb_incorporate_check(2, vo, vl, 2, lo, obs, NULL, 0, 2, pair, 1, NULL, 0, NULL, 0) == CVB_EINVAL);   /* a and b share view 1 */
    CHECK(cvb_incorporate_check(2, vo, vl, 2, lo, obs, NULL, 0, 0, NULL, 0, vs, 2, os, 3) == 0);
    CHECK(cvb_incorporate_check(2, vo, vl, 2, lo, obs, NULL, 0, 0, NULL, 0, vs, 1, os, 3) == CVB_EINVAL);
    vs[1] = CVB_RECON_VIEW_NO_EDGES;
    CHECK(cvb_incorporate_check(2, vo, vl, 2, lo, obs, NULL, 0, 0, NULL, 0, vs, 2, os, 3) == CVB_EINVAL);      /* kept obs of a removed view */
    os[1] = os[2] = CVB_RECON_OBS_DROPPED;
    CHECK(cvb_incorporate_check(2, vo, vl, 2, lo, obs, NULL, 0, 0, NULL, 0, vs, 2, os, 3) == 0);
    cvb_register_cfg rcfg;
    cvb_register_cfg_default(&rcfg);
    cvb_constraints_cfg ccfg;
    cvb_constraints_cfg_default(&ccfg);
    cvb_recon_cfg ocfg;
    cvb_recon_cfg_default(&ocfg);
    cvb_triangulator tri;
    cvb_triangulator_default(&tri, CVB_TRI_LINEAR_EIGEN);
    cvb_arrsac_cfg ars;
    cvb_arrsac_default_cfg(&ars, 1e-5);
    cvb_rng rng;
    cvb_rng_seed_xoshiro256pp(&rng, 7);
    /* outputs with the incorporate capacities: V + 1 views, n_features + N rows, L + N + n_obs + N landmarks, n_obs + N observations */
    cvb_pose p_out[3];
    uint32_t vo_out[4], vl_out[5], lo_out[11], obs_out[10], vmap[2], lmap[2];
    double bear_out[15];
    uint8_t desc_out[5 * 64], col_out[15];
    cvb_view_constraint cons_out[64];
    cvb_register_match m_out[2];
    cvb_incorporate_counts cnt;
    cvb_incorporate_result res;
    CHECK(cvb_add_view(NULL, 2, poses, vo, vl, bear, NULL, NULL, 2, lo, obs, poses, new_bear, NULL, NULL, 2, m, 1, p_out, vo_out, vl_out,
                       bear_out, NULL, NULL, lo_out, obs_out, lmap, &cnt) == CVB_EINVAL);
    CHECK(cvb_add_view_dev(NULL, 2, poses, vo, vl, bear, NULL, NULL, 3, 2, lo, obs, 3, poses, new_bear, NULL, NULL, 2, m, 1, p_out, vo_out,
                           vl_out, bear_out, NULL, NULL, lo_out, obs_out, lmap, &cnt) == CVB_EINVAL);
    CHECK(cvb_apply_optimization(NULL, 2, poses, vo, vl, bear, NULL, NULL, 2, lo, obs, NULL, 0, vs, os, p_out, vo_out, vl_out, bear_out, NULL,
                                 NULL, lo_out, obs_out, cons_out, vmap, lmap, &cnt) == CVB_EINVAL);
    CHECK(cvb_apply_optimization_dev(NULL, 2, poses, vo, vl, bear, NULL, NULL, 3, 2, lo, obs, 3, NULL, 0, vs, os, p_out, vo_out, vl_out,
                                     bear_out, NULL, NULL, lo_out, obs_out, cons_out, vmap, lmap, &cnt) == CVB_EINVAL);
    CHECK(cvb_incorporate_frame(NULL, &rcfg, &ccfg, &ocfg, &tri, &ars, &rng, 2, poses, vo, vl, bear, desc, NULL, 2, lo, obs, NULL, 0, new_desc,
                                new_bear, NULL, 2, vm, 2, p_out, vo_out, vl_out, bear_out, desc_out, NULL, lo_out, obs_out, cons_out, vmap, lmap,
                                m_out, &res) == CVB_EINVAL);
    CHECK(cvb_incorporate_frame_dev(NULL, &rcfg, &ccfg, &ocfg, &tri, &ars, &rng, 2, poses, vo, vl, bear, desc, NULL, 3, 2, lo, obs, 3, NULL, 0,
                                    new_desc, new_bear, NULL, 2, vm, 2, p_out, vo_out, vl_out, bear_out, desc_out, NULL, lo_out, obs_out,
                                    cons_out, vmap, lmap, m_out, &res) == CVB_EINVAL);
    (void)col_out;
    cvb_ctx *ctx = NULL;
    int rc = cvb_ctx_create(0, &ctx);
    if (!gpu) {
        CHECK(rc == CVB_ENODEV && ctx == NULL);
        printf("no-device checks ok\n");
        return 0;
    }
    CHECK(rc == 0 && ctx);
    /* add_view: feature 1 joins landmark 0, feature 0 starts landmark 2 */
    CHECK(cvb_add_view(ctx, 2, poses, vo, vl, bear, NULL, NULL, 2, lo, obs, poses, new_bear, NULL, NULL, 2, m, 1, p_out, vo_out, vl_out, bear_out,
                       NULL, NULL, lo_out, obs_out, lmap, &cnt) == 0);
    CHECK(cnt.V == 3 && cnt.n_features == 5 && cnt.L == 3 && cnt.n_observations == 5 && cnt.merges == 0);
    CHECK(vl_out[3] == 2 && vl_out[4] == 0 && lo_out[1] == 3 && obs_out[4] == 2 && obs_out[5] == 1);
    /* remove_view of the new view gives the input back */
    uint32_t vo2[4], vl2[5], lo2[9], obs2[10], vo3[4], vl3[5], lo3[9], obs3[10];
    memcpy(vo2, vo_out, sizeof(vo2)); memcpy(vl2, vl_out, sizeof(vl2)); memcpy(lo2, lo_out, 4 * sizeof(uint32_t)); memcpy(obs2, obs_out, sizeof(obs2));
    double bear2[15];
    memcpy(bear2, bear_out, sizeof(bear2));
    cvb_pose p2[3];
    memcpy(p2, p_out, sizeof(p2));
    uint8_t vs3[3] = {0, 0, CVB_RECON_VIEW_NO_EDGES}, os3[5];
    for (int o = 0; o < 5; o++) os3[o] = obs2[2 * o] == 2 ? CVB_RECON_OBS_DROPPED : CVB_RECON_OBS_KEPT;
    uint32_t vmap3[3], lmap3[3];
    CHECK(cvb_apply_optimization(ctx, 3, p2, vo2, vl2, bear2, NULL, NULL, 3, lo2, obs2, NULL, 0, vs3, os3, p_out, vo3, vl3, bear_out, NULL, NULL,
                                 lo3, obs3, cons_out, vmap3, lmap3, &cnt) == 0);
    CHECK(cnt.V == 2 && cnt.L == 2 && memcmp(vo3, vo, sizeof(vo)) == 0 && memcmp(vl3, vl, sizeof(vl)) == 0 && memcmp(lo3, lo, sizeof(lo)) == 0 &&
          memcmp(obs3, obs, sizeof(obs)) == 0 && vmap3[2] == CVB_INCORPORATE_NONE);
    /* a frame whose features cannot reach three candidate landmarks: the register panic */
    CHECK(cvb_incorporate_frame(ctx, &rcfg, &ccfg, &ocfg, &tri, &ars, &rng, 2, poses, vo, vl, bear, desc, NULL, 2, lo, obs, NULL, 0, new_desc,
                                new_bear, NULL, 2, vm, 2, p_out, vo_out, vl_out, bear_out, desc_out, NULL, lo_out, obs_out, cons_out, vmap, lmap,
                                m_out, &res) == 0);
    CHECK(res.status == CVB_INCORPORATE_REGISTER_PANIC && res.new_view == CVB_INCORPORATE_NONE && res.counts.V == 0 &&
          vmap[0] == CVB_INCORPORATE_NONE && lmap[0] == CVB_INCORPORATE_NONE);
    cvb_triangulator dlt;
    cvb_triangulator_default(&dlt, CVB_TRI_RELATIVE_DLT);
    CHECK(cvb_incorporate_frame(ctx, &rcfg, &ccfg, &ocfg, &dlt, &ars, &rng, 2, poses, vo, vl, bear, desc, NULL, 2, lo, obs, NULL, 0, new_desc,
                                new_bear, NULL, 2, vm, 2, p_out, vo_out, vl_out, bear_out, desc_out, NULL, lo_out, obs_out, cons_out, vmap, lmap,
                                m_out, &res) == CVB_EUNSUPPORTED);
    cvb_ctx_destroy(ctx);
    printf("GPU workflow ok: add_view then remove_view gives the input back, a frame without three candidate landmarks is the register panic\n");
    return 0;
}
