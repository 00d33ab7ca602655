/* Test infrastructure: a plain C translation unit against include/cvb200_merge.h that calls EVERY entry point that header declares, so
 * that the prototypes a Rust / cgo / JNI binding transcribes are checked by a C compiler (ctypes never sees the header).
 *   mode 0 (no GPU): the host validator accepts a well-formed merge and refuses broken ones, context creation reports no device, and the
 *                    entries return CVB_EINVAL for the missing context.
 *   mode 1 (GPU):    moving a two-view reconstruction whose views get no constraints refuses both moved views, one per constraints call,
 *                    and gives the destination back; a merge whose frame cannot reach three candidate landmarks is the register panic.
 *                    (tests/test_gpu_merge.py holds every result to the oracle.)
 * Build: gcc -std=c11 -Wall -Wextra -Werror abi_smoke_merge.c -I../../include -L../../cv_b200 -lcvb200_merge -lcvb200_register
 *        -lcvb200_constraints -lcvb200_reconstruction -lcvb200 -lm */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "cvb200_merge.h"

#define CHECK(cond) do { if (!(cond)) { fprintf(stderr, "abi_smoke_merge: %s:%d: %s\n", __FILE__, __LINE__, #cond); return 1; } } while (0)

int main(int argc, char **argv) {
    const int gpu = argc > 1 && atoi(argv[1]) == 1;
    /* D and S alike: two views of one landmark (feature 0 of each), and a second landmark seen by view 1 only */
    uint32_t vo[3] = {0, 1, 3}, vl[3] = {0, 0, 1}, lo[3] = {0, 2, 3}, obs[6] = {0, 0, 1, 0, 1, 1}, vm[2] = {0, 1};
    cvb_pose poses[2] = {{{1, 0, 0, 0, 1, 0, 0, 0, 1}, {0, 0, 0}}, {{1, 0, 0, 0, 1, 0, 0, 0, 1}, {-1, 0, 0}}};
    cvb_pose wt = {{1, 0, 0, 0, 1, 0, 0, 0, 1}, {0, 0, 0}};
    double bear[9] = {0, 0, 1, 0, 0, 1, 0, 0, 1};
    uint8_t desc[3 * 64];
    memset(desc, 0, sizeof(desc));
    uint32_t lmap[2] = {0, CVB_MERGE_NONE}, dup[2] = {0, 0}, far[2] = {2, CVB_MERGE_NONE};
    CHECK(cvb_merge_check(2, vo, vl, 2, lo, obs, NULL, 0, 2, vo, vl, 2, lo, obs, 1, lmap, 0, 0) == 0);
    CHECK(cvb_merge_check(2, vo, vl, 2, lo, obs, NULL, 0, 2, vo, vl, 2, lo, obs, CVB_MERGE_NONE, lmap, 0, 0) == 0);
    CHECK(cvb_merge_check(2, vo, vl, 2, lo, obs, NULL, 0, 2, vo, vl, 2, lo, obs, 2, lmap, 0, 0) == CVB_EINVAL);      /* view >= V_S */
    CHECK(cvb_merge_check(2, vo, vl, 2, lo, obs, NULL, 0, 2, vo, vl, 2, lo, obs, 1, dup, 0, 0) == CVB_EINVAL);       /* not injective */
    CHECK(cvb_merge_check(2, vo, vl, 2, lo, obs, NULL, 0, 2, vo, vl, 2, lo, obs, 1, far, 0, 0) == CVB_EINVAL);       /* entry >= L_D */
    CHECK(cvb_merge_check(2, vo, vl, 2, lo, obs, NULL, 0, 2, vo, vl, 2, lo, obs, 1, lmap, 1, 0) == CVB_EINVAL);      /* colours */
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
    /* outputs with the merge capacities: V + V_S views, nf + nf_S rows, L + n_obs + 4 nf_S landmarks, n_obs + 2 nf_S observations */
    cvb_pose p_out[4];
    uint32_t vo_out[5], vl_out[6], lo_out[18], obs_out[18], dvmap[2], dlmap[2], svmap[2], slmap[2];
    double bear_out[18];
    uint8_t desc_out[6 * 64];
    cvb_view_constraint cons_out[3 * 64];
    cvb_view_constraints_result cres[2];
    cvb_move_result mres;
    cvb_merge_result res;
    CHECK(cvb_incorporate_reconstruction(NULL, &ccfg, &tri, 2, poses, vo, vl, bear, NULL, NULL, 2, lo, obs, NULL, 0, 2, poses, vo, vl, bear, NULL,
                                         NULL, 2, lo, obs, CVB_MERGE_NONE, &wt, lmap, p_out, vo_out, vl_out, bear_out, NULL, NULL, lo_out, obs_out,
                                         cons_out, svmap, slmap, cres, &mres) == CVB_EINVAL);
    CHECK(cvb_incorporate_reconstruction_dev(NULL, &ccfg, &tri, 2, poses, vo, vl, bear, NULL, NULL, 3, 2, lo, obs, 3, NULL, 0, 2, poses, vo, vl,
                                             bear, NULL, NULL, 3, 2, lo, obs, 3, CVB_MERGE_NONE, &wt, lmap, p_out, vo_out, vl_out, bear_out, NULL,
                                             NULL, lo_out, obs_out, cons_out, svmap, slmap, cres, &mres) == CVB_EINVAL);
    CHECK(cvb_merge_reconstructions(NULL, &rcfg, &ccfg, &ocfg, &tri, &ars, &rng, 2, poses, vo, vl, bear, desc, NULL, 2, lo, obs, NULL, 0, 2, poses,
                                    vo, vl, bear, desc, NULL, 2, lo, obs, 1, vm, 2, p_out, vo_out, vl_out, bear_out, desc_out, NULL, lo_out,
                                    obs_out, cons_out, dvmap, dlmap, svmap, slmap, cres, &res) == CVB_EINVAL);
    CHECK(cvb_merge_reconstructions_dev(NULL, &rcfg, &ccfg, &ocfg, &tri, &ars, &rng, 2, poses, vo, vl, bear, desc, NULL, 3, 2, lo, obs, 3, NULL, 0,
                                        2, poses, vo, vl, bear, desc, NULL, 3, 2, lo, obs, 3, 1, vm, 2, p_out, vo_out, vl_out, bear_out, desc_out,
                                        NULL, lo_out, obs_out, cons_out, dvmap, dlmap, svmap, slmap, cres, &res) == CVB_EINVAL);
    cvb_ctx *ctx = NULL;
    int rc = cvb_ctx_create(0, &ctx);
    if (!gpu) {
        CHECK(rc == CVB_ENODEV && ctx == NULL);
        printf("no-device checks ok\n");
        return 0;
    }
    CHECK(rc == 0 && ctx);
    /* the move: S's landmark 0 joins D's landmark 0, its landmark 1 is created; neither moved view gets a constraint, and with four and
     * then three views both are refused, one per constraints call, which gives D back */
    CHECK(cvb_incorporate_reconstruction(ctx, &ccfg, &tri, 2, poses, vo, vl, bear, NULL, NULL, 2, lo, obs, NULL, 0, 2, poses, vo, vl, bear, NULL,
                                         NULL, 2, lo, obs, CVB_MERGE_NONE, &wt, lmap, p_out, vo_out, vl_out, bear_out, NULL, NULL, lo_out, obs_out,
                                         cons_out, svmap, slmap, cres, &mres) == 0);
    CHECK(mres.moved_views == 2 && mres.refused_views == 2 && mres.created_landmarks == 1 && mres.constraint_calls == 2);
    CHECK(mres.counts.V == 2 && mres.counts.L == 2 && mres.counts.n_observations == 3 && mres.counts.C == 0);
    CHECK(memcmp(vo_out, vo, sizeof(vo)) == 0 && memcmp(vl_out, vl, sizeof(vl)) == 0 && memcmp(lo_out, lo, sizeof(lo)) == 0 &&
          memcmp(obs_out, obs, sizeof(obs)) == 0);
    CHECK(svmap[0] == CVB_MERGE_NONE && svmap[1] == CVB_MERGE_NONE && slmap[0] == 0 && slmap[1] == CVB_MERGE_NONE);
    /* a frame whose features cannot reach three candidate landmarks: the register panic, no snapshot */
    CHECK(cvb_merge_reconstructions(ctx, &rcfg, &ccfg, &ocfg, &tri, &ars, &rng, 2, poses, vo, vl, bear, desc, NULL, 2, lo, obs, NULL, 0, 2, poses,
                                    vo, vl, bear, desc, NULL, 2, lo, obs, 1, vm, 2, p_out, vo_out, vl_out, bear_out, desc_out, NULL, lo_out,
                                    obs_out, cons_out, dvmap, dlmap, svmap, slmap, cres, &res) == 0);
    CHECK(res.status == CVB_MERGE_REGISTER_PANIC && res.dest_view == CVB_MERGE_NONE && res.counts.V == 0 && dvmap[0] == CVB_MERGE_NONE &&
          svmap[1] == CVB_MERGE_NONE);
    cvb_ctx_destroy(ctx);
    printf("GPU workflow ok: two refused moved views give the destination back, a frame without three candidate landmarks is the register panic\n");
    return 0;
}
