// cv_b200/csrc/try_init_abi.cu -- libcvb200_try_init.so, the module that exports the C ABI of include/cvb200_try_init.h (cv-sfm's
// reconstruction creation).  The kernels (try_init_dev.cuh) and their drivers live in geom.cu inside libcvb200.so; this module only gives
// them their C names, so that libcvb200.so's own exports stay exactly those of cvb200.h, cvb200_sfm.h and cvb200_tri.h.  It links
// libcvb200.so (rpath $ORIGIN) and takes that library's contexts.
#include "../../include/cvb200_try_init.h"

int try_init_check(uint32_t nc, uint32_t n1, uint32_t n2, uint32_t center, uint32_t first, uint32_t second, const uint32_t *comb, uint32_t K,
                   const uint32_t *fm, uint32_t K1, const uint32_t *sm, uint32_t K2);
int add_reconstruction_dev(cvb_ctx *ctx, const uint8_t *desc, const uint32_t *n, const double *bear, const uint8_t *col, uint32_t frames,
                           uint32_t cap, uint32_t center, uint32_t first, uint32_t second, const cvb_init_result *ir, const uint32_t *comb,
                           const uint32_t *fm, const uint32_t *sm, cvb_pose *poses_out, uint32_t *vo_out, uint32_t *vl_out, double *bear_out,
                           uint8_t *desc_out, uint8_t *col_out, uint32_t *lo_out, uint32_t *obs_out, cvb_view_constraint *cons_out,
                           cvb_incorporate_counts *counts);
int add_reconstruction(cvb_ctx *ctx, const uint8_t *desc, const uint32_t *n, const double *bear, const uint8_t *col, uint32_t frames, uint32_t cap,
                       uint32_t center, uint32_t first, uint32_t second, const cvb_init_result *ir, const uint32_t *comb, const uint32_t *fm,
                       const uint32_t *sm, cvb_pose *poses_out, uint32_t *vo_out, uint32_t *vl_out, double *bear_out, uint8_t *desc_out,
                       uint8_t *col_out, uint32_t *lo_out, uint32_t *obs_out, cvb_view_constraint *cons_out, cvb_incorporate_counts *counts);
int try_init_dev(cvb_ctx *ctx, const cvb_init_cfg *icfg, const cvb_triangulator *tri, const cvb_arrsac_cfg *arrsac, cvb_rng *rngs,
                 uint32_t better_by, const uint8_t *desc, const uint32_t *n, const double *bear, const uint8_t *col, uint32_t frames, uint32_t cap,
                 uint32_t center, const uint32_t *options, uint32_t F, cvb_pose *poses_out, uint32_t *vo_out, uint32_t *vl_out, double *bear_out,
                 uint8_t *desc_out, uint8_t *col_out, uint32_t *lo_out, uint32_t *obs_out, cvb_view_constraint *cons_out,
                 cvb_try_init_result *res_dev);
int try_init(cvb_ctx *ctx, const cvb_init_cfg *icfg, const cvb_triangulator *tri, const cvb_arrsac_cfg *arrsac, cvb_rng *rngs, uint32_t better_by,
             const uint8_t *desc, const uint32_t *n, const double *bear, const uint8_t *col, uint32_t frames, uint32_t cap, uint32_t center,
             const uint32_t *options, uint32_t F, cvb_pose *poses_out, uint32_t *vo_out, uint32_t *vl_out, double *bear_out, uint8_t *desc_out,
             uint8_t *col_out, uint32_t *lo_out, uint32_t *obs_out, cvb_view_constraint *cons_out, cvb_try_init_result *res);

extern "C" {

int cvb_try_init_check(uint32_t n_center, uint32_t n_first, uint32_t n_second, uint32_t center, uint32_t first, uint32_t second,
                       const uint32_t *combined, uint32_t n_combined, const uint32_t *first_matches, uint32_t n_first_matches,
                       const uint32_t *second_matches, uint32_t n_second_matches) {
    return try_init_check(n_center, n_first, n_second, center, first, second, combined, n_combined, first_matches, n_first_matches,
                          second_matches, n_second_matches);
}

int cvb_add_reconstruction_dev(cvb_ctx *ctx, const uint8_t *a0, const uint32_t *a1, const double *a2, const uint8_t *a3, uint32_t a4, uint32_t a5,
                               uint32_t a6, uint32_t a7, uint32_t a8, const cvb_init_result *a9, const uint32_t *a10, const uint32_t *a11,
                               const uint32_t *a12, cvb_pose *a13, uint32_t *a14, uint32_t *a15, double *a16, uint8_t *a17, uint8_t *a18,
                               uint32_t *a19, uint32_t *a20, cvb_view_constraint *a21, cvb_incorporate_counts *a22) {
    return add_reconstruction_dev(ctx, a0, a1, a2, a3, a4, a5, a6, a7, a8, a9, a10, a11, a12, a13, a14, a15, a16, a17, a18, a19, a20, a21, a22);
}

int cvb_add_reconstruction(cvb_ctx *ctx, const uint8_t *a0, const uint32_t *a1, const double *a2, const uint8_t *a3, uint32_t a4, uint32_t a5,
                           uint32_t a6, uint32_t a7, uint32_t a8, const cvb_init_result *a9, const uint32_t *a10, const uint32_t *a11,
                           const uint32_t *a12, cvb_pose *a13, uint32_t *a14, uint32_t *a15, double *a16, uint8_t *a17, uint8_t *a18,
                           uint32_t *a19, uint32_t *a20, cvb_view_constraint *a21, cvb_incorporate_counts *a22) {
    return add_reconstruction(ctx, a0, a1, a2, a3, a4, a5, a6, a7, a8, a9, a10, a11, a12, a13, a14, a15, a16, a17, a18, a19, a20, a21, a22);
}

int cvb_try_init_dev(cvb_ctx *ctx, const cvb_init_cfg *a0, const cvb_triangulator *a1, const cvb_arrsac_cfg *a2, cvb_rng *a3, uint32_t a4,
                     const uint8_t *a5, const uint32_t *a6, const double *a7, const uint8_t *a8, uint32_t a9, uint32_t a10, uint32_t a11,
                     const uint32_t *a12, uint32_t a13, cvb_pose *a14, uint32_t *a15, uint32_t *a16, double *a17, uint8_t *a18, uint8_t *a19,
                     uint32_t *a20, uint32_t *a21, cvb_view_constraint *a22, cvb_try_init_result *a23) {
    return try_init_dev(ctx, a0, a1, a2, a3, a4, a5, a6, a7, a8, a9, a10, a11, a12, a13, a14, a15, a16, a17, a18, a19, a20, a21, a22, a23);
}

int cvb_try_init(cvb_ctx *ctx, const cvb_init_cfg *a0, const cvb_triangulator *a1, const cvb_arrsac_cfg *a2, cvb_rng *a3, uint32_t a4,
                 const uint8_t *a5, const uint32_t *a6, const double *a7, const uint8_t *a8, uint32_t a9, uint32_t a10, uint32_t a11,
                 const uint32_t *a12, uint32_t a13, cvb_pose *a14, uint32_t *a15, uint32_t *a16, double *a17, uint8_t *a18, uint8_t *a19,
                 uint32_t *a20, uint32_t *a21, cvb_view_constraint *a22, cvb_try_init_result *a23) {
    return try_init(ctx, a0, a1, a2, a3, a4, a5, a6, a7, a8, a9, a10, a11, a12, a13, a14, a15, a16, a17, a18, a19, a20, a21, a22, a23);
}

}  // extern "C"
