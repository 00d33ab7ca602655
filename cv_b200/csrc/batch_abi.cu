// cv_b200/csrc/batch_abi.cu -- libcvb200_batch.so, the module that exports the C ABI of include/cvb200_batch.h (B independent ARRSAC
// problems in one set of launches, and cv-sfm's two-view initialisation against F option frames).  The kernels (arrsac_dev.cuh) and their driver live in geom.cu inside libcvb200.so; this module
// only gives them their C names, so that libcvb200.so's own exports stay exactly those of cvb200.h, cvb200_sfm.h and cvb200_tri.h.
// It links libcvb200.so (rpath $ORIGIN) and takes that library's contexts.
#include "../../include/cvb200_batch.h"

int ars_batch_dev(cvb_ctx *ctx, const cvb_arrsac_cfg *cfg, int kind, int row0, const double *a_dev, const double *b_dev, const uint32_t *n_dev,
                  uint32_t n_max, uint32_t B, const cvb_rng *rngs, cvb_pose *model_out_dev, uint32_t *inliers_out_dev, uint32_t cap,
                  uint32_t *n_inliers_dev, int32_t *found_dev);
int ars_batch_host(cvb_ctx *ctx, const cvb_arrsac_cfg *cfg, int kind, int row0, const double *a, const double *b, const uint32_t *offsets,
                   uint32_t B, cvb_rng *rngs, cvb_pose *models_out, uint32_t *inliers_out, uint32_t *n_inliers_out, int32_t *found_out);
int ars_commit_rng_batch(cvb_ctx *ctx, cvb_rng *rngs, uint32_t B, uint32_t *stats_out);
int two_view_options_dev(cvb_ctx *ctx, const uint8_t *desc_dev, const uint32_t *n_dev, const double *bearings_dev, uint32_t frames, uint32_t cap,
                         uint32_t center, const uint32_t *options, uint32_t F, uint32_t better_by, const cvb_arrsac_cfg *cfg, const cvb_rng *rngs,
                         uint32_t *pairs_out_dev, uint32_t *n_pairs_dev, cvb_pose *model_out_dev, uint32_t *inliers_out_dev,
                         uint32_t *n_inliers_dev, int32_t *found_dev);

extern "C" {

int cvb_arrsac_batch_dev(cvb_ctx *ctx, const cvb_arrsac_cfg *cfg, int32_t kind, int32_t eigenvector_row0, const double *a_dev,
                         const double *b_dev, const uint32_t *n_dev, uint32_t n_max, uint32_t B, const cvb_rng *rngs,
                         cvb_pose *model_out_dev, uint32_t *inliers_out_dev, uint32_t cap, uint32_t *n_inliers_dev, int32_t *found_dev) {
    return ars_batch_dev(ctx, cfg, kind, eigenvector_row0, a_dev, b_dev, n_dev, n_max, B, rngs, model_out_dev, inliers_out_dev, cap,
                         n_inliers_dev, found_dev);
}

int cvb_arrsac_batch(cvb_ctx *ctx, const cvb_arrsac_cfg *cfg, int32_t kind, int32_t eigenvector_row0, const double *a, const double *b,
                     const uint32_t *offsets, uint32_t B, cvb_rng *rngs, cvb_pose *models_out, uint32_t *inliers_out,
                     uint32_t *n_inliers_out, int32_t *found_out) {
    return ars_batch_host(ctx, cfg, kind, eigenvector_row0, a, b, offsets, B, rngs, models_out, inliers_out, n_inliers_out, found_out);
}

int cvb_arrsac_commit_rng_batch(cvb_ctx *ctx, cvb_rng *rngs, uint32_t B, uint32_t *stats_out) {
    return ars_commit_rng_batch(ctx, rngs, B, stats_out);
}

int cvb_two_view_options_dev(cvb_ctx *ctx, const uint8_t *desc_dev, const uint32_t *n_dev, const double *bearings_dev, uint32_t frames,
                             uint32_t cap, uint32_t center, const uint32_t *options, uint32_t F, uint32_t better_by, const cvb_arrsac_cfg *cfg,
                             const cvb_rng *rngs, uint32_t *pairs_out_dev, uint32_t *n_pairs_dev, cvb_pose *model_out_dev,
                             uint32_t *inliers_out_dev, uint32_t *n_inliers_dev, int32_t *found_dev) {
    return two_view_options_dev(ctx, desc_dev, n_dev, bearings_dev, frames, cap, center, options, F, better_by, cfg, rngs, pairs_out_dev,
                                n_pairs_dev, model_out_dev, inliers_out_dev, n_inliers_dev, found_dev);
}

}  // extern "C"
