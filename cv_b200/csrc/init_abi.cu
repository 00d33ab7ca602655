// cv_b200/csrc/init_abi.cu -- libcvb200_init.so, the module that exports the C ABI of include/cvb200_init.h (cv-sfm's three-view
// initialisation over the two-view options).  The kernels (init_dev.cuh) and their driver live in geom.cu inside libcvb200.so; this module
// only gives them their C names, so that libcvb200.so's own exports stay exactly those of cvb200.h, cvb200_sfm.h and cvb200_tri.h.
// It links libcvb200.so (rpath $ORIGIN) and takes that library's contexts.
#include "../../include/cvb200_init.h"

void init_cfg_default(cvb_init_cfg *c);
int init_reconstruction_dev(cvb_ctx *ctx, const cvb_init_cfg *cfg, const cvb_triangulator *tri, const double *bearings_dev, uint32_t frames,
                            uint32_t cap, uint32_t center, const uint32_t *options, uint32_t F, const uint32_t *pairs_dev,
                            const uint32_t *n_pairs_dev, const cvb_pose *model_dev, const uint32_t *inliers_dev, const uint32_t *n_inliers_dev,
                            const int32_t *found_dev, cvb_init_result *result_dev, uint32_t *combined_dev, uint32_t *first_matches_dev,
                            uint32_t *second_matches_dev, cvb_init_pair_stats *stats_dev);

extern "C" {

void cvb_init_cfg_default(cvb_init_cfg *cfg) { init_cfg_default(cfg); }

int cvb_init_reconstruction_dev(cvb_ctx *ctx, const cvb_init_cfg *cfg, const cvb_triangulator *tri, const double *bearings_dev, uint32_t frames,
                                uint32_t cap, uint32_t center, const uint32_t *options, uint32_t F, const uint32_t *pairs_dev,
                                const uint32_t *n_pairs_dev, const cvb_pose *model_dev, const uint32_t *inliers_dev,
                                const uint32_t *n_inliers_dev, const int32_t *found_dev, cvb_init_result *result_dev, uint32_t *combined_dev,
                                uint32_t *first_matches_dev, uint32_t *second_matches_dev, cvb_init_pair_stats *stats_dev) {
    return init_reconstruction_dev(ctx, cfg, tri, bearings_dev, frames, cap, center, options, F, pairs_dev, n_pairs_dev, model_dev, inliers_dev,
                                   n_inliers_dev, found_dev, result_dev, combined_dev, first_matches_dev, second_matches_dev, stats_dev);
}

}  // extern "C"
