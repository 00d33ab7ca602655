// cv_b200/csrc/register_abi.cu -- libcvb200_register.so, the module that exports the C ABI of include/cvb200_register.h (cv-sfm's frame
// registration).  The kernels (register_dev.cuh) and their driver live in geom.cu inside libcvb200.so; this module only gives them their C
// names, so that libcvb200.so's own exports stay exactly those of cvb200.h, cvb200_sfm.h and cvb200_tri.h.  It links libcvb200.so (rpath
// $ORIGIN) and takes that library's contexts.
#include "../../include/cvb200_register.h"

void register_cfg_default(cvb_register_cfg *c);
int register_check(uint32_t V, const uint32_t *vo, const uint32_t *vl, uint32_t L, const uint32_t *lo, const uint32_t *obs,
                   const uint32_t *view_matches, uint32_t H);
int register_frame_dev(cvb_ctx *ctx, const cvb_register_cfg *cfg, const cvb_triangulator *tri, const cvb_arrsac_cfg *arrsac, cvb_rng *rng,
                       uint32_t V, const cvb_pose *poses_dev, const uint32_t *view_off_dev, const uint32_t *view_lm_dev, const double *bear_dev,
                       const uint8_t *desc_dev, uint32_t n_features, uint32_t L, const uint32_t *lm_off_dev, const uint32_t *obs_dev,
                       uint32_t n_obs, const uint8_t *new_desc_dev, const double *new_bear_dev, uint32_t N, const uint32_t *view_matches,
                       uint32_t H, cvb_register_result *res_dev, cvb_register_match *matches_dev, uint32_t *inliers_dev,
                       cvb_register_stats *stats_dev);
int register_frame(cvb_ctx *ctx, const cvb_register_cfg *cfg, const cvb_triangulator *tri, const cvb_arrsac_cfg *arrsac, cvb_rng *rng,
                   uint32_t V, const cvb_pose *poses, const uint32_t *vo, const uint32_t *vl, const double *bear, const uint8_t *desc, uint32_t L,
                   const uint32_t *lo, const uint32_t *obs, const uint8_t *new_desc, const double *new_bear, uint32_t N,
                   const uint32_t *view_matches, uint32_t H, cvb_register_result *res, cvb_register_match *matches, uint32_t *inliers,
                   cvb_register_stats *stats);

extern "C" {

void cvb_register_cfg_default(cvb_register_cfg *cfg) { register_cfg_default(cfg); }

int cvb_register_check(uint32_t V, const uint32_t *view_offsets, const uint32_t *view_landmarks, uint32_t L, const uint32_t *landmark_offsets,
                       const uint32_t *observations, const uint32_t *view_matches, uint32_t H) {
    return register_check(V, view_offsets, view_landmarks, L, landmark_offsets, observations, view_matches, H);
}

int cvb_register_frame_dev(cvb_ctx *ctx, const cvb_register_cfg *cfg, const cvb_triangulator *tri, const cvb_arrsac_cfg *arrsac,
                           cvb_rng *rng, uint32_t V, const cvb_pose *poses_dev, const uint32_t *view_offsets_dev,
                           const uint32_t *view_landmarks_dev, const double *bearings_dev, const uint8_t *descriptors_dev, uint32_t n_features,
                           uint32_t L, const uint32_t *landmark_offsets_dev, const uint32_t *observations_dev, uint32_t n_observations,
                           const uint8_t *new_descriptors_dev, const double *new_bearings_dev, uint32_t N, const uint32_t *view_matches,
                           uint32_t H, cvb_register_result *result_dev, cvb_register_match *matches_dev, uint32_t *inliers_dev,
                           cvb_register_stats *stats_dev) {
    return register_frame_dev(ctx, cfg, tri, arrsac, rng, V, poses_dev, view_offsets_dev, view_landmarks_dev, bearings_dev, descriptors_dev,
                              n_features, L, landmark_offsets_dev, observations_dev, n_observations, new_descriptors_dev, new_bearings_dev, N,
                              view_matches, H, result_dev, matches_dev, inliers_dev, stats_dev);
}

int cvb_register_frame(cvb_ctx *ctx, const cvb_register_cfg *cfg, const cvb_triangulator *tri, const cvb_arrsac_cfg *arrsac, cvb_rng *rng,
                       uint32_t V, const cvb_pose *poses, const uint32_t *view_offsets, const uint32_t *view_landmarks, const double *bearings,
                       const uint8_t *descriptors, uint32_t L, const uint32_t *landmark_offsets, const uint32_t *observations,
                       const uint8_t *new_descriptors, const double *new_bearings, uint32_t N, const uint32_t *view_matches, uint32_t H,
                       cvb_register_result *result, cvb_register_match *matches, uint32_t *inliers,
                       cvb_register_stats *stats) {
    return register_frame(ctx, cfg, tri, arrsac, rng, V, poses, view_offsets, view_landmarks, bearings, descriptors, L, landmark_offsets,
                          observations, new_descriptors, new_bearings, N, view_matches, H, result, matches, inliers, stats);
}

}  // extern "C"
