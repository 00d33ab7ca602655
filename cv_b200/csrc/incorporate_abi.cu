// cv_b200/csrc/incorporate_abi.cu -- libcvb200_incorporate.so, the module that exports the C ABI of include/cvb200_incorporate.h (cv-sfm's
// frame incorporation).  The kernels (incorporate_dev.cuh) and their drivers live in geom.cu inside libcvb200.so; this module only gives
// them their C names, so that libcvb200.so's own exports stay exactly those of cvb200.h, cvb200_sfm.h and cvb200_tri.h.  It links
// libcvb200.so (rpath $ORIGIN) and takes that library's contexts.
#include "../../include/cvb200_incorporate.h"

int incorporate_check(uint32_t V, const uint32_t *vo, const uint32_t *vl, uint32_t L, const uint32_t *lo, const uint32_t *obs,
                      const cvb_view_constraint *cons, uint32_t C, uint32_t N, const cvb_register_match *matches, uint32_t M,
                      const uint8_t *view_state, uint32_t n_view_state, const uint8_t *obs_state, uint32_t n_obs_state);
int add_view_dev(cvb_ctx *ctx, uint32_t V, const cvb_pose *poses_dev, const uint32_t *view_off_dev, const uint32_t *view_lm_dev,
                 const double *bear_dev, const uint8_t *desc_dev, const uint8_t *col_dev, uint32_t nf, uint32_t L, const uint32_t *lm_off_dev,
                 const uint32_t *obs_dev, uint32_t n_obs, const cvb_pose *new_pose_dev, const double *new_bear_dev, const uint8_t *new_desc_dev,
                 const uint8_t *new_col_dev, uint32_t N, const cvb_register_match *matches_dev, uint32_t M, cvb_pose *poses_out,
                 uint32_t *view_off_out, uint32_t *view_lm_out, double *bear_out, uint8_t *desc_out, uint8_t *col_out, uint32_t *lm_off_out,
                 uint32_t *obs_out, uint32_t *lmap, cvb_incorporate_counts *counts);
int add_view(cvb_ctx *ctx, uint32_t V, const cvb_pose *poses, const uint32_t *vo, const uint32_t *vl, const double *bear, const uint8_t *desc,
             const uint8_t *col, uint32_t L, const uint32_t *lo, const uint32_t *obs, const cvb_pose *new_pose, const double *new_bear,
             const uint8_t *new_desc, const uint8_t *new_col, uint32_t N, const cvb_register_match *matches, uint32_t M, cvb_pose *poses_out,
             uint32_t *vo_out, uint32_t *vl_out, double *bear_out, uint8_t *desc_out, uint8_t *col_out, uint32_t *lo_out, uint32_t *obs_out,
             uint32_t *lmap, cvb_incorporate_counts *counts);
int apply_optimization_dev(cvb_ctx *ctx, uint32_t V, const cvb_pose *poses_dev, const uint32_t *view_off_dev, const uint32_t *view_lm_dev,
                           const double *bear_dev, const uint8_t *desc_dev, const uint8_t *col_dev, uint32_t nf, uint32_t L,
                           const uint32_t *lm_off_dev, const uint32_t *obs_dev, uint32_t n_obs, const cvb_view_constraint *cons_dev, uint32_t C,
                           const uint8_t *vstate, const uint8_t *ostate, cvb_pose *poses_out, uint32_t *view_off_out, uint32_t *view_lm_out,
                           double *bear_out, uint8_t *desc_out, uint8_t *col_out, uint32_t *lm_off_out, uint32_t *obs_out,
                           cvb_view_constraint *cons_out, uint32_t *vmap, uint32_t *lmap, cvb_incorporate_counts *counts);
int apply_optimization(cvb_ctx *ctx, uint32_t V, const cvb_pose *poses, const uint32_t *vo, const uint32_t *vl, const double *bear,
                       const uint8_t *desc, const uint8_t *col, uint32_t L, const uint32_t *lo, const uint32_t *obs, const cvb_view_constraint *cons,
                       uint32_t C, const uint8_t *vstate, const uint8_t *ostate, cvb_pose *poses_out, uint32_t *vo_out, uint32_t *vl_out,
                       double *bear_out, uint8_t *desc_out, uint8_t *col_out, uint32_t *lo_out, uint32_t *obs_out, cvb_view_constraint *cons_out,
                       uint32_t *vmap, uint32_t *lmap, cvb_incorporate_counts *counts);
int incorporate_frame_dev(cvb_ctx *ctx, const cvb_register_cfg *rcfg, const cvb_constraints_cfg *ccfg, const cvb_recon_cfg *ocfg,
                          const cvb_triangulator *tri, const cvb_arrsac_cfg *arrsac, cvb_rng *rng, uint32_t V, const cvb_pose *poses_dev,
                          const uint32_t *view_off_dev, const uint32_t *view_lm_dev, const double *bear_dev, const uint8_t *desc_dev,
                          const uint8_t *col_dev, uint32_t nf, uint32_t L, const uint32_t *lm_off_dev, const uint32_t *obs_dev, uint32_t n_obs,
                          const cvb_view_constraint *cons_dev, uint32_t C, const uint8_t *new_desc_dev, const double *new_bear_dev,
                          const uint8_t *new_col_dev, uint32_t N, const uint32_t *view_matches, uint32_t H, cvb_pose *poses_out,
                          uint32_t *view_off_out, uint32_t *view_lm_out, double *bear_out, uint8_t *desc_out, uint8_t *col_out,
                          uint32_t *lm_off_out, uint32_t *obs_out, cvb_view_constraint *cons_out, uint32_t *vmap, uint32_t *lmap,
                          cvb_register_match *matches_out, cvb_incorporate_result *res_dev);
int incorporate_frame(cvb_ctx *ctx, const cvb_register_cfg *rcfg, const cvb_constraints_cfg *ccfg, const cvb_recon_cfg *ocfg,
                      const cvb_triangulator *tri, const cvb_arrsac_cfg *arrsac, cvb_rng *rng, uint32_t V, const cvb_pose *poses, const uint32_t *vo,
                      const uint32_t *vl, const double *bear, const uint8_t *desc, const uint8_t *col, uint32_t L, const uint32_t *lo,
                      const uint32_t *obs, const cvb_view_constraint *cons, uint32_t C, const uint8_t *new_desc, const double *new_bear,
                      const uint8_t *new_col, uint32_t N, const uint32_t *view_matches, uint32_t H, cvb_pose *poses_out, uint32_t *vo_out,
                      uint32_t *vl_out, double *bear_out, uint8_t *desc_out, uint8_t *col_out, uint32_t *lo_out, uint32_t *obs_out,
                      cvb_view_constraint *cons_out, uint32_t *vmap, uint32_t *lmap, cvb_register_match *matches, cvb_incorporate_result *res);

extern "C" {

int cvb_incorporate_check(uint32_t V, const uint32_t *view_offsets, const uint32_t *view_landmarks, uint32_t L, const uint32_t *landmark_offsets,
                          const uint32_t *observations, const cvb_view_constraint *constraints, uint32_t C, uint32_t N,
                          const cvb_register_match *matches, uint32_t M, const uint8_t *view_state, uint32_t n_view_state,
                          const uint8_t *obs_state, uint32_t n_obs_state) {
    return incorporate_check(V, view_offsets, view_landmarks, L, landmark_offsets, observations, constraints, C, N, matches, M, view_state,
                             n_view_state, obs_state, n_obs_state);
}

int cvb_add_view_dev(cvb_ctx *ctx, uint32_t V, const cvb_pose *poses_dev, const uint32_t *view_offsets_dev, const uint32_t *view_landmarks_dev,
                     const double *bearings_dev, const uint8_t *descriptors_dev, const uint8_t *colors_dev, uint32_t n_features, uint32_t L,
                     const uint32_t *landmark_offsets_dev, const uint32_t *observations_dev, uint32_t n_observations, const cvb_pose *new_pose_dev,
                     const double *new_bearings_dev, const uint8_t *new_descriptors_dev, const uint8_t *new_colors_dev, uint32_t N,
                     const cvb_register_match *matches_dev, uint32_t M, cvb_pose *poses_out_dev, uint32_t *view_offsets_out_dev,
                     uint32_t *view_landmarks_out_dev, double *bearings_out_dev, uint8_t *descriptors_out_dev, uint8_t *colors_out_dev,
                     uint32_t *landmark_offsets_out_dev, uint32_t *observations_out_dev, uint32_t *landmark_map_dev,
                     cvb_incorporate_counts *counts_dev) {
    return add_view_dev(ctx, V, poses_dev, view_offsets_dev, view_landmarks_dev, bearings_dev, descriptors_dev, colors_dev, n_features, L,
                        landmark_offsets_dev, observations_dev, n_observations, new_pose_dev, new_bearings_dev, new_descriptors_dev, new_colors_dev,
                        N, matches_dev, M, poses_out_dev, view_offsets_out_dev, view_landmarks_out_dev, bearings_out_dev, descriptors_out_dev,
                        colors_out_dev, landmark_offsets_out_dev, observations_out_dev, landmark_map_dev, counts_dev);
}

int cvb_add_view(cvb_ctx *ctx, uint32_t V, const cvb_pose *poses, const uint32_t *view_offsets, const uint32_t *view_landmarks,
                 const double *bearings, const uint8_t *descriptors, const uint8_t *colors, uint32_t L, const uint32_t *landmark_offsets,
                 const uint32_t *observations, const cvb_pose *new_pose, const double *new_bearings, const uint8_t *new_descriptors,
                 const uint8_t *new_colors, uint32_t N, const cvb_register_match *matches, uint32_t M, cvb_pose *poses_out,
                 uint32_t *view_offsets_out, uint32_t *view_landmarks_out, double *bearings_out, uint8_t *descriptors_out, uint8_t *colors_out,
                 uint32_t *landmark_offsets_out, uint32_t *observations_out, uint32_t *landmark_map, cvb_incorporate_counts *counts) {
    return add_view(ctx, V, poses, view_offsets, view_landmarks, bearings, descriptors, colors, L, landmark_offsets, observations, new_pose,
                    new_bearings, new_descriptors, new_colors, N, matches, M, poses_out, view_offsets_out, view_landmarks_out, bearings_out,
                    descriptors_out, colors_out, landmark_offsets_out, observations_out, landmark_map, counts);
}

int cvb_apply_optimization_dev(cvb_ctx *ctx, uint32_t V, const cvb_pose *poses_dev, const uint32_t *view_offsets_dev,
                               const uint32_t *view_landmarks_dev, const double *bearings_dev, const uint8_t *descriptors_dev,
                               const uint8_t *colors_dev, uint32_t n_features, uint32_t L, const uint32_t *landmark_offsets_dev,
                               const uint32_t *observations_dev, uint32_t n_observations, const cvb_view_constraint *constraints_dev, uint32_t C,
                               const uint8_t *view_state_dev, const uint8_t *obs_state_dev, cvb_pose *poses_out_dev, uint32_t *view_offsets_out_dev,
                               uint32_t *view_landmarks_out_dev, double *bearings_out_dev, uint8_t *descriptors_out_dev, uint8_t *colors_out_dev,
                               uint32_t *landmark_offsets_out_dev, uint32_t *observations_out_dev, cvb_view_constraint *constraints_out_dev,
                               uint32_t *view_map_dev, uint32_t *landmark_map_dev, cvb_incorporate_counts *counts_dev) {
    return apply_optimization_dev(ctx, V, poses_dev, view_offsets_dev, view_landmarks_dev, bearings_dev, descriptors_dev, colors_dev, n_features,
                                  L, landmark_offsets_dev, observations_dev, n_observations, constraints_dev, C, view_state_dev, obs_state_dev,
                                  poses_out_dev, view_offsets_out_dev, view_landmarks_out_dev, bearings_out_dev, descriptors_out_dev,
                                  colors_out_dev, landmark_offsets_out_dev, observations_out_dev, constraints_out_dev, view_map_dev,
                                  landmark_map_dev, counts_dev);
}

int cvb_apply_optimization(cvb_ctx *ctx, uint32_t V, const cvb_pose *poses, const uint32_t *view_offsets, const uint32_t *view_landmarks,
                           const double *bearings, const uint8_t *descriptors, const uint8_t *colors, uint32_t L, const uint32_t *landmark_offsets,
                           const uint32_t *observations, const cvb_view_constraint *constraints, uint32_t C, const uint8_t *view_state,
                           const uint8_t *obs_state, cvb_pose *poses_out, uint32_t *view_offsets_out, uint32_t *view_landmarks_out,
                           double *bearings_out, uint8_t *descriptors_out, uint8_t *colors_out, uint32_t *landmark_offsets_out,
                           uint32_t *observations_out, cvb_view_constraint *constraints_out, uint32_t *view_map, uint32_t *landmark_map,
                           cvb_incorporate_counts *counts) {
    return apply_optimization(ctx, V, poses, view_offsets, view_landmarks, bearings, descriptors, colors, L, landmark_offsets, observations,
                              constraints, C, view_state, obs_state, poses_out, view_offsets_out, view_landmarks_out, bearings_out,
                              descriptors_out, colors_out, landmark_offsets_out, observations_out, constraints_out, view_map, landmark_map,
                              counts);
}

int cvb_incorporate_frame_dev(cvb_ctx *ctx, const cvb_register_cfg *register_cfg, const cvb_constraints_cfg *constraints_cfg,
                              const cvb_recon_cfg *recon_cfg, const cvb_triangulator *tri, const cvb_arrsac_cfg *arrsac, cvb_rng *rng, uint32_t V,
                              const cvb_pose *poses_dev, const uint32_t *view_offsets_dev, const uint32_t *view_landmarks_dev,
                              const double *bearings_dev, const uint8_t *descriptors_dev, const uint8_t *colors_dev, uint32_t n_features,
                              uint32_t L, const uint32_t *landmark_offsets_dev, const uint32_t *observations_dev, uint32_t n_observations,
                              const cvb_view_constraint *constraints_dev, uint32_t C, const uint8_t *new_descriptors_dev,
                              const double *new_bearings_dev, const uint8_t *new_colors_dev, uint32_t N, const uint32_t *view_matches, uint32_t H,
                              cvb_pose *poses_out_dev, uint32_t *view_offsets_out_dev, uint32_t *view_landmarks_out_dev, double *bearings_out_dev,
                              uint8_t *descriptors_out_dev, uint8_t *colors_out_dev, uint32_t *landmark_offsets_out_dev,
                              uint32_t *observations_out_dev, cvb_view_constraint *constraints_out_dev, uint32_t *view_map_dev,
                              uint32_t *landmark_map_dev, cvb_register_match *matches_dev, cvb_incorporate_result *result_dev) {
    return incorporate_frame_dev(ctx, register_cfg, constraints_cfg, recon_cfg, tri, arrsac, rng, V, poses_dev, view_offsets_dev,
                                 view_landmarks_dev, bearings_dev, descriptors_dev, colors_dev, n_features, L, landmark_offsets_dev, observations_dev,
                                 n_observations, constraints_dev, C, new_descriptors_dev, new_bearings_dev, new_colors_dev, N, view_matches, H,
                                 poses_out_dev, view_offsets_out_dev, view_landmarks_out_dev, bearings_out_dev, descriptors_out_dev, colors_out_dev,
                                 landmark_offsets_out_dev, observations_out_dev, constraints_out_dev, view_map_dev, landmark_map_dev, matches_dev,
                                 result_dev);
}

int cvb_incorporate_frame(cvb_ctx *ctx, const cvb_register_cfg *register_cfg, const cvb_constraints_cfg *constraints_cfg,
                          const cvb_recon_cfg *recon_cfg, const cvb_triangulator *tri, const cvb_arrsac_cfg *arrsac, cvb_rng *rng, uint32_t V,
                          const cvb_pose *poses, const uint32_t *view_offsets, const uint32_t *view_landmarks, const double *bearings,
                          const uint8_t *descriptors, const uint8_t *colors, uint32_t L, const uint32_t *landmark_offsets,
                          const uint32_t *observations, const cvb_view_constraint *constraints, uint32_t C, const uint8_t *new_descriptors,
                          const double *new_bearings, const uint8_t *new_colors, uint32_t N, const uint32_t *view_matches, uint32_t H,
                          cvb_pose *poses_out, uint32_t *view_offsets_out, uint32_t *view_landmarks_out, double *bearings_out,
                          uint8_t *descriptors_out, uint8_t *colors_out, uint32_t *landmark_offsets_out, uint32_t *observations_out,
                          cvb_view_constraint *constraints_out, uint32_t *view_map, uint32_t *landmark_map, cvb_register_match *matches,
                          cvb_incorporate_result *result) {
    return incorporate_frame(ctx, register_cfg, constraints_cfg, recon_cfg, tri, arrsac, rng, V, poses, view_offsets, view_landmarks, bearings,
                             descriptors, colors, L, landmark_offsets, observations, constraints, C, new_descriptors, new_bearings, new_colors, N,
                             view_matches, H, poses_out, view_offsets_out, view_landmarks_out, bearings_out, descriptors_out, colors_out,
                             landmark_offsets_out, observations_out, constraints_out, view_map, landmark_map, matches, result);
}

}  // extern "C"
