// cv_b200/csrc/export_abi.cu -- libcvb200_export.so, the module that exports the C ABI of include/cvb200_export.h (cv-sfm's
// reconstruction export).  The kernels (export_dev.cuh) and their drivers live in geom.cu inside libcvb200.so; this module only gives them
// their C names, so that libcvb200.so's own exports stay exactly those of cvb200.h, cvb200_sfm.h and cvb200_tri.h.  It links
// libcvb200.so (rpath $ORIGIN) and takes that library's contexts.
#include "../../include/cvb200_export.h"

void export_cfg_default(cvb_export_cfg *c);
int export_check(uint32_t V, const uint32_t *vo, const uint32_t *vl, uint32_t L, const uint32_t *lo, const uint32_t *obs,
                 const cvb_view_constraint *cons, uint32_t C, uint32_t first_view);
int robust_landmarks_dev(cvb_ctx *ctx, const cvb_export_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses_dev,
                         const uint32_t *view_off_dev, const uint32_t *view_lm_dev, const double *bear_dev, uint32_t n_features, uint32_t L,
                         const uint32_t *lm_off_dev, const uint32_t *obs_dev, uint32_t n_obs, double *points_dev, uint8_t *state_dev);
int robust_landmarks(cvb_ctx *ctx, const cvb_export_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses,
                     const uint32_t *vo, const uint32_t *vl, const double *bear, uint32_t L, const uint32_t *lo, const uint32_t *obs,
                     double *points, uint8_t *state);
int export_reconstruction_dev(cvb_ctx *ctx, const cvb_export_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses_dev,
                              const uint32_t *view_off_dev, const uint32_t *view_lm_dev, const double *bear_dev, const uint8_t *colors_dev,
                              uint32_t n_features, uint32_t L, const uint32_t *lm_off_dev, const uint32_t *obs_dev, uint32_t n_obs,
                              double *points_dev, uint8_t *colors_out_dev, uint32_t *n_points_dev, cvb_export_camera *cameras_dev,
                              double *mean_dev);
int export_reconstruction(cvb_ctx *ctx, const cvb_export_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses,
                          const uint32_t *vo, const uint32_t *vl, const double *bear, const uint8_t *colors, uint32_t L, const uint32_t *lo,
                          const uint32_t *obs, double *points, uint8_t *point_colors, uint32_t *n_points, cvb_export_camera *cameras,
                          double *mean);
int normalize_reconstruction_dev(cvb_ctx *ctx, const cvb_export_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses_dev,
                                 const uint32_t *view_off_dev, const uint32_t *view_lm_dev, const double *bear_dev, uint32_t n_features,
                                 uint32_t L, const uint32_t *lm_off_dev, const uint32_t *obs_dev, uint32_t n_obs,
                                 const cvb_view_constraint *cons_dev, uint32_t C, uint32_t first_view, cvb_pose *poses_out_dev,
                                 cvb_view_constraint *cons_out_dev, cvb_normalize_result *res_dev);
int normalize_reconstruction(cvb_ctx *ctx, const cvb_export_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses,
                             const uint32_t *vo, const uint32_t *vl, const double *bear, uint32_t L, const uint32_t *lo, const uint32_t *obs,
                             const cvb_view_constraint *cons, uint32_t C, uint32_t first_view, cvb_pose *poses_out,
                             cvb_view_constraint *cons_out, cvb_normalize_result *res);

extern "C" {

void cvb_export_cfg_default(cvb_export_cfg *cfg) { export_cfg_default(cfg); }

int cvb_export_check(uint32_t V, const uint32_t *view_offsets, const uint32_t *view_landmarks, uint32_t L, const uint32_t *landmark_offsets,
                     const uint32_t *observations, const cvb_view_constraint *constraints, uint32_t C, uint32_t first_view) {
    return export_check(V, view_offsets, view_landmarks, L, landmark_offsets, observations, constraints, C, first_view);
}

int cvb_robust_landmarks_dev(cvb_ctx *ctx, const cvb_export_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses_dev,
                             const uint32_t *view_offsets_dev, const uint32_t *view_landmarks_dev, const double *bearings_dev,
                             uint32_t n_features, uint32_t L, const uint32_t *landmark_offsets_dev, const uint32_t *observations_dev,
                             uint32_t n_observations, double *points_dev, uint8_t *state_dev) {
    return robust_landmarks_dev(ctx, cfg, tri, V, poses_dev, view_offsets_dev, view_landmarks_dev, bearings_dev, n_features, L,
                                landmark_offsets_dev, observations_dev, n_observations, points_dev, state_dev);
}

int cvb_robust_landmarks(cvb_ctx *ctx, const cvb_export_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses,
                         const uint32_t *view_offsets, const uint32_t *view_landmarks, const double *bearings, uint32_t L,
                         const uint32_t *landmark_offsets, const uint32_t *observations, double *points, uint8_t *state) {
    return robust_landmarks(ctx, cfg, tri, V, poses, view_offsets, view_landmarks, bearings, L, landmark_offsets, observations, points, state);
}

int cvb_export_reconstruction_dev(cvb_ctx *ctx, const cvb_export_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses_dev,
                                  const uint32_t *view_offsets_dev, const uint32_t *view_landmarks_dev, const double *bearings_dev,
                                  const uint8_t *colors_dev, uint32_t n_features, uint32_t L, const uint32_t *landmark_offsets_dev,
                                  const uint32_t *observations_dev, uint32_t n_observations, double *points_dev, uint8_t *point_colors_dev,
                                  uint32_t *n_points_dev, cvb_export_camera *cameras_dev, double *mean_distance_dev) {
    return export_reconstruction_dev(ctx, cfg, tri, V, poses_dev, view_offsets_dev, view_landmarks_dev, bearings_dev, colors_dev, n_features, L,
                                     landmark_offsets_dev, observations_dev, n_observations, points_dev, point_colors_dev, n_points_dev,
                                     cameras_dev, mean_distance_dev);
}

int cvb_export_reconstruction(cvb_ctx *ctx, const cvb_export_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses,
                              const uint32_t *view_offsets, const uint32_t *view_landmarks, const double *bearings, const uint8_t *colors,
                              uint32_t L, const uint32_t *landmark_offsets, const uint32_t *observations, double *points,
                              uint8_t *point_colors, uint32_t *n_points, cvb_export_camera *cameras, double *mean_distance) {
    return export_reconstruction(ctx, cfg, tri, V, poses, view_offsets, view_landmarks, bearings, colors, L, landmark_offsets, observations,
                                 points, point_colors, n_points, cameras, mean_distance);
}

int cvb_normalize_reconstruction_dev(cvb_ctx *ctx, const cvb_export_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses_dev,
                                     const uint32_t *view_offsets_dev, const uint32_t *view_landmarks_dev, const double *bearings_dev,
                                     uint32_t n_features, uint32_t L, const uint32_t *landmark_offsets_dev, const uint32_t *observations_dev,
                                     uint32_t n_observations, const cvb_view_constraint *constraints_dev, uint32_t C, uint32_t first_view,
                                     cvb_pose *poses_out_dev, cvb_view_constraint *constraints_out_dev, cvb_normalize_result *result_dev) {
    return normalize_reconstruction_dev(ctx, cfg, tri, V, poses_dev, view_offsets_dev, view_landmarks_dev, bearings_dev, n_features, L,
                                        landmark_offsets_dev, observations_dev, n_observations, constraints_dev, C, first_view, poses_out_dev,
                                        constraints_out_dev, result_dev);
}

int cvb_normalize_reconstruction(cvb_ctx *ctx, const cvb_export_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses,
                                 const uint32_t *view_offsets, const uint32_t *view_landmarks, const double *bearings, uint32_t L,
                                 const uint32_t *landmark_offsets, const uint32_t *observations, const cvb_view_constraint *constraints,
                                 uint32_t C, uint32_t first_view, cvb_pose *poses_out, cvb_view_constraint *constraints_out,
                                 cvb_normalize_result *result) {
    return normalize_reconstruction(ctx, cfg, tri, V, poses, view_offsets, view_landmarks, bearings, L, landmark_offsets, observations,
                                    constraints, C, first_view, poses_out, constraints_out, result);
}

}  // extern "C"
