// cv_b200/csrc/constraints_abi.cu -- libcvb200_constraints.so, the module that exports the C ABI of include/cvb200_constraints.h
// (cv-sfm's three-view constraints of many views).  The kernels (constraints_dev.cuh, k_three_view_opt_warp) and their driver live in
// geom.cu inside libcvb200.so; this module only gives them their C names, so that libcvb200.so's own exports stay exactly those of
// cvb200.h, cvb200_sfm.h and cvb200_tri.h.  It links libcvb200.so (rpath $ORIGIN) and takes that library's contexts.
#include "../../include/cvb200_constraints.h"

void constraints_cfg_default(cvb_constraints_cfg *c);
int view_constraints_check(uint32_t V, const uint32_t *vo, const uint32_t *vl, uint32_t L, const uint32_t *lo, const uint32_t *obs,
                           const uint32_t *queries, uint32_t Q);
int view_constraints_dev(cvb_ctx *ctx, const cvb_constraints_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses_dev,
                         const uint32_t *view_off_dev, const uint32_t *view_lm_dev, const double *bear_dev, uint32_t n_features, uint32_t L,
                         const uint32_t *lm_off_dev, const uint32_t *obs_dev, uint32_t n_obs, const uint32_t *queries, uint32_t Q,
                         cvb_view_constraint *out_dev, cvb_view_constraints_result *res_dev, cvb_view_constraints_stats *stats_dev);
int view_constraints(cvb_ctx *ctx, const cvb_constraints_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses,
                     const uint32_t *vo, const uint32_t *vl, const double *bear, uint32_t L, const uint32_t *lo, const uint32_t *obs,
                     const uint32_t *queries, uint32_t Q, cvb_view_constraint *out, cvb_view_constraints_result *res,
                     cvb_view_constraints_stats *stats);
int three_view_adaptive_optimize_l2_dev(cvb_ctx *ctx, const cvb_pose *poses_dev, uint32_t B, const double *obs_dev, const uint32_t *offsets_dev,
                                        uint32_t iterations, cvb_pose *poses_out_dev, uint32_t *updates_dev);

extern "C" {

void cvb_constraints_cfg_default(cvb_constraints_cfg *cfg) { constraints_cfg_default(cfg); }

int cvb_view_constraints_check(uint32_t V, const uint32_t *view_offsets, const uint32_t *view_landmarks, uint32_t L,
                               const uint32_t *landmark_offsets, const uint32_t *observations, const uint32_t *queries, uint32_t Q) {
    return view_constraints_check(V, view_offsets, view_landmarks, L, landmark_offsets, observations, queries, Q);
}

int cvb_view_constraints_dev(cvb_ctx *ctx, const cvb_constraints_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses_dev,
                             const uint32_t *view_offsets_dev, const uint32_t *view_landmarks_dev, const double *bearings_dev,
                             uint32_t n_features, uint32_t L, const uint32_t *landmark_offsets_dev, const uint32_t *observations_dev,
                             uint32_t n_observations, const uint32_t *queries, uint32_t Q, cvb_view_constraint *constraints_dev,
                             cvb_view_constraints_result *results_dev, cvb_view_constraints_stats *stats_dev) {
    return view_constraints_dev(ctx, cfg, tri, V, poses_dev, view_offsets_dev, view_landmarks_dev, bearings_dev, n_features, L, landmark_offsets_dev,
                                observations_dev, n_observations, queries, Q, constraints_dev, results_dev, stats_dev);
}

int cvb_view_constraints(cvb_ctx *ctx, const cvb_constraints_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses,
                         const uint32_t *view_offsets, const uint32_t *view_landmarks, const double *bearings, uint32_t L,
                         const uint32_t *landmark_offsets, const uint32_t *observations, const uint32_t *queries, uint32_t Q,
                         cvb_view_constraint *constraints, cvb_view_constraints_result *results, cvb_view_constraints_stats *stats) {
    return view_constraints(ctx, cfg, tri, V, poses, view_offsets, view_landmarks, bearings, L, landmark_offsets, observations, queries, Q,
                            constraints, results, stats);
}

int cvb_three_view_adaptive_optimize_l2_dev(cvb_ctx *ctx, const cvb_pose *poses_dev, uint32_t B, const double *obs_dev,
                                            const uint32_t *offsets_dev, uint32_t iterations, cvb_pose *poses_out_dev, uint32_t *updates_dev) {
    return three_view_adaptive_optimize_l2_dev(ctx, poses_dev, B, obs_dev, offsets_dev, iterations, poses_out_dev, updates_dev);
}

}  // extern "C"
