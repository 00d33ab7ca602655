// cv_b200/csrc/reconstruction_abi.cu -- libcvb200_reconstruction.so, the module that exports the C ABI of include/cvb200_reconstruction.h
// (cv-sfm's reconstruction optimisation).  The kernels (reconstruction_dev.cuh) and their driver live in geom.cu inside libcvb200.so; this
// module only gives them their C names, so that libcvb200.so's own exports stay exactly those of cvb200.h, cvb200_sfm.h and
// cvb200_tri.h.  It links libcvb200.so (rpath $ORIGIN) and takes that library's contexts.
#include "../../include/cvb200_reconstruction.h"

void recon_cfg_default(cvb_recon_cfg *c);
int optimize_reconstruction_check(uint32_t V, const uint32_t *vo, const uint32_t *vl, uint32_t L, const uint32_t *lo, const uint32_t *obs,
                                  const cvb_view_constraint *cons, uint32_t C);
int optimize_reconstruction_dev(cvb_ctx *ctx, const cvb_recon_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses_dev,
                                const uint32_t *view_off_dev, const uint32_t *view_lm_dev, const double *bear_dev, uint32_t n_features,
                                uint32_t L, const uint32_t *lm_off_dev, const uint32_t *obs_dev, uint32_t n_obs,
                                const cvb_view_constraint *cons_dev, uint32_t C, cvb_recon_result *res_dev, cvb_pose *poses_out_dev,
                                uint8_t *view_state_dev, uint8_t *obs_state_dev);
int optimize_reconstruction(cvb_ctx *ctx, const cvb_recon_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses,
                            const uint32_t *vo, const uint32_t *vl, const double *bear, uint32_t L, const uint32_t *lo, const uint32_t *obs,
                            const cvb_view_constraint *cons, uint32_t C, cvb_recon_result *res, cvb_pose *poses_out, uint8_t *view_state,
                            uint8_t *obs_state);

extern "C" {

void cvb_recon_cfg_default(cvb_recon_cfg *cfg) { recon_cfg_default(cfg); }

int cvb_optimize_reconstruction_check(uint32_t V, const uint32_t *view_offsets, const uint32_t *view_landmarks, uint32_t L,
                                      const uint32_t *landmark_offsets, const uint32_t *observations, const cvb_view_constraint *constraints,
                                      uint32_t C) {
    return optimize_reconstruction_check(V, view_offsets, view_landmarks, L, landmark_offsets, observations, constraints, C);
}

int cvb_optimize_reconstruction_dev(cvb_ctx *ctx, const cvb_recon_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses_dev,
                                    const uint32_t *view_offsets_dev, const uint32_t *view_landmarks_dev, const double *bearings_dev,
                                    uint32_t n_features, uint32_t L, const uint32_t *landmark_offsets_dev, const uint32_t *observations_dev,
                                    uint32_t n_observations, const cvb_view_constraint *constraints_dev, uint32_t C,
                                    cvb_recon_result *result_dev, cvb_pose *poses_out_dev, uint8_t *view_state_dev, uint8_t *obs_state_dev) {
    return optimize_reconstruction_dev(ctx, cfg, tri, V, poses_dev, view_offsets_dev, view_landmarks_dev, bearings_dev, n_features, L,
                                       landmark_offsets_dev, observations_dev, n_observations, constraints_dev, C, result_dev, poses_out_dev,
                                       view_state_dev, obs_state_dev);
}

int cvb_optimize_reconstruction(cvb_ctx *ctx, const cvb_recon_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses,
                                const uint32_t *view_offsets, const uint32_t *view_landmarks, const double *bearings, uint32_t L,
                                const uint32_t *landmark_offsets, const uint32_t *observations, const cvb_view_constraint *constraints,
                                uint32_t C, cvb_recon_result *result, cvb_pose *poses_out, uint8_t *view_state, uint8_t *obs_state) {
    return optimize_reconstruction(ctx, cfg, tri, V, poses, view_offsets, view_landmarks, bearings, L, landmark_offsets, observations,
                                   constraints, C, result, poses_out, view_state, obs_state);
}

}  // extern "C"
