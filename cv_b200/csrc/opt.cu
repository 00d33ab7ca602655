// cv_b200/csrc/opt.cu -- libcvb200_opt.so, the module that exports the C ABI of include/cvb200_opt.h (cv-optimize's L1 optimizers).
// The kernels and their host code live in geom.cu next to the L2 optimizers they share their device functions with; this module only
// gives them their C names, so that libcvb200.so's own exports stay exactly those of cvb200.h, cvb200_sfm.h and cvb200_tri.h.
// It links libcvb200.so (rpath $ORIGIN) and takes that library's contexts.
#include "../../include/cvb200_opt.h"

int opt_single_view_l1(cvb_ctx *ctx, const cvb_pose *poses, uint32_t B, double epsilon, double optimization_rate, uint32_t iterations,
                       const double *bearings, const double *world, const uint32_t *offsets, cvb_pose *poses_out, uint32_t *updates_out);
int opt_three_view_l1(cvb_ctx *ctx, const cvb_pose *poses, uint32_t B, double epsilon, double optimization_rate, uint32_t iterations,
                      const double *observations, const uint32_t *offsets, cvb_pose *poses_out, uint32_t *updates_out);

extern "C" {

int cvb_single_view_optimize_l1(cvb_ctx *ctx, const cvb_pose *poses, uint32_t B, double epsilon, double optimization_rate,
                                uint32_t iterations, const double *bearings, const double *world, const uint32_t *offsets,
                                cvb_pose *poses_out, uint32_t *updates_out) {
    return opt_single_view_l1(ctx, poses, B, epsilon, optimization_rate, iterations, bearings, world, offsets, poses_out, updates_out);
}

int cvb_three_view_optimize_l1(cvb_ctx *ctx, const cvb_pose *poses, uint32_t B, double epsilon, double optimization_rate,
                               uint32_t iterations, const double *observations, const uint32_t *offsets, cvb_pose *poses_out,
                               uint32_t *updates_out) {
    return opt_three_view_l1(ctx, poses, B, epsilon, optimization_rate, iterations, observations, offsets, poses_out, updates_out);
}

}  // extern "C"
