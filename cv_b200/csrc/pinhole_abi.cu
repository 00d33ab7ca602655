// cv_b200/csrc/pinhole_abi.cu -- libcvb200_pinhole.so, the module that exports the C ABI of include/cvb200_pinhole.h (cv-pinhole's
// reprojection error and EssentialMatrix model).  The kernels and their host code live in geom.cu next to the triangulators and the
// eight-point / essential device functions they share; this module only gives them their C names, so that libcvb200.so's own exports
// stay exactly those of cvb200.h, cvb200_sfm.h and cvb200_tri.h.  It links libcvb200.so (rpath $ORIGIN) and takes that library's contexts.
#include "../../include/cvb200_pinhole.h"

int pin_pose_reprojection_error(cvb_ctx *ctx, const cvb_triangulator *tri, const cvb_pose *poses, uint32_t npose, const double *a,
                                const double *b, uint32_t n, double *err_out, double *avg_out, uint8_t *ok_out);
int pin_pose_reprojection_error_dev(cvb_ctx *ctx, const cvb_triangulator *tri, const cvb_pose *poses_dev, uint32_t npose,
                                    const double *a_dev, const double *b_dev, const uint32_t *n_dev, uint32_t n_max,
                                    const int32_t *found_dev, double *err_out_dev, double *avg_out_dev, uint8_t *ok_out_dev);
int pin_eight_point_essential_batch(cvb_ctx *ctx, double epsilon, uint32_t iterations, const double *a, const double *b, uint32_t n,
                                    const uint32_t *samples, uint32_t H, double *E_out, uint8_t *ok_out);
int pin_residuals_essential(cvb_ctx *ctx, const double *E, uint32_t m, const double *a, const double *b, uint32_t n, double *out);
int pin_essential_recondition(cvb_ctx *ctx, const double *E, uint32_t m, double epsilon, uint32_t max_iterations, double *E_out,
                              uint8_t *ok_out);
int pin_essential_decompose(cvb_ctx *ctx, const double *E, uint32_t m, double epsilon, uint32_t max_iterations, double *rot_a_out,
                            double *rot_b_out, double *t_out, uint8_t *ok_out);

extern "C" {

int cvb_pose_reprojection_error(cvb_ctx *ctx, const cvb_triangulator *tri, const cvb_pose *poses, uint32_t npose, const double *a,
                                const double *b, uint32_t n, double *err_out, double *avg_out, uint8_t *ok_out) {
    return pin_pose_reprojection_error(ctx, tri, poses, npose, a, b, n, err_out, avg_out, ok_out);
}

int cvb_pose_reprojection_error_dev(cvb_ctx *ctx, const cvb_triangulator *tri, const cvb_pose *poses_dev, uint32_t npose,
                                    const double *a_dev, const double *b_dev, const uint32_t *n_dev, uint32_t n_max,
                                    const int32_t *found_dev, double *err_out_dev, double *avg_out_dev, uint8_t *ok_out_dev) {
    return pin_pose_reprojection_error_dev(ctx, tri, poses_dev, npose, a_dev, b_dev, n_dev, n_max, found_dev, err_out_dev, avg_out_dev,
                                           ok_out_dev);
}

int cvb_eight_point_essential_batch(cvb_ctx *ctx, double epsilon, uint32_t iterations, const double *a, const double *b, uint32_t n,
                                    const uint32_t *samples, uint32_t H, double *E_out, uint8_t *ok_out) {
    return pin_eight_point_essential_batch(ctx, epsilon, iterations, a, b, n, samples, H, E_out, ok_out);
}

int cvb_residuals_essential(cvb_ctx *ctx, const double *E, uint32_t m, const double *a, const double *b, uint32_t n, double *out) {
    return pin_residuals_essential(ctx, E, m, a, b, n, out);
}

int cvb_essential_recondition(cvb_ctx *ctx, const double *E, uint32_t m, double epsilon, uint32_t max_iterations, double *E_out,
                              uint8_t *ok_out) {
    return pin_essential_recondition(ctx, E, m, epsilon, max_iterations, E_out, ok_out);
}

int cvb_essential_decompose(cvb_ctx *ctx, const double *E, uint32_t m, double epsilon, uint32_t max_iterations, double *rot_a_out,
                            double *rot_b_out, double *t_out, uint8_t *ok_out) {
    return pin_essential_decompose(ctx, E, m, epsilon, max_iterations, rot_a_out, rot_b_out, t_out, ok_out);
}

}  // extern "C"
