/* include/cvb200_pinhole.h -- C ABI of cv-pinhole's reprojection error and EssentialMatrix model, batched on the device.
 *
 *   cvb_pose_reprojection_error(_dev)   <- pose_reprojection_error + average_pose_reprojection_error   cv-pinhole/src/lib.rs:314-372
 *   cvb_eight_point_essential_batch     <- EightPoint::from_matches                eight-point/src/lib.rs:11-58
 *   cvb_residuals_essential             <- impl Model<FeatureMatch> for EssentialMatrix   cv-pinhole/src/essential.rs:266-275
 *   cvb_essential_recondition           <- EssentialMatrix::recondition            essential.rs:64-77
 *   cvb_essential_decompose             <- possible_rotations_unscaled_translation essential.rs:114-162
 *
 * possible_rotations, possible_unscaled_poses ((t, Ra), (t, Rb), (-t, Ra), (-t, Rb)) and possible_unscaled_poses_bearing
 * (essential.rs:183-262) are reshuffles of cvb_essential_decompose's output; From<CameraToCamera> is [t]x R.  The bindings build them.
 *
 * Library: libcvb200_pinhole.so, a module over libcvb200.so that takes its contexts (link with -lcvb200_pinhole -lcvb200).
 * The conventions of include/cvb200.h hold: return codes, HOST pointers unless the name ends in _dev, no CPU fallback (no device: no
 * context, CVB_ENODEV).  Matrices (E, rotations) are row-major double[9], like cvb_pose.r.  Where the reference returns None the row's
 * ok is 0 and every double of the row is NaN (not zero, so that an unchecked mean is visibly wrong).
 *
 * epsilon / max_iterations are those of the reference's SVD and symmetric eigen solver.  Here they bound a cyclic Jacobi solver, as
 * cvb_triangulator's do for RelativeDlt: the solver stops when the off-diagonal mass is below epsilon^2 times the diagonal's, or fails
 * (ok = 0) after max_iterations sweeps; values above INT32_MAX are clamped, and max_iterations = 0 runs no sweep and so never gives a
 * result (nalgebra reads 0 as unbounded).  The 3x3 SVD of recondition and decompose is the one the eight-point and five-point estimators
 * use: it comes from the eigen-decomposition of E^T E and returns no result when s1 <= 1e-12 s0 (rank <= 1), where nalgebra would still
 * decompose.  The third left singular vector is u1 x u2 (its sign is fixed by the det(U) > 0 rule of essential.rs:139-143). */
#ifndef CVB200_PINHOLE_H
#define CVB200_PINHOLE_H
#include "cvb200_tri.h"

#ifdef __cplusplus
extern "C" {
#endif

/* pose_reprojection_error for n FeatureMatches (a, b: bearings in cameras A and B, n x 3) and relative poses (CameraToCamera from A to B;
 * npose = 1: one pose for every match, npose = n: one per match, else CVB_EINVAL).  tri: any of the six triangulators (TriangulatorRelative).
 * err_out (n x 4): a_norm - reproject_a, b_norm - reproject_b, where x_norm = x.xy / x.z of the input bearing and reproject = the
 * bearing's xy / z of the triangulated CameraPoint, then of pose * point.  The reference returns None (ok = 0) when the triangulator
 * does, or when either bearing's z has its sign bit set: +0.0 and +NaN pass, so infinities and NaNs can reach err with ok = 1.
 * avg_out (n, may be NULL): average_pose_reprojection_error = (|e_a| + |e_b|) * 0.5. */
int cvb_pose_reprojection_error(cvb_ctx *ctx, const cvb_triangulator *tri, const cvb_pose *poses, uint32_t npose, const double *a,
                                const double *b, uint32_t n, double *err_out, double *avg_out, uint8_t *ok_out);

/* The same on device data, asynchronous on the context's stream: the outputs of cvb_arrsac_eight_point_dev (model_out_dev, found_dev)
 * and of cvb_pair_bearings(_k1)_dev / cvb_two_view_pair_dev (bearings, count).  Rows i < min(*n_dev, n_max) are written; the rows
 * behind them are left untouched.  npose is 1 or n_max.  When found_dev is non-NULL and *found_dev == 0, every written row gets ok = 0
 * (and NaN).  tri is a HOST pointer; avg_out_dev may be NULL. */
int cvb_pose_reprojection_error_dev(cvb_ctx *ctx, const cvb_triangulator *tri, const cvb_pose *poses_dev, uint32_t npose,
                                    const double *a_dev, const double *b_dev, const uint32_t *n_dev, uint32_t n_max,
                                    const int32_t *found_dev, double *err_out_dev, double *avg_out_dev, uint8_t *ok_out_dev);

/* EightPoint { epsilon, iterations }::from_matches for H samples of 8 match indices into (a, b) (n x 3 bearings each; an index >= n is
 * CVB_EINVAL).  Only the 8 matches of a sample enter, and b is divided by a.z, as in the reference (lib.rs:16).  E_out: H x 9. */
int cvb_eight_point_essential_batch(cvb_ctx *ctx, double epsilon, uint32_t iterations, const double *a, const double *b, uint32_t n,
                                    const uint32_t *samples, uint32_t H, double *E_out, uint8_t *ok_out);

/* EssentialMatrix::residual of every (E, FeatureMatch): |b_norm^T E a_norm| with x_norm = x / x.z.  E: m x 9; out: m x n (row = E). */
int cvb_residuals_essential(cvb_ctx *ctx, const double *E, uint32_t m, const double *a, const double *b, uint32_t n, double *out);

/* EssentialMatrix::recondition of m matrices: U diag(s, s, 0) V^T with s = (s0 + s1) / 2.  E_out: m x 9. */
int cvb_essential_recondition(cvb_ctx *ctx, const double *E, uint32_t m, double epsilon, uint32_t max_iterations, double *E_out,
                              uint8_t *ok_out);

/* EssentialMatrix::possible_rotations_unscaled_translation of m matrices: rot_a = U W V^T, rot_b = U W^T V^T (m x 9 each) and
 * t = the third column of U (m x 3), after the det(U), det(V^T) > 0 fix-ups. */
int cvb_essential_decompose(cvb_ctx *ctx, const double *E, uint32_t m, double epsilon, uint32_t max_iterations, double *rot_a_out,
                            double *rot_b_out, double *t_out, uint8_t *ok_out);

#ifdef __cplusplus
}
#endif
#endif /* CVB200_PINHOLE_H */
