/* include/cvb200_tri.h -- C ABI of libcvb200.so for the triangulators of cv-geom (cv-geom/src/triangulation.rs), batched on the device.
 *
 *   CVB_TRI_LINEAR_EIGEN  <- LinearEigenTriangulator       TriangulatorObservations   triangulation.rs:39-130
 *   CVB_TRI_SINE_L1       <- SineL1Triangulator            TriangulatorObservations   :163-276
 *   CVB_TRI_MEAN_MEAN     <- MeanMeanTriangulator          TriangulatorObservations   :389-442
 *   CVB_TRI_RELATIVE_DLT  <- RelativeDltTriangulator       TriangulatorRelative only  :279-363
 *   CVB_TRI_ANGULAR_L1    <- AngularL1Triangulator         TriangulatorRelative only  :469-530
 *   CVB_TRI_ANGULAR_LINF  <- AngularLInfinityTriangulator  TriangulatorRelative only  :555-606
 *
 * cv-sfm is generic over its triangulator (VSlam<C, EF, T: TriangulatorObservations + Clone>, cv-sfm/src/lib.rs:737-751); these entry
 * points let any of cv-geom's triangulators run on the device, including inside cv-sfm's robustness filters
 * (cvb_observation_losses_tri, cvb_tri_landmarks_robust_tri), where the entry points of cvb200.h always use LinearEigen.
 *
 * The conventions of include/cvb200.h hold: return codes, HOST pointers, no CPU fallback (no device: no context, CVB_ENODEV).
 * Outputs: homogeneous points normalised as Projective::from_homogeneous does (w >= 0, |xyz| = 1); ok = 0 where the reference returns
 * None, and that row of xyzw is zero.  The relative entry point returns the point in camera A's frame (CameraPoint). */
#ifndef CVB200_TRI_H
#define CVB200_TRI_H
#include "cvb200.h"

#ifdef __cplusplus
extern "C" {
#endif

#define CVB_TRI_LINEAR_EIGEN 0 /* TriangulatorObservations */
#define CVB_TRI_SINE_L1 1      /* TriangulatorObservations */
#define CVB_TRI_MEAN_MEAN 2    /* TriangulatorObservations */
#define CVB_TRI_RELATIVE_DLT 3 /* TriangulatorRelative only */
#define CVB_TRI_ANGULAR_L1 4   /* TriangulatorRelative only */
#define CVB_TRI_ANGULAR_LINF 5 /* TriangulatorRelative only */

/* One triangulator and its builder settings.  epsilon and max_iterations are those of the eigen solver (LinearEigen, and SineL1's
 * initial guess), of SineL1's refinement loop and of RelativeDlt's SVD; optimization_rate is SineL1's.  Fields a method does not have
 * are ignored. */
typedef struct {
    int32_t method;
    uint32_t max_iterations;
    double epsilon, optimization_rate;
} cvb_triangulator;

/* The reference's Default impls: LinearEigen 1e-12 / 1000; SineL1 1e-12 / 1000 / rate 1.0 (its doc comment says 0.01, :197-199);
 * RelativeDlt 1e-12 / 1000 (its doc comments say 1e-9 and 100, :293-305).  An unknown method leaves *t zeroed with that method. */
void cvb_triangulator_default(cvb_triangulator *t, int32_t method);

/* TriangulatorObservations::triangulate_observations for L landmarks; methods 0-2.  Landmark l has the observations
 * offsets[l] .. offsets[l + 1] - 1 of poses (WorldToCamera) and bearings (unit, f64 x 3); offsets (L + 1 entries) must be
 * non-decreasing.  xyzw_out: L x 4 homogeneous WorldPoints, ok_out: L flags. */
int cvb_triangulate_observations(cvb_ctx *ctx, const cvb_triangulator *tri, const cvb_pose *poses, const double *bearings,
                                 const uint32_t *offsets, uint32_t L, double *xyzw_out, uint8_t *ok_out);

/* TriangulatorRelative::triangulate_relative for n (relative pose, a, b) triples; all six methods.  poses: CameraToCamera from camera A
 * to camera B, npose = 1 (one pose shared by every triple, cv-sfm's case) or npose = n (one per triple).  a, b: unit bearings in A and B
 * (n x 3).  Methods 0-2 go through the reference's blanket impl (cv-core/src/triangulation.rs:52-67): the observations
 * [(identity, a), (pose, b)], then CameraPoint::from_homogeneous once more.  xyzw_out: n x 4 CameraPoints, ok_out: n flags. */
int cvb_triangulate_relative(cvb_ctx *ctx, const cvb_triangulator *tri, const cvb_pose *poses, uint32_t npose, const double *a,
                             const double *b, uint32_t n, double *xyzw_out, uint8_t *ok_out);

/* cvb_observation_losses (include/cvb200.h) with the caller's triangulator (methods 0-2) where cv-sfm calls self.triangulator
 * (cv-sfm/src/lib.rs:2613,2641).  A LinearEigen triangulator in its default configuration gives cvb_observation_losses' bits. */
int cvb_observation_losses_tri(cvb_ctx *ctx, const cvb_triangulator *tri, const cvb_pose *poses, const double *bearings,
                               const uint32_t *offsets, uint32_t L, double *loss_out);

/* cvb_tri_landmarks_robust (include/cvb200.h) with the caller's triangulator (methods 0-2; cv-sfm/src/lib.rs:1332). */
int cvb_tri_landmarks_robust_tri(cvb_ctx *ctx, const cvb_triangulator *tri, const cvb_pose *first_pose, const cvb_pose *second_pose,
                                 const double *observations, uint32_t n, double maximum_cosine_distance,
                                 double incidence_minimum_cosine_distance, uint8_t *robust_out);

#ifdef __cplusplus
}
#endif
#endif /* CVB200_TRI_H */
