/* include/cvb200_export.h -- C ABI of cv-sfm's reconstruction export on the device.
 *
 *   cvb_robust_landmarks_dev          <- VSlam::triangulate_landmark_robust (cv-sfm/src/lib.rs:2907-2934, 2975-3000) for every landmark of a
 *                                        reconstruction snapshot
 *   cvb_export_reconstruction_dev     <- VSlam::export_reconstruction (lib.rs:2285-2340) without the file: the point cloud with its colours
 *                                        and the cameras (cv-sfm/src/export.rs's ExportCamera)
 *   cvb_normalize_reconstruction_dev  <- VSlam::normalize_reconstruction (lib.rs:2241-2283)
 *   cvb_robust_landmarks, cvb_export_reconstruction, cvb_normalize_reconstruction
 *                                     <- the same on host inputs, validated first, with one synchronisation
 *   cvb_export_check                  <- that validation alone (host, no device needed)
 *   cvb_export_cfg_default            <- the defaults of the settings they read (cv-sfm/src/settings.rs)
 *
 * Library: libcvb200_export.so, a module over libcvb200.so that takes its contexts (link with -lcvb200_export -lcvb200).  The conventions
 * of include/cvb200.h hold: return codes, HOST pointers unless the name ends in _dev, no CPU fallback.
 *
 * Inputs.  The snapshot has exactly the layout of include/cvb200_constraints.h: poses[V] (WorldToCamera), the view CSR view_offsets /
 * view_landmarks with bearings, and the landmark CSR landmark_offsets / observations of (view, feature), whose order is the caller's
 * (UNPINNED: Landmark.observations is a HashMap upstream).  colors[n_features][3] are the features' colours on the view CSR, as
 * cvb_frame_features_batch returns them.  The triangulator `tri` is one of methods 0-2 (VSlam's triangulator is a TriangulatorObservations);
 * methods 3-5 are CVB_EUNSUPPORTED.
 *
 * Robust landmarks (triangulate_landmark_robust).  state[l] is
 *   CVB_EXPORT_POINT        the triangulator's homogeneous WorldPoint is in points[l] and its w is not zero;
 *   CVB_EXPORT_NOT_ROBUST   are_observations_robust is false: fewer than min(robust_minimum_observations, V) observations, or no pair
 *                           i < j of world-frame bearings (pose^-1's rotation applied to the bearing), in tuple_combinations order, with
 *                           1 - a.b > robust_observation_incidence_minimum_cosine_distance;
 *   CVB_EXPORT_TRI_FAILED   the triangulator over (pose, bearing) in observation order returns None;
 *   CVB_EXPORT_AT_INFINITY  the point is Some but its w is zero (Projective::point is None); it is in points[l].
 * points[l] of the other two states is zero.
 *
 * The mean distance of a view (the `Mean` of lib.rs:2252-2257 and 2315-2324) folds, in the view's feature order, one value per feature
 * whose landmark has a point (POINT or AT_INFINITY; filter_map skips the others): pose.transform(h) is pose.to_homogeneous() h, every
 * row, w' included, as ((m0 x + m1 y) + m2 z) + m3 w (so w' is computed, not copied: 0 * inf is NaN), made a CameraPoint by
 * Projective::from_homogeneous (cv-core/src/point.rs:20-25: negated when w' has its sign bit set, then every component divided by
 * sqrt((x^2 + y^2) + z^2)); a w that is then zero (-0 too) is skipped (Point3::from_homogeneous is None); otherwise the value is the norm
 * sqrt((x^2 + y^2) + z^2) of xyz / w.
 * The reference triangulates a landmark again for every view that observes it; triangulation is deterministic, so computing each
 * landmark's point once and reusing it gives the same bits.
 *
 * Crates outside the reference's tree, restated here and UNPINNED against them:
 *   average 0.13.1's Mean: n += 1; avg += (x - avg) / n, from avg = 0; the mean of no values is NaN (believed to be what 0.13 returns).
 *     A view with no value therefore gets focal_length NaN, which the PLY writer prints as NaN.
 *   nalgebra: Point3::from_homogeneous divides x, y and z by w; Isometry::inverse is (R^T, R^T (-t)); A * B is (A.R B.R, A.t + A.R B.t);
 *     a matrix times a vector sums the columns in order; the norm is sqrt((x^2 + y^2) + z^2).
 *
 * Export.  The points are the POINT landmarks, compacted in landmark index order, each x, y and z divided by w; the colour of a point is
 * that of its landmark's first observation in the caller's order (observations.iter().next() on a HashMap upstream, so UNPINNED).
 * cameras[v], in view order: with c2w = pose^-1, optical_center = c2w.R (0, 0, 0) + c2w.t, up_direction = c2w.R (-0, -1, -0) (the
 * negated unit y, signed zeros included), forward_direction = c2w.R (0, 0, 1), focal_length = mean distance * 0.01.
 *
 * Normalisation.  first_view is the view normalize_reconstruction takes (views.values().next() of a DenseSlotMap whose removals swap,
 * so UNPINNED: the caller passes its index).  Only its landmarks are triangulated.  If its mean distance is not normal (is_normal: zero,
 * subnormal, infinite or NaN), the outputs are the inputs unchanged and normalized = 0.  Otherwise, with T = P_first^-1 and
 * s = 1.0 / mean: every view's pose is P_v * T with its translation then multiplied by s, and both translations of every constraint are
 * multiplied by s (every other field is copied). */
#ifndef CVB200_EXPORT_H
#define CVB200_EXPORT_H
#include "cvb200.h"
#include "cvb200_tri.h"
#include "cvb200_constraints.h"

#ifdef __cplusplus
extern "C" {
#endif

/* state of a landmark */
#define CVB_EXPORT_POINT 0
#define CVB_EXPORT_NOT_ROBUST 1
#define CVB_EXPORT_TRI_FAILED 2
#define CVB_EXPORT_AT_INFINITY 3

/* the cv-sfm settings these calls read (cv-sfm/src/settings.rs).  vslam-sandbox exports with robust_minimum_observations from its
 * --export-robust-minimum-observations (default 3) */
typedef struct {
    double robust_observation_incidence_minimum_cosine_distance;   /* 1e-3  settings.rs:348-350 */
    uint32_t robust_minimum_observations;                          /* 3     settings.rs:344-346 */
} cvb_export_cfg;

/* cv-sfm/src/export.rs's ExportCamera */
typedef struct {
    double optical_center[3];
    double up_direction[3];
    double forward_direction[3];
    double focal_length;
} cvb_export_camera;

typedef struct {
    int32_t normalized;            /* 1 when the mean distance was normal and the reconstruction was transformed */
    uint32_t robust_points;        /* the values folded into the first view's mean distance */
    double mean_distance;          /* the first view's mean distance (NaN when robust_points = 0) */
} cvb_normalize_result;

void cvb_export_cfg_default(cvb_export_cfg *cfg);

/* Validates a snapshot on the host: cvb_optimize_reconstruction_check of the CSRs and the C constraints (constraints may be NULL when
 * C = 0), and first_view < V.  0, or CVB_EINVAL. */
int cvb_export_check(uint32_t V, const uint32_t *view_offsets, const uint32_t *view_landmarks, uint32_t L, const uint32_t *landmark_offsets,
                     const uint32_t *observations, const cvb_view_constraint *constraints, uint32_t C, uint32_t first_view);

/* Device inputs as in cvb_view_constraints_dev.  Outputs (device): points_dev [L][4], state_dev [L].  A NULL argument, V = 0 or
 * view_offsets[V] != n_features is CVB_EINVAL.  Returns when the outputs are written. */
int cvb_robust_landmarks_dev(cvb_ctx *ctx, const cvb_export_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses_dev,
                             const uint32_t *view_offsets_dev, const uint32_t *view_landmarks_dev, const double *bearings_dev,
                             uint32_t n_features, uint32_t L, const uint32_t *landmark_offsets_dev, const uint32_t *observations_dev,
                             uint32_t n_observations, double *points_dev, uint8_t *state_dev);

/* The same on HOST arrays (validated by cvb_export_check first); outputs are host arrays as above. */
int cvb_robust_landmarks(cvb_ctx *ctx, const cvb_export_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses,
                         const uint32_t *view_offsets, const uint32_t *view_landmarks, const double *bearings, uint32_t L,
                         const uint32_t *landmark_offsets, const uint32_t *observations, double *points, uint8_t *state);

/* Device inputs as in cvb_robust_landmarks_dev plus colors_dev [n_features][3].  Outputs (device): points_dev [L][3] and
 * point_colors_dev [L][3], of which the first *n_points_dev are written; n_points_dev [1]; cameras_dev [V]; mean_distance_dev [V] (may be
 * NULL).  Errors as cvb_robust_landmarks_dev.  Returns when the outputs are written. */
int cvb_export_reconstruction_dev(cvb_ctx *ctx, const cvb_export_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses_dev,
                                  const uint32_t *view_offsets_dev, const uint32_t *view_landmarks_dev, const double *bearings_dev,
                                  const uint8_t *colors_dev, uint32_t n_features, uint32_t L, const uint32_t *landmark_offsets_dev,
                                  const uint32_t *observations_dev, uint32_t n_observations, double *points_dev, uint8_t *point_colors_dev,
                                  uint32_t *n_points_dev, cvb_export_camera *cameras_dev, double *mean_distance_dev);

/* The same on HOST arrays (validated by cvb_export_check first); outputs are host arrays as above. */
int cvb_export_reconstruction(cvb_ctx *ctx, const cvb_export_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses,
                              const uint32_t *view_offsets, const uint32_t *view_landmarks, const double *bearings, const uint8_t *colors,
                              uint32_t L, const uint32_t *landmark_offsets, const uint32_t *observations, double *points,
                              uint8_t *point_colors, uint32_t *n_points, cvb_export_camera *cameras, double *mean_distance);

/* Device inputs as in cvb_robust_landmarks_dev plus constraints_dev [C] and first_view.  Outputs (device): poses_out_dev [V],
 * constraints_out_dev [C], result_dev [1].  A NULL argument, V = 0, first_view >= V or view_offsets[V] != n_features is CVB_EINVAL.
 * Returns when the outputs are written. */
int cvb_normalize_reconstruction_dev(cvb_ctx *ctx, const cvb_export_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses_dev,
                                     const uint32_t *view_offsets_dev, const uint32_t *view_landmarks_dev, const double *bearings_dev,
                                     uint32_t n_features, uint32_t L, const uint32_t *landmark_offsets_dev, const uint32_t *observations_dev,
                                     uint32_t n_observations, const cvb_view_constraint *constraints_dev, uint32_t C, uint32_t first_view,
                                     cvb_pose *poses_out_dev, cvb_view_constraint *constraints_out_dev, cvb_normalize_result *result_dev);

/* The same on HOST arrays (validated by cvb_export_check first); outputs are host arrays as above. */
int cvb_normalize_reconstruction(cvb_ctx *ctx, const cvb_export_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses,
                                 const uint32_t *view_offsets, const uint32_t *view_landmarks, const double *bearings, uint32_t L,
                                 const uint32_t *landmark_offsets, const uint32_t *observations, const cvb_view_constraint *constraints,
                                 uint32_t C, uint32_t first_view, cvb_pose *poses_out, cvb_view_constraint *constraints_out,
                                 cvb_normalize_result *result);

#ifdef __cplusplus
}
#endif
#endif /* CVB200_EXPORT_H */
