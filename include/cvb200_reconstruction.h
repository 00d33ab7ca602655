/* include/cvb200_reconstruction.h -- C ABI of cv-sfm's reconstruction optimisation on the device.
 *
 *   cvb_optimize_reconstruction_dev    <- VSlam::optimize_reconstruction (cv-sfm/src/lib.rs:2343-2355): apply_constraints (lib.rs:2358-2414,
 *                                         constrain_view :1892-1936, flatten_constraints :2519-2532, edge_constraints :167-180) and
 *                                         filter_non_robust_observations (lib.rs:2657-2757), as a pure function of a reconstruction
 *                                         snapshot and its three-view constraints
 *   cvb_optimize_reconstruction        <- the same on host inputs, validated first, with one synchronisation
 *   cvb_optimize_reconstruction_check  <- that validation alone (host, no device needed)
 *   cvb_recon_cfg_default              <- the defaults of the settings it reads (cv-sfm/src/settings.rs)
 *
 * Library: libcvb200_reconstruction.so, a module over libcvb200.so that takes its contexts (link with -lcvb200_reconstruction -lcvb200).
 * The conventions of include/cvb200.h hold: return codes, HOST pointers unless the name ends in _dev, no CPU fallback.
 *
 * Inputs.  The snapshot has exactly the layout of include/cvb200_constraints.h: poses[V] (WorldToCamera), the view CSR view_offsets /
 * view_landmarks with bearings, and the landmark CSR landmark_offsets / observations of (view, feature).  The C constraints are
 * cvb_view_constraint in the caller's order: Reconstruction::constraints.values(), a DenseSlotMap whose removals swap, so that order is
 * UNPINNED; their `landmarks` field is ignored.  Every constraint's views are < V and pairwise distinct (cvb_optimize_reconstruction checks
 * it; for cvb_optimize_reconstruction_dev it is a precondition, and the device ignores a constraint that breaks it rather than reading out
 * of bounds).  The triangulator `tri` is one of methods 0-2.
 *
 * Semantics.  For each of reconstruction_optimization_iterations rounds:
 *   1. flatten: the constraints that contain no view removed so far (remove_view drops them, lib.rs:541-543) give their six edges each,
 *      in edge_constraints' order: (v0 <- v2, second^-1), (v0 <- v1, first^-1), (v1 <- v0, first), (v1 <- v2, (second first^-1)^-1),
 *      (v2 <- v1, second first^-1), (v2 <- v0, second).  A view's edge list is in (constraint order, edge order).  The transforms are
 *      computed once per round.
 *   2. optimization_iterations Jacobi steps; every present view computes its update from the poses of the previous step:
 *        - a view with no edges is removed;
 *        - otherwise delta = graph_optimization_rate * sum_e se3(T_e * P_other * P_v^-1), the sum starting from zero and adding the
 *          edges in list order (Iterator::sum over Vector6).  se3 is the translation followed by Skew3::from(rotation): scaled_axis with
 *          NaN mapped to zero (cv-core/src/so3.rs:263-275);
 *        - a non-finite delta removes the view;
 *        - otherwise the new pose is from_se3(delta) * P_v.  The exp map (so3.rs:248-261) takes rotation_small -- Rotation3::from_matrix
 *          (I + hat(w)), nalgebra's iterative projection onto SO(3) -- when |w|^2 <= f64::EPSILON, and from_axis_angle otherwise.
 *      A step in which fewer than 3 views are updated removes the reconstruction (status CVB_RECON_REMOVED_CONSTRAINTS); that step's
 *      updates and removals are not applied.  A view removed for a non-finite delta stays in this round's edge lists, and in the next
 *      step the reference indexes its removed slot-map key and panics: the call stops there with CVB_RECON_PANIC, before that step
 *      changes anything.  Non-finite constraint poses come from optimize_three_view's unguarded rescale, so this is reachable.
 *   3. filter_non_robust_observations over the new poses.  Observations of removed views are dropped (remove_view).  Landmarks are taken
 *      in index order, their observations in the caller's order (UNPINNED: a HashMap upstream).  One observation: skipped.  Two:
 *      is_bi_landmark_robust (epipolar loss of second * first^-1 below maximum_sine_distance), else split_landmark, which keeps the FIRST.
 *      Three or more: the triangulator; on failure split_landmark (keeps the first); otherwise, in observation order, split_observation
 *      of every observation with 1 - cos > maximum_cosine_distance (strict), which refuses to split the last remaining observation, so
 *      when all fail the LAST one stays.  Then the robust landmarks are counted (is_landmark_robust, lib.rs:2907-2934, 2975-2988: at least
 *      min(robust_minimum_observations, views remaining) observations and some pair of world-frame bearings with
 *      1 - a.b > robust_observation_incidence_minimum_cosine_distance); fewer than minimum_robust_landmarks removes the reconstruction
 *      (status CVB_RECON_REMOVED_FILTER).  A split observation forms a landmark of one observation, which is never robust.
 *
 * nalgebra 0.30.1 is not in the reference's tree; these are restated from that version and UNPINNED against the crate:
 *   Rotation3::angle = acos((m00 + m11 + m22 - 1) / 2); axis = Unit::try_new((m21 - m12, m02 - m20, m10 - m01), f64::EPSILON), None when
 *   the squared norm is <= epsilon^2; scaled_axis = axis * angle, or zero without an axis; from_axis_angle as Rodrigues' formula;
 *   from_matrix = from_matrix_eps(m, f64::EPSILON, unbounded, identity): rot <- from_axis_angle(a / |a|, |a|) * rot with
 *   a = sum_i rot_col_i x m_col_i / (|sum_i rot_col_i . m_col_i| + f64::EPSILON), until |a|^2 <= f64::EPSILON^2.  The loop here stops after
 *   CVB_RECON_FROM_MATRIX_MAX_ITERATIONS, a bound the inputs it sees (|w|^2 <= f64::EPSILON) converge far below.
 * The device's FP64 sin, cos and acos are not glibc's, so poses after one or more steps agree with a host restatement to rounding, not
 * bit for bit; with optimization_iterations = 0 the call is bit for bit.
 *
 * Outputs: the result header; poses_out[V], the poses at the end (also when the reconstruction is removed or the call stops);
 * view_state[V] (CVB_RECON_VIEW_*); obs_state[n_observations] on the input CSR (CVB_RECON_OBS_*).  An observation split in one round whose
 * view is removed in a later one is dropped.  With these the caller replays the slot-map edits; the device does no bookkeeping. */
#ifndef CVB200_RECONSTRUCTION_H
#define CVB200_RECONSTRUCTION_H
#include "cvb200.h"
#include "cvb200_tri.h"
#include "cvb200_constraints.h"

#ifdef __cplusplus
extern "C" {
#endif

#define CVB_RECON_FROM_MATRIX_MAX_ITERATIONS 64

/* cvb_recon_result.status */
#define CVB_RECON_KEPT 0                  /* optimize_reconstruction returns Some */
#define CVB_RECON_REMOVED_CONSTRAINTS 1   /* apply_constraints: fewer than 3 views updated in a step */
#define CVB_RECON_REMOVED_FILTER 2        /* filter_non_robust_observations: fewer than minimum_robust_landmarks */
#define CVB_RECON_PANIC 3                 /* a step would index a view removed in an earlier step of the round (the reference panics) */
/* view_state */
#define CVB_RECON_VIEW_KEPT 0
#define CVB_RECON_VIEW_NO_EDGES 1         /* removed: no edges in its round */
#define CVB_RECON_VIEW_NON_FINITE 2       /* removed: a non-finite update */
/* obs_state */
#define CVB_RECON_OBS_KEPT 0              /* stays in its landmark */
#define CVB_RECON_OBS_SPLIT 1             /* split into a landmark of its own */
#define CVB_RECON_OBS_DROPPED 2           /* dropped with its view */

/* the cv-sfm settings optimize_reconstruction reads (cv-sfm/src/settings.rs) */
typedef struct {
    double graph_optimization_rate;                                /* 0.001  settings.rs:477-479 */
    double maximum_sine_distance;                                  /* 0.1    settings.rs:328-330 */
    double maximum_cosine_distance;                                /* 1e-5   settings.rs:324-326 */
    double robust_observation_incidence_minimum_cosine_distance;   /* 1e-3   settings.rs:348-350 */
    uint32_t optimization_iterations;                              /* 1024   settings.rs:461-463 */
    uint32_t reconstruction_optimization_iterations;               /* 1      settings.rs:429-431 */
    uint32_t robust_minimum_observations;                          /* 3      settings.rs:344-346 */
    uint32_t minimum_robust_landmarks;                             /* 32     settings.rs:340-342 */
} cvb_recon_cfg;

typedef struct {
    int32_t status;                /* CVB_RECON_* */
    uint32_t round, step;          /* where it stopped (0-based; statuses 1 and 3); status 2: the round, step = optimization_iterations;
                                      status 0: round = reconstruction_optimization_iterations, step = 0 */
    uint32_t views_removed;        /* view_state != CVB_RECON_VIEW_KEPT */
    uint32_t robust_before;        /* robust landmarks before the last filter that ran (0 if none ran) */
    uint32_t robust_after;         /* and after it */
    uint32_t observations_split;   /* split_observation calls that split, over all rounds */
    uint32_t small_angle_updates;  /* applied view updates whose exp map took rotation_small */
} cvb_recon_result;

void cvb_recon_cfg_default(cvb_recon_cfg *cfg);

/* Validates a snapshot and its constraints on the host: cvb_view_constraints_check of the CSRs (no queries), then every constraint's
 * views < V and pairwise distinct.  0, or CVB_EINVAL (also for constraints == NULL with C > 0). */
int cvb_optimize_reconstruction_check(uint32_t V, const uint32_t *view_offsets, const uint32_t *view_landmarks, uint32_t L,
                                      const uint32_t *landmark_offsets, const uint32_t *observations, const cvb_view_constraint *constraints,
                                      uint32_t C);

/* Device inputs as in cvb_view_constraints_dev (view_landmarks_dev is part of the layout; the device reads only view_offsets_dev and
 * bearings_dev of the view CSR), constraints_dev [C].  Outputs (device): result_dev [1], poses_out_dev [V], view_state_dev [V],
 * obs_state_dev [n_observations].  Triangulator methods 3-5 are CVB_EUNSUPPORTED; a NULL argument, V = 0 or
 * view_offsets[V] != n_features is CVB_EINVAL.  Returns when the outputs are written. */
int cvb_optimize_reconstruction_dev(cvb_ctx *ctx, const cvb_recon_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses_dev,
                                    const uint32_t *view_offsets_dev, const uint32_t *view_landmarks_dev, const double *bearings_dev,
                                    uint32_t n_features, uint32_t L, const uint32_t *landmark_offsets_dev, const uint32_t *observations_dev,
                                    uint32_t n_observations, const cvb_view_constraint *constraints_dev, uint32_t C,
                                    cvb_recon_result *result_dev, cvb_pose *poses_out_dev, uint8_t *view_state_dev, uint8_t *obs_state_dev);

/* The same on HOST arrays (validated by cvb_optimize_reconstruction_check first); outputs are host arrays as above. */
int cvb_optimize_reconstruction(cvb_ctx *ctx, const cvb_recon_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses,
                                const uint32_t *view_offsets, const uint32_t *view_landmarks, const double *bearings, uint32_t L,
                                const uint32_t *landmark_offsets, const uint32_t *observations, const cvb_view_constraint *constraints,
                                uint32_t C, cvb_recon_result *result, cvb_pose *poses_out, uint8_t *view_state, uint8_t *obs_state);

#ifdef __cplusplus
}
#endif
#endif /* CVB200_RECONSTRUCTION_H */
