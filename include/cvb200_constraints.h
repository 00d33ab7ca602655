/* include/cvb200_constraints.h -- C ABI of cv-sfm's three-view constraints on the device.
 *
 *   cvb_view_constraints_dev     <- VSlam::generate_view_constraints (cv-sfm/src/lib.rs:2438-2516) and the acceptance of
 *                                   record_view_constraints (lib.rs:2092-2109) for Q query views of one reconstruction snapshot
 *   cvb_view_constraints         <- the same on host inputs, validated first, with one synchronisation
 *   cvb_view_constraints_check   <- that validation alone (host, no device needed)
 *   cvb_three_view_adaptive_optimize_l2_dev <- three_view_adaptive_optimize_l2 (cv-optimize/src/three_view_optimizer.rs:203-272), many
 *                                   problems of at most 512 landmarks, one warp each (the constraints run it on batches larger than one
 *                                   CTA per SM, and cvb_three_view_optimize_l2's kernel, which gives the same bits, on smaller ones)
 *   cvb_constraints_cfg_default  <- the defaults of the settings they read (cv-sfm/src/settings.rs:332-350, 453-483)
 *
 * Library: libcvb200_constraints.so, a module over libcvb200.so that takes its contexts (link with -lcvb200_constraints -lcvb200).  The
 * conventions of include/cvb200.h hold: return codes, HOST pointers unless the name ends in _dev, no CPU fallback.
 *
 * The snapshot mirrors VSlamData's reconstruction, with views numbered 0 .. V in ascending ViewKey order:
 *   poses[v]                        View.pose, WorldToCamera;
 *   view_offsets[V + 1], view_landmarks[view_offsets[V]]
 *                                   View.landmarks as CSR: feature j of view v (j < view_offsets[v + 1] - view_offsets[v]) belongs to
 *                                   landmark view_landmarks[view_offsets[v] + j];
 *   bearings[view_offsets[V]][3]    the feature bearings, on the same CSR;
 *   landmark_offsets[L + 1], observations[landmark_offsets[L]][2]
 *                                   Landmark.observations as CSR of (view, feature), in the order the caller gives them.
 * The two CSRs must agree: feature j of view v belongs to landmark l exactly when l observes (v, j), and no landmark observes a view twice.
 * cvb_view_constraints checks that (CVB_EINVAL); for cvb_view_constraints_dev it is a precondition.
 *
 * Semantics, for each query view q (duplicates allowed; queries are independent given the snapshot):
 *   1. robust landmarks (triangulate_landmark_robust, lib.rs:2907-2934, 2975-3000): at least min(robust_minimum_observations, V)
 *      observations, some pair of world-frame bearings (the inverse pose's rotation applied to the bearing) with
 *      1 - a.b > robust_observation_incidence_minimum_cosine_distance, and the triangulator `tri` (methods 0-2) returns a point over
 *      (pose, bearing) in observation order;
 *   2. covisibilities (view_covisibilities, lib.rs:2535-2556): q's robust landmarks in feature order, appended to the list of every other
 *      view observing them; the coviews with at least optimization_robust_covisibility_minimum_landmarks are kept;
 *   3. triples (lib.rs:2463-2481): every pair (a, b) of kept coviews in combination order, with a's list filtered to the landmarks b
 *      observes, kept when it still has the minimum; its views are canonical_view_order([q, a, b]) (lib.rs:54-57), ascending;
 *   4. order (lib.rs:2483-2515): the triples sorted by descending landmark count; the "unique" ones -- those for which
 *      views.iter().any(|v| already_visited.insert(v)) holds, up to optimization_maximum_three_view_constraints; `any` stops at the first
 *      new view, so the triple's later views are not marked -- come first, then the rest in sorted order; optimize_three_view runs over
 *      that sequence until optimization_maximum_three_view_constraints of them succeed;
 *   5. optimize_three_view (lib.rs:1939-2062): fewer than optimization_minimum_landmarks landmarks is None; otherwise the landmarks are
 *      sorted by descending observation count and the first optimization_maximum_landmarks taken; fewer than
 *      robust_view_num_robust_bearing_pair robust bearing pairs (i < j, 1 - a.b > robust_view_bearing_pair_minimum_cosine_distance in all
 *      three views) is None; otherwise first = P1 P0^-1 and second = P2 P0^-1 go through three_view_adaptive_optimize_l2 for
 *      constraint_patience iterations and both translations are scaled by (|t1| + |t2|) before / after (pose.rs:37-41, unguarded);
 *   6. acceptance (record_view_constraints, lib.rs:2097-2102): accepted unless n < optimization_minimum_new_constraints && n + 1 < V.
 * UNPINNED, where the reference's order is not defined: coviews are taken in ascending view index (HashMap order upstream); both sorts are
 * stable (ties keep combination order, and the query's feature order); there is no shuffle of the landmarks (lib.rs:1968 shuffles them with
 * VSlam's shared generator); observations are taken in the caller's order.  Parity with a run of the reference is therefore pinned only
 * up to these orders.
 *
 * A call over every view equals regenerate_reconstruction's constraint pass (lib.rs:2418-2435), which removes nothing.
 * incorporate_reconstruction removes views between its calls to record_view_constraints; include/cvb200_merge.h runs it as one call over
 * every moved view, repeated after each refusal for the views after it, which gives the results of the one-view-at-a-time loop. */
#ifndef CVB200_CONSTRAINTS_H
#define CVB200_CONSTRAINTS_H
#include "cvb200.h"
#include "cvb200_tri.h"

#ifdef __cplusplus
extern "C" {
#endif

/* the largest optimization_maximum_landmarks (and landmarks per problem of cvb_three_view_adaptive_optimize_l2_dev) */
#define CVB_CONSTRAINTS_MAX_LANDMARKS 512

/* the cv-sfm settings generate_view_constraints and record_view_constraints read (cv-sfm/src/settings.rs) */
typedef struct {
    double robust_observation_incidence_minimum_cosine_distance;   /* 1e-3  settings.rs:348-350 */
    double robust_view_bearing_pair_minimum_cosine_distance;       /* 1e-2  settings.rs:332-334 */
    uint32_t robust_minimum_observations;                          /* 3     settings.rs:344-346 */
    uint32_t robust_view_num_robust_bearing_pair;                  /* 3     settings.rs:336-338 */
    uint32_t optimization_robust_covisibility_minimum_landmarks;   /* 16    settings.rs:473-475 */
    uint32_t optimization_minimum_landmarks;                       /* 24    settings.rs:465-467 */
    uint32_t optimization_maximum_landmarks;                       /* 64    settings.rs:469-471 (at most 512) */
    uint32_t optimization_maximum_three_view_constraints;          /* 64    settings.rs:453-455 */
    uint32_t optimization_minimum_new_constraints;                 /* 4     settings.rs:457-459 */
    uint32_t constraint_patience;                                  /* 4096  settings.rs:481-483 */
} cvb_constraints_cfg;

/* one constraint: its views ascending, poses CameraToCamera views[0] -> views[1] / views[2] */
typedef struct {
    uint32_t views[3];
    uint32_t landmarks;            /* landmarks in its optimisation */
    cvb_pose poses[2];
} cvb_view_constraint;

/* per query */
typedef struct {
    uint32_t n_constraints;        /* constraints written, at most optimization_maximum_three_view_constraints */
    int32_t accepted;              /* record_view_constraints' return */
} cvb_view_constraints_result;

/* optional per-query statistics */
typedef struct {
    uint32_t robust_landmarks;     /* the query's robust landmarks */
    uint32_t coviews;              /* coviews kept */
    uint32_t triples;              /* triples kept */
    uint32_t unique_triples;
    uint32_t candidates;           /* triples passed to optimize_three_view */
    uint32_t few_landmarks;        /* None: fewer than optimization_minimum_landmarks */
    uint32_t few_bearing_pairs;    /* None: too few robust bearing pairs */
    uint32_t updates;              /* optimiser pose updates, summed */
} cvb_view_constraints_stats;

void cvb_constraints_cfg_default(cvb_constraints_cfg *cfg);

/* Validates a snapshot and its queries on the host (the layout above): 0, or CVB_EINVAL for a NULL array, a non-monotone offset array,
 * an offset array that does not start at 0, a landmark, view, feature or query out of range, or two CSRs that disagree. */
int cvb_view_constraints_check(uint32_t V, const uint32_t *view_offsets, const uint32_t *view_landmarks, uint32_t L,
                               const uint32_t *landmark_offsets, const uint32_t *observations, const uint32_t *queries, uint32_t Q);

/* Device inputs: poses_dev [V], view_offsets_dev [V + 1], view_landmarks_dev and bearings_dev [n_features] (n_features = view_offsets[V]),
 * landmark_offsets_dev [L + 1], observations_dev [n_observations][2] (n_observations = landmark_offsets[L]); queries: HOST [Q].
 * Outputs (device): constraints_dev [Q][optimization_maximum_three_view_constraints] in the reference's evaluation order,
 * results_dev [Q], stats_dev [Q] (may be NULL).  Queries are processed in chunks that keep the workspace bounded; results do not depend on
 * the chunking.  Triangulator methods 3-5 and optimization_maximum_landmarks above CVB_CONSTRAINTS_MAX_LANDMARKS are CVB_EUNSUPPORTED; a
 * NULL argument not marked optional, V = 0 or a query >= V is CVB_EINVAL.  Returns when the outputs are written. */
int cvb_view_constraints_dev(cvb_ctx *ctx, const cvb_constraints_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses_dev,
                             const uint32_t *view_offsets_dev, const uint32_t *view_landmarks_dev, const double *bearings_dev,
                             uint32_t n_features, uint32_t L, const uint32_t *landmark_offsets_dev, const uint32_t *observations_dev,
                             uint32_t n_observations, const uint32_t *queries, uint32_t Q, cvb_view_constraint *constraints_dev,
                             cvb_view_constraints_result *results_dev, cvb_view_constraints_stats *stats_dev);

/* The same on HOST arrays (validated by cvb_view_constraints_check first); outputs are host arrays as above. */
int cvb_view_constraints(cvb_ctx *ctx, const cvb_constraints_cfg *cfg, const cvb_triangulator *tri, uint32_t V, const cvb_pose *poses,
                         const uint32_t *view_offsets, const uint32_t *view_landmarks, const double *bearings, uint32_t L,
                         const uint32_t *landmark_offsets, const uint32_t *observations, const uint32_t *queries, uint32_t Q,
                         cvb_view_constraint *constraints, cvb_view_constraints_result *results, cvb_view_constraints_stats *stats);

/* B problems of three_view_adaptive_optimize_l2 on device arrays, one warp per problem: poses_dev [2 B] (CameraToCamera centre -> first,
 * centre -> second), obs_dev [offsets[B]][9] (centre, first, second bearings), offsets_dev [B + 1] (HOST n_rows = offsets[B]),
 * `iterations` adaptive steps.  Outputs poses_out_dev [2 B] and updates_dev [B].  Bit for bit cvb_three_view_optimize_l2 with
 * adaptive = 1 (include/cvb200_opt.h) for every problem of at most CVB_CONSTRAINTS_MAX_LANDMARKS landmarks; a larger problem is
 * CVB_EUNSUPPORTED (the offsets are read back to check it). */
int cvb_three_view_adaptive_optimize_l2_dev(cvb_ctx *ctx, const cvb_pose *poses_dev, uint32_t B, const double *obs_dev,
                                            const uint32_t *offsets_dev, uint32_t iterations, cvb_pose *poses_out_dev, uint32_t *updates_dev);

#ifdef __cplusplus
}
#endif
#endif /* CVB200_CONSTRAINTS_H */
