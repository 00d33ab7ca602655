/* include/cvb200_register.h -- C ABI of cv-sfm's frame registration on the device.
 *
 *   cvb_register_frame_dev    <- VSlam::register_frame / register_frame_subset (cv-sfm/src/lib.rs:1452-1812) for one new frame against
 *                                one reconstruction snapshot, from the frame's descriptors and bearings to Some((pose, matches)) / None
 *   cvb_register_frame        <- the same on host inputs, validated first
 *   cvb_register_check        <- that validation alone (host, no device needed)
 *   cvb_register_cfg_default  <- the defaults of the settings it reads (cv-sfm/src/settings.rs:324-387)
 *
 * Library: libcvb200_register.so, a module over libcvb200.so that takes its contexts (link with -lcvb200_register -lcvb200).  The
 * conventions of include/cvb200.h hold: return codes, HOST pointers unless the name ends in _dev, no CPU fallback.
 *
 * The snapshot is laid out as in include/cvb200_constraints.h (poses, the view CSR with its bearings, the landmark CSR of (view, feature)),
 * plus descriptors[view_offsets[V]][64] on the view CSR: a view's features are its frame's features.  The new frame comes as
 * cvb_frame_features_batch produces it: descriptors[N][64] and unit bearings[N][3].  view_matches[H] (HOST, duplicates allowed) are the
 * views matched against.  The caller's cvb_arrsac_cfg and cvb_rng are VSlam's single_view_consensus; the cvb_triangulator (methods 0-2)
 * is VSlam's triangulator.
 *
 * Semantics, step by step:
 *   1. subsets (register_frame, lib.rs:1789-1811): features 0 .. min(single_view_initial_features, N), then end .. min(2 end, N), until
 *      a subset succeeds or end == N; the status is that of the last subset tried;
 *   2. original_matches accumulates across subsets (lib.rs:1458, 1533-1540): only the new range is matched each time, and the claim filter
 *      and the sort of step 4 run over the whole list;
 *   3. per feature of the range (lib.rs:1468-1541): the 3 nearest features of every view in view_matches; each landmark keeps its best
 *      distance; the best three landmarks; d0 + single_view_match_better_by <= d1 is a unique match (l0); otherwise
 *      d1 + better_by <= d2 makes the merge pair (l0, l1) when the two share no view (are_landmarks_sharing_view, lib.rs:1435-1449);
 *      fewer than three distinct landmarks is where the reference panics (lib.rs:1510-1514): CVB_REGISTER_PANIC;
 *   4. claim filter and order (lib.rs:1551-1576): every match one of whose landmarks is claimed by more than one match is dropped; the
 *      rest are stable-sorted by descending summed observation count;
 *   5. robust points (lib.rs:1583-1602): triangulate_landmark_robust (lib.rs:2975-3000) for a single landmark,
 *      triangulate_merged_landmark_robust (lib.rs:2940-2972) for a pair: the two landmarks' observations concatenated, a's first, with
 *      min(robust_minimum_observations, V); matches_3d are the (feature bearing, homogeneous world point) of the matches that have one,
 *      in list order; fewer than single_view_minimum_landmarks of them is CVB_REGISTER_FEW_ROBUST_LANDMARKS;
 *   6. consensus (lib.rs:1619-1641): P3P ARRSAC over matches_3d (cvb_arrsac_p3p_dev), None is CVB_REGISTER_NO_CONSENSUS; its inliers,
 *      in the order it returns them, up to single_view_optimization_num_matches; robust_minimum_matches = that count / 2;
 *   7. the filter loop (lib.rs:1643-1693), single_view_filter_loop_iterations times: at most robust_minimum_matches left is
 *      CVB_REGISTER_FILTER_HALF (result.iteration = the iteration); single_view_simple_optimize_l2 (rate, single_view_patience); the
 *      matches consistent under the new pose whose robust point exists, in list order, up to single_view_optimization_num_matches;
 *   8. the final stage (lib.rs:1701-1775): at most robust_minimum_matches left is CVB_REGISTER_FINAL_HALF; one more optimisation; the
 *      consistent matches with a robust point at most robust_minimum_matches is CVB_REGISTER_FINAL_ROBUST_HALF; the consistent matches
 *      (robust point or not) are the result, fewer than single_view_minimum_robust_landmarks of them is CVB_REGISTER_FEW_MATCHES.
 * is_observation_consistent (lib.rs:2622-2655): with one other observation, is_bi_landmark_robust (lib.rs:1306-1318) of
 * other_pose * pose^-1 with maximum_sine_distance; otherwise the other observations followed by the new (pose, bearing) are triangulated
 * and every one's cosine distance must be strictly below maximum_cosine_distance (a failed triangulation is inconsistent).
 * The generator advances as the reference's model_inliers calls advance it: once per subset that reaches the consensus.
 *
 * UNPINNED, where the reference's order is not defined: the k-NN is exact (the reference's HggLite::knn is approximate) and ties go to
 * the lower feature index, as cvb_hamming_knn does; the best three landmarks are taken by (distance, landmark index) (HashMap order
 * upstream); observations are taken in the caller's order.  The result matches are listed ascending by feature; the reference returns
 * a HashMap, whose order is immaterial: it is add_view's existing_landmark closure. */
#ifndef CVB200_REGISTER_H
#define CVB200_REGISTER_H
#include "cvb200.h"
#include "cvb200_tri.h"

#ifdef __cplusplus
extern "C" {
#endif

/* result.status: one per `return None` of the reference, and its panic */
#define CVB_REGISTER_OK 0
#define CVB_REGISTER_FEW_ROBUST_LANDMARKS 1   /* matches_3d < single_view_minimum_landmarks (lib.rs:1604) */
#define CVB_REGISTER_NO_CONSENSUS 2           /* model_inliers is None (lib.rs:1623) */
#define CVB_REGISTER_FILTER_HALF 3            /* at most half left in filter iteration result.iteration (lib.rs:1650) */
#define CVB_REGISTER_FINAL_HALF 4             /* at most half left before the final optimisation (lib.rs:1701) */
#define CVB_REGISTER_FINAL_ROBUST_HALF 5      /* final robust count at most half (lib.rs:1738) */
#define CVB_REGISTER_FEW_MATCHES 6            /* final matches < single_view_minimum_robust_landmarks (lib.rs:1768) */
#define CVB_REGISTER_PANIC 7                  /* a feature with fewer than three distinct candidate landmarks (lib.rs:1511-1513) */

#define CVB_REGISTER_NONE 0xffffffffu         /* landmark_b of a single-landmark match */
#define CVB_REGISTER_STATS_ITERATIONS 16      /* filter-loop iterations whose match count the statistics record */

/* the cv-sfm settings register_frame reads (cv-sfm/src/settings.rs) */
typedef struct {
    double single_view_optimization_rate;                            /* 1e-3    settings.rs:373-375 */
    double maximum_sine_distance;                                    /* 0.1     settings.rs:328-330 */
    double maximum_cosine_distance;                                  /* 1e-5    settings.rs:324-326 */
    double robust_observation_incidence_minimum_cosine_distance;     /* 1e-3    settings.rs:348-350 */
    uint32_t single_view_match_better_by;                            /* 24      settings.rs:385-387 */
    uint32_t single_view_initial_features;                           /* 8192    settings.rs:369-371 */
    uint32_t single_view_minimum_landmarks;                          /* 32      settings.rs:377-379 */
    uint32_t single_view_optimization_num_matches;                   /* 2048    settings.rs:357-359 */
    uint32_t single_view_filter_loop_iterations;                     /* 5       settings.rs:361-363 */
    uint32_t single_view_patience;                                   /* 100000  settings.rs:365-367 */
    uint32_t single_view_minimum_robust_landmarks;                   /* 64      settings.rs:381-383 */
    uint32_t robust_minimum_observations;                            /* 3       settings.rs:344-346 */
} cvb_register_cfg;

/* one final match: landmark_b is CVB_REGISTER_NONE for a single landmark */
typedef struct {
    uint32_t feature, landmark_a, landmark_b;
} cvb_register_match;

typedef struct {
    int32_t status;                /* CVB_REGISTER_* of the last subset tried */
    uint32_t iteration;            /* the filter iteration of CVB_REGISTER_FILTER_HALF, else 0 */
    uint32_t n_matches;            /* matches written (CVB_REGISTER_OK only, else 0) */
    uint32_t n_inliers;            /* the consensus' inliers in the last subset tried (0 when it found nothing or did not run) */
    cvb_pose pose;                 /* WorldToCamera (CVB_REGISTER_OK only) */
} cvb_register_result;

/* optional statistics, of the last subset tried */
typedef struct {
    uint32_t subsets;              /* subsets tried */
    uint32_t matches;              /* original_matches accumulated */
    uint32_t claimed;              /* after the claim filter */
    uint32_t matches_3d;           /* with a robust point */
    uint32_t inliers;              /* the consensus' inliers (before the cap) */
    uint32_t final_robust;         /* final_num_robust_matches */
    uint32_t final_matches;        /* the consistent matches after the final optimisation */
    uint32_t iterations;           /* filter iterations entered (the final stage not counted) */
    uint32_t filter_matches[CVB_REGISTER_STATS_ITERATIONS];   /* matches_3d.len() checked at the start of iteration i (the first 16) */
    uint32_t final_stage_matches;  /* matches_3d.len() checked before the final optimisation */
    uint32_t reserved[3];
} cvb_register_stats;

void cvb_register_cfg_default(cvb_register_cfg *cfg);

/* Validates a snapshot and the view matches on the host: cvb_view_constraints_check's snapshot rules with view_matches as the queries
 * (0, or CVB_EINVAL for a NULL array, a malformed snapshot or a view out of range). */
int cvb_register_check(uint32_t V, const uint32_t *view_offsets, const uint32_t *view_landmarks, uint32_t L,
                       const uint32_t *landmark_offsets, const uint32_t *observations, const uint32_t *view_matches, uint32_t H);

/* Device inputs: the snapshot (poses_dev [V], view_offsets_dev [V + 1], view_landmarks_dev, bearings_dev and descriptors_dev on the view
 * CSR (n_features = view_offsets[V] rows), landmark_offsets_dev [L + 1], observations_dev [n_observations][2]); the new frame's
 * new_descriptors_dev [N][64] and new_bearings_dev [N][3]; view_matches HOST [H].  The descriptor arrays must be 16-byte aligned.
 * arrsac, rng: HOST; *rng is advanced past the draws of every consensus run.  Outputs (device): result_dev, matches_dev [N] (the first
 * result.n_matches written), inliers_dev [N] (may be NULL: the last subset's consensus inliers, indices into its matches_3d in the order
 * the consensus returns them, the first result.n_inliers written), stats_dev (may be NULL).  The view offsets are read back once; then the host waits once per subset, for
 * the generator commit and the status.  Triangulator methods 3-5 are CVB_EUNSUPPORTED; a NULL argument not marked optional, V = 0, a
 * view match >= V, view_offsets[V] != n_features, or single_view_initial_features = 0 with N > 0 (the reference's loop never ends
 * there) is CVB_EINVAL.  The two CSRs must agree (a precondition here; cvb_register_frame
 * checks it).  Returns when the outputs are written. */
int cvb_register_frame_dev(cvb_ctx *ctx, const cvb_register_cfg *cfg, const cvb_triangulator *tri, const cvb_arrsac_cfg *arrsac,
                           cvb_rng *rng, uint32_t V, const cvb_pose *poses_dev, const uint32_t *view_offsets_dev,
                           const uint32_t *view_landmarks_dev, const double *bearings_dev, const uint8_t *descriptors_dev, uint32_t n_features,
                           uint32_t L, const uint32_t *landmark_offsets_dev, const uint32_t *observations_dev, uint32_t n_observations,
                           const uint8_t *new_descriptors_dev, const double *new_bearings_dev, uint32_t N, const uint32_t *view_matches,
                           uint32_t H, cvb_register_result *result_dev, cvb_register_match *matches_dev, uint32_t *inliers_dev,
                           cvb_register_stats *stats_dev);

/* The same on HOST arrays (validated by cvb_register_check first); outputs are host arrays as above. */
int cvb_register_frame(cvb_ctx *ctx, const cvb_register_cfg *cfg, const cvb_triangulator *tri, const cvb_arrsac_cfg *arrsac, cvb_rng *rng,
                       uint32_t V, const cvb_pose *poses, const uint32_t *view_offsets, const uint32_t *view_landmarks, const double *bearings,
                       const uint8_t *descriptors, uint32_t L, const uint32_t *landmark_offsets, const uint32_t *observations,
                       const uint8_t *new_descriptors, const double *new_bearings, uint32_t N, const uint32_t *view_matches, uint32_t H,
                       cvb_register_result *result, cvb_register_match *matches, uint32_t *inliers,
                       cvb_register_stats *stats);

#ifdef __cplusplus
}
#endif
#endif /* CVB200_REGISTER_H */
