/* include/cvb200_init.h -- C ABI of cv-sfm's three-view initialisation on the device.
 *
 *   cvb_init_reconstruction_dev  <- VSlam::init_reconstruction's choice of the three-view initialisation over every pair of two-view
 *                                   options (cv-sfm/src/lib.rs:986-1303), on the outputs of cvb_two_view_options_dev
 *                                   (include/cvb200_batch.h, which is lib.rs:966-985)
 *   cvb_init_cfg_default         <- the defaults of the settings it reads (cv-sfm/src/settings.rs:320-428)
 *
 * Library: libcvb200_init.so, a module over libcvb200.so that takes its contexts (link with -lcvb200_init -lcvb200).  The conventions of
 * include/cvb200.h hold: return codes, HOST pointers unless the name ends in _dev, no CPU fallback.
 *
 * Semantics, for the options that take part -- found_dev[f] != 0 and n_inliers_dev[f] >= two_view_minimum_robust_matches (lib.rs:977-985
 * with the rule of lib.rs:1421) -- taken in pairs (first, second) in itertools' tuple_combinations order of their option indices:
 *   - option f's matches are pairs_dev[f][inliers_dev[f][i]], i < n_inliers_dev[f], in inlier order (lib.rs:1412);
 *   - common: the first option's matches, in order, whose center feature is also matched by the second option, as (c, f, s) triples.
 *     The reference shuffles them with VSlam's shared generator (lib.rs:999); here they stay in first-match order, so parity with the
 *     shuffled order is UNPINNED (the relative scale's median, the take-limited optimisation sets and every result downstream of them
 *     can differ from a run of the reference);
 *   - relative scales (lib.rs:1002-1059), the first optimisation set and its robust bearing pairs (lib.rs:1064-1106; too few pairs makes
 *     the WHOLE call None, not just the pair), the filter loop (lib.rs:1108-1187) and the final lists and counts (lib.rs:1189-1300) are
 *     restated exactly, with the triangulator `tri` (cv-sfm's TriangulatorObservations: methods 0-2) and three_view_simple_optimize_l2
 *     at rate 0.001 for three_view_patience iterations (k_three_view_opt of cvb_three_view_optimize_l2);
 *   - the result is the first pair that is accepted or that hits the bearing-pair None; no such pair: None.
 * The pairs run speculatively in waves of as many pairs as the device has streaming multiprocessors; the host reads one word after each
 * wave and stops at the first wave that holds a decisive pair.  Results do not depend on the wave size.
 *
 * The call returns once the decision is known; the gather of the winner's lists is enqueued on the context's stream after it. */
#ifndef CVB200_INIT_H
#define CVB200_INIT_H
#include "cvb200.h"
#include "cvb200_tri.h"
#include "cvb200_batch.h"

#ifdef __cplusplus
extern "C" {
#endif

/* cvb_init_result.status */
#define CVB_INIT_NONE 0                /* no pair decided (lib.rs:1302-1303), or fewer than two options take part */
#define CVB_INIT_ACCEPTED 1            /* lib.rs:1294-1300 */
#define CVB_INIT_NONE_BEARING_PAIRS 2  /* lib.rs:1100-1106: the decisive pair has too few robust bearing pairs; the call is None */

/* cvb_init_pair_stats.outcome */
#define CVB_INIT_PAIR_NOT_EVALUATED 0  /* after the decisive pair, or beyond the pairs that exist */
#define CVB_INIT_PAIR_ACCEPTED 1
#define CVB_INIT_PAIR_BEARING_PAIRS 2  /* decisive None, lib.rs:1105 */
#define CVB_INIT_PAIR_FEW_SCALES 3     /* fewer than three_view_minimum_relative_scales ratios, lib.rs:1039-1048 */
#define CVB_INIT_PAIR_FEW_MATCHES 4    /* an optimisation set of fewer than 32 triples, lib.rs:1118-1124, 1167-1173 */
#define CVB_INIT_PAIR_HALF_MATCHES 5   /* an optimisation set of at most half the first one's size, lib.rs:1126-1129, 1175-1178 */
#define CVB_INIT_PAIR_HALF_ROBUST 6    /* final robust count at most half the first set's size, lib.rs:1281-1284 */
#define CVB_INIT_PAIR_FEW_ROBUST 7     /* final robust count below three_view_minimum_robust_matches, lib.rs:1286-1292 */

/* the cv-sfm settings init_reconstruction reads (cv-sfm/src/settings.rs) */
typedef struct {
    double robust_observation_incidence_minimum_cosine_distance;   /* 1e-3  settings.rs:348-350 */
    double robust_view_bearing_pair_minimum_cosine_distance;       /* 1e-2  settings.rs:332-334 */
    double maximum_cosine_distance;                                /* 1e-5  settings.rs:324-326 */
    double maximum_sine_distance;                                  /* 0.1   settings.rs:328-330 */
    uint32_t two_view_minimum_robust_matches;                      /* 256   settings.rs:393-395 */
    uint32_t three_view_minimum_relative_scales;                   /* 16    settings.rs:413-415 */
    uint32_t three_view_optimization_landmarks;                    /* 1024  settings.rs:421-423 */
    uint32_t robust_view_num_robust_bearing_pair;                  /* 3     settings.rs:336-338 */
    uint32_t three_view_filter_loop_iterations;                    /* 8     settings.rs:417-419 */
    uint32_t three_view_patience;                                  /* 65536 settings.rs:409-411 */
    uint32_t three_view_minimum_robust_matches;                    /* 32    settings.rs:425-427 */
    uint32_t reserved;                                             /* 0 */
} cvb_init_cfg;

/* the decision; first / second are positions in options[] */
typedef struct {
    int32_t status;
    uint32_t pair;                 /* the decisive pair's index in combination order (status != CVB_INIT_NONE) */
    uint32_t first, second;
    uint32_t n_pairs;              /* pairs of the options that take part */
    uint32_t n_combined, n_first_matches, n_second_matches;
    cvb_pose first_pose, second_pose;   /* CameraToCamera center -> first / second (status == CVB_INIT_ACCEPTED) */
} cvb_init_result;

/* what happened to one pair (indexed by the pair's position in combination order) */
typedef struct {
    int32_t outcome;               /* CVB_INIT_PAIR_* */
    uint32_t first, second;        /* positions in options[] */
    uint32_t scales;               /* relative scales kept */
    double median_scale;           /* the scale applied to the second pose (0 when too few scales) */
    uint64_t bearing_pairs;        /* robust bearing pairs of the first optimisation set */
    uint32_t common;               /* common triples */
    uint32_t opti;                 /* size of the first optimisation set */
    uint32_t updates;              /* pose updates of all the pair's optimisations */
    uint32_t robust;               /* final robust count (accepted or rejected at lib.rs:1281-1292) */
} cvb_init_pair_stats;

void cvb_init_cfg_default(cvb_init_cfg *cfg);

/* The three-view initialisation of frame `center` over the two-view options options[0 .. F) (HOST array of frame indices):
 *   bearings_dev: frames x cap x 3 f64, frame b at b * cap (cvb_frame_features_batch_dev);
 *   pairs_dev (F x cap x 2), n_pairs_dev (F), model_dev (F), inliers_dev (F x cap), n_inliers_dev (F), found_dev (F): the outputs of
 *   cvb_two_view_options_dev for the same center, options and cap;
 *   tri: the triangulator (methods 0-2; 3-5 are CVB_EUNSUPPORTED).
 * Outputs (device): result_dev; combined_dev (cap x 3: center, first, second feature), first_matches_dev and second_matches_dev (cap x 2:
 * center feature, option feature), in the reference's order, filled when accepted; stats_dev (may be NULL): F * (F - 1) / 2 entries.
 * F = 0 or fewer than two taking part: result None.  F above CVB_ARRSAC_BATCH_MAX and methods 3-5 are CVB_EUNSUPPORTED; a NULL argument
 * not marked optional, cap = 0, center or an option >= frames are CVB_EINVAL. */
int cvb_init_reconstruction_dev(cvb_ctx *ctx, const cvb_init_cfg *cfg, const cvb_triangulator *tri, const double *bearings_dev, uint32_t frames,
                                uint32_t cap, uint32_t center, const uint32_t *options, uint32_t F, const uint32_t *pairs_dev,
                                const uint32_t *n_pairs_dev, const cvb_pose *model_dev, const uint32_t *inliers_dev,
                                const uint32_t *n_inliers_dev, const int32_t *found_dev, cvb_init_result *result_dev, uint32_t *combined_dev,
                                uint32_t *first_matches_dev, uint32_t *second_matches_dev, cvb_init_pair_stats *stats_dev);

#ifdef __cplusplus
}
#endif
#endif /* CVB200_INIT_H */
