/* include/cvb200_try_init.h -- C ABI of cv-sfm's reconstruction creation on the device: a frame and its free frames to the first snapshot
 * of a new reconstruction, so that a reconstruction is born where cvb_incorporate_frame_dev and the other snapshot calls take it over.
 *
 *   cvb_add_reconstruction_dev  <- VSlamData::add_reconstruction (cv-sfm/src/lib.rs:377-427): the chosen frames, the two init poses and the
 *                                  three match lists of init_reconstruction to a three-view snapshot
 *   cvb_try_init_dev            <- VSlam::try_init (lib.rs:814-839): cvb_two_view_options_dev, cvb_init_reconstruction_dev and, when
 *                                  accepted, add_reconstruction, with no host copy of the lists or the snapshot
 *   cvb_add_reconstruction, cvb_try_init
 *                               <- the same on host inputs, validated first
 *   cvb_try_init_check          <- that validation alone (host, no device needed)
 *
 * Library: libcvb200_try_init.so, a module over libcvb200.so that takes its contexts (link with -lcvb200_try_init -lcvb200).  The
 * conventions of include/cvb200.h hold: return codes, HOST pointers unless the name ends in _dev, no CPU fallback.
 *
 * The frame store is cvb_frame_features_batch_dev's: descriptors [frames][cap][64], counts [frames], bearings [frames][cap][3] and
 * optional colours [frames][cap][3], frame b at row b * cap; a count above cap is read as cap.  The output is the snapshot of
 * include/cvb200_incorporate.h with its counts (merges = 0).
 *
 * add_reconstruction(center, first, second, first_pose, second_pose, combined, first_matches, second_matches):
 *   views         0 = center with the identity pose, 1 = first with first_pose, 2 = second with second_pose (the CameraToCamera poses of
 *                 the init, used as WorldToCamera poses: the center is the world, lib.rs:400-418); each view has all counts[frame]
 *                 features of its frame in feature order (add_view iterates descriptor_features), with their bearings, descriptors and
 *                 colours;
 *   landmarks     landmark c for each center feature c, in feature order; then one new landmark per feature of the first view that is
 *                 not mapped, in feature order, where feature f is mapped to landmark c when [c, f] is in first_matches or (c, f, _) in
 *                 combined; then the same for the second view with second_matches and (c, _, s);
 *   observations  of a landmark in view order: (0, c), then (1, f), then (2, s); so n_observations = n_features;
 *   constraints   exactly one: views (0, 1, 2), poses [first_pose, second_pose], landmarks 0 (ignored downstream).
 * The reconstruction is fresh, so its DenseSlotMaps have seen no removal and iterate in insertion order: the view, landmark, view-CSR and
 * constraint orders EQUAL the reference's.  Only the order of the observations inside a landmark comes from a HashMap there; it is
 * UNPINNED in the reference and PINNED here as view order.  A caller's keys follow the output directly: view i is frames[i], landmark
 * index = slot-map insertion order.
 *
 * The lists are init_reconstruction's (cvb_init_reconstruction_dev's combined_dev / first_matches_dev / second_matches_dev, their lengths
 * in its cvb_init_result).  cvb_try_init_check and the host forms refuse with CVB_EINVAL:
 *   - a c, f or s out of range of its frame's count (the reference would index out of bounds);
 *   - a feature of the first view that appears twice across first_matches and combined, or a center feature mapped twice into the first
 *     view (the reference's HashMap insert would silently drop an entry or an observation); the same two for the second view;
 *   - two equal frames.
 * The lists of cvb_init_reconstruction_dev satisfy all of these (symmetric matching is one-to-one, and first_matches / second_matches
 * exclude the common centers, lib.rs:1212-1246).  For the _dev forms they are preconditions, and a broken one never makes a call read or
 * write out of bounds.
 *
 * try_init(center, options[F]): cvb_two_view_options_dev over center and the options with generator rngs[f] for option f, committed as
 * cvb_arrsac_commit_rng_batch commits them (every rngs[f] is advanced, whatever the outcome); cvb_init_reconstruction_dev; and, when its
 * status is CVB_INIT_ACCEPTED, add_reconstruction of (center, options[first], options[second]).  No snapshot is written otherwise.  The
 * host waits are the generators' commit, the init's (one word per wave), one read of its result and the final one; the lists and the
 * snapshot never leave the device.
 *
 * Output capacities (rows): poses 3, view_offsets 4, features (view_landmarks, bearings, descriptors, colours) and observations 3 cap,
 * landmark_offsets 3 cap + 1, constraints 1. */
#ifndef CVB200_TRY_INIT_H
#define CVB200_TRY_INIT_H
#include "cvb200.h"
#include "cvb200_tri.h"
#include "cvb200_batch.h"
#include "cvb200_init.h"
#include "cvb200_constraints.h"
#include "cvb200_reconstruction.h"
#include "cvb200_register.h"
#include "cvb200_incorporate.h"

#ifdef __cplusplus
extern "C" {
#endif

#define CVB_TRY_INIT_NO_FRAME 0xffffffffu   /* frames[1], frames[2] when no pair was decided */

/* cvb_try_init_result.status */
#define CVB_TRY_INIT_CREATED 0                /* accepted: the snapshot is written */
#define CVB_TRY_INIT_NONE 1                   /* init_reconstruction returned None (CVB_INIT_NONE): no snapshot */
#define CVB_TRY_INIT_NONE_BEARING_PAIRS 2     /* ... through the bearing-pair abort (CVB_INIT_NONE_BEARING_PAIRS): no snapshot */

typedef struct {
    int32_t status;                /* CVB_TRY_INIT_* */
    uint32_t frames[3];            /* the frames of views 0, 1, 2: center, options[init.first], options[init.second] (decided pair) */
    cvb_init_result init;          /* cvb_init_reconstruction_dev's result */
    cvb_incorporate_counts counts; /* of the snapshot (all 0 when there is none) */
} cvb_try_init_result;

/* Validates on the host: n_center, n_first, n_second the three frames' feature counts; combined [n_combined][3], first_matches
 * [n_first_matches][2], second_matches [n_second_matches][2] (each may be NULL when its length is 0).  0, or CVB_EINVAL. */
int cvb_try_init_check(uint32_t n_center, uint32_t n_first, uint32_t n_second, uint32_t center, uint32_t first, uint32_t second,
                       const uint32_t *combined, uint32_t n_combined, const uint32_t *first_matches, uint32_t n_first_matches,
                       const uint32_t *second_matches, uint32_t n_second_matches);

/* add_reconstruction on device arrays: the frame store (colors_dev may be NULL, and then colors_out_dev too), center / first / second
 * (host), init_result_dev [1] (its n_combined, n_first_matches, n_second_matches, first_pose and second_pose are read on the device),
 * combined_dev [cap][3], first_matches_dev and second_matches_dev [cap][2].  Outputs as in the capacity table and counts_dev [1].  A NULL
 * argument not marked optional, cap = 0, a frame index >= frames or two equal frames is CVB_EINVAL.  Returns when the outputs are
 * written. */
int cvb_add_reconstruction_dev(cvb_ctx *ctx, const uint8_t *descriptors_dev, const uint32_t *counts_dev, const double *bearings_dev,
                               const uint8_t *colors_dev, uint32_t frames, uint32_t cap, uint32_t center, uint32_t first, uint32_t second,
                               const cvb_init_result *init_result_dev, const uint32_t *combined_dev, const uint32_t *first_matches_dev,
                               const uint32_t *second_matches_dev, cvb_pose *poses_out_dev, uint32_t *view_offsets_out_dev,
                               uint32_t *view_landmarks_out_dev, double *bearings_out_dev, uint8_t *descriptors_out_dev, uint8_t *colors_out_dev,
                               uint32_t *landmark_offsets_out_dev, uint32_t *observations_out_dev, cvb_view_constraint *constraints_out_dev,
                               cvb_incorporate_counts *snapshot_counts_dev);

/* The same on HOST arrays (validated by cvb_try_init_check first): the frame store [frames][cap][...], init_result HOST [1], the lists
 * with the lengths it gives; outputs are host arrays, and *snapshot_counts says how many rows of each are valid.  Returns when they are
 * written. */
int cvb_add_reconstruction(cvb_ctx *ctx, const uint8_t *descriptors, const uint32_t *counts, const double *bearings, const uint8_t *colors,
                           uint32_t frames, uint32_t cap, uint32_t center, uint32_t first, uint32_t second, const cvb_init_result *init_result,
                           const uint32_t *combined, const uint32_t *first_matches, const uint32_t *second_matches, cvb_pose *poses_out,
                           uint32_t *view_offsets_out, uint32_t *view_landmarks_out, double *bearings_out, uint8_t *descriptors_out,
                           uint8_t *colors_out, uint32_t *landmark_offsets_out, uint32_t *observations_out, cvb_view_constraint *constraints_out,
                           cvb_incorporate_counts *snapshot_counts);

/* try_init on device arrays: init_cfg, tri (methods 0-2; 3-5 are CVB_EUNSUPPORTED), arrsac and better_by as cvb_two_view_options_dev
 * takes them, rngs HOST [F] (advanced), the frame store, center and options HOST [F] (F above CVB_ARRSAC_BATCH_MAX is CVB_EUNSUPPORTED).
 * Outputs as in the capacity table (written only when the status is CVB_TRY_INIT_CREATED) and result_dev [1].  Arguments are refused as
 * by cvb_two_view_options_dev, cvb_init_reconstruction_dev and cvb_add_reconstruction_dev.  Returns when the outputs are written. */
int cvb_try_init_dev(cvb_ctx *ctx, const cvb_init_cfg *init_cfg, const cvb_triangulator *tri, const cvb_arrsac_cfg *arrsac, cvb_rng *rngs,
                     uint32_t better_by, const uint8_t *descriptors_dev, const uint32_t *counts_dev, const double *bearings_dev,
                     const uint8_t *colors_dev, uint32_t frames, uint32_t cap, uint32_t center, const uint32_t *options, uint32_t F,
                     cvb_pose *poses_out_dev, uint32_t *view_offsets_out_dev, uint32_t *view_landmarks_out_dev, double *bearings_out_dev,
                     uint8_t *descriptors_out_dev, uint8_t *colors_out_dev, uint32_t *landmark_offsets_out_dev, uint32_t *observations_out_dev,
                     cvb_view_constraint *constraints_out_dev, cvb_try_init_result *result_dev);

/* The same on HOST arrays: the frame store [frames][cap][...] is uploaded, the outputs are host arrays. */
int cvb_try_init(cvb_ctx *ctx, const cvb_init_cfg *init_cfg, const cvb_triangulator *tri, const cvb_arrsac_cfg *arrsac, cvb_rng *rngs,
                 uint32_t better_by, const uint8_t *descriptors, const uint32_t *counts, const double *bearings, const uint8_t *colors,
                 uint32_t frames, uint32_t cap, uint32_t center, const uint32_t *options, uint32_t F, cvb_pose *poses_out,
                 uint32_t *view_offsets_out, uint32_t *view_landmarks_out, double *bearings_out, uint8_t *descriptors_out, uint8_t *colors_out,
                 uint32_t *landmark_offsets_out, uint32_t *observations_out, cvb_view_constraint *constraints_out, cvb_try_init_result *result);

#ifdef __cplusplus
}
#endif
#endif /* CVB200_TRY_INIT_H */
