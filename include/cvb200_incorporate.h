/* include/cvb200_incorporate.h -- C ABI of cv-sfm's frame incorporation on the device: the reconstruction edits between register_frame,
 * record_view_constraints and optimize_reconstruction, so that a reconstruction can stay on the device from one tracked frame to the next.
 *
 *   cvb_add_view_dev            <- VSlamData::add_view with merge_landmarks (cv-sfm/src/lib.rs:432-483, 699-721), one new view
 *   cvb_apply_optimization_dev  <- the slot-map edits optimize_reconstruction makes (remove_view lib.rs:517-546, split_landmark and
 *                                  split_observation lib.rs:552-588), replayed from cvb_optimize_reconstruction's view and observation states
 *   cvb_incorporate_frame_dev   <- VSlam::incorporate_frame (lib.rs:2067-2087) followed by the optimize_reconstruction that try_localize /
 *                                  try_localize_and_incorporate run right after it (lib.rs:882-890, 940-945): register_frame, add_view,
 *                                  record_view_constraints (remove_view when refused), optimize_reconstruction and its edits
 *   cvb_add_view, cvb_apply_optimization, cvb_incorporate_frame
 *                               <- the same on host inputs, validated first
 *   cvb_incorporate_check       <- that validation alone (host, no device needed)
 *
 * Library: libcvb200_incorporate.so, a module over libcvb200.so that takes its contexts (link with -lcvb200_incorporate -lcvb200).  The
 * conventions of include/cvb200.h hold: return codes, HOST pointers unless the name ends in _dev, no CPU fallback.  The settings are the
 * existing ones: cvb_register_cfg, cvb_constraints_cfg, cvb_recon_cfg, a cvb_triangulator of methods 0-2, cvb_arrsac_cfg and its cvb_rng.
 *
 * The snapshot is register_frame's (include/cvb200_register.h): poses[V], the view CSR view_offsets / view_landmarks with bearings[][3]
 * and descriptors[][64], the landmark CSR landmark_offsets / observations of (view, feature), plus optional colors[][3] on the view CSR
 * (so that cvb_export_reconstruction can run on the result), and the constraints cvb_view_constraint[C] in the caller's order.  Every call
 * is a pure function from one snapshot to the next: nothing is kept on the device between calls, the caller's slot-map keys stay the
 * caller's, and the index maps returned (old index -> new index, or CVB_INCORPORATE_NONE) let the caller follow.  descriptors and colors
 * are optional in add_view and apply (NULL in, NULL out); the outputs never alias the inputs.
 *
 * add_view, in these PINNED orders (the reference's come from a DenseSlotMap and HashMaps, so its own are unpinned):
 *   views         the old views keep their indices; the new view is V, its N features appended to the view CSR;
 *   landmarks     the old landmarks in index order minus every match's landmark_b, then one new singleton per unmatched feature, in
 *                 feature order;
 *   observations  a survivor keeps its observations in order; a merged landmark_a takes a's, then b's, then (V, feature); a single match
 *                 its own, then (V, feature); a singleton (V, feature);
 *   view CSR      every old entry remapped (b's features now name a), then the new view's entries;
 *   landmark_map  [L] old -> new; b maps to a's new index.
 * Matches are register_frame's cvb_register_match list: ascending by feature, each feature < N, landmark_b = CVB_REGISTER_NONE for a
 * single landmark, a != b and both < L, no landmark in two matches, and a merged pair sharing no view (merge_landmarks' assert!,
 * lib.rs:714-718).  cvb_add_view and cvb_incorporate_check refuse a list that breaks one of these; for cvb_add_view_dev they are
 * preconditions, and a broken one never makes it read or write out of bounds.
 *
 * apply_optimization, from cvb_optimize_reconstruction(_dev)'s poses_out, view_state and obs_state with status CVB_RECON_KEPT:
 *   views         the kept views (CVB_RECON_VIEW_KEPT) in order, with their poses from poses_out; a removed view loses its features,
 *                 bearings, descriptors and colours;
 *   observations  CVB_RECON_OBS_KEPT stays in its landmark, in order; CVB_RECON_OBS_SPLIT becomes a landmark of its own;
 *                 CVB_RECON_OBS_DROPPED is gone (it must be exactly the observations of the removed views);
 *   landmarks     the old landmarks with at least one KEPT observation, in index order, then the split singletons in observation-CSR order.
 *                 This is exactly what the reference's remove_view + split_landmark + split_observation leave: remove_view deletes a
 *                 landmark when its last observation goes and otherwise only the observation; split_observation never splits a landmark's
 *                 last observation, and split_landmark keeps the first; so an old landmark survives exactly when one of its observations
 *                 was neither split off nor dropped;
 *   constraints   a constraint that contains a removed view is dropped (lib.rs:541-543); the rest keep their order with their views
 *                 renumbered, which keeps them ascending;
 *   view_map [V], landmark_map [L]: old -> new, or CVB_INCORPORATE_NONE.
 * Useful on its own after cvb_optimize_reconstruction or cv_b200's regenerate_reconstruction; incorporate_frame uses it for both of its
 * edits.
 *
 * incorporate_frame:
 *   1. register_frame (cvb_register_frame_dev: its per-subset host waits; the generator advances exactly as there); a failure returns the
 *      input snapshot unchanged (status CVB_INCORPORATE_NOT_REGISTERED, result.reg.status says why); its panic returns none;
 *   2. add_view of the registered pose and matches;
 *   3. cvb_view_constraints_dev of the new view (Q = 1); when record_view_constraints refuses it, remove_view of the new view, which is
 *      apply_optimization with the new view removed and every other state KEPT: the merges of step 2 persist, as in the reference
 *      (status CVB_INCORPORATE_REJECTED);
 *   4. otherwise cvb_optimize_reconstruction_dev over the old constraints followed by the new ones (a slot-map insert appends), then
 *      apply_optimization of its states (status CVB_INCORPORATE_KEPT); a removed reconstruction or the optimisation's panic returns none.
 * The view and landmark maps are composed from the input to the output; result.new_view is the new view's output index, or NONE.
 * The host reads back once per stage: the registration result with its matches (add_view's landmark count, L - merges + (N - matches),
 * follows from them on the host, without a wait of its own), the constraint result, the optimisation result and the output counts.
 *
 * Output capacities of the _dev forms (rows):
 *                 poses / view_map   view_offsets   features (view_landmarks, bearings, descriptors, colors)   landmark_offsets
 *                 observations       constraints
 *   add_view      V + 1              V + 2          n_features + N                                             L + N + 1
 *                 n_observations + N  -
 *   apply         V                  V + 1          n_features                                                 L + n_observations + 1
 *                 n_observations     C
 *   incorporate   V + 1              V + 2          n_features + N                                             L + N + n_observations + N + 1
 *                 n_observations + N  C + optimization_maximum_three_view_constraints
 * landmark_map has L rows and view_map V rows in every form; the counts written say how many rows of each output are valid. */
#ifndef CVB200_INCORPORATE_H
#define CVB200_INCORPORATE_H
#include "cvb200.h"
#include "cvb200_tri.h"
#include "cvb200_constraints.h"
#include "cvb200_reconstruction.h"
#include "cvb200_register.h"

#ifdef __cplusplus
extern "C" {
#endif

#define CVB_INCORPORATE_NONE 0xffffffffu   /* a map entry with no image */

/* cvb_incorporate_result.status */
#define CVB_INCORPORATE_KEPT 0                  /* accepted and optimised: the final snapshot */
#define CVB_INCORPORATE_NOT_REGISTERED 1        /* register_frame returned None (reg.status): the input snapshot */
#define CVB_INCORPORATE_REGISTER_PANIC 2        /* register_frame's panic: no snapshot */
#define CVB_INCORPORATE_REJECTED 3              /* record_view_constraints refused the view: add_view followed by remove_view */
#define CVB_INCORPORATE_REMOVED_CONSTRAINTS 4   /* optimize_reconstruction removed the reconstruction (CVB_RECON_REMOVED_CONSTRAINTS) */
#define CVB_INCORPORATE_REMOVED_FILTER 5        /* ... (CVB_RECON_REMOVED_FILTER) */
#define CVB_INCORPORATE_RECON_PANIC 6           /* optimize_reconstruction's panic (CVB_RECON_PANIC): no snapshot */

/* the sizes of a snapshot */
typedef struct {
    uint32_t V, n_features, L, n_observations, C;
    uint32_t merges;               /* add_view: the matches that merged two landmarks; apply: 0 */
} cvb_incorporate_counts;

typedef struct {
    int32_t status;                /* CVB_INCORPORATE_* */
    uint32_t new_view;             /* the new view's output index, or CVB_INCORPORATE_NONE */
    cvb_incorporate_counts counts; /* of the output snapshot (all 0 when there is none) */
    cvb_register_result reg;       /* step 1 */
    cvb_register_stats reg_stats;
    cvb_view_constraints_result con;   /* step 3 (zero when it did not run) */
    cvb_recon_result recon;        /* step 4 (zero when it did not run) */
    uint32_t reserved[2];
} cvb_incorporate_result;

/* Validates on the host, with cvb_optimize_reconstruction_check's snapshot and constraint rules: 0, or CVB_EINVAL.  With M > 0 it checks
 * an add_view's matches against N new features as above.  With view_state or obs_state given it checks an apply: n_view_state must be V
 * and n_obs_state n_observations, every state in range, an observation DROPPED exactly when its view is removed, and no landmark with
 * every observation SPLIT.  The two may be checked in one call; a NULL snapshot array, constraints == NULL with C > 0, matches == NULL
 * with M > 0, or one state array without the other is CVB_EINVAL. */
int cvb_incorporate_check(uint32_t V, const uint32_t *view_offsets, const uint32_t *view_landmarks, uint32_t L, const uint32_t *landmark_offsets,
                          const uint32_t *observations, const cvb_view_constraint *constraints, uint32_t C, uint32_t N,
                          const cvb_register_match *matches, uint32_t M, const uint8_t *view_state, uint32_t n_view_state,
                          const uint8_t *obs_state, uint32_t n_obs_state);

/* add_view on device arrays: the snapshot (n_features = view_offsets[V], n_observations = landmark_offsets[L], both checked against the
 * device), new_pose_dev [1], new_bearings_dev [N][3], new_descriptors_dev [N][64] and new_colors_dev [N][3] (each optional with its
 * snapshot array), matches_dev [M].  Outputs as in the capacity table; counts_dev [1].  A NULL argument not marked optional is
 * CVB_EINVAL.  Returns when the outputs are written. */
int cvb_add_view_dev(cvb_ctx *ctx, uint32_t V, const cvb_pose *poses_dev, const uint32_t *view_offsets_dev, const uint32_t *view_landmarks_dev,
                     const double *bearings_dev, const uint8_t *descriptors_dev, const uint8_t *colors_dev, uint32_t n_features, uint32_t L,
                     const uint32_t *landmark_offsets_dev, const uint32_t *observations_dev, uint32_t n_observations, const cvb_pose *new_pose_dev,
                     const double *new_bearings_dev, const uint8_t *new_descriptors_dev, const uint8_t *new_colors_dev, uint32_t N,
                     const cvb_register_match *matches_dev, uint32_t M, cvb_pose *poses_out_dev, uint32_t *view_offsets_out_dev,
                     uint32_t *view_landmarks_out_dev, double *bearings_out_dev, uint8_t *descriptors_out_dev, uint8_t *colors_out_dev,
                     uint32_t *landmark_offsets_out_dev, uint32_t *observations_out_dev, uint32_t *landmark_map_dev,
                     cvb_incorporate_counts *counts_dev);

/* The same on HOST arrays (validated by cvb_incorporate_check first); outputs are host arrays with the same capacities, counts [1]. */
int cvb_add_view(cvb_ctx *ctx, uint32_t V, const cvb_pose *poses, const uint32_t *view_offsets, const uint32_t *view_landmarks,
                 const double *bearings, const uint8_t *descriptors, const uint8_t *colors, uint32_t L, const uint32_t *landmark_offsets,
                 const uint32_t *observations, const cvb_pose *new_pose, const double *new_bearings, const uint8_t *new_descriptors,
                 const uint8_t *new_colors, uint32_t N, const cvb_register_match *matches, uint32_t M, cvb_pose *poses_out,
                 uint32_t *view_offsets_out, uint32_t *view_landmarks_out, double *bearings_out, uint8_t *descriptors_out, uint8_t *colors_out,
                 uint32_t *landmark_offsets_out, uint32_t *observations_out, uint32_t *landmark_map, cvb_incorporate_counts *counts);

/* apply_optimization on device arrays: the snapshot with poses_dev = optimize_reconstruction's poses_out, constraints_dev [C],
 * view_state_dev [V], obs_state_dev [n_observations].  Outputs as in the capacity table, view_map_dev [V], landmark_map_dev [L],
 * counts_dev [1].  Descriptor arrays must be 16-byte aligned; V = 0 is CVB_EINVAL.  The states are preconditions (cvb_apply_optimization checks them); an out-of-range one never makes the call read or
 * write out of bounds.  Returns when the outputs are written. */
int cvb_apply_optimization_dev(cvb_ctx *ctx, uint32_t V, const cvb_pose *poses_dev, const uint32_t *view_offsets_dev,
                               const uint32_t *view_landmarks_dev, const double *bearings_dev, const uint8_t *descriptors_dev,
                               const uint8_t *colors_dev, uint32_t n_features, uint32_t L, const uint32_t *landmark_offsets_dev,
                               const uint32_t *observations_dev, uint32_t n_observations, const cvb_view_constraint *constraints_dev, uint32_t C,
                               const uint8_t *view_state_dev, const uint8_t *obs_state_dev, cvb_pose *poses_out_dev, uint32_t *view_offsets_out_dev,
                               uint32_t *view_landmarks_out_dev, double *bearings_out_dev, uint8_t *descriptors_out_dev, uint8_t *colors_out_dev,
                               uint32_t *landmark_offsets_out_dev, uint32_t *observations_out_dev, cvb_view_constraint *constraints_out_dev,
                               uint32_t *view_map_dev, uint32_t *landmark_map_dev, cvb_incorporate_counts *counts_dev);

/* The same on HOST arrays (validated by cvb_incorporate_check first). */
int cvb_apply_optimization(cvb_ctx *ctx, uint32_t V, const cvb_pose *poses, const uint32_t *view_offsets, const uint32_t *view_landmarks,
                           const double *bearings, const uint8_t *descriptors, const uint8_t *colors, uint32_t L, const uint32_t *landmark_offsets,
                           const uint32_t *observations, const cvb_view_constraint *constraints, uint32_t C, const uint8_t *view_state,
                           const uint8_t *obs_state, cvb_pose *poses_out, uint32_t *view_offsets_out, uint32_t *view_landmarks_out,
                           double *bearings_out, uint8_t *descriptors_out, uint8_t *colors_out, uint32_t *landmark_offsets_out,
                           uint32_t *observations_out, cvb_view_constraint *constraints_out, uint32_t *view_map, uint32_t *landmark_map,
                           cvb_incorporate_counts *counts);

/* incorporate_frame on device arrays: the snapshot (descriptors required, colors optional with new_colors_dev and colors_out_dev),
 * constraints_dev [C], the new frame's new_descriptors_dev [N][64] (16-byte aligned), new_bearings_dev [N][3], new_colors_dev [N][3];
 * view_matches HOST [H]; arrsac and rng HOST (*rng advanced as cvb_register_frame advances it).  Outputs as in the capacity table, plus
 * view_map_dev [V], landmark_map_dev [L], matches_dev [N] (may be NULL: register_frame's matches, result.reg.n_matches of them) and
 * result_dev [1].  Arguments are refused as by cvb_register_frame_dev.  Returns when the outputs are written. */
int cvb_incorporate_frame_dev(cvb_ctx *ctx, const cvb_register_cfg *register_cfg, const cvb_constraints_cfg *constraints_cfg,
                              const cvb_recon_cfg *recon_cfg, const cvb_triangulator *tri, const cvb_arrsac_cfg *arrsac, cvb_rng *rng, uint32_t V,
                              const cvb_pose *poses_dev, const uint32_t *view_offsets_dev, const uint32_t *view_landmarks_dev,
                              const double *bearings_dev, const uint8_t *descriptors_dev, const uint8_t *colors_dev, uint32_t n_features,
                              uint32_t L, const uint32_t *landmark_offsets_dev, const uint32_t *observations_dev, uint32_t n_observations,
                              const cvb_view_constraint *constraints_dev, uint32_t C, const uint8_t *new_descriptors_dev,
                              const double *new_bearings_dev, const uint8_t *new_colors_dev, uint32_t N, const uint32_t *view_matches, uint32_t H,
                              cvb_pose *poses_out_dev, uint32_t *view_offsets_out_dev, uint32_t *view_landmarks_out_dev, double *bearings_out_dev,
                              uint8_t *descriptors_out_dev, uint8_t *colors_out_dev, uint32_t *landmark_offsets_out_dev,
                              uint32_t *observations_out_dev, cvb_view_constraint *constraints_out_dev, uint32_t *view_map_dev,
                              uint32_t *landmark_map_dev, cvb_register_match *matches_dev, cvb_incorporate_result *result_dev);

/* The same on HOST arrays (validated by cvb_incorporate_check first); outputs are host arrays with the same capacities. */
int cvb_incorporate_frame(cvb_ctx *ctx, const cvb_register_cfg *register_cfg, const cvb_constraints_cfg *constraints_cfg,
                          const cvb_recon_cfg *recon_cfg, const cvb_triangulator *tri, const cvb_arrsac_cfg *arrsac, cvb_rng *rng, uint32_t V,
                          const cvb_pose *poses, const uint32_t *view_offsets, const uint32_t *view_landmarks, const double *bearings,
                          const uint8_t *descriptors, const uint8_t *colors, uint32_t L, const uint32_t *landmark_offsets,
                          const uint32_t *observations, const cvb_view_constraint *constraints, uint32_t C, const uint8_t *new_descriptors,
                          const double *new_bearings, const uint8_t *new_colors, uint32_t N, const uint32_t *view_matches, uint32_t H,
                          cvb_pose *poses_out, uint32_t *view_offsets_out, uint32_t *view_landmarks_out, double *bearings_out,
                          uint8_t *descriptors_out, uint8_t *colors_out, uint32_t *landmark_offsets_out, uint32_t *observations_out,
                          cvb_view_constraint *constraints_out, uint32_t *view_map, uint32_t *landmark_map, cvb_register_match *matches,
                          cvb_incorporate_result *result);

#ifdef __cplusplus
}
#endif
#endif /* CVB200_INCORPORATE_H */
