/* include/cvb200_merge.h -- C ABI of cv-sfm's reconstruction merging on the device: two reconstruction snapshots to one, so that the
 * merge branch of try_localize needs no round trip to the host either.
 *
 *   cvb_incorporate_reconstruction_dev  <- VSlam::incorporate_reconstruction (cv-sfm/src/lib.rs:1817-1887): every view of a source
 *                                          reconstruction S moved into a destination D under a WorldToWorld, its landmarks mapped or
 *                                          created, then record_view_constraints of each moved view in order, remove_view on refusal
 *   cvb_merge_reconstructions_dev       <- VSlam::try_merge_reconstructions (lib.rs:2116-2193) followed by the optimize_reconstruction(D)
 *                                          that try_localize runs after it (lib.rs:867-877)
 *   cvb_incorporate_reconstruction, cvb_merge_reconstructions
 *                                       <- the same on host inputs, validated first
 *   cvb_merge_check                     <- that validation alone (host, no device needed)
 *
 * Library: libcvb200_merge.so, a module over libcvb200.so that takes its contexts (link with -lcvb200_merge -lcvb200).  The conventions
 * of include/cvb200.h hold: return codes, HOST pointers unless the name ends in _dev, no CPU fallback.  Snapshots are those of
 * include/cvb200_incorporate.h (poses, view CSR with bearings, descriptors and optional colours, landmark CSR, constraints); D and S must
 * both have colours or both not.  S's constraints are never read: incorporate_reconstruction does not carry them over, and D gets only
 * the constraints recorded by the call.
 *
 * incorporate_reconstruction(D, S, skip_view, world_transform, landmark_map):
 *   the moved views are S's views in index order without skip_view (CVB_MERGE_NONE: none skipped), which expresses
 *   try_merge_reconstructions' direct removal of src_view from S's view map (no remove_view: S's landmarks are not edited);
 *   1. moved view v gets the pose P_v * world_transform^-1 and S's features, bearings, descriptors and colours of v;
 *   2. feature f of v, of S landmark l, joins D landmark landmark_map[l] when l is mapped, and otherwise the landmark created for l by
 *      the first moved (view, feature) that observes it; landmark_map must be injective (HashMap::insert would otherwise overwrite an
 *      observation of the same view), each entry < L_D or CVB_MERGE_NONE;
 *   3. after every view moved: view_constraints of each moved view in order, against the snapshot as it stands; a refused view is
 *      removed (remove_view: its observations go, a landmark left without one goes, a constraint that contains it goes);
 *   D's own views and landmarks keep their indices; only moved views can be refused and only landmarks created from S can vanish.
 *
 * Step 3 is speculative and exact: one view_constraints call over every moved view still undecided, its results walked in order on the
 * host.  Every view before the first refusal saw exactly the snapshot the sequential loop gives it, so its result is final; the first
 * refused view is removed and the call is repeated for the views after it, against the new snapshot (whose view count, which the
 * acceptance reads, is one lower).  The results are those of the sequential loop; a call with r refusals makes at most r + 1 constraint
 * calls (result.constraint_calls).
 *
 * PINNED orders (the reference's come from a DenseSlotMap, whose remove of src_view swaps the last view into its slot, and from
 * HashMaps, so its own orders are UNPINNED against these):
 *   views         D's views, then (merge only) the new dest view of add_view, then the moved views in S index order without skip_view;
 *   landmarks     D's landmarks (merge: in add_view's order), then the landmarks created from S in creation order: moved-view order, then
 *                 feature order;
 *   observations  a landmark's existing observations, then the appended ones in moved-view order;
 *   constraints   D's constraints, then (merge only) the dest view's, then each accepted moved view's in order; a removal drops the
 *                 constraints that contain the removed view and renumbers the rest (cvb_apply_optimization's rule).
 * PINNED arithmetic: world_transform = dest^-1 * src is formed as that product, then inverted (not as a product of inverses), and the
 * moved pose is P_v * world_transform^-1.  A * B is (A.R B.R, A.t + A.R B.t); every 3x3 product and matrix-vector product sums
 * k = 0, 1, 2 left to right, without fused multiply-adds; the inverse is (R^T, R^T (-t)).
 *
 * merge_reconstructions(D, S, s_view, dest_view_matches):
 *   1. register_frame of s_view's frame against D: its descriptors, bearings and colours are s_view's rows of S's view CSR;
 *      cvb_register_frame_dev's waits, and *rng advances exactly as there; a failure returns D unchanged (NOT_REGISTERED), its panic none;
 *   2. add_view of that frame into D with the registered pose and matches (merged pairs merge; landmark_a survives);
 *   3. the dest view's constraints (Q = 1); on refusal remove_view of it: D keeps the merges of step 2, S is untouched (REJECTED);
 *   4. landmark_map: S landmark of s_view's feature f -> add_view's landmark_a of the match of f; world_transform from S's pose of
 *      s_view and the dest view's pose;
 *   5. incorporate_reconstruction with skip_view = s_view; S is consumed;
 *   6. optimize_reconstruction of the result and its edits (cvb_apply_optimization's rule): MERGED, or REMOVED_* / RECON_PANIC, after which
 *      neither reconstruction remains.
 *   The maps run from both inputs to the output; src_view_map[s_view] is the dest view, so a caller's frames[frame].view can follow.
 *
 * Output capacities (rows), with N = s_view's features and maxc = optimization_maximum_three_view_constraints:
 *                  poses         features           landmark_offsets                 observations        constraints
 *   incorporate    V + V_S       nf + nf_S          L + nf_S + 1                     n_obs + nf_S         C + V_S maxc
 *   merge          V + V_S       nf + nf_S          L + n_obs + 4 nf_S + 1           n_obs + 2 nf_S       C + (V_S + 1) maxc
 * (view_offsets one row more than poses).  The counts written say how many rows of each output are valid. */
#ifndef CVB200_MERGE_H
#define CVB200_MERGE_H
#include "cvb200.h"
#include "cvb200_tri.h"
#include "cvb200_constraints.h"
#include "cvb200_reconstruction.h"
#include "cvb200_register.h"
#include "cvb200_incorporate.h"

#ifdef __cplusplus
extern "C" {
#endif

#define CVB_MERGE_NONE 0xffffffffu   /* a map entry with no image, or no skip_view */

/* cvb_merge_result.status */
#define CVB_MERGE_MERGED 0                /* merged and optimised: one snapshot */
#define CVB_MERGE_NOT_REGISTERED 1        /* register_frame returned None (reg.status): D unchanged, S untouched */
#define CVB_MERGE_REGISTER_PANIC 2        /* register_frame's panic: no snapshot */
#define CVB_MERGE_REJECTED 3              /* the dest view's constraints refused: D after add_view + remove_view, S untouched */
#define CVB_MERGE_REMOVED_CONSTRAINTS 4   /* optimize_reconstruction removed the merged reconstruction: none remains */
#define CVB_MERGE_REMOVED_FILTER 5        /* ... (CVB_RECON_REMOVED_FILTER) */
#define CVB_MERGE_RECON_PANIC 6           /* optimize_reconstruction's panic: no snapshot */

/* incorporate_reconstruction's result */
typedef struct {
    cvb_incorporate_counts counts; /* of its output snapshot (merges = 0) */
    uint32_t moved_views;          /* S's views without skip_view */
    uint32_t refused_views;        /* moved views refused and removed */
    uint32_t created_landmarks;    /* landmarks created from S before the removals */
    uint32_t constraint_calls;     /* view_constraints calls of the speculative loop: refused_views + 1, one fewer when the last moved
                                      view is refused, 0 when no view is moved */
} cvb_move_result;

typedef struct {
    int32_t status;                /* CVB_MERGE_* */
    uint32_t dest_view;            /* the dest view's output index, or CVB_MERGE_NONE */
    cvb_incorporate_counts counts; /* of the output snapshot (all 0 when there is none) */
    cvb_register_result reg;       /* step 1 */
    cvb_register_stats reg_stats;
    cvb_view_constraints_result con;   /* step 3, the dest view (zero when it did not run) */
    cvb_move_result move;          /* step 5 (zero when it did not run) */
    cvb_recon_result recon;        /* step 6 (zero when it did not run) */
} cvb_merge_result;

/* Validates on the host: D and S as cvb_incorporate_check's snapshots (D with its constraints), S_view = s_view or skip_view < V_S
 * (CVB_MERGE_NONE allowed for skip_view only when landmark_map is given), landmark_map [L_S] (may be NULL) with every entry < L_D or
 * CVB_MERGE_NONE and no two entries equal, and has_colors_D == has_colors_S (1 or 0).  0, or CVB_EINVAL. */
int cvb_merge_check(uint32_t V, const uint32_t *view_offsets, const uint32_t *view_landmarks, uint32_t L, const uint32_t *landmark_offsets,
                    const uint32_t *observations, const cvb_view_constraint *constraints, uint32_t C, uint32_t V_S,
                    const uint32_t *view_offsets_S, const uint32_t *view_landmarks_S, uint32_t L_S, const uint32_t *landmark_offsets_S,
                    const uint32_t *observations_S, uint32_t view_S, const uint32_t *landmark_map, int has_colors, int has_colors_S);

/* incorporate_reconstruction on device arrays: D (poses_dev .. constraints_dev [C]), S (poses_S_dev .. observations_S_dev; descriptors
 * both given or both NULL, colours likewise), skip_view, world_transform_dev [1], landmark_map_dev [L_S].  Outputs as in the capacity
 * table, src_view_map_dev [V_S], src_landmark_map_dev [L_S] (the D landmark S's landmark became: landmark_map's entry, the created one,
 * or NONE), con_results_dev [V_S] (moved view v's constraint result; skip_view's zero) and result_dev [1].  A NULL argument not marked
 * optional, V = 0 or skip_view >= V_S other than NONE is CVB_EINVAL; triangulator methods 3-5 are CVB_EUNSUPPORTED.  The rules of
 * cvb_merge_check are preconditions: a broken one never makes the call read or write out of bounds.  Returns when the outputs are
 * written. */
int cvb_incorporate_reconstruction_dev(cvb_ctx *ctx, const cvb_constraints_cfg *constraints_cfg, const cvb_triangulator *tri, uint32_t V,
                                       const cvb_pose *poses_dev, const uint32_t *view_offsets_dev, const uint32_t *view_landmarks_dev,
                                       const double *bearings_dev, const uint8_t *descriptors_dev, const uint8_t *colors_dev, uint32_t n_features,
                                       uint32_t L, const uint32_t *landmark_offsets_dev, const uint32_t *observations_dev, uint32_t n_observations,
                                       const cvb_view_constraint *constraints_dev, uint32_t C, uint32_t V_S, const cvb_pose *poses_S_dev,
                                       const uint32_t *view_offsets_S_dev, const uint32_t *view_landmarks_S_dev, const double *bearings_S_dev,
                                       const uint8_t *descriptors_S_dev, const uint8_t *colors_S_dev, uint32_t n_features_S, uint32_t L_S,
                                       const uint32_t *landmark_offsets_S_dev, const uint32_t *observations_S_dev, uint32_t n_observations_S,
                                       uint32_t skip_view, const cvb_pose *world_transform_dev, const uint32_t *landmark_map_dev,
                                       cvb_pose *poses_out_dev, uint32_t *view_offsets_out_dev, uint32_t *view_landmarks_out_dev,
                                       double *bearings_out_dev, uint8_t *descriptors_out_dev, uint8_t *colors_out_dev,
                                       uint32_t *landmark_offsets_out_dev, uint32_t *observations_out_dev, cvb_view_constraint *constraints_out_dev,
                                       uint32_t *src_view_map_dev, uint32_t *src_landmark_map_dev, cvb_view_constraints_result *con_results_dev,
                                       cvb_move_result *result_dev);

/* The same on HOST arrays (validated by cvb_merge_check first); world_transform HOST [1]; outputs are host arrays. */
int cvb_incorporate_reconstruction(cvb_ctx *ctx, const cvb_constraints_cfg *constraints_cfg, const cvb_triangulator *tri, uint32_t V,
                                   const cvb_pose *poses, const uint32_t *view_offsets, const uint32_t *view_landmarks, const double *bearings,
                                   const uint8_t *descriptors, const uint8_t *colors, uint32_t L, const uint32_t *landmark_offsets,
                                   const uint32_t *observations, const cvb_view_constraint *constraints, uint32_t C, uint32_t V_S,
                                   const cvb_pose *poses_S, const uint32_t *view_offsets_S, const uint32_t *view_landmarks_S,
                                   const double *bearings_S, const uint8_t *descriptors_S, const uint8_t *colors_S, uint32_t L_S,
                                   const uint32_t *landmark_offsets_S, const uint32_t *observations_S, uint32_t skip_view,
                                   const cvb_pose *world_transform, const uint32_t *landmark_map, cvb_pose *poses_out, uint32_t *view_offsets_out,
                                   uint32_t *view_landmarks_out, double *bearings_out, uint8_t *descriptors_out, uint8_t *colors_out,
                                   uint32_t *landmark_offsets_out, uint32_t *observations_out, cvb_view_constraint *constraints_out,
                                   uint32_t *src_view_map, uint32_t *src_landmark_map, cvb_view_constraints_result *con_results,
                                   cvb_move_result *result);

/* merge_reconstructions on device arrays: D with descriptors (colours optional, with S's and the output's), S likewise, s_view,
 * dest_view_matches HOST [H]; arrsac and rng HOST (*rng advanced as cvb_register_frame advances it).  Outputs as in the capacity table,
 * dest_view_map_dev [V], dest_landmark_map_dev [L], src_view_map_dev [V_S], src_landmark_map_dev [L_S], con_results_dev [V_S] (the moved
 * views' results, as in incorporate_reconstruction) and result_dev [1].  Arguments are refused as by cvb_register_frame_dev and
 * cvb_incorporate_reconstruction_dev.  Returns when the outputs are written. */
int cvb_merge_reconstructions_dev(cvb_ctx *ctx, const cvb_register_cfg *register_cfg, const cvb_constraints_cfg *constraints_cfg,
                                  const cvb_recon_cfg *recon_cfg, const cvb_triangulator *tri, const cvb_arrsac_cfg *arrsac, cvb_rng *rng,
                                  uint32_t V, const cvb_pose *poses_dev, const uint32_t *view_offsets_dev, const uint32_t *view_landmarks_dev,
                                  const double *bearings_dev, const uint8_t *descriptors_dev, const uint8_t *colors_dev, uint32_t n_features,
                                  uint32_t L, const uint32_t *landmark_offsets_dev, const uint32_t *observations_dev, uint32_t n_observations,
                                  const cvb_view_constraint *constraints_dev, uint32_t C, uint32_t V_S, const cvb_pose *poses_S_dev,
                                  const uint32_t *view_offsets_S_dev, const uint32_t *view_landmarks_S_dev, const double *bearings_S_dev,
                                  const uint8_t *descriptors_S_dev, const uint8_t *colors_S_dev, uint32_t n_features_S, uint32_t L_S,
                                  const uint32_t *landmark_offsets_S_dev, const uint32_t *observations_S_dev, uint32_t n_observations_S,
                                  uint32_t s_view, const uint32_t *dest_view_matches, uint32_t H, cvb_pose *poses_out_dev,
                                  uint32_t *view_offsets_out_dev, uint32_t *view_landmarks_out_dev, double *bearings_out_dev,
                                  uint8_t *descriptors_out_dev, uint8_t *colors_out_dev, uint32_t *landmark_offsets_out_dev,
                                  uint32_t *observations_out_dev, cvb_view_constraint *constraints_out_dev, uint32_t *dest_view_map_dev,
                                  uint32_t *dest_landmark_map_dev, uint32_t *src_view_map_dev, uint32_t *src_landmark_map_dev,
                                  cvb_view_constraints_result *con_results_dev, cvb_merge_result *result_dev);

/* The same on HOST arrays (validated by cvb_merge_check and cvb_register_frame's view-match rule first); outputs are host arrays. */
int cvb_merge_reconstructions(cvb_ctx *ctx, const cvb_register_cfg *register_cfg, const cvb_constraints_cfg *constraints_cfg,
                              const cvb_recon_cfg *recon_cfg, const cvb_triangulator *tri, const cvb_arrsac_cfg *arrsac, cvb_rng *rng, uint32_t V,
                              const cvb_pose *poses, const uint32_t *view_offsets, const uint32_t *view_landmarks, const double *bearings,
                              const uint8_t *descriptors, const uint8_t *colors, uint32_t L, const uint32_t *landmark_offsets,
                              const uint32_t *observations, const cvb_view_constraint *constraints, uint32_t C, uint32_t V_S,
                              const cvb_pose *poses_S, const uint32_t *view_offsets_S, const uint32_t *view_landmarks_S, const double *bearings_S,
                              const uint8_t *descriptors_S, const uint8_t *colors_S, uint32_t L_S, const uint32_t *landmark_offsets_S,
                              const uint32_t *observations_S, uint32_t s_view, const uint32_t *dest_view_matches, uint32_t H,
                              cvb_pose *poses_out, uint32_t *view_offsets_out, uint32_t *view_landmarks_out, double *bearings_out,
                              uint8_t *descriptors_out, uint8_t *colors_out, uint32_t *landmark_offsets_out, uint32_t *observations_out,
                              cvb_view_constraint *constraints_out, uint32_t *dest_view_map, uint32_t *dest_landmark_map, uint32_t *src_view_map,
                              uint32_t *src_landmark_map, cvb_view_constraints_result *con_results, cvb_merge_result *result);

#ifdef __cplusplus
}
#endif
#endif /* CVB200_MERGE_H */
