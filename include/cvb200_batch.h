/* include/cvb200_batch.h -- C ABI of batched consensus on the device: B independent ARRSAC problems in one set of launches.
 *
 *   cvb_arrsac_batch_dev / cvb_arrsac_batch  <- B calls of arrsac::Arrsac::model_inliers (Consensus<EightPoint, FeatureMatch>,
 *                                               Consensus<LambdaTwist, FeatureWorldMatch>, Consensus<NisterStewenius, FeatureMatch>),
 *                                               such as the per-candidate two-view runs of cv-sfm's VSlam::init_reconstruction
 *                                               (cv-sfm/src/lib.rs:966-985 -> init_two_view, lib.rs:1365-1432)
 *   cvb_arrsac_commit_rng_batch              <- the generator state each of those calls leaves behind
 *   cvb_two_view_options_dev                 <- VSlam::init_reconstruction's init_two_view(center, option) for every option frame
 *                                               (cv-sfm/src/lib.rs:966-985 -> init_two_view, lib.rs:1365-1432): symmetric_matching,
 *                                               the matches' bearings, model_inliers, on the device for all options at once
 *
 * Library: libcvb200_batch.so, a module over libcvb200.so that takes its contexts (link with -lcvb200_batch -lcvb200).  The conventions
 * of include/cvb200.h hold: return codes, HOST pointers unless the name ends in _dev, asynchronous _dev variants on the context's
 * stream, no CPU fallback.
 *
 * kind: 0 eight-point (a, b: unit bearings, 3 doubles per row), 1 P3P (a: unit bearings, b: homogeneous world points, 4 doubles per
 * row), 2 five-point (as 0; eigenvector_row0 5 or 6 as in cvb_arrsac_five_point, ignored for the other kinds).
 *
 * Semantics: problem b's result -- pose, inlier list, found, and its generator after the commit -- is bit for bit the result of the
 * single-problem call on the same rows with generator rngs[b] (cvb_arrsac_eight_point_dev / cvb_arrsac_p3p_dev, and the five-point
 * solver's cvb_arrsac_five_point, of which kind 2 is also the device-resident form).  Each problem has its OWN generator: the
 * reference runs its candidates one after the other on one shared generator, so candidate i starts where candidate i - 1 stopped,
 * and a batch cannot know those start states (the draws a run consumes are known only when it ends).  Parity with cv-sfm's
 * shared-generator sequence, and with the shuffle cv-sfm applies to the matches in front of consensus (lib.rs:1386), is UNPINNED.
 *
 * Limits: 1 <= B <= CVB_ARRSAC_BATCH_MAX; B = 0 is a no-op (nothing is enqueued, no run is pending); B above the maximum is
 * CVB_EUNSUPPORTED; a NULL argument that is not marked optional is CVB_EINVAL.  The configuration limits are those of the single
 * entries.  The undecided-predicate queue of the consensus filter is split between the problems; predicates beyond a problem's share
 * are evaluated in place, so the split changes time, never results. */
#ifndef CVB200_BATCH_H
#define CVB200_BATCH_H
#include "cvb200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* the most problems in one batch (cv-sfm's default tracking_recent_frames = 32 gives up to 31 candidates per frame) */
#define CVB_ARRSAC_BATCH_MAX 64

/* Device data: problem b owns rows [b * n_max, b * n_max + n_dev[b]) of a_dev / b_dev (n_dev may be NULL: every problem has n_max
 * rows; counts above n_max are clamped).  cfg and rngs (B generators) are HOST pointers; the generators are read, not advanced:
 * cvb_arrsac_commit_rng_batch does that once the stream has drained.  Outputs per problem b: model_out_dev[b], found_dev[b]
 * (0 -> None), n_inliers_dev[b], and inliers_out_dev[b * cap ..] (may be NULL): ascending datum indices within the problem, at most
 * cap written. */
int cvb_arrsac_batch_dev(cvb_ctx *ctx, const cvb_arrsac_cfg *cfg, int32_t kind, int32_t eigenvector_row0, const double *a_dev,
                         const double *b_dev, const uint32_t *n_dev, uint32_t n_max, uint32_t B, const cvb_rng *rngs,
                         cvb_pose *model_out_dev, uint32_t *inliers_out_dev, uint32_t cap, uint32_t *n_inliers_dev, int32_t *found_dev);

/* Host data in CSR form: problem b owns rows offsets[b] .. offsets[b + 1] of a / b (offsets: B + 1 non-decreasing entries).  One
 * synchronisation at the end; every rngs[b] is advanced.  Outputs: models_out[b], found_out[b], n_inliers_out[b], and problem b's
 * inliers (indices within the problem) at inliers_out[offsets[b] - offsets[0] ..] (may be NULL; offsets[B] - offsets[0] entries
 * always suffice). */
int cvb_arrsac_batch(cvb_ctx *ctx, const cvb_arrsac_cfg *cfg, int32_t kind, int32_t eigenvector_row0, const double *a, const double *b,
                     const uint32_t *offsets, uint32_t B, cvb_rng *rngs, cvb_pose *models_out, uint32_t *inliers_out,
                     uint32_t *n_inliers_out, int32_t *found_out);

/* Synchronises the context stream and advances rngs[0 .. B) past the draws each problem of the pending cvb_arrsac_batch_dev run
 * consumed.  stats_out (may be NULL): B x 16 words, problem b's at b * 16, the words of cvb_arrsac_commit_rng.  A pending run that is
 * not a batch, a batch of another size, or no pending run: CVB_EINVAL, and no generator moves (likewise cvb_arrsac_commit_rng
 * refuses a pending batch). */
int cvb_arrsac_commit_rng_batch(cvb_ctx *ctx, cvb_rng *rngs, uint32_t B, uint32_t *stats_out);

/* cv-sfm's init_two_view of frame `center` against the F frames options[0 .. F) (HOST array of frame indices), on what
 * cvb_frame_features_batch_dev produced for `frames` frames: descriptors desc_dev (frames x cap x 64 bytes), counts n_dev (frames) and
 * bearings_dev (frames x cap x 3 f64), frame b at b * cap.  For option f:
 *   1. the symmetric match of the center's and the option's descriptors with better_by (cvb_match_symmetric_pairs_dev, n_max = cap):
 *      pairs_out_dev[f * cap * 2 ..] (center feature, option feature), n_pairs_dev[f];
 *   2. one gather launch for all options copies the matched bearing rows into the consensus input;
 *   3. one batched eight-point ARRSAC over the F problems with generator rngs[f]: model_out_dev[f], found_dev[f], n_inliers_dev[f],
 *      inliers_out_dev[f * cap ..] (may be NULL): indices into option f's pairs.
 * Option f's outputs are bit for bit those of cvb_two_view_pair_k1_dev on the center's and the option's keypoints, descriptors and counts
 * with n_max = cap, the camera the bearings were made with and generator rngs[f].  Commit the generators with
 * cvb_arrsac_commit_rng_batch(ctx, rngs, F, ...).  Not applied on the device: cv-sfm's two_view_minimum_robust_matches (an option with
 * fewer inliers is None; the Python and Rust wrappers apply it) and its pre-consensus shuffle of the matches (unpinned, as in the other
 * fused entries).  F = 0 is a no-op; F above CVB_ARRSAC_BATCH_MAX is CVB_EUNSUPPORTED; center or an option >= frames, cap = 0 or a NULL
 * argument not marked optional is CVB_EINVAL. */
int cvb_two_view_options_dev(cvb_ctx *ctx, const uint8_t *desc_dev, const uint32_t *n_dev, const double *bearings_dev, uint32_t frames,
                             uint32_t cap, uint32_t center, const uint32_t *options, uint32_t F, uint32_t better_by, const cvb_arrsac_cfg *cfg,
                             const cvb_rng *rngs, uint32_t *pairs_out_dev, uint32_t *n_pairs_dev, cvb_pose *model_out_dev,
                             uint32_t *inliers_out_dev, uint32_t *n_inliers_dev, int32_t *found_dev);

#ifdef __cplusplus
}
#endif
#endif /* CVB200_BATCH_H */
