/* include/cvb200_stages.h -- C ABI of AKAZE's staged surface on the device: a resident scale space, keypoint detection without
 * descriptors, and descriptors at caller keypoints.  These are the parts of akaze::Akaze the akaze crate exposes for clients that
 * want only a portion of the pipeline (akaze/src/lib.rs:341-345):
 *
 *   cvb_akaze_scale_space(_dev)            <- allocate_evolutions (evolution.rs:80-126) + create_nonlinear_scale_space
 *                                             (lib.rs:193-258) + detector_response (detector_response.rs:8-85), the sequence
 *                                             inside extract_from_gray_float_image (lib.rs:309-339); the multiscale Lx / Ly
 *                                             of detector_response (detector_response.rs:63-64) are what descriptors read
 *   cvb_akaze_evolutions                   <- the scalar fields of the EvolutionStep table (evolution.rs:8-44)
 *   cvb_akaze_find_image_keypoints(_dev)   <- Akaze::find_image_keypoints (lib.rs:268-276) minus detector_response, i.e.
 *                                             detect_keypoints = find_scale_space_extrema + do_subpixel_refinement
 *   cvb_akaze_extract_descriptors(_dev)    <- Akaze::extract_descriptors(&evolutions, &keypoints) (descriptors.rs:16-45)
 *
 * Library: libcvb200_stages.so, a module over libcvb200.so that takes its contexts (link with -lcvb200_stages -lcvb200).  The
 * conventions of include/cvb200.h hold: return codes, HOST pointers unless the name ends in _dev, asynchronous _dev variants on the
 * context's stream, no CPU fallback.
 *
 * Ticket: a scale space lives in the context's AKAZE workspace, and the call returns a ticket for it (never 0).  Every call that
 * rewrites that workspace's planes -- any extract entry point, two-view frames, frame features, a new scale space, or a call that
 * rebuilds the workspace for another size or config -- makes earlier tickets stale.  find / evolutions / describe with a stale
 * or unknown ticket return CVB_EINVAL ("scale space replaced"); they never answer from other planes.
 *
 * find: keypoints of frame b go to kp_out[b * cap ..], in the reference's order (the order of the extractor's "refined" stage),
 * NOT sorted by response and NOT truncated: maximum_features is ignored, as in find_image_keypoints.  Detection uses the config the
 * scale space was built with (detector_threshold, derivative_factor, ...): the detector response, computed with the scale space,
 * already depends on it.  The reference reads them from find_image_keypoints' &self, so a caller must build the scale space with
 * the Akaze it detects with.  n_out[b] is the count.  More
 * than cap keypoints: the host call returns CVB_ECAP with n_out[b] = the required count; the _dev call writes the first cap and
 * sets flag 3 of cvb_akaze_dev_overflow.  Every call runs detection again.  When a frame exceeds an internal capacity there, the host
 * call grows the capacity and detects again on the same planes (the ticket stays valid); the _dev call sets flag 1 or 2 (see
 * cvb_akaze_dev_overflow in cvb200.h).  An image too small for one octave (no evolutions)
 * gives 0 keypoints.
 *
 * describe: the keypoints of frame b are kp_in[offsets[b] .. offsets[b + 1]) (offsets: batch + 1 non-decreasing entries, CSR).
 * The kept ones are copied bit for bit, in input order, to kp_out[offsets[b] ..], their 64-byte descriptors to
 * desc_out[offsets[b] * 64 ..], and n_out[b] is their count; the rest of each frame's slots is left as it was.  A keypoint is
 * dropped when a sample of its pattern falls outside its level (descriptors.rs:131-140); duplicates are kept.  The output is never
 * longer than the input, so there is no CVB_ECAP.
 *   - Config: only descriptor_channels (1..3) and descriptor_pattern_size (its lattice at most 21 points per axis) are read, like
 *     the reference's &self.  Another descriptor config than the scale space's does not touch the scale space or its ticket.
 *   - Level: the pattern ratio comes from keypoint.octave, the planes and bounds from evolutions[class_id], as in the reference,
 *     even when the two disagree.
 *   - Sample positions: `f32::round(v) as isize` (descriptors.rs:129-130) is Rust's saturating cast, so a NaN position reads
 *     row / column 0 and the keypoint is kept, while +-inf and huge values are out of bounds.
 *   - Angles: sin and cos are glibc 2.39's sinf / cosf (what Rust's f32::sin / cos call on linux-gnu) over the whole float range:
 *     any finite angle, in radians or not, is reduced exactly; +-inf and NaN give NaN, hence NaN positions.
 *   - Invalid keypoints: class_id >= the number of evolutions (an out-of-bounds index in the reference) or octave >= 32 (a shift
 *     overflow).  The host call returns CVB_EINVAL naming the first one; the _dev call drops them and sets flag 4 ("invalid input
 *     keypoint") of cvb_akaze_dev_overflow.  With no evolutions every keypoint is invalid.
 *   - _dev: offsets_dev is read on the device; total_max bounds the launch, and offsets are clamped to it.  kp_in_dev and the
 *     outputs must not overlap.  Flags 1-3 of cvb_akaze_dev_overflow keep their meaning. */
#ifndef CVB200_STAGES_H
#define CVB200_STAGES_H
#include "cvb200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* the scalar fields of akaze's EvolutionStep (evolution.rs:8-44), with the level size and the length of fed_tau_steps.
 * sigma_size is the reference's `esigma.round() as u32` (evolution.rs:58), rounding half away from zero. */
typedef struct {
    uint32_t octave;
    uint32_t sublevel;
    double esigma;
    double etime;
    uint32_t sigma_size;
    uint32_t width;
    uint32_t height;
    uint32_t n_fed_steps;
} cvb_akaze_evolution;

/* builds the scale space of `batch` frames of w x h f32 (host images: batch * w * h floats) */
int cvb_akaze_scale_space(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, const float *images, uint32_t batch, uint32_t w, uint32_t h,
                          uint64_t *scale_space_out);
int cvb_akaze_scale_space_dev(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, const float *images_dev, uint32_t batch, uint32_t w, uint32_t h,
                              uint64_t *scale_space_out);

/* the evolution table: *n_out = its length, the first min(cap, length) entries written to out (out may be NULL when cap is 0) */
int cvb_akaze_evolutions(cvb_ctx *ctx, uint64_t scale_space, cvb_akaze_evolution *out, uint32_t cap, uint32_t *n_out);

/* kp_out: batch x cap keypoints, n_out: batch counts */
int cvb_akaze_find_image_keypoints(cvb_ctx *ctx, uint64_t scale_space, cvb_keypoint *kp_out, uint32_t cap, uint32_t *n_out);
int cvb_akaze_find_image_keypoints_dev(cvb_ctx *ctx, uint64_t scale_space, cvb_keypoint *kp_out_dev, uint32_t cap,
                                       uint32_t *n_out_dev);

/* kp_in / kp_out: offsets[batch] keypoints, desc_out: offsets[batch] x 64 bytes, offsets: batch + 1, n_out: batch */
int cvb_akaze_extract_descriptors(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, uint64_t scale_space, const cvb_keypoint *kp_in,
                                  const uint32_t *offsets, cvb_keypoint *kp_out, uint8_t *desc_out, uint32_t *n_out);
int cvb_akaze_extract_descriptors_dev(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, uint64_t scale_space, const cvb_keypoint *kp_in_dev,
                                      const uint32_t *offsets_dev, uint32_t total_max, cvb_keypoint *kp_out_dev, uint8_t *desc_out_dev,
                                      uint32_t *n_out_dev);

#ifdef __cplusplus
}
#endif
#endif /* CVB200_STAGES_H */
