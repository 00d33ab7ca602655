/* include/cvb200_sfm.h -- C ABI of libcvb200.so for cv-sfm integration: the reference's camera with radial distortion
 * (cv_pinhole::CameraIntrinsicsK1Distortion) in the fused two-view entry points, and cv-sfm's per-frame feature ingestion
 * (VSlam::kps_descriptors).  Every camera of the reference's applications has a k1 coefficient: VSlam::add_feed takes a
 * CameraIntrinsicsK1Distortion (cv-sfm/src/lib.rs:125,777), vslam-sandbox builds one (vslam-sandbox/src/main.rs:71-78) and tutorial
 * chapter 5 uses one (tutorial-code/chapter5-geometric-verification/src/main.rs:36-42).
 *
 *   cvb_intrinsics_k1            <- CameraIntrinsicsK1Distortion          cv-pinhole/src/lib.rs:150-153, calibrate :191-202
 *   cvb_pair_bearings_k1_dev     <- FeatureMatch bearings with that camera cv-sfm/src/lib.rs:1400
 *   cvb_two_view_pair_k1_dev,
 *   cvb_two_view_frames_k1       <- cv-sfm's two-view initialisation      cv-sfm/src/lib.rs:1375-1412
 *   cvb_frame_features_batch*    <- VSlam::kps_descriptors                cv-sfm/src/lib.rs:2195-2235
 *
 * The conventions of include/cvb200.h hold (return codes, HOST pointers unless `_dev`, asynchronous `_dev` variants, no CPU fallback).
 * The entry points of cvb200.h that take a cvb_intrinsics are these with k1 = 0: the distortion step then divides by exactly 1.0, so
 * their results are the same bits as the undistorted camera's (CameraIntrinsics::calibrate, cv-pinhole/src/lib.rs:108-116). */
#ifndef CVB200_SFM_H
#define CVB200_SFM_H
#include "cvb200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* CameraIntrinsicsK1Distortion (cv-pinhole/src/lib.rs:150-153): simple_intrinsics + one radial coefficient k1.  Its calibrate
 * (:191-202) centres, divides by the focals, removes skew, then divides both components by 1 + k1 r^2 (r^2 = x^2 + y^2) before
 * normalising. */
typedef struct { double fx, fy, cx, cy, skew, k1; } cvb_intrinsics_k1;

/* cvb_pair_bearings_dev (include/cvb200.h) with the K1 camera */
int cvb_pair_bearings_k1_dev(cvb_ctx *ctx, const cvb_keypoint *kp_a_dev, const cvb_keypoint *kp_b_dev, const uint32_t *pairs_dev,
                             const uint32_t *n_pairs_dev, uint32_t cap, const cvb_intrinsics_k1 *intrinsics /* host */, double *a_out_dev,
                             double *b_out_dev);

/* cvb_two_view_pair_dev / cvb_two_view_frames (include/cvb200.h) with the K1 camera */
int cvb_two_view_pair_k1_dev(cvb_ctx *ctx, const cvb_keypoint *kp_a_dev, const uint8_t *desc_a_dev, const uint32_t *n_a_dev,
                             const cvb_keypoint *kp_b_dev, const uint8_t *desc_b_dev, const uint32_t *n_b_dev, uint32_t n_max,
                             uint32_t better_by, const cvb_intrinsics_k1 *intrinsics, const cvb_arrsac_cfg *cfg, const cvb_rng *rng,
                             uint32_t *pairs_out_dev, uint32_t cap, uint32_t *n_pairs_dev, cvb_pose *model_out_dev,
                             uint32_t *inliers_out_dev, uint32_t *n_inliers_dev, int32_t *found_dev);
int cvb_two_view_frames_k1(cvb_ctx *ctx, const cvb_akaze_cfg *akaze, const float *frames, uint32_t w, uint32_t h, uint32_t better_by,
                           const cvb_intrinsics_k1 *intrinsics, const cvb_arrsac_cfg *cfg, cvb_rng *rng, cvb_keypoint *kp_out,
                           uint8_t *desc_out, uint32_t cap, uint32_t *n_out, uint32_t *pairs_out, uint32_t *n_pairs, cvb_pose *model_out,
                           uint32_t *inliers_out, uint32_t *n_inliers, int32_t *found);

/* ---- cv-sfm frame ingestion: VSlam::kps_descriptors (cv-sfm/src/lib.rs:2195-2235) for B frames of one size ------------------------
 * Per frame: AKAZE (cv-sfm sets maximum_features = tracking_features in the configuration), the colour of every keypoint sampled from
 * the RGB frame by bicubic interpolation (cv-sfm/src/bicubic.rs:13-68, black outside the reference's border rule
 * left < 0 || left + 4 >= w || top < 0 || top + 4 >= h; every row blend is clamped to u8 before the column blend), and its K1 bearing.
 * The clamp is imageproc 0.23's Clamp<f32> for u8 (x < 255 ? (x > 0 ? (u8)x : 0) : 255), an external crate restated from its published
 * source: parity unpinned beyond that restatement.
 * Order: kps_descriptors ends with sort_unstable_by_key(Reverse(FloatOrd(response))) (:2234).  AKAZE's output is already in that
 * order (akaze/src/lib.rs:326-327; extract_descriptors only drops keypoints, akaze/src/descriptors.rs:16-30), and the standard
 * library's unstable sort (pdqsort, and the later ipnsort) returns an already sorted slice unchanged, so the reference's order is
 * AKAZE's order: feature i is keypoint i, and no sort runs here.
 * rgb: B frames of h rows of w interleaved R, G, B bytes (image::RgbImage, i.e. DynamicImage::to_rgb8()).
 * Outputs per frame b at offset b * cap: keypoints and descriptors exactly as cvb_akaze_extract_batch writes them, unit bearings
 * (f64 x 3) and colours (u8 x 3) of the same keypoints; n_out[b] their number. */
int cvb_frame_features_batch(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, const float *images, const uint8_t *rgb, uint32_t batch, uint32_t w,
                             uint32_t h, const cvb_intrinsics_k1 *intrinsics, cvb_keypoint *kp_out, uint8_t *desc_out, double *bearings_out,
                             uint8_t *colors_out, uint32_t cap, uint32_t *n_out);
/* Device-resident variant on the outputs of cvb_akaze_extract_batch_dev (kp_dev: batch x cap, n_dev: batch) and device RGB frames:
 * writes bearings_out_dev (batch x cap x 3 f64) and colors_out_dev (batch x cap x 3 u8) for the first min(n_dev[b], cap) keypoints of
 * each frame; rows beyond are left untouched.  intrinsics is a HOST pointer.  Asynchronous on the context stream. */
int cvb_frame_features_batch_dev(cvb_ctx *ctx, const cvb_keypoint *kp_dev, const uint32_t *n_dev, uint32_t batch, uint32_t cap,
                                 const uint8_t *rgb_dev, uint32_t w, uint32_t h, const cvb_intrinsics_k1 *intrinsics, double *bearings_out_dev,
                                 uint8_t *colors_out_dev);

#ifdef __cplusplus
}
#endif
#endif /* CVB200_SFM_H */
