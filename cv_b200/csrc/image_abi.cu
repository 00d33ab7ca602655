// cv_b200/csrc/image_abi.cu -- libcvb200_image.so, the module that exports the C ABI of include/cvb200_image.h (8- and 16-bit frames into
// the extractor, frame ingestion and the two-view entry).  The kernel and its host code live in image.cu inside libcvb200.so, next to the
// f32 paths they take; this module only gives them their C names, so that libcvb200.so's own exports stay exactly those of cvb200.h,
// cvb200_sfm.h and cvb200_tri.h.  It links libcvb200.so (rpath $ORIGIN) and takes that library's contexts.
#include "../../include/cvb200_image.h"

int img_gray_float_from_dynamic_dev(cvb_ctx *ctx, cvb_pixel_format format, const void *pixels_dev, uint32_t batch, uint32_t w, uint32_t h,
                                    float *gray_out_dev, uint8_t *rgb_out_dev);
int img_akaze_extract_dynamic_batch(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, cvb_pixel_format format, const void *pixels, uint32_t batch,
                                    uint32_t w, uint32_t h, cvb_keypoint *kp_out, uint8_t *desc_out, uint32_t cap, uint32_t *n_out);
int img_akaze_extract_dynamic_batch_dev(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, cvb_pixel_format format, const void *pixels_dev,
                                        uint32_t batch, uint32_t w, uint32_t h, cvb_keypoint *kp_out_dev, uint8_t *desc_out_dev, uint32_t cap,
                                        uint32_t *n_out_dev);
int img_frame_features_dynamic_batch(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, cvb_pixel_format format, const void *pixels, uint32_t batch,
                                     uint32_t w, uint32_t h, const cvb_intrinsics_k1 *intrinsics, cvb_keypoint *kp_out, uint8_t *desc_out,
                                     double *bearings_out, uint8_t *colors_out, uint32_t cap, uint32_t *n_out);
int img_two_view_frames_dynamic_k1(cvb_ctx *ctx, const cvb_akaze_cfg *akaze, cvb_pixel_format format, const void *frames, uint32_t w,
                                   uint32_t h, uint32_t better_by, const cvb_intrinsics_k1 *intrinsics, const cvb_arrsac_cfg *cfg, cvb_rng *rng,
                                   cvb_keypoint *kp_out, uint8_t *desc_out, uint32_t cap, uint32_t *n_out, uint32_t *pairs_out,
                                   uint32_t *n_pairs, cvb_pose *model_out, uint32_t *inliers_out, uint32_t *n_inliers, int32_t *found);

extern "C" {

int cvb_gray_float_from_dynamic_dev(cvb_ctx *ctx, cvb_pixel_format format, const void *pixels_dev, uint32_t batch, uint32_t w, uint32_t h,
                                    float *gray_out_dev, uint8_t *rgb_out_dev) {
    return img_gray_float_from_dynamic_dev(ctx, format, pixels_dev, batch, w, h, gray_out_dev, rgb_out_dev);
}

int cvb_akaze_extract_dynamic_batch(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, cvb_pixel_format format, const void *pixels, uint32_t batch,
                                    uint32_t w, uint32_t h, cvb_keypoint *kp_out, uint8_t *desc_out, uint32_t cap, uint32_t *n_out) {
    return img_akaze_extract_dynamic_batch(ctx, cfg, format, pixels, batch, w, h, kp_out, desc_out, cap, n_out);
}

int cvb_akaze_extract_dynamic_batch_dev(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, cvb_pixel_format format, const void *pixels_dev,
                                        uint32_t batch, uint32_t w, uint32_t h, cvb_keypoint *kp_out_dev, uint8_t *desc_out_dev, uint32_t cap,
                                        uint32_t *n_out_dev) {
    return img_akaze_extract_dynamic_batch_dev(ctx, cfg, format, pixels_dev, batch, w, h, kp_out_dev, desc_out_dev, cap, n_out_dev);
}

int cvb_frame_features_dynamic_batch(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, cvb_pixel_format format, const void *pixels, uint32_t batch,
                                     uint32_t w, uint32_t h, const cvb_intrinsics_k1 *intrinsics, cvb_keypoint *kp_out, uint8_t *desc_out,
                                     double *bearings_out, uint8_t *colors_out, uint32_t cap, uint32_t *n_out) {
    return img_frame_features_dynamic_batch(ctx, cfg, format, pixels, batch, w, h, intrinsics, kp_out, desc_out, bearings_out, colors_out, cap,
                                            n_out);
}

int cvb_two_view_frames_dynamic_k1(cvb_ctx *ctx, const cvb_akaze_cfg *akaze, cvb_pixel_format format, const void *frames, uint32_t w,
                                   uint32_t h, uint32_t better_by, const cvb_intrinsics_k1 *intrinsics, const cvb_arrsac_cfg *cfg, cvb_rng *rng,
                                   cvb_keypoint *kp_out, uint8_t *desc_out, uint32_t cap, uint32_t *n_out, uint32_t *pairs_out,
                                   uint32_t *n_pairs, cvb_pose *model_out, uint32_t *inliers_out, uint32_t *n_inliers, int32_t *found) {
    return img_two_view_frames_dynamic_k1(ctx, akaze, format, frames, w, h, better_by, intrinsics, cfg, rng, kp_out, desc_out, cap, n_out,
                                          pairs_out, n_pairs, model_out, inliers_out, n_inliers, found);
}

}  // extern "C"
