// cv_b200/csrc/stages_abi.cu -- libcvb200_stages.so, the module that exports the C ABI of include/cvb200_stages.h (AKAZE's staged
// surface: a resident scale space, find_image_keypoints, extract_descriptors at caller keypoints).  The kernels and their host code
// live in akaze.cu inside libcvb200.so; this module only gives them their C names, so that libcvb200.so's own exports stay exactly
// those of cvb200.h, cvb200_sfm.h and cvb200_tri.h.  It links libcvb200.so (rpath $ORIGIN) and takes that library's contexts.
#include "../../include/cvb200_stages.h"

int stages_scale_space(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, const float *images, bool on_device, uint32_t batch, uint32_t w,
                       uint32_t h, uint64_t *ticket_out);
int stages_evolutions(cvb_ctx *ctx, uint64_t ticket, cvb_akaze_evolution *out, uint32_t cap, uint32_t *n_out);
int stages_find(cvb_ctx *ctx, uint64_t ticket, cvb_keypoint *kp_out, uint32_t cap, uint32_t *n_out, bool on_device);
int stages_describe(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, uint64_t ticket, const cvb_keypoint *kp_in, const uint32_t *offsets,
                    uint32_t total_max, cvb_keypoint *kp_out, uint8_t *desc_out, uint32_t *n_out, bool on_device);

extern "C" {

int cvb_akaze_scale_space(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, const float *images, uint32_t batch, uint32_t w, uint32_t h,
                          uint64_t *scale_space_out) {
    return stages_scale_space(ctx, cfg, images, false, batch, w, h, scale_space_out);
}

int cvb_akaze_scale_space_dev(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, const float *images_dev, uint32_t batch, uint32_t w, uint32_t h,
                              uint64_t *scale_space_out) {
    return stages_scale_space(ctx, cfg, images_dev, true, batch, w, h, scale_space_out);
}

int cvb_akaze_evolutions(cvb_ctx *ctx, uint64_t scale_space, cvb_akaze_evolution *out, uint32_t cap, uint32_t *n_out) {
    return stages_evolutions(ctx, scale_space, out, cap, n_out);
}

int cvb_akaze_find_image_keypoints(cvb_ctx *ctx, uint64_t scale_space, cvb_keypoint *kp_out, uint32_t cap, uint32_t *n_out) {
    return stages_find(ctx, scale_space, kp_out, cap, n_out, false);
}

int cvb_akaze_find_image_keypoints_dev(cvb_ctx *ctx, uint64_t scale_space, cvb_keypoint *kp_out_dev, uint32_t cap,
                                       uint32_t *n_out_dev) {
    return stages_find(ctx, scale_space, kp_out_dev, cap, n_out_dev, true);
}

int cvb_akaze_extract_descriptors(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, uint64_t scale_space, const cvb_keypoint *kp_in,
                                  const uint32_t *offsets, cvb_keypoint *kp_out, uint8_t *desc_out, uint32_t *n_out) {
    return stages_describe(ctx, cfg, scale_space, kp_in, offsets, 0, kp_out, desc_out, n_out, false);
}

int cvb_akaze_extract_descriptors_dev(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, uint64_t scale_space, const cvb_keypoint *kp_in_dev,
                                      const uint32_t *offsets_dev, uint32_t total_max, cvb_keypoint *kp_out_dev, uint8_t *desc_out_dev,
                                      uint32_t *n_out_dev) {
    return stages_describe(ctx, cfg, scale_space, kp_in_dev, offsets_dev, total_max, kp_out_dev, desc_out_dev, n_out_dev, true);
}

}  // extern "C"
