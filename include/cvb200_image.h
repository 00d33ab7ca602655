/* include/cvb200_image.h -- C ABI of the extractor's input on the device: 8- and 16-bit luma / RGB(A) frames, converted the way
 * akaze::Akaze::extract converts its DynamicImage (GrayFloatImage::from_dynamic, akaze/src/image.rs:45-109) and, for cv-sfm's frame
 * ingestion, the way DynamicImage::to_rgb8() gives the colour plane.
 *
 *   cvb_gray_float_from_dynamic_dev     <- GrayFloatImage::from_dynamic (+ to_rgb8)          image.rs:45-109
 *   cvb_akaze_extract_dynamic_batch(_dev) <- Akaze::extract(&DynamicImage)                   akaze/src/lib.rs:295-298
 *   cvb_frame_features_dynamic_batch    <- VSlam::kps_descriptors(&DynamicImage)            cv-sfm/src/lib.rs:2195-2235
 *   cvb_two_view_frames_dynamic_k1      <- cv-sfm's two-view initialisation on two frames    cv-sfm/src/lib.rs:1375-1412
 *
 * Library: libcvb200_image.so, a module over libcvb200.so that takes its contexts (link with -lcvb200_image -lcvb200).  The conventions
 * of include/cvb200.h hold: return codes, HOST pointers unless the name ends in _dev, asynchronous _dev variants, no CPU fallback (no
 * device: no context, CVB_ENODEV).  A null context, an unknown format or an empty frame or batch is CVB_EINVAL.
 *
 * Frames: `batch` frames of one size, each h rows of w pixels, tightly packed and interleaved, in the layout of ImageBuffer::as_bytes()
 * (16-bit channels in native, i.e. little-endian, byte order), frame after frame.  The host forms upload these bytes (about a quarter of
 * the f32 plane for LUMA8) and convert them on the device into a buffer of the context, reused across calls, so that the extractor's
 * CUDA graph, cached per input buffer, is replayed.  Their results and return codes are those of the f32 entry points (cvb200.h,
 * cvb200_sfm.h) called on the converted planes, CVB_ECAP and the capacity flag included.
 *
 * Semantics, from_dynamic(img) = grayscale(img), then channel 0 / 255f32 (8-bit) or / 65535f32 (16-bit), one correctly rounded f32
 * division (image.rs:53-86):
 *   LUMA8, LUMA_A8, LUMA16, LUMA_A16: grayscale() returns the image unchanged; the luma is divided, alpha is never read.  Pinned by the
 *     reference tree itself.
 *   RGB8, RGBA8, RGB16, RGBA16: grayscale() applies the image crate's rgb_to_luma (image 0.24, color.rs; an external crate restated from
 *     its published source):  Y = (2126 R + 7152 G + 722 B) / 10000  with u32 intermediates and truncating integer division (the
 *     coefficients sum to 10000, so Y never exceeds the channel's maximum; a gray pixel R = G = B = v gives exactly v).  Alpha is dropped.
 *     Parity unpinned beyond that restatement (as imageproc's clamp in cvb200_sfm.h): no image-crate build checks it here.  The formula
 *     lives in one device function (rgb_to_luma, cv_b200/csrc/image.cu) and one oracle function (oracle/ref_image.c).
 *   RGB32F, RGBA32F: CVB_EUNSUPPORTED (their grayscale() / to_luma() clamping is not restated; a gray f32 plane has its own entry points).
 * The RGB8 plane of frame ingestion follows to_rgb8(): LUMA8 and LUMA_A8 copy the luma into all three channels, RGBA8 drops alpha, RGB8
 * is used as it is.  to_rgb8()'s 16 -> 8-bit conversion is image-crate internal and unpinned, so frame ingestion takes the four 8-bit
 * formats only; the 16-bit ones are CVB_EUNSUPPORTED there. */
#ifndef CVB200_IMAGE_H
#define CVB200_IMAGE_H
#include "cvb200_sfm.h"

#ifdef __cplusplus
extern "C" {
#endif

/* image::ColorType / the DynamicImage variants, in the image crate's order (bytes per pixel in brackets) */
typedef uint32_t cvb_pixel_format;
#define CVB_PIXEL_LUMA8 0      /* [1] */
#define CVB_PIXEL_LUMA_A8 1    /* [2] */
#define CVB_PIXEL_RGB8 2       /* [3] */
#define CVB_PIXEL_RGBA8 3      /* [4] */
#define CVB_PIXEL_LUMA16 4     /* [2] */
#define CVB_PIXEL_LUMA_A16 5   /* [4] */
#define CVB_PIXEL_RGB16 6      /* [6] */
#define CVB_PIXEL_RGBA16 7     /* [8] */
#define CVB_PIXEL_RGB32F 8     /* [12] CVB_EUNSUPPORTED */
#define CVB_PIXEL_RGBA32F 9    /* [16] CVB_EUNSUPPORTED */

/* The conversion on its own: pixels_dev (batch frames) -> gray_out_dev (batch x h x w f32, frame b at b * w * h: the layout
 * cvb_akaze_extract_batch_dev reads) and, when rgb_out_dev is non-NULL, the to_rgb8() plane (batch x h x w x 3 u8, the layout
 * cvb_frame_features_batch_dev reads; 8-bit formats only).  One kernel launch, asynchronous on the context's stream. */
int cvb_gray_float_from_dynamic_dev(cvb_ctx *ctx, cvb_pixel_format format, const void *pixels_dev, uint32_t batch, uint32_t w, uint32_t h,
                                    float *gray_out_dev, uint8_t *rgb_out_dev);

/* cvb_akaze_extract_batch(_dev) (include/cvb200.h) on batch frames of one pixel format */
int cvb_akaze_extract_dynamic_batch(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, cvb_pixel_format format, const void *pixels, uint32_t batch,
                                    uint32_t w, uint32_t h, cvb_keypoint *kp_out, uint8_t *desc_out, uint32_t cap, uint32_t *n_out);
int cvb_akaze_extract_dynamic_batch_dev(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, cvb_pixel_format format, const void *pixels_dev,
                                        uint32_t batch, uint32_t w, uint32_t h, cvb_keypoint *kp_out_dev, uint8_t *desc_out_dev, uint32_t cap,
                                        uint32_t *n_out_dev);

/* cvb_frame_features_batch (include/cvb200_sfm.h) from one image per frame: the extractor's plane and the colour plane both come from
 * `pixels` (8-bit formats only) */
int cvb_frame_features_dynamic_batch(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, cvb_pixel_format format, const void *pixels, uint32_t batch,
                                     uint32_t w, uint32_t h, const cvb_intrinsics_k1 *intrinsics, cvb_keypoint *kp_out, uint8_t *desc_out,
                                     double *bearings_out, uint8_t *colors_out, uint32_t cap, uint32_t *n_out);

/* cvb_two_view_frames_k1 (include/cvb200_sfm.h) on two host frames of one size and pixel format, frame a then frame b */
int cvb_two_view_frames_dynamic_k1(cvb_ctx *ctx, const cvb_akaze_cfg *akaze, cvb_pixel_format format, const void *frames, uint32_t w,
                                   uint32_t h, uint32_t better_by, const cvb_intrinsics_k1 *intrinsics, const cvb_arrsac_cfg *cfg, cvb_rng *rng,
                                   cvb_keypoint *kp_out, uint8_t *desc_out, uint32_t cap, uint32_t *n_out, uint32_t *pairs_out,
                                   uint32_t *n_pairs, cvb_pose *model_out, uint32_t *inliers_out, uint32_t *n_inliers, int32_t *found);

#ifdef __cplusplus
}
#endif
#endif /* CVB200_IMAGE_H */
