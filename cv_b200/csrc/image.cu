// cv_b200/csrc/image.cu -- the extractor's input on the device (include/cvb200_image.h): 8- and 16-bit luma / RGB(A) frames converted
// as GrayFloatImage::from_dynamic (akaze/src/image.rs:45-109) converts a DynamicImage, and for frame ingestion into the to_rgb8() plane.
// k_from_dynamic is one pass over the packed bytes; the host entry points then take the f32 paths of akaze.cu, frame.cu and pair.cu on
// the converted planes.  The C names are given by image_abi.cu (libcvb200_image.so), so libcvb200.so's exports stay as they are.
#include <algorithm>
#include "common.cuh"
#include "../../include/cvb200_image.h"

struct ImageWorkspace {
    uint8_t *raw = nullptr; size_t raw_bytes = 0;   // uploaded frames of the host forms
    float *gray = nullptr; size_t gray_px = 0;      // converted planes: the extractor's input, reused so that its graph replays
    uint8_t *rgb = nullptr; size_t rgb_px = 0;      // to_rgb8() planes of frame ingestion
};

void image_workspace_free(ImageWorkspace *w) {
    if (!w) return;
    cudaFree(w->raw); cudaFree(w->gray); cudaFree(w->rgb);
    delete w;
}

namespace {

// image 0.24 rgb_to_luma (color.rs; external crate, restated from its published source): integer sRGB luma coefficients over 10000,
// u32 intermediates (T::Larger of u8 and u16), truncating division.  The one device copy of the formula (see include/cvb200_image.h).
__device__ __forceinline__ uint32_t rgb_to_luma(uint32_t r, uint32_t g, uint32_t b) { return (2126u * r + 7152u * g + 722u * b) / 10000u; }

// C channels of 8 or 16 bits per pixel; channel 0..2 are R, G, B when C >= 3, the luma otherwise; a trailing alpha is never read.
template <int C, bool W16>
struct Px {
    static constexpr int BPP = C * (W16 ? 2 : 1);
    static constexpr int VEC = BPP % 3 == 0 ? 3 : 1;            // 16-byte loads per group: 48 bytes for 3 and 6 bytes per pixel
    static constexpr int GP = 16 * VEC / BPP;                    // pixels per group (16, 8, 16, 4, 8, 4, 8, 2)
    __device__ __forceinline__ static uint32_t ch(const uint8_t *p, int c) {
        if constexpr (W16) return (uint32_t)p[2 * c] | ((uint32_t)p[2 * c + 1] << 8);
        else return p[c];
    }
    __device__ __forceinline__ static uint32_t luma(const uint8_t *p) {
        if constexpr (C >= 3) return rgb_to_luma(ch(p, 0), ch(p, 1), ch(p, 2));
        else return ch(p, 0);
    }
    // from_dynamic: one correctly rounded f32 division (image.rs:53-86); not __fdividef, not a reciprocal multiply
    __device__ __forceinline__ static float gray(const uint8_t *p) { return __fdiv_rn((float)luma(p), W16 ? 65535.0f : 255.0f); }
};

// to_rgb8() of one 8-bit pixel: a luma is copied into all three channels, alpha is dropped
template <int C>
__device__ __forceinline__ void rgb8(const uint8_t *p, uint8_t *o) {
    o[0] = p[0]; o[1] = C >= 3 ? p[1] : p[0]; o[2] = C >= 3 ? p[2] : p[0];
}

// One thread per group of GP pixels.  The frames are packed, so the batch is one stream of npx pixels whose groups start at multiples
// of 16 bytes: with 16-byte aligned buffers a group is read with 16-byte loads and written with 16-byte (gray) and 4-byte (rgb) stores.
// The last, partial group (a row width whose bytes are not a multiple of 16 leaves one at the end of the batch) and unaligned caller
// buffers go pixel by pixel.  gray: npx f32; rgb (8-bit formats, may be null): 3 * npx u8 of to_rgb8().
template <int C, bool W16>
__global__ void __launch_bounds__(256) k_from_dynamic(const uint8_t *__restrict__ src, size_t npx, bool aligned, float *__restrict__ gray,
                                                      uint8_t *__restrict__ rgb) {
    using P = Px<C, W16>;
    const size_t p0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * P::GP;
    if (p0 >= npx) return;
    if (aligned && p0 + P::GP <= npx) {
        uint4 v[P::VEC];
        const uint4 *s = reinterpret_cast<const uint4 *>(src + p0 * P::BPP);
#pragma unroll
        for (int k = 0; k < P::VEC; k++) v[k] = __ldg(s + k);
        const uint8_t *b = reinterpret_cast<const uint8_t *>(v);
        float g[P::GP];
#pragma unroll
        for (int k = 0; k < P::GP; k++) g[k] = P::gray(b + k * P::BPP);
        if constexpr (P::GP % 4 == 0) {
#pragma unroll
            for (int k = 0; k < P::GP; k += 4) *reinterpret_cast<float4 *>(gray + p0 + k) = make_float4(g[k], g[k + 1], g[k + 2], g[k + 3]);
        } else {
#pragma unroll
            for (int k = 0; k < P::GP; k++) gray[p0 + k] = g[k];
        }
        if constexpr (!W16) {   // every 8-bit group has a multiple of 4 pixels: 3 * GP bytes at 3 * p0, a multiple of 12
            if (rgb) {
                uint32_t o[3 * P::GP / 4];
#pragma unroll
                for (int k = 0; k < P::GP; k++) rgb8<C>(b + k * P::BPP, reinterpret_cast<uint8_t *>(o) + 3 * k);
                uint32_t *d = reinterpret_cast<uint32_t *>(rgb + 3 * p0);
#pragma unroll
                for (int k = 0; k < 3 * P::GP / 4; k++) d[k] = o[k];
            }
        }
    } else {
        const size_t end = p0 + P::GP < npx ? p0 + P::GP : npx;
        for (size_t i = p0; i < end; i++) {
            const uint8_t *p = src + i * P::BPP;
            gray[i] = P::gray(p);
            if constexpr (!W16) {
                if (rgb) rgb8<C>(p, rgb + 3 * i);
            }
        }
    }
}

int bytes_per_pixel(cvb_pixel_format f) {
    static const int bpp[10] = {1, 2, 3, 4, 2, 4, 6, 8, 12, 16};
    return f < 10 ? bpp[f] : 0;
}

// the argument checks every entry point shares: 0 or the error code (set on the context)
int check_format(cvb_ctx *ctx, cvb_pixel_format format, bool rgb, uint32_t batch, uint32_t w, uint32_t h) {
    if (format > CVB_PIXEL_RGBA32F) return cvb_set_error(ctx, CVB_EINVAL, "unknown pixel format %u", format);
    if (format >= CVB_PIXEL_RGB32F) return cvb_set_error(ctx, CVB_EUNSUPPORTED, "float pixel formats are not supported");
    if (rgb && format >= CVB_PIXEL_LUMA16) return cvb_set_error(ctx, CVB_EUNSUPPORTED, "the RGB8 plane is made from 8-bit formats only");
    if (batch == 0 || w == 0 || h == 0) return cvb_set_error(ctx, CVB_EINVAL, "empty image or batch");
    if ((uint64_t)w * h > (1ull << 28)) return cvb_set_error(ctx, CVB_EUNSUPPORTED, "image too large");
    return 0;
}

ImageWorkspace *workspace(cvb_ctx *ctx) {
    if (!ctx->image) ctx->image = new ImageWorkspace();
    return ctx->image;
}

int launch_from_dynamic(cvb_ctx *ctx, cvb_pixel_format format, const void *pixels_dev, size_t npx, float *gray, uint8_t *rgb) {
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    const uint8_t *src = (const uint8_t *)pixels_dev;
    const bool aligned = ((uintptr_t)src & 15) == 0 && ((uintptr_t)gray & 15) == 0 && ((uintptr_t)rgb & 3) == 0;
    const int bpp = bytes_per_pixel(format);
    CVB_PROF(ctx, "k_from_dynamic", (double)npx * (bpp + 4 + (rgb ? 3 : 0)));
    const int gp = 16 * (bpp % 3 == 0 ? 3 : 1) / bpp;
    const size_t groups = (npx + gp - 1) / gp;
    if (groups > (size_t)INT32_MAX * 256) return cvb_set_error(ctx, CVB_EUNSUPPORTED, "batch too large");
    const unsigned grid = (unsigned)((groups + 255) / 256);
    cudaStream_t st = ctx->stream;
    switch (format) {
    case CVB_PIXEL_LUMA8: k_from_dynamic<1, false><<<grid, 256, 0, st>>>(src, npx, aligned, gray, rgb); break;
    case CVB_PIXEL_LUMA_A8: k_from_dynamic<2, false><<<grid, 256, 0, st>>>(src, npx, aligned, gray, rgb); break;
    case CVB_PIXEL_RGB8: k_from_dynamic<3, false><<<grid, 256, 0, st>>>(src, npx, aligned, gray, rgb); break;
    case CVB_PIXEL_RGBA8: k_from_dynamic<4, false><<<grid, 256, 0, st>>>(src, npx, aligned, gray, rgb); break;
    case CVB_PIXEL_LUMA16: k_from_dynamic<1, true><<<grid, 256, 0, st>>>(src, npx, aligned, gray, nullptr); break;
    case CVB_PIXEL_LUMA_A16: k_from_dynamic<2, true><<<grid, 256, 0, st>>>(src, npx, aligned, gray, nullptr); break;
    case CVB_PIXEL_RGB16: k_from_dynamic<3, true><<<grid, 256, 0, st>>>(src, npx, aligned, gray, nullptr); break;
    case CVB_PIXEL_RGBA16: k_from_dynamic<4, true><<<grid, 256, 0, st>>>(src, npx, aligned, gray, nullptr); break;
    default: return cvb_set_error(ctx, CVB_EINVAL, "unknown pixel format %u", format);
    }
    CVB_LAUNCH_CHECK(ctx);
    return 0;
}

// host frames -> the context's converted planes (and RGB8 planes when `rgb`)
int upload_and_convert(cvb_ctx *ctx, cvb_pixel_format format, const void *pixels, uint32_t batch, uint32_t w, uint32_t h, bool rgb) {
    ImageWorkspace *iw = workspace(ctx);
    const size_t npx = (size_t)batch * w * h, bytes = npx * bytes_per_pixel(format);
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    int rc;
    if ((rc = ws_grow(ctx, &iw->raw, &iw->raw_bytes, bytes)) || (rc = ws_grow(ctx, &iw->gray, &iw->gray_px, npx))) return rc;
    if (rgb && (rc = ws_grow(ctx, &iw->rgb, &iw->rgb_px, 3 * npx))) return rc;
    CVB_CUDA(ctx, cudaMemcpyAsync(iw->raw, pixels, bytes, cudaMemcpyHostToDevice, ctx->stream));
    return launch_from_dynamic(ctx, format, iw->raw, npx, iw->gray, rgb ? iw->rgb : nullptr);
}

}  // namespace

int img_gray_float_from_dynamic_dev(cvb_ctx *ctx, cvb_pixel_format format, const void *pixels_dev, uint32_t batch, uint32_t w, uint32_t h,
                                    float *gray_out_dev, uint8_t *rgb_out_dev) {
    if (!ctx) return CVB_EINVAL;
    int rc = check_format(ctx, format, rgb_out_dev != nullptr, batch, w, h);
    if (rc) return rc;
    if (!pixels_dev || !gray_out_dev) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    return launch_from_dynamic(ctx, format, pixels_dev, (size_t)batch * w * h, gray_out_dev, rgb_out_dev);
}

int img_akaze_extract_dynamic_batch(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, cvb_pixel_format format, const void *pixels, uint32_t batch,
                                    uint32_t w, uint32_t h, cvb_keypoint *kp_out, uint8_t *desc_out, uint32_t cap, uint32_t *n_out) {
    if (!ctx) return CVB_EINVAL;
    int rc = check_format(ctx, format, false, batch, w, h);
    if (rc) return rc;
    if (!cfg || !pixels) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (!n_out || (cap && (!kp_out || !desc_out))) return cvb_set_error(ctx, CVB_EINVAL, "null output");
    if ((rc = upload_and_convert(ctx, format, pixels, batch, w, h, false))) return rc;
    return akaze_extract_batch_host(ctx, cfg, ctx->image->gray, true, batch, w, h, kp_out, desc_out, cap, n_out);
}

int img_akaze_extract_dynamic_batch_dev(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, cvb_pixel_format format, const void *pixels_dev,
                                        uint32_t batch, uint32_t w, uint32_t h, cvb_keypoint *kp_out_dev, uint8_t *desc_out_dev, uint32_t cap,
                                        uint32_t *n_out_dev) {
    if (!ctx) return CVB_EINVAL;
    int rc = check_format(ctx, format, false, batch, w, h);
    if (rc) return rc;
    if (!cfg || !pixels_dev) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (!kp_out_dev || !desc_out_dev || !n_out_dev) return cvb_set_error(ctx, CVB_EINVAL, "null output");
    ImageWorkspace *iw = workspace(ctx);
    const size_t npx = (size_t)batch * w * h;
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    if ((rc = ws_grow(ctx, &iw->gray, &iw->gray_px, npx))) return rc;
    if ((rc = launch_from_dynamic(ctx, format, pixels_dev, npx, iw->gray, nullptr))) return rc;
    return cvb_akaze_extract_batch_dev(ctx, cfg, iw->gray, batch, w, h, kp_out_dev, desc_out_dev, cap, n_out_dev);
}

int img_frame_features_dynamic_batch(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, cvb_pixel_format format, const void *pixels, uint32_t batch,
                                     uint32_t w, uint32_t h, const cvb_intrinsics_k1 *intrinsics, cvb_keypoint *kp_out, uint8_t *desc_out,
                                     double *bearings_out, uint8_t *colors_out, uint32_t cap, uint32_t *n_out) {
    if (!ctx) return CVB_EINVAL;
    int rc = check_format(ctx, format, true, batch, w, h);
    if (rc) return rc;
    if (!cfg || !pixels || !intrinsics || !n_out || (cap && (!kp_out || !desc_out || !bearings_out || !colors_out)))
        return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if ((rc = upload_and_convert(ctx, format, pixels, batch, w, h, true))) return rc;
    return frame_features_batch_host(ctx, cfg, ctx->image->gray, ctx->image->rgb, true, batch, w, h, intrinsics, kp_out, desc_out,
                                     bearings_out, colors_out, cap, n_out);
}

int img_two_view_frames_dynamic_k1(cvb_ctx *ctx, const cvb_akaze_cfg *akaze, cvb_pixel_format format, const void *frames, uint32_t w,
                                   uint32_t h, uint32_t better_by, const cvb_intrinsics_k1 *intrinsics, const cvb_arrsac_cfg *cfg, cvb_rng *rng,
                                   cvb_keypoint *kp_out, uint8_t *desc_out, uint32_t cap, uint32_t *n_out, uint32_t *pairs_out,
                                   uint32_t *n_pairs, cvb_pose *model_out, uint32_t *inliers_out, uint32_t *n_inliers, int32_t *found) {
    if (!ctx) return CVB_EINVAL;
    int rc = check_format(ctx, format, false, 2, w, h);
    if (rc) return rc;
    if (!akaze || !frames || !intrinsics || !cfg || !rng || !kp_out || !desc_out || !n_out || !pairs_out || !n_pairs || !model_out ||
        !inliers_out || !n_inliers || !found)
        return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (cap == 0) return cvb_set_error(ctx, CVB_EINVAL, "empty image or zero capacity");
    if ((rc = upload_and_convert(ctx, format, frames, 2, w, h, false))) return rc;
    return two_view_frames_k1_host(ctx, akaze, ctx->image->gray, true, w, h, better_by, intrinsics, cfg, rng, kp_out, desc_out, cap, n_out,
                                   pairs_out, n_pairs, model_out, inliers_out, n_inliers, found);
}
