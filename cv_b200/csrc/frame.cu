// cv_b200/csrc/frame.cu -- cv-sfm frame ingestion, VSlam::kps_descriptors (cv-sfm/src/lib.rs:2195-2235): AKAZE, then per keypoint its
// K1 bearing and its bicubic RGB colour.  The extractor is cvb_akaze_extract_batch_dev unchanged; k_frame_features adds the rest.
#include <algorithm>
#include "common.cuh"
#include "pinhole.cuh"

struct FrameWorkspace {
    float *img = nullptr; uint8_t *rgb = nullptr; size_t px = 0;   // px = batch * w * h
    cvb_keypoint *kp = nullptr; uint8_t *desc = nullptr; double *bear = nullptr; uint8_t *col = nullptr; size_t slots = 0;   // batch * cap
    uint32_t *n = nullptr; uint32_t batch = 0;
};

void frame_workspace_free(FrameWorkspace *w) {
    if (!w) return;
    cudaFree(w->img); cudaFree(w->rgb); cudaFree(w->kp); cudaFree(w->desc); cudaFree(w->bear); cudaFree(w->col); cudaFree(w->n);
    delete w;
}

namespace {

// imageproc 0.23 `Clamp<f32> for u8` (definitions.rs; external crate, restated from its published source): truncating cast inside
// (0, 255), saturating outside.
__device__ __forceinline__ uint8_t clamp_u8(float x) { return x < 255.0f ? (x > 0.0f ? (uint8_t)x : (uint8_t)0) : (uint8_t)255; }

// cv-sfm/src/bicubic.rs:13-31 blend_cubic for one channel, f32, in the source's association order (-fmad=false: no contraction).
__device__ __forceinline__ float blend_cubic(float p0, float p1, float p2, float p3, float x) {
    return p1 + 0.5f * x * (p2 - p0 + x * (2.0f * p0 - 5.0f * p1 + 4.0f * p2 - p3 + x * (3.0f * (p1 - p2) + p3 - p0)));
}

// cv-sfm/src/bicubic.rs:33-68 interpolate_bicubic on an RgbImage with default Rgb([0, 0, 0]).  The border test uses right = left + 4
// (not left + 3, the last column read) exactly as the reference does; each row blend is clamped to u8 because it is stored in a Pixel.
__device__ __forceinline__ void bicubic_rgb8(const uint8_t *__restrict__ rgb, uint32_t w, uint32_t h, float x, float y, uint8_t *out) {
    const float left = floorf(x) - 1.0f, right = left + 4.0f, top = floorf(y) - 1.0f, bottom = top + 4.0f;
    const float xw = x - (left + 1.0f), yw = y - (top + 1.0f);
    if (left < 0.0f || right >= (float)w || top < 0.0f || bottom >= (float)h) { out[0] = out[1] = out[2] = 0; return; }
    const uint32_t l = (uint32_t)left, t = (uint32_t)top;
    float col[3][4];
    for (int r = 0; r < 4; r++) {
        const uint8_t *p = rgb + ((size_t)(t + r) * w + l) * 3;
        for (int c = 0; c < 3; c++) col[c][r] = (float)clamp_u8(blend_cubic((float)p[c], (float)p[3 + c], (float)p[6 + c], (float)p[9 + c], xw));
    }
    for (int c = 0; c < 3; c++) out[c] = clamp_u8(blend_cubic(col[c][0], col[c][1], col[c][2], col[c][3], yw));
}

// One thread per keypoint, frame on grid.y.  Keypoint i of frame b is feature i (see the order note in include/cvb200.h).
__global__ void __launch_bounds__(128) k_frame_features(const cvb_keypoint *__restrict__ kp, const uint32_t *__restrict__ n, uint32_t cap,
                                                        const uint8_t *__restrict__ rgb, uint32_t w, uint32_t h, cvb_intrinsics_k1 K,
                                                        double *__restrict__ bearings, uint8_t *__restrict__ colors) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (i >= min(n[b], cap)) return;
    const size_t s = (size_t)b * cap + i;
    const cvb_keypoint k = kp[s];
    calibrate_k1(K, (double)k.x, (double)k.y, bearings + 3 * s);       // ImagePoint of akaze::KeyPoint: (x as f64, y as f64)
    uint8_t c[3];
    bicubic_rgb8(rgb + (size_t)b * w * h * 3, w, h, k.x, k.y, c);
    colors[3 * s] = c[0]; colors[3 * s + 1] = c[1]; colors[3 * s + 2] = c[2];
}

template <typename T>
int grow(cvb_ctx *ctx, T **p, size_t n) {
    if (*p) { cvb_wait(ctx, ctx->stream); cudaFree(*p); *p = nullptr; }
    const cudaError_t e = cudaMalloc((void **)p, std::max<size_t>(n, 1) * sizeof(T));
    if (e != cudaSuccess) return cvb_set_error(ctx, CVB_ENOMEM, "cudaMalloc: %s", cudaGetErrorString(e));
    return 0;
}

int ensure_frame(cvb_ctx *ctx, uint32_t batch, size_t px, size_t slots) {
    if (!ctx->frame) ctx->frame = new FrameWorkspace();
    FrameWorkspace *w = ctx->frame;
    int rc;
    if (w->px < px) {
        if ((rc = grow(ctx, &w->img, px)) || (rc = grow(ctx, &w->rgb, 3 * px))) return rc;
        w->px = px;
    }
    if (w->slots < slots) {
        if ((rc = grow(ctx, &w->kp, slots)) || (rc = grow(ctx, &w->desc, 64 * slots)) || (rc = grow(ctx, &w->bear, 3 * slots)) ||
            (rc = grow(ctx, &w->col, 3 * slots)))
            return rc;
        w->slots = slots;
    }
    if (w->batch < batch) { if ((rc = grow(ctx, &w->n, batch))) return rc; w->batch = batch; }
    return 0;
}

}  // namespace

extern "C" {

int cvb_frame_features_batch_dev(cvb_ctx *ctx, const cvb_keypoint *kp_dev, const uint32_t *n_dev, uint32_t batch, uint32_t cap,
                                 const uint8_t *rgb_dev, uint32_t w, uint32_t h, const cvb_intrinsics_k1 *intrinsics, double *bearings_out_dev,
                                 uint8_t *colors_out_dev) {
    if (!ctx) return CVB_EINVAL;
    if (!kp_dev || !n_dev || !rgb_dev || !intrinsics || !bearings_out_dev || !colors_out_dev) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (batch == 0 || cap == 0) return 0;
    if (w == 0 || h == 0) return cvb_set_error(ctx, CVB_EINVAL, "empty image");
    if (batch > 65535) return cvb_set_error(ctx, CVB_EUNSUPPORTED, "batch > 65535");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    CVB_PROF(ctx, "k_frame_features", 0);
    k_frame_features<<<dim3(cdiv(cap, 128), batch), 128, 0, ctx->stream>>>(kp_dev, n_dev, cap, rgb_dev, w, h, *intrinsics, bearings_out_dev,
                                                                          colors_out_dev);
    CVB_LAUNCH_CHECK(ctx);
    return 0;
}

int cvb_frame_features_batch(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, const float *images, const uint8_t *rgb, uint32_t batch, uint32_t w,
                             uint32_t h, const cvb_intrinsics_k1 *intrinsics, cvb_keypoint *kp_out, uint8_t *desc_out, double *bearings_out,
                             uint8_t *colors_out, uint32_t cap, uint32_t *n_out) {
    return frame_features_batch_host(ctx, cfg, images, rgb, false, batch, w, h, intrinsics, kp_out, desc_out, bearings_out, colors_out, cap,
                                     n_out);
}

}  // extern "C"

int frame_features_batch_host(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, const float *images, const uint8_t *rgb, bool planes_on_device,
                              uint32_t batch, uint32_t w, uint32_t h, const cvb_intrinsics_k1 *intrinsics, cvb_keypoint *kp_out,
                              uint8_t *desc_out, double *bearings_out, uint8_t *colors_out, uint32_t cap, uint32_t *n_out) {
    if (!ctx) return CVB_EINVAL;
    if (!cfg || !images || !rgb || !intrinsics || !n_out || (cap && (!kp_out || !desc_out || !bearings_out || !colors_out)))
        return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (batch == 0 || w == 0 || h == 0) return cvb_set_error(ctx, CVB_EINVAL, "empty image or batch");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    const size_t px = (size_t)batch * w * h, slots = (size_t)batch * std::max<uint32_t>(cap, 1);
    int rc = ensure_frame(ctx, batch, planes_on_device ? 0 : px, slots);
    if (rc) return rc;
    FrameWorkspace *fw = ctx->frame;
    const uint32_t cd = std::max<uint32_t>(cap, 1);
    cudaStream_t st = ctx->stream;
    if (!planes_on_device) {
        CVB_CUDA(ctx, cudaMemcpyAsync(fw->img, images, sizeof(float) * px, cudaMemcpyHostToDevice, st));
        CVB_CUDA(ctx, cudaMemcpyAsync(fw->rgb, rgb, 3 * px, cudaMemcpyHostToDevice, st));
        images = fw->img; rgb = fw->rgb;
    }
    // a frame that exceeds the extractor's keypoint capacities is run again in a grown workspace (the planes stay resident)
    if ((rc = akaze_clear_overflow(ctx))) return rc;
    for (int attempt = 0;; attempt++) {
        if ((rc = cvb_akaze_extract_batch_dev(ctx, cfg, images, batch, w, h, fw->kp, fw->desc, cd, fw->n))) return rc;
        if ((rc = cvb_frame_features_batch_dev(ctx, fw->kp, fw->n, batch, cd, rgb, w, h, intrinsics, fw->bear, fw->col))) return rc;
        // counts behind word 0 of the page-locked scratch, which cvb_akaze_dev_overflow fills with the flag (and then synchronises)
        uint32_t *hs = (uint32_t *)cvb_pinned(ctx, sizeof(uint32_t) * ((size_t)batch + 1));
        if (!hs) return cvb_set_error(ctx, CVB_ENOMEM, "page-locked scratch");
        CVB_CUDA(ctx, cudaMemcpyAsync(hs + 1, fw->n, sizeof(uint32_t) * batch, cudaMemcpyDeviceToHost, st));
        uint32_t ovf = 0;
        if ((rc = cvb_akaze_dev_overflow(ctx, &ovf))) return rc;
        for (uint32_t b = 0; b < batch; b++) n_out[b] = hs[1 + b];
        if (!ovf) break;
        bool rerun = false;
        if ((rc = akaze_capacity_rerun(ctx, batch, attempt, &rerun))) return rc;
        if (rerun) continue;
        if (ovf == 3) return cvb_set_error(ctx, CVB_ECAP, "output capacity %u too small", cap);
        break;
    }
    for (uint32_t b = 0; b < batch; b++) {
        const size_t n = std::min<uint32_t>(n_out[b], cap), o = (size_t)b * cap, od = (size_t)b * cd;
        if (!n) continue;
        CVB_CUDA(ctx, cudaMemcpyAsync(kp_out + o, fw->kp + od, sizeof(cvb_keypoint) * n, cudaMemcpyDeviceToHost, st));
        CVB_CUDA(ctx, cudaMemcpyAsync(desc_out + 64 * o, fw->desc + 64 * od, 64 * n, cudaMemcpyDeviceToHost, st));
        CVB_CUDA(ctx, cudaMemcpyAsync(bearings_out + 3 * o, fw->bear + 3 * od, sizeof(double) * 3 * n, cudaMemcpyDeviceToHost, st));
        CVB_CUDA(ctx, cudaMemcpyAsync(colors_out + 3 * o, fw->col + 3 * od, 3 * n, cudaMemcpyDeviceToHost, st));
    }
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    return 0;
}
