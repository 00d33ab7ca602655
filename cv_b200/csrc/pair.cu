// cv_b200/csrc/pair.cu -- one frame pair end to end: AKAZE extract x2 -> symmetric match -> bearings -> ARRSAC + eight-point.
// The sequence of cv-sfm's two-view initialisation (cv-sfm/src/lib.rs:1375-1412; extraction at :2200-2204) composed from the
// device-resident entry points of this library: one enqueue, one synchronisation, no intermediate host round trip.
#include <string.h>
#include <algorithm>
#include "common.cuh"
#include "pinhole.cuh"

struct PairWorkspace {
    float *img = nullptr; size_t img_floats = 0;
    cvb_keypoint *kp = nullptr; uint8_t *desc = nullptr; uint32_t *n = nullptr; uint32_t cap = 0;
    double *a = nullptr, *b = nullptr;
    unsigned char *res = nullptr;     // [n_pairs u32 | n_inliers u32 | found i32 | pad | model | pairs cap*2 | inliers cap]
    uint32_t res_cap = 0;
};

void pair_workspace_free(PairWorkspace *w) {
    if (!w) return;
    cudaFree(w->img); cudaFree(w->kp); cudaFree(w->desc); cudaFree(w->n); cudaFree(w->a); cudaFree(w->b); cudaFree(w->res);
    delete w;
}

namespace {

struct ResLayout { size_t model, pairs, inliers, bytes; };
ResLayout res_layout(uint32_t cap) {
    ResLayout L;
    L.model = 16;
    L.pairs = L.model + sizeof(cvb_pose);
    L.inliers = L.pairs + sizeof(uint32_t) * 2 * (size_t)cap;
    L.bytes = L.inliers + sizeof(uint32_t) * (size_t)cap;
    return L;
}

template <typename T>
int regrow(cvb_ctx *ctx, T **p, size_t n) {
    if (*p) { cvb_wait(ctx, ctx->stream); cudaFree(*p); *p = nullptr; }
    cudaError_t e = cudaMalloc((void **)p, std::max<size_t>(n, 1) * sizeof(T));
    if (e != cudaSuccess) return cvb_set_error(ctx, CVB_ENOMEM, "cudaMalloc: %s", cudaGetErrorString(e));
    return 0;
}

int ensure_pair(cvb_ctx *ctx, uint32_t cap, size_t img_floats) {
    if (!ctx->pair) ctx->pair = new PairWorkspace();
    PairWorkspace *w = ctx->pair;
    int rc;
    if (w->img_floats < img_floats) { if ((rc = regrow(ctx, &w->img, img_floats))) return rc; w->img_floats = img_floats; }
    if (w->cap < cap) {
        if ((rc = regrow(ctx, &w->kp, 2 * (size_t)cap))) return rc;
        if ((rc = regrow(ctx, &w->desc, 2 * (size_t)cap * 64))) return rc;
        if ((rc = regrow(ctx, &w->n, 2))) return rc;
        if ((rc = regrow(ctx, &w->a, 3 * (size_t)cap))) return rc;
        if ((rc = regrow(ctx, &w->b, 3 * (size_t)cap))) return rc;
        w->cap = cap;
    }
    if (w->res_cap < cap) { if ((rc = regrow(ctx, &w->res, res_layout(cap).bytes))) return rc; w->res_cap = cap; }
    return 0;
}

}  // namespace

extern "C" {

// The entry points taking cvb_intrinsics are the K1 ones with k1 = 0 (bit-identical bearings, pinhole.cuh).
int cvb_two_view_pair_dev(cvb_ctx *ctx, const cvb_keypoint *kp_a_dev, const uint8_t *desc_a_dev, const uint32_t *n_a_dev,
                          const cvb_keypoint *kp_b_dev, const uint8_t *desc_b_dev, const uint32_t *n_b_dev, uint32_t n_max,
                          uint32_t better_by, const cvb_intrinsics *intrinsics, const cvb_arrsac_cfg *cfg, const cvb_rng *rng,
                          uint32_t *pairs_out_dev, uint32_t cap, uint32_t *n_pairs_dev, cvb_pose *model_out_dev,
                          uint32_t *inliers_out_dev, uint32_t *n_inliers_dev, int32_t *found_dev) {
    const cvb_intrinsics_k1 K = intrinsics ? intrinsics_k1(*intrinsics) : cvb_intrinsics_k1{};
    return cvb_two_view_pair_k1_dev(ctx, kp_a_dev, desc_a_dev, n_a_dev, kp_b_dev, desc_b_dev, n_b_dev, n_max, better_by, intrinsics ? &K : nullptr,
                                    cfg, rng, pairs_out_dev, cap, n_pairs_dev, model_out_dev, inliers_out_dev, n_inliers_dev, found_dev);
}

int cvb_two_view_frames(cvb_ctx *ctx, const cvb_akaze_cfg *akaze, const float *frames, uint32_t w, uint32_t h, uint32_t better_by,
                        const cvb_intrinsics *intrinsics, const cvb_arrsac_cfg *cfg, cvb_rng *rng, cvb_keypoint *kp_out, uint8_t *desc_out,
                        uint32_t cap, uint32_t *n_out, uint32_t *pairs_out, uint32_t *n_pairs, cvb_pose *model_out, uint32_t *inliers_out,
                        uint32_t *n_inliers, int32_t *found) {
    const cvb_intrinsics_k1 K = intrinsics ? intrinsics_k1(*intrinsics) : cvb_intrinsics_k1{};
    return cvb_two_view_frames_k1(ctx, akaze, frames, w, h, better_by, intrinsics ? &K : nullptr, cfg, rng, kp_out, desc_out, cap, n_out,
                                  pairs_out, n_pairs, model_out, inliers_out, n_inliers, found);
}

int cvb_two_view_pair_k1_dev(cvb_ctx *ctx, const cvb_keypoint *kp_a_dev, const uint8_t *desc_a_dev, const uint32_t *n_a_dev,
                             const cvb_keypoint *kp_b_dev, const uint8_t *desc_b_dev, const uint32_t *n_b_dev, uint32_t n_max,
                             uint32_t better_by, const cvb_intrinsics_k1 *intrinsics, const cvb_arrsac_cfg *cfg, const cvb_rng *rng,
                             uint32_t *pairs_out_dev, uint32_t cap, uint32_t *n_pairs_dev, cvb_pose *model_out_dev,
                             uint32_t *inliers_out_dev, uint32_t *n_inliers_dev, int32_t *found_dev) {
    if (!ctx) return CVB_EINVAL;
    if (!kp_a_dev || !desc_a_dev || !n_a_dev || !kp_b_dev || !desc_b_dev || !n_b_dev || !intrinsics || !cfg || !rng || !pairs_out_dev ||
        !n_pairs_dev || !model_out_dev || !n_inliers_dev || !found_dev)
        return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (cap == 0 || n_max == 0) return cvb_set_error(ctx, CVB_EINVAL, "zero capacity");
    int rc = ensure_pair(ctx, cap, 0);
    if (rc) return rc;
    PairWorkspace *w = ctx->pair;
    if ((rc = cvb_match_symmetric_pairs_dev(ctx, desc_a_dev, n_a_dev, n_max, desc_b_dev, n_b_dev, n_max, better_by, pairs_out_dev, cap, n_pairs_dev)))
        return rc;
    if ((rc = cvb_pair_bearings_k1_dev(ctx, kp_a_dev, kp_b_dev, pairs_out_dev, n_pairs_dev, cap, intrinsics, w->a, w->b))) return rc;
    return cvb_arrsac_eight_point_dev(ctx, cfg, w->a, w->b, n_pairs_dev, cap, rng, model_out_dev, inliers_out_dev, cap, n_inliers_dev, found_dev);
}

int cvb_two_view_frames_k1(cvb_ctx *ctx, const cvb_akaze_cfg *akaze, const float *frames, uint32_t w, uint32_t h, uint32_t better_by,
                           const cvb_intrinsics_k1 *intrinsics, const cvb_arrsac_cfg *cfg, cvb_rng *rng, cvb_keypoint *kp_out,
                           uint8_t *desc_out, uint32_t cap, uint32_t *n_out, uint32_t *pairs_out, uint32_t *n_pairs, cvb_pose *model_out,
                           uint32_t *inliers_out, uint32_t *n_inliers, int32_t *found) {
    return two_view_frames_k1_host(ctx, akaze, frames, false, w, h, better_by, intrinsics, cfg, rng, kp_out, desc_out, cap, n_out, pairs_out,
                                   n_pairs, model_out, inliers_out, n_inliers, found);
}

}  // extern "C"

int two_view_frames_k1_host(cvb_ctx *ctx, const cvb_akaze_cfg *akaze, const float *frames, bool frames_on_device, uint32_t w, uint32_t h,
                            uint32_t better_by, const cvb_intrinsics_k1 *intrinsics, const cvb_arrsac_cfg *cfg, cvb_rng *rng,
                            cvb_keypoint *kp_out, uint8_t *desc_out, uint32_t cap, uint32_t *n_out, uint32_t *pairs_out, uint32_t *n_pairs,
                            cvb_pose *model_out, uint32_t *inliers_out, uint32_t *n_inliers, int32_t *found) {
    if (!ctx) return CVB_EINVAL;
    if (!akaze || !frames || !intrinsics || !cfg || !rng || !kp_out || !desc_out || !n_out || !pairs_out || !n_pairs || !model_out ||
        !inliers_out || !n_inliers || !found)
        return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (cap == 0 || w == 0 || h == 0) return cvb_set_error(ctx, CVB_EINVAL, "empty image or zero capacity");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    const size_t px = (size_t)w * h;
    int rc = ensure_pair(ctx, cap, frames_on_device ? 0 : 2 * px);
    if (rc) return rc;
    PairWorkspace *pw = ctx->pair;
    cudaStream_t st = ctx->stream;
    const ResLayout L = res_layout(pw->res_cap);
    uint32_t *n_pairs_dev = (uint32_t *)pw->res, *n_inl_dev = n_pairs_dev + 1;
    int32_t *found_dev = (int32_t *)(n_pairs_dev + 2);
    cvb_pose *model_dev = (cvb_pose *)(pw->res + L.model);
    uint32_t *pairs_dev = (uint32_t *)(pw->res + L.pairs), *inl_dev = (uint32_t *)(pw->res + L.inliers);
    if (!frames_on_device) CVB_CUDA(ctx, cudaMemcpyAsync(pw->img, frames, sizeof(float) * 2 * px, cudaMemcpyHostToDevice, st));
    if ((rc = cvb_akaze_extract_batch_dev(ctx, akaze, frames_on_device ? frames : pw->img, 2, w, h, pw->kp, pw->desc, pw->cap, pw->n)))
        return rc;
    if ((rc = cvb_two_view_pair_k1_dev(ctx, pw->kp, pw->desc, pw->n, pw->kp + pw->cap, pw->desc + (size_t)pw->cap * 64, pw->n + 1, pw->cap,
                                       better_by, intrinsics, cfg, rng, pairs_dev, cap, n_pairs_dev, model_dev, inl_dev, n_inl_dev, found_dev)))
        return rc;
    // results by capacity (the counts are only known on the device): one synchronisation at the very end
    unsigned char *hs = (unsigned char *)cvb_pinned(ctx, L.model + sizeof(cvb_pose) + 16);
    if (!hs) return cvb_set_error(ctx, CVB_ENOMEM, "page-locked scratch");
    CVB_CUDA(ctx, cudaMemcpyAsync(hs, pw->res, L.model + sizeof(cvb_pose), cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(hs + L.model + sizeof(cvb_pose), pw->n, 8, cudaMemcpyDeviceToHost, st));
    for (int f = 0; f < 2; f++) {
        CVB_CUDA(ctx, cudaMemcpyAsync(kp_out + (size_t)f * cap, pw->kp + (size_t)f * pw->cap, sizeof(cvb_keypoint) * cap, cudaMemcpyDeviceToHost, st));
        CVB_CUDA(ctx, cudaMemcpyAsync(desc_out + (size_t)f * cap * 64, pw->desc + (size_t)f * pw->cap * 64, (size_t)cap * 64, cudaMemcpyDeviceToHost, st));
    }
    CVB_CUDA(ctx, cudaMemcpyAsync(pairs_out, pairs_dev, sizeof(uint32_t) * 2 * cap, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(inliers_out, inl_dev, sizeof(uint32_t) * cap, cudaMemcpyDeviceToHost, st));
    if ((rc = cvb_arrsac_commit_rng(ctx, rng, nullptr))) return rc;      // synchronises the stream
    const uint32_t *hw = (const uint32_t *)hs;
    *n_pairs = hw[0]; *n_inliers = hw[1]; *found = (int32_t)hw[2];
    memcpy(model_out, hs + L.model, sizeof(cvb_pose));
    const uint32_t *hn = (const uint32_t *)(hs + L.model + sizeof(cvb_pose));
    n_out[0] = hn[0]; n_out[1] = hn[1];
    return 0;
}
