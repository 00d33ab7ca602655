// cv_b200/csrc/common.cuh -- shared declarations for libcvb200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <algorithm>
#include <string>
#include <vector>
#include "../../include/cvb200_sfm.h"   // includes cvb200.h

struct AkazeWorkspace;
struct MatchWorkspace;
struct GeomWorkspace;
struct PairWorkspace;
struct FrameWorkspace;
struct ImageWorkspace;
struct FilterWorkspace;
struct LshWorkspace;

struct cvb_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = true;
    std::string err;
    uint64_t launches = 0;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    cudaEvent_t ev_wait = nullptr;   // blocking-sync event of cvb_wait
    int num_sms = 132;
    AkazeWorkspace *akaze = nullptr;
    MatchWorkspace *match = nullptr;
    GeomWorkspace *geom = nullptr;
    PairWorkspace *pair = nullptr;
    FrameWorkspace *frame = nullptr;
    ImageWorkspace *image = nullptr;
    FilterWorkspace *filter = nullptr;
    LshWorkspace *lsh = nullptr;
    // page-locked host scratch for the small device->host results of the host API (a D2H copy into pageable memory is
    // staged synchronously inside the driver and stalls the other contexts' launches)
    void *pinned = nullptr;
    size_t pinned_bytes = 0;
    // optional per-kernel CUDA-event profiling (bench.py roofline pass); off by default
    bool prof = false;
    std::vector<cudaEvent_t> prof_pool;
    size_t prof_used = 0;
    struct ProfRec { const char *name; cudaEvent_t e0, e1; double bytes; };
    std::vector<ProfRec> prof_recs;
};

cudaEvent_t cvb_prof_event(cvb_ctx *ctx);
// Host wait for a stream.  Default: the thread sleeps on a blocking-sync event (a service runs one host thread per context and
// several ranks per box; spinning threads take the cores the launching threads need).  CVB_SYNC=spin: cudaStreamSynchronize.
cudaError_t cvb_wait(cvb_ctx *ctx, cudaStream_t st);
void *cvb_pinned(cvb_ctx *ctx, size_t bytes);   // >= bytes of page-locked scratch (nullptr on failure); valid until the next call
struct CvbProfScope {
    cvb_ctx *ctx; const char *name; double bytes; cudaEvent_t e0 = nullptr;
    CvbProfScope(cvb_ctx *c, const char *n, double b) : ctx(c), name(n), bytes(b) {
        if (ctx->prof) { e0 = cvb_prof_event(ctx); cudaEventRecord(e0, ctx->stream); }
    }
    ~CvbProfScope() {
        if (ctx->prof && e0) { cudaEvent_t e1 = cvb_prof_event(ctx); cudaEventRecord(e1, ctx->stream); ctx->prof_recs.push_back({name, e0, e1, bytes}); }
    }
};
// PROF(ctx, "kernel", algorithmic_bytes) brackets the launches that follow in the current scope
#define CVB_PROF(ctx, name, bytes) CvbProfScope prof_scope__((ctx), (name), (double)(bytes))

int cvb_set_error(cvb_ctx *ctx, int code, const char *fmt, ...);
void akaze_workspace_free(AkazeWorkspace *ws);
void match_workspace_free(MatchWorkspace *ws);
void geom_workspace_free(GeomWorkspace *ws);
void pair_workspace_free(PairWorkspace *ws);
void frame_workspace_free(FrameWorkspace *ws);
void image_workspace_free(ImageWorkspace *ws);
void filter_workspace_free(FilterWorkspace *ws);
void lsh_workspace_free(LshWorkspace *ws);

// Bodies of the host-API entry points cvb_akaze_extract_batch, cvb_frame_features_batch and cvb_two_view_frames_k1.  With the
// *_on_device flag set, the f32 planes (and the RGB8 plane) are already on the device and nothing is uploaded: the pixel-format entry
// points of image.cu (include/cvb200_image.h) convert into their own buffers, then take exactly these paths.
// The capacity reruns of the host calls (akaze.cu): clear the overflow flag before a run; after a run that raised it, grow the
// keypoint capacities to what the frames needed and set *rerun (CVB_ECAP once `attempt` reaches the limit).
int akaze_clear_overflow(cvb_ctx *ctx);
int akaze_capacity_rerun(cvb_ctx *ctx, unsigned B, int attempt, bool *rerun);
int akaze_extract_batch_host(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, const float *images, bool images_on_device, uint32_t batch, uint32_t w,
                             uint32_t h, cvb_keypoint *kp_out, uint8_t *desc_out, uint32_t cap, uint32_t *n_out);
int frame_features_batch_host(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, const float *images, const uint8_t *rgb, bool planes_on_device,
                              uint32_t batch, uint32_t w, uint32_t h, const cvb_intrinsics_k1 *intrinsics, cvb_keypoint *kp_out,
                              uint8_t *desc_out, double *bearings_out, uint8_t *colors_out, uint32_t cap, uint32_t *n_out);
int two_view_frames_k1_host(cvb_ctx *ctx, const cvb_akaze_cfg *akaze, const float *frames, bool frames_on_device, uint32_t w, uint32_t h,
                            uint32_t better_by, const cvb_intrinsics_k1 *intrinsics, const cvb_arrsac_cfg *cfg, cvb_rng *rng,
                            cvb_keypoint *kp_out, uint8_t *desc_out, uint32_t cap, uint32_t *n_out, uint32_t *pairs_out, uint32_t *n_pairs,
                            cvb_pose *model_out, uint32_t *inliers_out, uint32_t *n_inliers, int32_t *found);

// akaze.cu pieces the public image module (filter.cu, include/cvb200_filter.h) reuses: gaussian_kernel (image.rs:349-374) on the host, and
// one launch of the extractor's k_half_size over `batch` packed planes (out: batch planes of (w / 2) x (h / 2), both non-empty).
void gaussian_kernel_host(float r, int ks, float *out);
int half_size_launch(cvb_ctx *ctx, const float *in, float *out, uint32_t batch, uint32_t w, uint32_t h);

// A device buffer of the context's workspaces grown to >= n elements (contents not kept); waits for the stream before freeing.
template <typename T>
int ws_grow(cvb_ctx *ctx, T **p, size_t *have, size_t n) {
    if (*have >= n) return 0;
    if (*p) { cvb_wait(ctx, ctx->stream); cudaFree(*p); *p = nullptr; *have = 0; }
    const cudaError_t e = cudaMalloc((void **)p, std::max<size_t>(n, 1) * sizeof(T));
    if (e != cudaSuccess) return cvb_set_error(ctx, CVB_ENOMEM, "cudaMalloc: %s", cudaGetErrorString(e));
    *have = n;
    return 0;
}

#define CVB_CUDA(ctx, call)                                                                          \
    do {                                                                                             \
        cudaError_t e__ = (call);                                                                    \
        if (e__ != cudaSuccess)                                                                      \
            return cvb_set_error((ctx), CVB_ECUDA, "%s:%d %s: %s", __FILE__, __LINE__, #call,        \
                                 cudaGetErrorString(e__));                                           \
    } while (0)

#define CVB_LAUNCH_CHECK(ctx)                                                                        \
    do {                                                                                             \
        (ctx)->launches++;                                                                           \
        cudaError_t e__ = cudaPeekAtLastError();                                                     \
        if (e__ != cudaSuccess)                                                                      \
            return cvb_set_error((ctx), CVB_ECUDA, "%s:%d launch: %s", __FILE__, __LINE__,           \
                                 cudaGetErrorString(e__));                                           \
    } while (0)

static inline unsigned cdiv(unsigned a, unsigned b) { return (a + b - 1) / b; }
