// cv_b200/csrc/ctx.cu -- context, error reporting, stream/event plumbing of libcvb200.so.
#include <stdarg.h>
#include <stdio.h>
#include <string.h>
#include <algorithm>
#include <vector>
#include "common.cuh"

int cvb_set_error(cvb_ctx *ctx, int code, const char *fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    if (ctx) ctx->err = buf;
    return code;
}

cudaEvent_t cvb_prof_event(cvb_ctx *ctx) {
    if (ctx->prof_used == ctx->prof_pool.size()) {
        cudaEvent_t e;
        cudaEventCreate(&e);
        ctx->prof_pool.push_back(e);
    }
    return ctx->prof_pool[ctx->prof_used++];
}

cudaError_t cvb_wait(cvb_ctx *ctx, cudaStream_t st) {
    static const bool spin = [] { const char *e = getenv("CVB_SYNC"); return e && !strcmp(e, "spin"); }();
    if (spin || !ctx) return cudaStreamSynchronize(st);
    if (!ctx->ev_wait) {
        const cudaError_t e = cudaEventCreateWithFlags(&ctx->ev_wait, cudaEventBlockingSync | cudaEventDisableTiming);
        if (e != cudaSuccess) { ctx->ev_wait = nullptr; cudaGetLastError(); return cudaStreamSynchronize(st); }
    }
    const cudaError_t e = cudaEventRecord(ctx->ev_wait, st);
    if (e != cudaSuccess) return e;
    return cudaEventSynchronize(ctx->ev_wait);
}

void *cvb_pinned(cvb_ctx *ctx, size_t bytes) {
    if (ctx->pinned && ctx->pinned_bytes >= bytes) return ctx->pinned;
    if (ctx->pinned) { cvb_wait(ctx, ctx->stream); cudaFreeHost(ctx->pinned); ctx->pinned = nullptr; ctx->pinned_bytes = 0; }
    const size_t n = std::max<size_t>(bytes, 64 * 1024);
    if (cudaHostAlloc(&ctx->pinned, n, cudaHostAllocDefault) != cudaSuccess) { ctx->pinned = nullptr; return nullptr; }
    ctx->pinned_bytes = n;
    return ctx->pinned;
}

extern "C" {

int cvb_ctx_profile(cvb_ctx *ctx, int enable) {
    if (!ctx) return CVB_EINVAL;
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    ctx->prof = enable != 0;
    ctx->prof_recs.clear();
    ctx->prof_used = 0;
    return 0;
}

// Text report: one line per kernel name: "name launches total_ms algorithmic_bytes"
int cvb_ctx_profile_report(cvb_ctx *ctx, char *buf, size_t cap) {
    if (!ctx || !buf || !cap) return CVB_EINVAL;
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    struct Agg { const char *name; int n; double ms, bytes; };
    std::vector<Agg> agg;
    for (auto &r : ctx->prof_recs) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, r.e0, r.e1);
        size_t i = 0;
        for (; i < agg.size(); i++) if (agg[i].name == r.name || !strcmp(agg[i].name, r.name)) break;
        if (i == agg.size()) agg.push_back({r.name, 0, 0.0, 0.0});
        agg[i].n++; agg[i].ms += ms; agg[i].bytes += r.bytes;
    }
    size_t off = 0;
    buf[0] = 0;
    for (auto &a : agg) {
        int w = snprintf(buf + off, cap - off, "%s %d %.6f %.0f\n", a.name, a.n, a.ms, a.bytes);
        if (w < 0 || (size_t)w >= cap - off) break;
        off += (size_t)w;
    }
    ctx->prof_recs.clear();
    ctx->prof_used = 0;
    return 0;
}

const char *cvb_version(void) { return "cvb200 0.1.0 (sm_90a)"; }

int cvb_ctx_create_on_stream(int device, void *cuda_stream, cvb_ctx **out) {
    if (!out) return CVB_EINVAL;
    *out = nullptr;
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count <= 0 || device < 0 || device >= count) return CVB_ENODEV;   // no CPU fallback
    if (cudaSetDevice(device) != cudaSuccess) return CVB_ENODEV;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return CVB_ENODEV;
    if (prop.major != 9 || prop.minor != 0) return CVB_ENODEV;   // kernels are built for sm_90a only
    cvb_ctx *ctx = new cvb_ctx();
    ctx->device = device;
    ctx->num_sms = prop.multiProcessorCount;
    if (cuda_stream) { ctx->stream = (cudaStream_t)cuda_stream; ctx->own_stream = false; }
    else if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) { delete ctx; return CVB_ECUDA; }
    cudaEventCreate(&ctx->ev0);
    cudaEventCreate(&ctx->ev1);
    *out = ctx;
    return CVB_OK;
}

int cvb_ctx_create(int device, cvb_ctx **out) { return cvb_ctx_create_on_stream(device, nullptr, out); }

void cvb_ctx_destroy(cvb_ctx *ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cvb_wait(ctx, ctx->stream);
    akaze_workspace_free(ctx->akaze);
    match_workspace_free(ctx->match);
    geom_workspace_free(ctx->geom);
    pair_workspace_free(ctx->pair);
    frame_workspace_free(ctx->frame);
    image_workspace_free(ctx->image);
    filter_workspace_free(ctx->filter);
    lsh_workspace_free(ctx->lsh);
    if (ctx->ev0) cudaEventDestroy(ctx->ev0);
    if (ctx->ev_wait) cudaEventDestroy(ctx->ev_wait);
    if (ctx->ev1) cudaEventDestroy(ctx->ev1);
    for (cudaEvent_t e : ctx->prof_pool) cudaEventDestroy(e);
    if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
    if (ctx->pinned) cudaFreeHost(ctx->pinned);
    delete ctx;
}

int cvb_ctx_sync(cvb_ctx *ctx) {
    if (!ctx) return CVB_EINVAL;
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    return 0;
}

const char *cvb_last_error(const cvb_ctx *ctx) { return ctx ? ctx->err.c_str() : "null context"; }

uint64_t cvb_ctx_launch_count(const cvb_ctx *ctx) { return ctx ? ctx->launches : 0; }

int cvb_ctx_timer_begin(cvb_ctx *ctx) {
    if (!ctx) return CVB_EINVAL;
    CVB_CUDA(ctx, cudaEventRecord(ctx->ev0, ctx->stream));
    return 0;
}

int cvb_ctx_timer_end(cvb_ctx *ctx, float *ms_out) {
    if (!ctx || !ms_out) return CVB_EINVAL;
    CVB_CUDA(ctx, cudaEventRecord(ctx->ev1, ctx->stream));
    CVB_CUDA(ctx, cudaEventSynchronize(ctx->ev1));
    CVB_CUDA(ctx, cudaEventElapsedTime(ms_out, ctx->ev0, ctx->ev1));
    return 0;
}

}  // extern "C"
