// cv_b200/csrc/filter.cu -- akaze::image on the device (include/cvb200_filter.h): horizontal, vertical and separable correlation filters
// of any odd length up to CVB_FILTER_MAX_TAPS, gaussian_blur and half_size, on batches of packed planes.  Bit-exact to the reference's
// f32x4 loops (akaze/src/image.rs:202-340), zero-weighted tail taps included; the extractor keeps its own fused kernels
// (akaze_kernels.cuh), which skip those taps.  The C names are given by filter_abi.cu (libcvb200_filter.so), so libcvb200.so's exports
// stay as they are.
#include <math.h>
#include <string.h>
#include "common.cuh"
#include "../../include/cvb200_filter.h"

struct FilterWorkspace {
    float *in = nullptr; size_t in_px = 0;     // uploaded planes of the host forms
    float *mid = nullptr; size_t mid_px = 0;   // the horizontal result of separable_filter / gaussian_blur
    float *out = nullptr; size_t out_px = 0;   // results of the host forms
};

void filter_workspace_free(FilterWorkspace *w) {
    if (!w) return;
    cudaFree(w->in); cudaFree(w->mid); cudaFree(w->out);
    delete w;
}

namespace {

constexpr int MAX_CHUNKS = (CVB_FILTER_MAX_TAPS + 3) / 4;   // f32x4 chunks of the zero-padded kernel

// The kernel as the reference's Vec<f32x4>: chunk c holds taps 4c .. 4c+3, zero past ks.  Passed by value (4 KiB of the 32 764 B of
// kernel parameters CUDA 12.1+ allows): no upload, and the caller's taps are free again when the launch returns.
struct FilterTaps { float4 k[MAX_CHUNKS]; };

// Pixel p (= x + j - half) of the reference's scratch line [half x first][line][half x last][3 x 0.0], for p >= -half.
__device__ __forceinline__ float scratch_at(const float *__restrict__ line, size_t stride, int n, int half, int p) {
    if (p < 0) return __ldg(line);
    if (p < n) return __ldg(line + (size_t)p * stride);
    if (p < n + half) return __ldg(line + (size_t)(n - 1) * stride);
    return 0.0f;
}

// R consecutive outputs of one line from a sliding register window: win[t] holds scratch pixel base + 4c + t while chunk c is applied,
// so output r's tap 4c + u reads win[r + u].  Each output's four lanes and their reduction follow wide::f32x4 exactly: lane u
// accumulates (pixel * k) + acc from +0 (-fmad=false keeps the two roundings), then (l0 + l2) + (l1 + l3).  LOAD(i) gives scratch pixel
// base + i.
template <int R, typename Load>
__device__ __forceinline__ void correlate(const FilterTaps &taps, int chunks, Load load, float (&res)[R]) {
    float win[R + 3], a[R][4];
#pragma unroll
    for (int t = 0; t < R + 3; t++) win[t] = load(t);
#pragma unroll
    for (int r = 0; r < R; r++) a[r][0] = a[r][1] = a[r][2] = a[r][3] = 0.0f;
    for (int c = 0;;) {
        const float4 k = taps.k[c];
#pragma unroll
        for (int r = 0; r < R; r++) {
            a[r][0] = win[r] * k.x + a[r][0];
            a[r][1] = win[r + 1] * k.y + a[r][1];
            a[r][2] = win[r + 2] * k.z + a[r][2];
            a[r][3] = win[r + 3] * k.w + a[r][3];
        }
        if (++c == chunks) break;
#pragma unroll
        for (int t = 0; t + 4 < R + 3; t++) win[t] = win[t + 4];
#pragma unroll
        for (int t = R - 1; t < R + 3; t++) win[t] = load(4 * c + t);
    }
#pragma unroll
    for (int r = 0; r < R; r++) res[r] = (a[r][0] + a[r][2]) + (a[r][1] + a[r][3]);
}

// Horizontal pass.  One CTA per row segment of SEG_H outputs: the segment's scratch pixels (SEG_H + 4 chunks + 3, the window's reads
// past the last chunk included) are staged in shared memory with coalesced loads, each thread correlates RH consecutive outputs, and
// the results go back through shared memory so that the row is stored coalesced.  RH is odd, so the threads' stride-RH shared reads and
// writes are free of bank conflicts.  Blocks enumerate (line, segment) of the batch's B * h lines.
constexpr int NT_H = 128, RH = 9, SEG_H = NT_H * RH;
__global__ void __launch_bounds__(NT_H) k_filter_h(const float *__restrict__ in, float *__restrict__ out, int w, int half, int nseg,
                                                   int chunks, const __grid_constant__ FilterTaps taps) {
    extern __shared__ float sm[];
    float *s_out = sm;                // SEG_H results
    float *s_in = sm + SEG_H;         // SEG_H + 4 * chunks + 3 scratch pixels
    const unsigned line = blockIdx.x / (unsigned)nseg;
    const int x0 = (int)(blockIdx.x - line * (unsigned)nseg) * SEG_H;
    const float *src = in + (size_t)line * w;
    const int nout = min(SEG_H, w - x0);
    const int nin = nout + 4 * chunks - 1;
    for (int i = threadIdx.x; i < nin; i += NT_H) s_in[i] = scratch_at(src, 1, w, half, x0 + i - half);
    __syncthreads();
    const int base = threadIdx.x * RH;
    if (base < nout) {
        float res[RH];
        correlate<RH>(taps, chunks, [&](int i) { return s_in[base + i]; }, res);
#pragma unroll
        for (int r = 0; r < RH; r++) s_out[base + r] = res[r];
    }
    __syncthreads();
    float *dst = out + (size_t)line * w + x0;
    for (int i = threadIdx.x; i < nout; i += NT_H) dst[i] = s_out[i];
}

// Vertical pass.  One column per thread (a warp's loads and stores are 32 consecutive floats of a row), RV consecutive rows per thread
// from a sliding window down the column read through the read-only cache, with clamped row indices and the same tail-tap rule.  Blocks
// enumerate (plane, row band, column block).
constexpr int NT_V = 128, RV = 16;
__global__ void __launch_bounds__(NT_V) k_filter_v(const float *__restrict__ in, float *__restrict__ out, int w, int h, int half,
                                                   int nxb, int nyb, int chunks, const __grid_constant__ FilterTaps taps) {
    const unsigned xb = blockIdx.x % (unsigned)nxb, rest = blockIdx.x / (unsigned)nxb;
    const unsigned yb = rest % (unsigned)nyb, b = rest / (unsigned)nyb;
    const int x = (int)xb * NT_V + threadIdx.x;
    if (x >= w) return;
    const int y0 = (int)yb * RV;
    const size_t plane = (size_t)b * w * h;
    const float *col = in + plane + x;
    float res[RV];
    correlate<RV>(taps, chunks, [&](int i) { return scratch_at(col, (size_t)w, h, half, y0 + i - half); }, res);
    float *dst = out + plane + (size_t)y0 * w + x;
#pragma unroll
    for (int r = 0; r < RV; r++)
        if (y0 + r < h) dst[(size_t)r * w] = res[r];
}

enum Dir { H, V };
struct Pass { Dir dir; const float *k; uint32_t ks; };

int check_size(cvb_ctx *ctx, uint32_t ks) {
    if (ks % 2 == 0) return cvb_set_error(ctx, CVB_EINVAL, "kernel size %u is not odd", ks);
    if (ks > CVB_FILTER_MAX_TAPS) return cvb_set_error(ctx, CVB_EUNSUPPORTED, "kernel size %u > %d", ks, CVB_FILTER_MAX_TAPS);
    return 0;
}

int check_planes(cvb_ctx *ctx, uint32_t batch, uint32_t w, uint32_t h) {
    if (batch == 0 || w == 0 || h == 0) return cvb_set_error(ctx, CVB_EINVAL, "empty image or batch");
    const uint64_t lines_h = (uint64_t)batch * h * cdiv(w, SEG_H), blocks_v = (uint64_t)batch * cdiv(h, RV) * cdiv(w, NT_V);
    if (lines_h > INT32_MAX || blocks_v > INT32_MAX) return cvb_set_error(ctx, CVB_EUNSUPPORTED, "batch too large");
    return 0;
}

bool overlap(const void *a, size_t a_bytes, const void *b, size_t b_bytes) {
    const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
    return x < y + b_bytes && y < x + a_bytes;
}

FilterWorkspace *workspace(cvb_ctx *ctx) {
    if (!ctx->filter) ctx->filter = new FilterWorkspace();
    return ctx->filter;
}

int launch_pass(cvb_ctx *ctx, const Pass &p, const float *src, float *dst, uint32_t batch, uint32_t w, uint32_t h) {
    FilterTaps t;
    memset(&t, 0, sizeof(t));
    memcpy(t.k, p.k, sizeof(float) * p.ks);
    const int chunks = (int)(p.ks + 3) / 4, half = (int)p.ks / 2;
    cudaStream_t st = ctx->stream;
    if (p.dir == H) {
        const unsigned nseg = cdiv(w, SEG_H);
        const size_t smem = sizeof(float) * (2 * SEG_H + 4 * chunks + 3);
        CVB_PROF(ctx, "k_filter_h", 8.0 * batch * w * h);
        k_filter_h<<<(unsigned)((uint64_t)batch * h * nseg), NT_H, smem, st>>>(src, dst, (int)w, half, (int)nseg, chunks, t);
        CVB_LAUNCH_CHECK(ctx);
    } else {
        const unsigned nxb = cdiv(w, NT_V), nyb = cdiv(h, RV);
        CVB_PROF(ctx, "k_filter_v", 8.0 * batch * w * h);
        k_filter_v<<<(unsigned)((uint64_t)batch * nyb * nxb), NT_V, 0, st>>>(src, dst, (int)w, (int)h, half, (int)nxb, (int)nyb, chunks,
                                                                              t);
        CVB_LAUNCH_CHECK(ctx);
    }
    return 0;
}

// One or two passes in -> out.  Host forms upload `in` into the context, run the passes there and download the result; device forms
// run on the caller's buffers.  Two passes go through the context's intermediate plane.
int run_passes(cvb_ctx *ctx, const float *in, uint32_t batch, uint32_t w, uint32_t h, const Pass *passes, int npass, float *out, bool dev) {
    int rc = check_planes(ctx, batch, w, h);
    if (rc) return rc;
    for (int i = 0; i < npass; i++) {
        if (!passes[i].k) return cvb_set_error(ctx, CVB_EINVAL, "null kernel");
        if ((rc = check_size(ctx, passes[i].ks))) return rc;
    }
    if (!in || !out) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    const size_t npx = (size_t)batch * w * h;
    if (overlap(in, npx * sizeof(float), out, npx * sizeof(float))) return cvb_set_error(ctx, CVB_EINVAL, "input and output overlap");
    FilterWorkspace *fw = workspace(ctx);
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    const float *src = in;
    float *dst = out;
    if (!dev) {
        if ((rc = ws_grow(ctx, &fw->in, &fw->in_px, npx)) || (rc = ws_grow(ctx, &fw->out, &fw->out_px, npx))) return rc;
        CVB_CUDA(ctx, cudaMemcpyAsync(fw->in, in, npx * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
        src = fw->in;
        dst = fw->out;
    }
    if (npass == 2) {
        if ((rc = ws_grow(ctx, &fw->mid, &fw->mid_px, npx))) return rc;
        if ((rc = launch_pass(ctx, passes[0], src, fw->mid, batch, w, h))) return rc;
        if ((rc = launch_pass(ctx, passes[1], fw->mid, dst, batch, w, h))) return rc;
    } else if ((rc = launch_pass(ctx, passes[0], src, dst, batch, w, h))) {
        return rc;
    }
    if (!dev) {
        CVB_CUDA(ctx, cudaMemcpyAsync(out, dst, npx * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
        CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    }
    return 0;
}

// image.rs:383-389: ks = 2 * ceil(2 r) + 1 in f32
int blur_taps(cvb_ctx *ctx, float r, float *k, uint32_t *ks) {
    if (!(r > 0.0f)) return cvb_set_error(ctx, CVB_EINVAL, "gaussian_blur needs sigma > 0 (got %g)", (double)r);
    const float radius = ceilf(2.0f * r);
    if (radius > (float)(CVB_FILTER_MAX_TAPS / 2)) return cvb_set_error(ctx, CVB_EUNSUPPORTED, "sigma %g needs more than %d taps", (double)r,
                                                                         CVB_FILTER_MAX_TAPS);
    *ks = 2 * (uint32_t)radius + 1;
    gaussian_kernel_host(r, (int)*ks, k);
    return 0;
}

}  // namespace

int flt_gaussian_kernel(float r, uint32_t kernel_size, float *out) {
    if (kernel_size % 2 == 0 || !out) return CVB_EINVAL;
    gaussian_kernel_host(r, (int)kernel_size, out);
    return 0;
}

int flt_filter(cvb_ctx *ctx, bool vertical, const float *in, uint32_t batch, uint32_t w, uint32_t h, const float *kernel,
               uint32_t kernel_size, float *out, bool dev) {
    if (!ctx) return CVB_EINVAL;
    const Pass p{vertical ? V : H, kernel, kernel_size};
    return run_passes(ctx, in, batch, w, h, &p, 1, out, dev);
}

int flt_separable_filter(cvb_ctx *ctx, const float *in, uint32_t batch, uint32_t w, uint32_t h, const float *h_kernel, uint32_t h_size,
                         const float *v_kernel, uint32_t v_size, float *out, bool dev) {
    if (!ctx) return CVB_EINVAL;
    const Pass p[2] = {{H, h_kernel, h_size}, {V, v_kernel, v_size}};
    return run_passes(ctx, in, batch, w, h, p, 2, out, dev);
}

int flt_gaussian_blur(cvb_ctx *ctx, const float *in, uint32_t batch, uint32_t w, uint32_t h, float r, float *out, bool dev) {
    if (!ctx) return CVB_EINVAL;
    float k[CVB_FILTER_MAX_TAPS];
    uint32_t ks = 0;
    int rc = blur_taps(ctx, r, k, &ks);
    if (rc) return rc;
    const Pass p[2] = {{H, k, ks}, {V, k, ks}};
    return run_passes(ctx, in, batch, w, h, p, 2, out, dev);
}

int flt_half_size(cvb_ctx *ctx, const float *in, uint32_t batch, uint32_t w, uint32_t h, float *out, bool dev) {
    if (!ctx) return CVB_EINVAL;
    if (batch == 0 || w == 0 || h == 0) return cvb_set_error(ctx, CVB_EINVAL, "empty image or batch");
    if (!in || !out) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    const size_t npx = (size_t)batch * w * h, nout = (size_t)batch * (w / 2) * (h / 2);
    if (overlap(in, npx * sizeof(float), out, nout * sizeof(float))) return cvb_set_error(ctx, CVB_EINVAL, "input and output overlap");
    if (nout == 0) return 0;   // a 1-pixel dimension: the reference's result is empty
    if (batch > 65535 || cdiv(h / 2, 8) > 65535) return cvb_set_error(ctx, CVB_EUNSUPPORTED, "batch too large");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    if (dev) return half_size_launch(ctx, in, out, batch, w, h);
    FilterWorkspace *fw = workspace(ctx);
    int rc;
    if ((rc = ws_grow(ctx, &fw->in, &fw->in_px, npx)) || (rc = ws_grow(ctx, &fw->out, &fw->out_px, nout))) return rc;
    CVB_CUDA(ctx, cudaMemcpyAsync(fw->in, in, npx * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    if ((rc = half_size_launch(ctx, fw->in, fw->out, batch, w, h))) return rc;
    CVB_CUDA(ctx, cudaMemcpyAsync(out, fw->out, nout * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    return 0;
}
