// cv_b200/csrc/akaze_kernels.cuh -- sm_90a kernels of the AKAZE extractor.
//
// Parity contract: every f32 value produced here is bit-identical to what rust-cv `akaze` 0.7.0
// computes on a default x86-64 build (unfused multiply-add, wide::f32x4 lane sums reduced as
// (l0+l2)+(l1+l3)).  Stages may be FUSED (intermediates live in shared memory, never in HBM) but
// each intermediate is rounded to f32 exactly where the reference materialises it.
// Compile with -fmad=false.  Reference line numbers are relative to the reference's akaze/src.
#pragma once
#include <cuda.h>            // CUtensorMap (types only: the encode entry point is resolved at run time, no libcuda link dependency)
#include <cuda/barrier>      // cuda::barrier + the cp.async.bulk.tensor wrappers (libcu++, header only)
#include <cuda_runtime.h>
#include <stdint.h>
#include "device_libm.cuh"
#include "../../include/cvb200.h"

namespace akz {

constexpr int TW = 32;        // tile width  (outputs)
constexpr int TH = 32;        // tile height (outputs)
constexpr int NT = 256;       // threads per CTA for tile kernels (32 x 8)
constexpr int MAXK = 33;      // max taps of a generic separable kernel (sigma <= 8)
constexpr int MAX_EVO = 32;
constexpr int MAX_TAU = 64;
constexpr int FED_SMAX = 8, FED_FUSE_DEFAULT = 8;   // diffusion steps fused per launch (halo = steps)

struct Taps { int ks; float k[MAXK]; };

// per-evolution description used by the keypoint kernels
struct EvoDev {
    int w, h;
    unsigned long long off;   // offset (floats) of this level inside a per-frame pyramid plane
    int octave;
    float size;               // (esigma * derivative_factor) as f32      scale_space_extrema.rs:63
    int rowbase;              // first global row index of this evolution (extrema scan)
    int tilebase;             // first 32x32 tile index of this evolution (all-evolution launches)
    int sigma;                // derivative kernel half-size   detector_response.rs:13
    float norm, middle;       // Scharr off-kernel weights     derivatives.rs:57-61
    float quat;               // sigma^4                       detector_response.rs:39
    int pad;
};
struct EvoTable { int n; int total_rows; int total_tiles; int pad; EvoDev e[MAX_EVO]; };

struct Cand { int x, y, e; float v; };

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// wide::f32x4 lane-ordered correlation (image.rs:242-247 / 320-325): lane j&3 accumulates taps
// j, j+4, ... as (w*k)+acc from +0; reduce_add = (l0+l2)+(l1+l3).
__device__ __forceinline__ float lane_dot(const float *w, int stride, const float *k, int ks) {
    float l0 = 0.f, l1 = 0.f, l2 = 0.f, l3 = 0.f;
    int j = 0;
    for (; j + 4 <= ks; j += 4) {
        l0 = w[(j + 0) * stride] * k[j + 0] + l0;
        l1 = w[(j + 1) * stride] * k[j + 1] + l1;
        l2 = w[(j + 2) * stride] * k[j + 2] + l2;
        l3 = w[(j + 3) * stride] * k[j + 3] + l3;
    }
    if (j < ks) l0 = w[j * stride] * k[j] + l0;
    if (j + 1 < ks) l1 = w[(j + 1) * stride] * k[j + 1] + l1;
    if (j + 2 < ks) l2 = w[(j + 2) * stride] * k[j + 2] + l2;
    return (l0 + l2) + (l1 + l3);
}

// Sparse 2-/3-tap versions of the same sum for the Scharr kernels (derivatives.rs:3-11, 54-79).
// Only the non-zero taps are evaluated.  The reference adds every product to a lane that starts at +0 and reduces
// (l0+l2)+(l1+l3) with the empty lanes still +0; adding +0 changes a value only when it is -0 (-> +0), and a sum of
// values none of which is -0 is never -0.  So the reference's result equals the sum of the products ASSOCIATED the same
// way (products sharing a lane first, then lanes of the same pair {0,2} / {1,3}, two-term adds commute exactly), with one
// final "+ 0.0f" that maps a -0 result to the reference's +0: 3-4 flops less per dot, bit-identical.
template <int JA, int JB>
__device__ __forceinline__ float dot2(float a, float ka, float b, float kb) {
    return (a * ka + b * kb) + 0.f;
}
template <int JA, int JB, int JC>
__device__ __forceinline__ float dot3(float a, float ka, float b, float kb, float c, float kc) {
    const float pa = a * ka, pb = b * kb, pc = c * kc;
    float r;
    if (JA == JB) r = (JC == JA) ? pc + (pb + pa) : (pb + pa) + pc;      // lane JA holds pb + pa (then pc + it)
    else if (JA == JC) r = (pc + pa) + pb;
    else if (JB == JC) r = (pc + pb) + pa;
    else if ((JA ^ JB) == 2) r = (pa + pb) + pc;                          // distinct lanes: the same-pair two are added first
    else if ((JA ^ JC) == 2) r = (pa + pc) + pb;
    else r = (pb + pc) + pa;
    return r + 0.f;
}
// Scharr "main" kernel [-1, 0.., 1] of size 2s+1: taps 0 and 2s.  SM = s & 3.
template <int SM>
__device__ __forceinline__ float scharr_main(float first, float last) {
    return (last - first) + 0.f;   // (-1*first) + (1*last): both products exact, see dot2
}
// Scharr "off" kernel [norm, 0.., middle, 0.., norm]: taps 0, s, 2s.
template <int SM>
__device__ __forceinline__ float scharr_off(float first, float mid, float last, float norm, float middle) {
    return dot3<0, SM & 3, (2 * SM) & 3>(first, norm, mid, middle, last, norm);
}

// ---------------------------------------------------------------------------------------------
// Generic separable filter, H then V in one pass through shared memory (image.rs:333-340).
// grid = (ceil(w/TW), ceil(h/TH), B).
__global__ void __launch_bounds__(NT) k_separable(const float *__restrict__ in, float *__restrict__ out, int w, int h,
                                                  size_t in_bstride, size_t out_bstride, Taps hk, Taps vk) {
    extern __shared__ float sm[];
    const int rx = hk.ks / 2, ry = vk.ks / 2;
    const int sw = TW + 2 * rx, sh = TH + 2 * ry;
    float *s_in = sm;            // sh x sw
    float *s_h = sm + sh * sw;   // sh x TW
    const float *src = in + (size_t)blockIdx.z * in_bstride;
    float *dst = out + (size_t)blockIdx.z * out_bstride;
    const int x0 = blockIdx.x * TW, y0 = blockIdx.y * TH;
    for (int i = threadIdx.x; i < sw * sh; i += NT) {
        int ly = i / sw, lx = i - ly * sw;
        int gx = clampi(x0 + lx - rx, 0, w - 1), gy = clampi(y0 + ly - ry, 0, h - 1);
        s_in[i] = src[(size_t)gy * w + gx];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < TW * sh; i += NT) {
        int ly = i / TW, lx = i - ly * TW;
        s_h[i] = lane_dot(s_in + ly * sw + lx, 1, hk.k, hk.ks);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < TW * TH; i += NT) {
        int ly = i / TW, lx = i - ly * TW;
        int gx = x0 + lx, gy = y0 + ly;
        if (gx < w && gy < h) dst[(size_t)gy * w + gx] = lane_dot(s_h + ly * TW + lx, TW, vk.k, vk.ks);
    }
}

// ---------------------------------------------------------------------------------------------
// half_size (image.rs:154-199): 2x2 box (row sums first) * 0.25; odd tail rows/cols * 0.5; corner copy.
__global__ void k_half_size(const float *__restrict__ in, float *__restrict__ out, int w, int h, size_t in_bstride,
                            size_t out_bstride) {
    const int hw = w / 2, hh = h / 2;
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= hw || y >= hh) return;
    const float *p = in + (size_t)blockIdx.z * in_bstride;
    const bool oddw = hw * 2 != w, oddh = hh * 2 != h;
    float v;
    if (oddw && oddh && x == hw - 1 && y == hh - 1) v = p[(size_t)(h - 1) * w + (w - 1)];
    else if (oddw && x == hw - 1) v = (p[(size_t)(2 * y) * w + (w - 1)] + p[(size_t)(2 * y + 1) * w + (w - 1)]) * 0.5f;
    else if (oddh && y == hh - 1) v = (p[(size_t)(h - 1) * w + 2 * x] + p[(size_t)(h - 1) * w + 2 * x + 1]) * 0.5f;
    else {
        const float *q = p + (size_t)(2 * y) * w + 2 * x;
        v = ((q[0] + q[1]) + (q[w] + q[w + 1])) * 0.25f;
    }
    out[(size_t)blockIdx.z * out_bstride + (size_t)y * hw + x] = v;
}

// contrast_factor.rs:35-48 histogram of floor(nbins * modg/hmax) over interior pixels with modg != 0
__global__ void __launch_bounds__(NT) k_contrast_hist(const double *__restrict__ g2, const unsigned long long *gmax,
                                                      unsigned *hist, unsigned *npoints, int n, size_t bstride, int nbins) {
    extern __shared__ unsigned s_hist[];
    for (int i = threadIdx.x; i < nbins; i += NT) s_hist[i] = 0;
    __syncthreads();
    const double hmax = sqrt(__longlong_as_double((long long)gmax[blockIdx.z]));
    const double *p = g2 + (size_t)blockIdx.z * bstride;
    unsigned cnt = 0;
    for (int i = blockIdx.x * NT + threadIdx.x; i < n; i += gridDim.x * NT) {
        double v = p[i];
        if (v < 0.0) continue;
        double modg = sqrt(v);
        if (modg != 0.0) {
            long long bin = (long long)floor((double)nbins * (modg / hmax));
            if (bin == nbins) bin -= 1;
            if (bin >= 0 && bin < nbins) atomicAdd(&s_hist[bin], 1u);
            cnt++;
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < nbins; i += NT)
        if (s_hist[i]) atomicAdd(&hist[(size_t)blockIdx.z * nbins + i], s_hist[i]);
    // warp-aggregate the point count
    for (int o = 16; o; o >>= 1) cnt += __shfl_down_sync(0xffffffffu, cnt, o);
    if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(&npoints[blockIdx.z], cnt);
}

// contrast_factor.rs:49-63 + lib.rs:222,248: k, then per-evolution inverse_k = (1/(k_i*k_i)) as f32 with
// k_i = k * 0.75^(octave changes so far), multiplied sequentially in f64 as the reference does.
__global__ void k_contrast_final(const unsigned long long *gmax, const unsigned *hist, const unsigned *npoints, int nbins,
                                 double percentile, const int *evo_octave, int nevo, double *kc, float *inv_k) {
    const int b = blockIdx.x;
    if (threadIdx.x != 0) return;
    const double hmax = sqrt(__longlong_as_double((long long)gmax[b]));
    const double num_points = (double)npoints[b];
    const unsigned long long threshold = (unsigned long long)(num_points * percentile);
    unsigned long long k = 0, nel = 0;
    while (nel < threshold && k < (unsigned long long)nbins) { nel += hist[(size_t)b * nbins + k]; k++; }
    double c = (nel >= threshold) ? hmax * (double)k / (double)nbins : 0.03;
    kc[b] = c;
    for (int i = 1; i < nevo; i++) {
        if (evo_octave[i] > evo_octave[i - 1]) c *= 0.75;
        inv_k[(size_t)b * MAX_EVO + i] = (float)(1.0 / (c * c));
    }
}

struct FedSteps { int n; float tau[FED_SMAX]; };

// ---------------------------------------------------------------------------------------------
// FED diffusion: a CTA owns a 128 x 32 region; every thread owns a 4 x 2 PATCH of it whose values stay
// in registers across the fused steps.  The flow across an edge is the same number for both cells that share
// it (nonlinear_diffusion.rs:30-52: the pair sum c_a + c_b and the difference are the same expressions seen
// from either side), so a patch evaluates each of its 22 edges once: 3 flops per edge + 4 adds per cell
// (12.25 flop / cell / step instead of 16).  Horizontal neighbours come from the adjacent lane (4 shuffles),
// vertical ones from shared memory (2 LDS.128, 2 STS.128 per step and thread).  Regions that do not touch the
// image border run without any predicate; border regions skip the missing edges exactly like the reference.
// The x halo is rounded up to a multiple of 4 so that global loads / stores are aligned float4 (w % 4 == 0;
// other widths take the scalar path).
constexpr int F3_W = 128, F3_H = 32;   // region; 512 threads (one warp per pair of rows)
template <bool BORDER>
__device__ __forceinline__ void fed3_steps(float (&l)[2][4], const float (&cH)[2][5], const float (&cV)[3][4], float *cur,
                                           float *nxt, const float *s_hs, int S, int lx0, int ly0, int gx0, int gy0,
                                           int w, int h) {
    const int rowU = max(ly0 - 1, 0) * F3_W + lx0, rowD = min(ly0 + 2, F3_H - 1) * F3_W + lx0, row0 = ly0 * F3_W + lx0;
    for (int t = 0; t < S; t++) {
        const float hs = s_hs[t];
        float lL[2], lR[2];
#pragma unroll
        for (int r = 0; r < 2; r++) {
            lL[r] = __shfl_up_sync(0xffffffffu, l[r][3], 1);
            lR[r] = __shfl_down_sync(0xffffffffu, l[r][0], 1);
        }
        const float4 up4 = *reinterpret_cast<const float4 *>(cur + rowU), dn4 = *reinterpret_cast<const float4 *>(cur + rowD);
        const float up[4] = {up4.x, up4.y, up4.z, up4.w}, dn[4] = {dn4.x, dn4.y, dn4.z, dn4.w};
        float fh[2][5], fv[3][4];
#pragma unroll
        for (int r = 0; r < 2; r++) {
            fh[r][0] = (hs * cH[r][0]) * (l[r][0] - lL[r]);
#pragma unroll
            for (int e = 1; e < 4; e++) fh[r][e] = (hs * cH[r][e]) * (l[r][e] - l[r][e - 1]);
            fh[r][4] = (hs * cH[r][4]) * (lR[r] - l[r][3]);
        }
#pragma unroll
        for (int k = 0; k < 4; k++) {
            fv[0][k] = (hs * cV[0][k]) * (l[0][k] - up[k]);
            fv[1][k] = (hs * cV[1][k]) * (l[1][k] - l[0][k]);
            fv[2][k] = (hs * cV[2][k]) * (dn[k] - l[1][k]);
        }
#pragma unroll
        for (int r = 0; r < 2; r++)
#pragma unroll
            for (int k = 0; k < 4; k++) {
                float v = l[r][k];
                if (BORDER) {
                    const int gx = gx0 + k, gy = gy0 + r;
                    v = gx < w - 1 ? v + fh[r][k + 1] : v;
                    v = gx > 0 ? v - fh[r][k] : v;
                    v = gy < h - 1 ? v + fv[r + 1][k] : v;
                    v = gy > 0 ? v - fv[r][k] : v;
                } else {
                    v = v + fh[r][k + 1];
                    v = v - fh[r][k];
                    v = v + fv[r + 1][k];
                    v = v - fv[r][k];
                }
                l[r][k] = v;
            }
        if (t + 1 < S) {   // the last step is written to global memory straight from the registers
            *reinterpret_cast<float4 *>(nxt + row0) = make_float4(l[0][0], l[0][1], l[0][2], l[0][3]);
            *reinterpret_cast<float4 *>(nxt + row0 + F3_W) = make_float4(l[1][0], l[1][1], l[1][2], l[1][3]);
            __syncthreads();
            float *tmp = cur; cur = nxt; nxt = tmp;
        }
    }
}

__global__ void __launch_bounds__(F3_H * 16, 2) k_fed3(const float *__restrict__ Lin, const float *__restrict__ C,
                                                       float *__restrict__ Lout, int w, int h, size_t lin_bstride,
                                                       size_t c_bstride, size_t lout_bstride, FedSteps steps) {
    __shared__ __align__(16) float bufA[F3_H * F3_W], bufB[F3_H * F3_W];
    __shared__ float s_hs[FED_SMAX];
    const int S = steps.n, HX = (S + 3) & ~3;
    if (threadIdx.x < FED_SMAX) s_hs[threadIdx.x] = 0.5f * steps.tau[threadIdx.x];   // (0.5 * step_size), nonlinear_diffusion.rs:30
    const int tw = F3_W - 2 * HX, th = F3_H - 2 * S;
    const int lx0 = (threadIdx.x & 31) * 4, ly0 = (threadIdx.x >> 5) * 2;
    const int X0 = blockIdx.x * tw - HX, Y0 = blockIdx.y * th - S;
    const int gx0 = X0 + lx0, gy0 = Y0 + ly0;
    const float *lin = Lin + (size_t)blockIdx.z * lin_bstride;
    const float *cc = C + (size_t)blockIdx.z * c_bstride;
    const bool vec = (w & 3) == 0;
    float l[2][4], c[2][4];
#pragma unroll
    for (int r = 0; r < 2; r++) {
        const int gy = gy0 + r;
        const bool rowin = gy >= 0 && gy < h;
        const size_t g = (size_t)gy * w + gx0;
        if (vec) {
            float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
            if (rowin && gx0 >= 0 && gx0 < w) { a = *reinterpret_cast<const float4 *>(lin + g); b = *reinterpret_cast<const float4 *>(cc + g); }
            l[r][0] = a.x; l[r][1] = a.y; l[r][2] = a.z; l[r][3] = a.w;
            c[r][0] = b.x; c[r][1] = b.y; c[r][2] = b.z; c[r][3] = b.w;
        } else {
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const bool in = rowin && gx0 + k >= 0 && gx0 + k < w;
                l[r][k] = in ? lin[g + k] : 0.f;
                c[r][k] = in ? cc[g + k] : 0.f;
            }
        }
        *reinterpret_cast<float4 *>(bufA + (ly0 + r) * F3_W + lx0) = make_float4(l[r][0], l[r][1], l[r][2], l[r][3]);
        *reinterpret_cast<float4 *>(bufB + (ly0 + r) * F3_W + lx0) = make_float4(c[r][0], c[r][1], c[r][2], c[r][3]);
    }
    __syncthreads();
    // conductivity pair sums per edge, operand order as in the reference: (left + right), (upper + lower)
    float cH[2][5], cV[3][4];
    {
#pragma unroll
        for (int r = 0; r < 2; r++) {
            const float cl = __shfl_up_sync(0xffffffffu, c[r][3], 1), cr = __shfl_down_sync(0xffffffffu, c[r][0], 1);
            cH[r][0] = cl + c[r][0];
#pragma unroll
            for (int e = 1; e < 4; e++) cH[r][e] = c[r][e - 1] + c[r][e];
            cH[r][4] = c[r][3] + cr;
        }
        const float4 cu4 = *reinterpret_cast<const float4 *>(bufB + max(ly0 - 1, 0) * F3_W + lx0);
        const float4 cd4 = *reinterpret_cast<const float4 *>(bufB + min(ly0 + 2, F3_H - 1) * F3_W + lx0);
        const float cu[4] = {cu4.x, cu4.y, cu4.z, cu4.w}, cd[4] = {cd4.x, cd4.y, cd4.z, cd4.w};
#pragma unroll
        for (int k = 0; k < 4; k++) { cV[0][k] = cu[k] + c[0][k]; cV[1][k] = c[0][k] + c[1][k]; cV[2][k] = c[1][k] + cd[k]; }
    }
    __syncthreads();   // bufB becomes the write buffer of step 1
    const bool border = X0 <= 0 || Y0 <= 0 || X0 + F3_W >= w || Y0 + F3_H >= h;   // CTA-uniform
    if (border) fed3_steps<true>(l, cH, cV, bufA, bufB, s_hs, S, lx0, ly0, gx0, gy0, w, h);
    else fed3_steps<false>(l, cH, cV, bufA, bufB, s_hs, S, lx0, ly0, gx0, gy0, w, h);
    float *dst = Lout + (size_t)blockIdx.z * lout_bstride;
    if (lx0 >= HX && lx0 < F3_W - HX && gx0 < w) {
#pragma unroll
        for (int r = 0; r < 2; r++) {
            const int ly = ly0 + r, gy = gy0 + r;
            if (ly < S || ly >= F3_H - S || gy >= h) continue;
            const size_t g = (size_t)gy * w + gx0;
            if (vec) *reinterpret_cast<float4 *>(dst + g) = make_float4(l[r][0], l[r][1], l[r][2], l[r][3]);
            else {
#pragma unroll
                for (int k = 0; k < 4; k++) if (gx0 + k < w) dst[g + k] = l[r][k];
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Multiscale first derivatives from Lsmooth (detector_response.rs:60-65, derivatives.rs:23-49):
//   Lx = V_off(H_main(Ls)),  Ly = V_main(H_off(Ls)),  kernel size 2*sigma+1.
template <int SM>
__global__ void __launch_bounds__(NT) k_deriv1(const float *__restrict__ Ls, float *__restrict__ Lx,
                                               float *__restrict__ Ly, int w, int h, size_t bstride, int sigma,
                                               float norm, float middle) {
    extern __shared__ float sm[];
    const int sw = TW + 2 * sigma, sh = TH + 2 * sigma;
    float *s_in = sm;                 // sh x sw
    float *s_hm = sm + sh * sw;       // sh x TW   H_main
    float *s_ho = s_hm + sh * TW;     // sh x TW   H_off
    const float *src = Ls + (size_t)blockIdx.z * bstride;
    const int x0 = blockIdx.x * TW, y0 = blockIdx.y * TH;
    for (int i = threadIdx.x; i < sw * sh; i += NT) {
        int ly = i / sw, lx = i - ly * sw;
        int gx = clampi(x0 + lx - sigma, 0, w - 1), gy = clampi(y0 + ly - sigma, 0, h - 1);
        s_in[i] = src[(size_t)gy * w + gx];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < TW * sh; i += NT) {
        int ly = i / TW, lx = i - ly * TW;
        const float *p = s_in + ly * sw + lx;   // p[0] = x - sigma, p[sigma] = x, p[2 sigma] = x + sigma
        s_hm[i] = scharr_main<SM>(p[0], p[2 * sigma]);
        s_ho[i] = scharr_off<SM>(p[0], p[sigma], p[2 * sigma], norm, middle);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < TW * TH; i += NT) {
        int ly = i / TW, lx = i - ly * TW;
        int gx = x0 + lx, gy = y0 + ly;
        if (gx >= w || gy >= h) continue;
        const float *pm = s_hm + ly * TW + lx, *po = s_ho + ly * TW + lx;
        size_t g = (size_t)blockIdx.z * bstride + (size_t)gy * w + gx;
        Lx[g] = scharr_off<SM>(pm[0], pm[sigma * TW], pm[2 * sigma * TW], norm, middle);
        Ly[g] = scharr_main<SM>(po[0], po[2 * sigma * TW]);
    }
}

// Second derivatives + determinant of Hessian (detector_response.rs:40-47,66-68):
//   Lxx = V_off(H_main(Lx)), Lyy = V_main(H_off(Ly)), Lxy = V_main(H_off(Lx)),
//   Ldet = (Lxx*Lyy - Lxy*Lxy) * sigma^4.   Lxx/Lyy/Lxy never reach HBM.
template <int SM>
__global__ void __launch_bounds__(NT) k_deriv2_det(const float *__restrict__ Lx, const float *__restrict__ Ly,
                                                   float *__restrict__ Ldet, int w, int h, size_t bstride, int sigma,
                                                   float norm, float middle, float quat) {
    extern __shared__ float sm[];
    const int sw = TW + 2 * sigma, sh = TH + 2 * sigma;
    float *s_x = sm;                  // Lx tile sh x sw
    float *s_y = sm + sh * sw;        // Ly tile
    float *s_a = s_y + sh * sw;       // H_main(Lx)  sh x TW
    float *s_b = s_a + sh * TW;       // H_off(Ly)
    float *s_c = s_b + sh * TW;       // H_off(Lx)
    const float *px = Lx + (size_t)blockIdx.z * bstride, *py = Ly + (size_t)blockIdx.z * bstride;
    const int x0 = blockIdx.x * TW, y0 = blockIdx.y * TH;
    for (int i = threadIdx.x; i < sw * sh; i += NT) {
        int ly = i / sw, lx = i - ly * sw;
        int gx = clampi(x0 + lx - sigma, 0, w - 1), gy = clampi(y0 + ly - sigma, 0, h - 1);
        size_t g = (size_t)gy * w + gx;
        s_x[i] = px[g];
        s_y[i] = py[g];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < TW * sh; i += NT) {
        int ly = i / TW, lx = i - ly * TW;
        const float *p = s_x + ly * sw + lx, *q = s_y + ly * sw + lx;
        s_a[i] = scharr_main<SM>(p[0], p[2 * sigma]);
        s_b[i] = scharr_off<SM>(q[0], q[sigma], q[2 * sigma], norm, middle);
        s_c[i] = scharr_off<SM>(p[0], p[sigma], p[2 * sigma], norm, middle);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < TW * TH; i += NT) {
        int ly = i / TW, lx = i - ly * TW;
        int gx = x0 + lx, gy = y0 + ly;
        if (gx >= w || gy >= h) continue;
        const float *pa = s_a + ly * TW + lx, *pb = s_b + ly * TW + lx, *pc = s_c + ly * TW + lx;
        float lxx = scharr_off<SM>(pa[0], pa[sigma * TW], pa[2 * sigma * TW], norm, middle);
        float lyy = scharr_main<SM>(pb[0], pb[2 * sigma * TW]);
        float lxy = scharr_main<SM>(pc[0], pc[2 * sigma * TW]);
        Ldet[(size_t)blockIdx.z * bstride + (size_t)gy * w + gx] = (lxx * lyy - lxy * lxy) * quat;
    }
}

template <int KS>
__device__ __forceinline__ float lane_dot_static(const float *w, int stride, const float *k) {
    // same sum as lane_dot without the additions of +0 (first touch of a lane, empty lanes); the trailing + 0.0f restores
    // the reference's +0 where every product is -0 (see dot2 / dot3)
    float l[4];
#pragma unroll
    for (int j = 0; j < KS; j++) {
        const float p = w[j * stride] * k[j];
        l[j & 3] = j < 4 ? p : p + l[j & 3];
    }
    if (KS == 1) return l[0] + 0.f;
    if (KS == 2) return (l[0] + l[1]) + 0.f;
    if (KS == 3) return ((l[0] + l[2]) + l[1]) + 0.f;
    return ((l[0] + l[2]) + (l[1] + l[3])) + 0.f;
}
// the same for KS values already in registers (vertical passes of the column-strip kernels)
template <int KS>
__device__ __forceinline__ float lane_dot_regs(const float *v, const float *k) {
    float l[4];
#pragma unroll
    for (int j = 0; j < KS; j++) {
        const float p = v[j] * k[j];
        l[j & 3] = j < 4 ? p : p + l[j & 3];
    }
    if (KS == 1) return l[0] + 0.f;
    if (KS == 2) return (l[0] + l[1]) + 0.f;
    if (KS == 3) return ((l[0] + l[2]) + l[1]) + 0.f;
    return ((l[0] + l[2]) + (l[1] + l[3])) + 0.f;
}

// ---------------------------------------------------------------------------------------------
// v3 "column strip" tile kernels.  A 256-thread CTA owns a 32 x 64 output tile; thread (tx, ty) owns the
// column x0+tx of the 8-row strip ty.  The clamped input region is staged once in shared memory; each thread
// then walks down its column computing the horizontal pass of every row it needs ONCE, in registers, and emits
// an output row as soon as its vertical taps are complete.  No intermediate shared-memory pass, one barrier,
// ~4x fewer instructions per pixel than the two-pass tiles above (which stay as the generic fallback).
// The arithmetic of every output is unchanged (same helpers, same order) -> still bit-exact.
constexpr int SW3 = 32, SH3 = 64, STRIP = 8;

// ---- TMA staging of interior tiles (BASELINE north_star: "TMA-staged tiles in shared memory").  A tile whose halo lies inside the
// image is fetched by ONE 3-D cp.async.bulk.tensor (x, y, frame) issued by one thread and awaited on an mbarrier; tiles that touch the
// border keep the clamped path below, because TMA fills out-of-bounds elements with zero while the reference replicates the border
// (image.rs:233-235,289-296).  The box is `pitch3(R)` floats wide; the padding columns are never read.  Shared-memory contents of the halo region are identical in both paths.
// A box that starts at an x coordinate that is not a multiple of 16 bytes faults ("illegal instruction"; x = 64 loads, x = 190 faults,
// 2-D and 3-D alike, in a stand-alone probe), so the staged box starts xpad3(R) >= R floats left of the tile, a multiple of
// 4 floats, and the kernels read their halo region at column offset xoff3(R) inside it.
__host__ __device__ constexpr int xpad3(int r) { return r <= 4 ? 4 : 8; }
__host__ __device__ constexpr int xoff3(int r) { return xpad3(r) - r; }
__host__ __device__ constexpr int pitch3(int r) { return SW3 + 2 * xpad3(r); }
// The TMA path follows the CUDA programming guide's tensor-copy protocol through libcu++ (cuda::barrier in shared memory,
// fence.proxy.async after its initialisation, every thread arrives, the issuing thread adds the transaction bytes): a hand-written
// mbarrier.init / fence.mbarrier_init / expect_tx sequence that serves the 1-D bulk copies of the matcher raised "illegal
// instruction" on UTMALDG in a stand-alone probe, the guide's protocol does not.
using ak_barrier = cuda::barrier<cuda::thread_scope_block>;

template <int RX, int RY, int RW = SW3 + 2 * RX, int XOFF = 0>
__device__ __forceinline__ void stage_region(const float *__restrict__ src, int w, int h, int x0, int y0, float *s_base,
                                             const CUtensorMap *tm = nullptr, int frame = 0, ak_barrier *bar = nullptr, bool tm_global = false) {
    // all of a thread's global loads are issued before the first shared store (a rolled load->store loop waits one
    // DRAM latency per row: ncu showed 36 % of the blur kernel's stall samples on that store)
    constexpr int RH = SH3 + 2 * RY, NI = (RH + 7) / 8;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const bool interior = x0 - RX >= 0 && x0 + SW3 + RX <= w && y0 - RY >= 0 && y0 + SH3 + RY <= h;
    float *s_in = s_base + XOFF;              // the halo region (what the classic path fills and every consumer reads)
    if (tm != nullptr && interior && x0 - (RX + XOFF) >= 0 && x0 + SW3 + RX + XOFF <= w) {          // CTA-uniform; the whole box inside the image
        namespace cde = cuda::device::experimental;
        if (threadIdx.x == 0) {
            init(bar, blockDim.x);
            cde::fence_proxy_async_shared_cta();      // the initialised barrier becomes visible to the async proxy (TMA unit)
        }
        __syncthreads();
        ak_barrier::arrival_token token;
        if (threadIdx.x == 0) {
            // a descriptor that lives in global memory was written through the generic proxy (cudaMemcpy): acquire it for the
            // tensor-map proxy before the TMA unit reads it
            if (tm_global) asm volatile("fence.proxy.tensormap::generic.acquire.gpu [%0], 128;" ::"l"(tm) : "memory");
            cde::cp_async_bulk_tensor_3d_global_to_shared(s_base, tm, x0 - (RX + XOFF), y0 - RY, frame, *bar);
            token = cuda::device::barrier_arrive_tx(*bar, 1, (unsigned)(RW * RH * sizeof(float)));
        } else {
            token = bar->arrive();
        }
        bar->wait(std::move(token));
        return;
    }
    const bool tail = tx < 2 * RX;
    float a[NI], b[NI];
    if (interior) {
        const float *base = src + (size_t)(y0 - RY) * w + (x0 - RX) + tx;
#pragma unroll
        for (int k = 0; k < NI; k++) {
            const int ly = ty + 8 * k;
            if (ly < RH) {
                const float *row = base + (size_t)ly * w;
                a[k] = row[0];
                if (tail) b[k] = row[32];
            }
        }
    } else {
        const int cxa = clampi(x0 + tx - RX, 0, w - 1), cxb = clampi(x0 + 32 + tx - RX, 0, w - 1);
#pragma unroll
        for (int k = 0; k < NI; k++) {
            const int ly = ty + 8 * k;
            if (ly < RH) {
                const float *row = src + (size_t)clampi(y0 + ly - RY, 0, h - 1) * w;
                a[k] = row[cxa];
                if (tail) b[k] = row[cxb];
            }
        }
    }
#pragma unroll
    for (int k = 0; k < NI; k++) {
        const int ly = ty + 8 * k;
        if (ly < RH) {
            s_in[ly * RW + tx] = a[k];
            if (tail) s_in[ly * RW + 32 + tx] = b[k];
        }
    }
}

__device__ __forceinline__ void tile_origin_v3(const EvoDev &ev, int gtile, int &x0, int &y0) {
    const int tiles_x = (ev.w + SW3 - 1) / SW3, tile = gtile - ev.tilebase;
    const int tyi = tile / tiles_x;
    x0 = (tile - tyi * tiles_x) * SW3; y0 = tyi * SH3;
}

// first derivatives, sigma = S (detector_response.rs:60-65): Lx = V_off(H_main(Ls)), Ly = V_main(H_off(Ls))
template <int S>
__device__ __forceinline__ void deriv1_body(const float *__restrict__ src, float *__restrict__ Lx, float *__restrict__ Ly,
                                            const EvoDev &ev, int x0, int y0, float *s_in, const CUtensorMap *tm, ak_barrier *bar) {
    constexpr int RW = pitch3(S), XO = xoff3(S);
    stage_region<S, S, RW, XO>(src, ev.w, ev.h, x0, y0, s_in, tm, (int)blockIdx.z, bar, true);
    __syncthreads();
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int gx = x0 + tx;
    if (gx >= ev.w) return;
    const float *col = s_in + XO + (ty * STRIP) * RW + tx;   // col[r * RW + {0, S, 2S}] = input row (y - S + r), x - S / x / x + S
    float hm[STRIP + 2 * S], ho[STRIP + 2 * S];
#pragma unroll
    for (int r = 0; r < STRIP + 2 * S; r++) {
        const float a = col[r * RW], m = col[r * RW + S], z = col[r * RW + 2 * S];
        hm[r] = scharr_main<S & 3>(a, z);
        ho[r] = scharr_off<S & 3>(a, m, z, ev.norm, ev.middle);
        if (r >= 2 * S) {
            const int o = r - 2 * S, gy = y0 + ty * STRIP + o;
            if (gy < ev.h) {
                const size_t g = (size_t)gy * ev.w + gx;
                Lx[g] = scharr_off<S & 3>(hm[o], hm[o + S], hm[o + 2 * S], ev.norm, ev.middle);
                Ly[g] = scharr_main<S & 3>(ho[o], ho[o + 2 * S]);
            }
        }
    }
}

__global__ void __launch_bounds__(NT) k_deriv1_v3(const float *__restrict__ Ls, const float *__restrict__ Lt0,
                                                  float *__restrict__ Lx, float *__restrict__ Ly, size_t bstride, EvoTable T,
                                                  const unsigned char *__restrict__ tile_evo, int tile_offset,
                                                  const CUtensorMap *__restrict__ maps) {
    extern __shared__ __align__(128) float sm[];
#pragma nv_diag_suppress static_var_with_dynamic_init
    __shared__ ak_barrier s_bar[1];
    const int gtile = blockIdx.x + tile_offset;
    const int e = tile_evo[gtile];
    const EvoDev ev = T.e[e];
    int x0, y0;
    tile_origin_v3(ev, gtile, x0, y0);
    const size_t base = (size_t)blockIdx.z * bstride + ev.off;
    const float *src = (e == 0 ? Lt0 : Ls) + base;   // evolution 0: Lsmooth IS Lt (lib.rs:201)
    const CUtensorMap *tm = maps ? maps + e : nullptr;   // per-evolution map of the source plane (all frames)
    float *sma = (float *)(((uintptr_t)sm + 127) & ~(uintptr_t)127);      // TMA destinations are 128-byte aligned
    switch (ev.sigma) {
    case 1: deriv1_body<1>(src, Lx + base, Ly + base, ev, x0, y0, sma, tm, s_bar); break;
    case 2: deriv1_body<2>(src, Lx + base, Ly + base, ev, x0, y0, sma, tm, s_bar); break;
    case 3: deriv1_body<3>(src, Lx + base, Ly + base, ev, x0, y0, sma, tm, s_bar); break;
    case 4: deriv1_body<4>(src, Lx + base, Ly + base, ev, x0, y0, sma, tm, s_bar); break;
    default: deriv1_body<5>(src, Lx + base, Ly + base, ev, x0, y0, sma, tm, s_bar); break;
    }
}

// second derivatives + Hessian determinant (detector_response.rs:40-47,66-68)
template <int S>
__device__ __forceinline__ void deriv2_body(const float *__restrict__ px, const float *__restrict__ py, float *__restrict__ Ldet,
                                            const EvoDev &ev, int x0, int y0, float *sm, const CUtensorMap *tmx, const CUtensorMap *tmy,
                                            ak_barrier *bar) {
    constexpr int RW = pitch3(S), RH = SH3 + 2 * S, XO = xoff3(S);
    float *s_x = sm, *s_y = sm + ((RW * RH + 31) & ~31);      // second buffer 128-byte aligned
    stage_region<S, S, RW, XO>(px, ev.w, ev.h, x0, y0, s_x, tmx, (int)blockIdx.z, bar, true);
    stage_region<S, S, RW, XO>(py, ev.w, ev.h, x0, y0, s_y, tmy, (int)blockIdx.z, bar + 1, true);
    __syncthreads();
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int gx = x0 + tx;
    if (gx >= ev.w) return;
    const float *cx = s_x + XO + (ty * STRIP) * RW + tx, *cy = s_y + XO + (ty * STRIP) * RW + tx;
    float hmx[STRIP + 2 * S], hox[STRIP + 2 * S], hoy[STRIP + 2 * S];
#pragma unroll
    for (int r = 0; r < STRIP + 2 * S; r++) {
        const float a = cx[r * RW], m = cx[r * RW + S], z = cx[r * RW + 2 * S];
        hmx[r] = scharr_main<S & 3>(a, z);                                             // H_main(Lx)
        hox[r] = scharr_off<S & 3>(a, m, z, ev.norm, ev.middle);                       // H_off(Lx)
        hoy[r] = scharr_off<S & 3>(cy[r * RW], cy[r * RW + S], cy[r * RW + 2 * S], ev.norm, ev.middle);   // H_off(Ly)
        if (r >= 2 * S) {
            const int o = r - 2 * S, gy = y0 + ty * STRIP + o;
            if (gy < ev.h) {
                const float lxx = scharr_off<S & 3>(hmx[o], hmx[o + S], hmx[o + 2 * S], ev.norm, ev.middle);
                const float lyy = scharr_main<S & 3>(hoy[o], hoy[o + 2 * S]);
                const float lxy = scharr_main<S & 3>(hox[o], hox[o + 2 * S]);
                Ldet[(size_t)gy * ev.w + gx] = (lxx * lyy - lxy * lxy) * ev.quat;
            }
        }
    }
}

__global__ void __launch_bounds__(NT) k_deriv2_v3(const float *__restrict__ Lx, const float *__restrict__ Ly,
                                                  float *__restrict__ Ldet, size_t bstride, EvoTable T,
                                                  const unsigned char *__restrict__ tile_evo, int tile_offset,
                                                  const CUtensorMap *__restrict__ maps_x, const CUtensorMap *__restrict__ maps_y) {
    extern __shared__ __align__(128) float sm[];
#pragma nv_diag_suppress static_var_with_dynamic_init
    __shared__ ak_barrier s_bar[2];
    const int gtile = blockIdx.x + tile_offset;
    const int e = tile_evo[gtile];
    const EvoDev ev = T.e[e];
    int x0, y0;
    tile_origin_v3(ev, gtile, x0, y0);
    const size_t base = (size_t)blockIdx.z * bstride + ev.off;
    const CUtensorMap *tmx = maps_x ? maps_x + e : nullptr, *tmy = maps_y ? maps_y + e : nullptr;
    float *sma = (float *)(((uintptr_t)sm + 127) & ~(uintptr_t)127);
    switch (ev.sigma) {
    case 1: deriv2_body<1>(Lx + base, Ly + base, Ldet + base, ev, x0, y0, sma, tmx, tmy, s_bar); break;
    case 2: deriv2_body<2>(Lx + base, Ly + base, Ldet + base, ev, x0, y0, sma, tmx, tmy, s_bar); break;
    case 3: deriv2_body<3>(Lx + base, Ly + base, Ldet + base, ev, x0, y0, sma, tmx, tmy, s_bar); break;
    case 4: deriv2_body<4>(Lx + base, Ly + base, Ldet + base, ev, x0, y0, sma, tmx, tmy, s_bar); break;
    default: deriv2_body<5>(Lx + base, Ly + base, Ldet + base, ev, x0, y0, sma, tmx, tmy, s_bar); break;
    }
}

// Gaussian blur, column strips (image.rs:202-340, 383-389).  grid = (ceil(w/32), ceil(h/64), B)
template <int KS>
__global__ void __launch_bounds__(NT) k_blur_v3(const float *__restrict__ in, float *__restrict__ out, int w, int h,
                                                size_t in_bstride, size_t out_bstride, Taps tk,
                                                const __grid_constant__ CUtensorMap tmap, int use_tma) {
    constexpr int R = KS / 2, RW = pitch3(R), XO = xoff3(R);
    __shared__ __align__(128) float s_in[(SH3 + 2 * R) * RW];
#pragma nv_diag_suppress static_var_with_dynamic_init
    __shared__ ak_barrier s_bar[1];
    const int x0 = blockIdx.x * SW3, y0 = blockIdx.y * SH3;
    stage_region<R, R, RW, XO>(in + (size_t)blockIdx.z * in_bstride, w, h, x0, y0, s_in, use_tma ? &tmap : nullptr, (int)blockIdx.z, s_bar);
    __syncthreads();
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int gx = x0 + tx;
    if (gx >= w) return;
    float *dst = out + (size_t)blockIdx.z * out_bstride;
    const float *col = s_in + XO + (ty * STRIP) * RW + tx;
    float hv[STRIP + 2 * R];
#pragma unroll
    for (int r = 0; r < STRIP + 2 * R; r++) {
        hv[r] = lane_dot_static<KS>(col + r * RW, 1, tk.k);            // horizontal pass of input row (y - R + r)
        if (r >= 2 * R) {
            const int o = r - 2 * R, gy = y0 + ty * STRIP + o;
            if (gy < h) dst[(size_t)gy * w + gx] = lane_dot_regs<KS>(hv + o, tk.k);   // vertical pass, same lane order
        }
    }
}

// Simple Scharr + pm_g2 (MODE 0) / contrast gradient (MODE 1), column strips.
template <int MODE>
__global__ void __launch_bounds__(NT) k_scharr_pm_v3(const float *__restrict__ in, float *__restrict__ out_flow,
                                                     double *__restrict__ out_g2, unsigned long long *__restrict__ gmax,
                                                     int w, int h, size_t in_bstride, size_t out_bstride,
                                                     const float *__restrict__ inv_k, int inv_k_stride) {
    constexpr int RW = SW3 + 2;
    __shared__ float s_in[(SH3 + 2) * RW];
    __shared__ unsigned long long s_max;
    const int x0 = blockIdx.x * SW3, y0 = blockIdx.y * SH3;
    if (MODE == 1 && threadIdx.x == 0) s_max = 0ull;
    stage_region<1, 1>(in + (size_t)blockIdx.z * in_bstride, w, h, x0, y0, s_in);
    __syncthreads();
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int gx = x0 + tx;
    unsigned long long lmax = 0ull;
    if (gx < w) {
        float ik = 0.f;
        if (MODE == 0) ik = inv_k[(size_t)blockIdx.z * inv_k_stride];
        const float *col = s_in + (ty * STRIP) * RW + tx;
        float hm[STRIP + 2], ho[STRIP + 2];
#pragma unroll
        for (int r = 0; r < STRIP + 2; r++) {
            const float a = col[r * RW], m = col[r * RW + 1], z = col[r * RW + 2];
            hm[r] = dot2<0, 2>(a, -1.0f, z, 1.0f);                 // H [-1,0,1]
            ho[r] = dot3<0, 1, 2>(a, 3.0f, m, 10.0f, z, 3.0f);     // H [3,10,3]
            if (r >= 2) {
                const int o = r - 2, gy = y0 + ty * STRIP + o;
                if (gy < h) {
                    const float dx = dot3<0, 1, 2>(hm[o], 3.0f, hm[o + 1], 10.0f, hm[o + 2], 3.0f);   // V [3,10,3]
                    const float dy = dot2<0, 2>(ho[o], -1.0f, ho[o + 2], 1.0f);                        // V [-1,0,1]
                    const size_t g = (size_t)blockIdx.z * out_bstride + (size_t)gy * w + gx;
                    if (MODE == 0) out_flow[g] = 1.0f / (1.0f + ik * (dx * dx + dy * dy));
                    else {
                        double g2 = -1.0;
                        if (gx >= 1 && gx < w - 1 && gy >= 1 && gy < h - 1) {
                            g2 = (double)(dx * dx) + (double)(dy * dy);
                            const unsigned long long bits = (unsigned long long)__double_as_longlong(g2);
                            lmax = bits > lmax ? bits : lmax;
                        }
                        out_g2[g] = g2;
                    }
                }
            }
        }
    }
    if (MODE == 1) {
        atomicMax(&s_max, lmax);
        __syncthreads();
        if (threadIdx.x == 0 && s_max) atomicMax(gmax + blockIdx.z, s_max);
    }
}

// ---------------------------------------------------------------------------------------------
// Lsmooth = gaussian_blur(L, 1.0) and Lflow = pm_g2(scharr(Lsmooth)) of one evolution in ONE launch (lib.rs:225-246).
// The 5-tap blur runs over the 32 x 64 tile plus a one-pixel ring (34 x 66 values kept in shared memory, the tile part also
// written to the Lsmooth plane); the Scharr stage is the body of k_scharr_pm_v3<0> reading that ring tile.  Ring positions
// outside the image take the value of the clamped position, which is what the separate kernel's replicate-border staging of
// the Lsmooth plane reads.  Same helpers and orders as the two separate kernels -> same bits.
__global__ void __launch_bounds__(NT) k_blur_scharr_pm(const float *__restrict__ in, float *__restrict__ out_lsm,
                                                       float *__restrict__ out_flow, int w, int h, size_t in_bstride,
                                                       size_t lsm_bstride, size_t flow_bstride, Taps tk,
                                                       const float *__restrict__ inv_k, int inv_k_stride,
                                                       const __grid_constant__ CUtensorMap tmap, int use_tma) {
    constexpr int RWI = pitch3(3), RHI = SH3 + 6, LW = SW3 + 2, LH = SH3 + 2, XO = xoff3(3);
    constexpr int BSTRIP = 10, NSTRIPS = (LH + BSTRIP - 1) / BSTRIP;     // 34 columns x 7 strips = 238 blur tasks
    static_assert(LW * NSTRIPS <= NT, "one blur task per thread");
    __shared__ __align__(128) float s_in[RHI * RWI];
    __shared__ float s_l[LH * LW];
#pragma nv_diag_suppress static_var_with_dynamic_init
    __shared__ ak_barrier s_bar[1];
    const int x0 = blockIdx.x * SW3, y0 = blockIdx.y * SH3;
    stage_region<3, 3, RWI, XO>(in + (size_t)blockIdx.z * in_bstride, w, h, x0, y0, s_in, use_tma ? &tmap : nullptr, (int)blockIdx.z, s_bar);
    __syncthreads();
    if (threadIdx.x < LW * NSTRIPS) {
        const int sidx = threadIdx.x / LW, c = threadIdx.x - sidx * LW;
        const int gx = x0 - 1 + c;
        if (gx >= 0 && gx < w) {
            float *lsm = out_lsm + (size_t)blockIdx.z * lsm_bstride;
            const float *col = s_in + XO + (sidx * BSTRIP) * RWI + c;   // ring row lr needs staged rows lr .. lr + 4, columns c .. c + 4
            float hv[BSTRIP + 4];
#pragma unroll
            for (int r = 0; r < BSTRIP + 4; r++) {
                hv[r] = sidx * BSTRIP + r < RHI ? lane_dot_static<5>(col + r * RWI, 1, tk.k) : 0.f;
                if (r >= 4) {
                    const int lr = sidx * BSTRIP + r - 4, gy = y0 - 1 + lr;
                    if (lr < LH && gy >= 0 && gy < h) {
                        const float v = lane_dot_regs<5>(hv + (r - 4), tk.k);
                        s_l[lr * LW + c] = v;
                        if (lr >= 1 && lr <= SH3 && c >= 1 && c <= SW3) lsm[(size_t)gy * w + gx] = v;
                    }
                }
            }
        }
    }
    __syncthreads();
    if (x0 < 1 || y0 < 1 || x0 + SW3 + 1 > w || y0 + SH3 + 1 > h) {      // the ring leaves the image (CTA-uniform)
        for (int p = threadIdx.x; p < LH * LW; p += NT) {
            const int lr = p / LW, lc = p - lr * LW, gy = y0 - 1 + lr, gx = x0 - 1 + lc;
            if (gx < 0 || gx >= w || gy < 0 || gy >= h)
                s_l[p] = s_l[(clampi(gy, 0, h - 1) - (y0 - 1)) * LW + (clampi(gx, 0, w - 1) - (x0 - 1))];
        }
        __syncthreads();
    }
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int gx = x0 + tx;
    if (gx >= w) return;
    const float ik = inv_k[(size_t)blockIdx.z * inv_k_stride];
    const float *col = s_l + (ty * STRIP) * LW + tx;
    float hm[STRIP + 2], ho[STRIP + 2];
#pragma unroll
    for (int r = 0; r < STRIP + 2; r++) {
        const float a = col[r * LW], m = col[r * LW + 1], z = col[r * LW + 2];
        hm[r] = dot2<0, 2>(a, -1.0f, z, 1.0f);                 // H [-1,0,1]
        ho[r] = dot3<0, 1, 2>(a, 3.0f, m, 10.0f, z, 3.0f);     // H [3,10,3]
        if (r >= 2) {
            const int o = r - 2, gy = y0 + ty * STRIP + o;
            if (gy < h) {
                const float dx = dot3<0, 1, 2>(hm[o], 3.0f, hm[o + 1], 10.0f, hm[o + 2], 3.0f);   // V [3,10,3]
                const float dy = dot2<0, 2>(ho[o], -1.0f, ho[o + 2], 1.0f);                        // V [-1,0,1]
                out_flow[(size_t)blockIdx.z * flow_bstride + (size_t)gy * w + gx] = 1.0f / (1.0f + ik * (dx * dx + dy * dy));
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Extrema detection: one pass over Ldet in 32 x 64 column-strip tiles produces a 1-bit-per-pixel mask
// (strict 3x3 maximum above the threshold on interior pixels, scale_space_extrema.rs:49-59: v > each of the
// eight neighbours <=> v > their maximum) plus per-row counts; a second, tiny pass turns mask words into the
// ordered candidate list.  wordbase[e] = first mask word of evolution e; row r of evolution e owns
// ceil(w/32) consecutive words.
struct MaskLayout { int wordbase[MAX_EVO]; int total_words; };

__global__ void __launch_bounds__(NT) k_extrema_mask(const float *__restrict__ Ldet, size_t bstride, EvoTable T,
                                                     const unsigned char *__restrict__ tile_evo, MaskLayout ML, float thr,
                                                     unsigned *__restrict__ mask, unsigned *__restrict__ rowcount) {
    constexpr int RW = SW3 + 2;
    __shared__ float s_in[(SH3 + 2) * RW];
    const int e = tile_evo[blockIdx.x];
    const EvoDev ev = T.e[e];
    int x0, y0;
    tile_origin_v3(ev, blockIdx.x, x0, y0);
    stage_region<1, 1>(Ldet + (size_t)blockIdx.z * bstride + ev.off, ev.w, ev.h, x0, y0, s_in);
    __syncthreads();
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int gx = x0 + tx;
    const bool xin = gx >= 1 && gx < ev.w - 1;
    const float *col = s_in + (ty * STRIP) * RW + tx;
    const int wpr = (ev.w + 31) >> 5;
    unsigned *mrow = mask + (size_t)blockIdx.z * ML.total_words + ML.wordbase[e];
    unsigned *rc = rowcount + (size_t)blockIdx.z * T.total_rows + ev.rowbase;
    float m3[STRIP + 2], sd[STRIP + 2], cn[STRIP + 2];
#pragma unroll
    for (int r = 0; r < STRIP + 2; r++) {
        const float l = col[r * RW], c = col[r * RW + 1], rt = col[r * RW + 2];
        sd[r] = fmaxf(l, rt);
        m3[r] = fmaxf(sd[r], c);
        cn[r] = c;
        if (r >= 2) {
            const int o = r - 2, gy = y0 + ty * STRIP + o;
            const float v = cn[o + 1];
            const float m8 = fmaxf(fmaxf(m3[o], m3[o + 2]), sd[o + 1]);
            const bool hit = xin && gy >= 1 && gy < ev.h - 1 && v > thr && v > m8;
            const unsigned bits = __ballot_sync(0xffffffffu, hit);
            if (tx == 0 && gy < ev.h && x0 < ev.w) {
                mrow[(size_t)gy * wpr + (x0 >> 5)] = bits;
                if (bits) atomicAdd(&rc[gy], (unsigned)__popc(bits));
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Detector response of one tile in ONE pass (detector_response.rs:40-68 + scale_space_extrema.rs:49-59): the work of
// k_deriv1_v3 + k_deriv2_v3 + k_extrema_mask without the Lx / Ly / Ldet re-reads.  Lsmooth is staged with a halo of 2S+1;
// Lx, Ly are computed over the tile plus a ring of S+1 (the tile part written to the planes), Ldet over the tile plus a
// one-pixel ring (the tile part written to the plane), and the 3x3 test runs on that Ldet tile in shared memory.
// Ring positions of Lx / Ly outside the image take the value at the clamped position, which is what k_deriv2_v3's
// replicate-border staging of the Lx / Ly planes reads (as k_blur_scharr_pm does for Lsmooth).  Ldet ring positions outside
// the image only neighbour border pixels, which are never extrema.  Same helpers, same operand order -> same bits.
__host__ __device__ constexpr int det_smem_floats(int s) {
    return (SW3 + 4 * s + 2) * (SH3 + 4 * s + 2) + 2 * (SW3 + 2 * s + 2) * (SH3 + 2 * s + 2);
}

template <int S>
__device__ __forceinline__ void detector_response_body(const float *__restrict__ src, float *__restrict__ Lx, float *__restrict__ Ly,
                                                       float *__restrict__ Ldet, const EvoDev &ev, int x0, int y0, float *sm,
                                                       float thr, unsigned *__restrict__ mrow, unsigned *__restrict__ rc) {
    constexpr int R = 2 * S + 1, RW = SW3 + 2 * R, RH = SH3 + 2 * R;          // staged Lsmooth
    constexpr int LW = SW3 + 2 * (S + 1), LH = SH3 + 2 * (S + 1);             // Lx / Ly ring tile
    constexpr int DW = SW3 + 2, DH = SH3 + 2;                                 // Ldet ring tile
    constexpr int NS1 = NT / LW, BS1 = (LH + NS1 - 1) / NS1;                  // Lx / Ly tasks: LW columns x NS1 strips
    constexpr int NS2 = NT / DW, BS2 = (DH + NS2 - 1) / NS2;                  // Ldet tasks: DW columns x NS2 strips
    static_assert(2 * R <= 32 && DW * DH <= RW * RH, "halo fits stage_region's tail lanes; Ldet tile fits the staging buffer");
    float *s_in = sm, *s_x = sm + RW * RH, *s_y = s_x + LW * LH;
    float *s_d = sm;                                                          // reuses the staging buffer once Lx / Ly exist
    const int w = ev.w, h = ev.h;
    stage_region<R, R>(src, w, h, x0, y0, s_in);
    __syncthreads();
    // Strips start at min(sidx * BS, rows - BS): the last one overlaps its neighbour (both write the same values) instead of
    // ending in guarded rows, so the unrolled loops carry no bounds branches.
    if (threadIdx.x < LW * NS1) {   // Lx / Ly over the ring tile: ring (lr, c) is pixel (y0 - S - 1 + lr, x0 - S - 1 + c)
        const int sidx = threadIdx.x / LW, c = threadIdx.x - sidx * LW;
        const int r0 = min(sidx * BS1, LH - BS1);
        const int gx = x0 - (S + 1) + c;
        const bool xt = c > S && c <= S + SW3 && gx < w;      // a tile column inside the image
        const int yt0 = S + 1 - r0, yt1 = min(S + SH3, h - 1 - y0 + S + 1) - r0;   // tile rows inside the image: yt0 <= o <= yt1
        const float *col = s_in + r0 * RW + c;     // col[r * RW + {0, S, 2S}] = staged row r0 + r
        float *ox = s_x + r0 * LW + c, *oy = s_y + r0 * LW + c;
        int g = (y0 - (S + 1) + r0) * w + gx;
        float hm[BS1 + 2 * S], ho[BS1 + 2 * S];
#pragma unroll
        for (int r = 0; r < BS1 + 2 * S; r++) {
            const float a = col[r * RW], m = col[r * RW + S], z = col[r * RW + 2 * S];
            hm[r] = scharr_main<S & 3>(a, z);
            ho[r] = scharr_off<S & 3>(a, m, z, ev.norm, ev.middle);
            if (r >= 2 * S) {
                const int o = r - 2 * S;
                const float vx = scharr_off<S & 3>(hm[o], hm[o + S], hm[o + 2 * S], ev.norm, ev.middle);
                const float vy = scharr_main<S & 3>(ho[o], ho[o + 2 * S]);
                ox[o * LW] = vx;
                oy[o * LW] = vy;
                if (xt && o >= yt0 && o <= yt1) {
                    Lx[g] = vx;
                    Ly[g] = vy;
                }
                g += w;
            }
        }
    }
    __syncthreads();
    // ring rows above / below the image and ring columns left / right of it (the positions that copy are never copied from)
    const int rt = max(0, S + 1 - y0), rb = max(0, y0 + SH3 + S + 1 - h), cl = max(0, S + 1 - x0), cr = max(0, x0 + SW3 + S + 1 - w);
    if (rt + rb + cl + cr > 0) {      // the ring leaves the image (CTA-uniform)
        const int nc = cl + cr, nr = LH - rt - rb;
        for (int p = threadIdx.x; p < (rt + rb) * LW + nr * nc; p += NT) {
            int lr, lc;
            if (p < (rt + rb) * LW) {          // whole rows outside the image
                const int i = p / LW;
                lr = i < rt ? i : LH - rb + (i - rt); lc = p - i * LW;
            } else {                           // columns outside the image of the rows inside it
                const int i = (p - (rt + rb) * LW) / nc, j = p - (rt + rb) * LW - i * nc;
                lr = rt + i; lc = j < cl ? j : LW - cr + (j - cl);
            }
            const int gy = y0 - (S + 1) + lr, gx = x0 - (S + 1) + lc;
            const int q = (clampi(gy, 0, h - 1) - (y0 - (S + 1))) * LW + (clampi(gx, 0, w - 1) - (x0 - (S + 1)));
            s_x[lr * LW + lc] = s_x[q];
            s_y[lr * LW + lc] = s_y[q];
        }
        __syncthreads();
    }
    if (threadIdx.x < DW * NS2) {   // Ldet over the one-pixel ring: ring (dr, c) is pixel (y0 - 1 + dr, x0 - 1 + c) = Lx ring (dr + S, c + S)
        const int sidx = threadIdx.x / DW, c = threadIdx.x - sidx * DW;
        const int r0 = min(sidx * BS2, DH - BS2);
        const int gx = x0 - 1 + c;
        const bool xt = c >= 1 && c <= SW3 && gx < w;
        const int yt0 = 1 - r0, yt1 = min(SH3, h - y0) - r0;                 // tile rows inside the image: yt0 <= o <= yt1
        const float *cx = s_x + r0 * LW + c, *cy = s_y + r0 * LW + c;
        float *od = s_d + r0 * DW + c;
        int g = (y0 - 1 + r0) * w + gx;
        float hmx[BS2 + 2 * S], hox[BS2 + 2 * S], hoy[BS2 + 2 * S];
#pragma unroll
        for (int r = 0; r < BS2 + 2 * S; r++) {
            const float a = cx[r * LW], m = cx[r * LW + S], z = cx[r * LW + 2 * S];
            hmx[r] = scharr_main<S & 3>(a, z);                                                          // H_main(Lx)
            hox[r] = scharr_off<S & 3>(a, m, z, ev.norm, ev.middle);                                    // H_off(Lx)
            hoy[r] = scharr_off<S & 3>(cy[r * LW], cy[r * LW + S], cy[r * LW + 2 * S], ev.norm, ev.middle);   // H_off(Ly)
            if (r >= 2 * S) {
                const int o = r - 2 * S;
                const float lxx = scharr_off<S & 3>(hmx[o], hmx[o + S], hmx[o + 2 * S], ev.norm, ev.middle);
                const float lyy = scharr_main<S & 3>(hoy[o], hoy[o + 2 * S]);
                const float lxy = scharr_main<S & 3>(hox[o], hox[o + 2 * S]);
                const float v = (lxx * lyy - lxy * lxy) * ev.quat;
                od[o * DW] = v;
                if (xt && o >= yt0 && o <= yt1) Ldet[g] = v;
                g += w;
            }
        }
    }
    __syncthreads();
    // the body of k_extrema_mask on the shared Ldet tile
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int gx = x0 + tx;
    const bool xin = gx >= 1 && gx < w - 1;
    const float *col = s_d + (ty * STRIP) * DW + tx;
    const int wpr = (w + 31) >> 5;
    float m3[STRIP + 2], sd[STRIP + 2], cn[STRIP + 2];
#pragma unroll
    for (int r = 0; r < STRIP + 2; r++) {
        const float l = col[r * DW], c = col[r * DW + 1], rt = col[r * DW + 2];
        sd[r] = fmaxf(l, rt);
        m3[r] = fmaxf(sd[r], c);
        cn[r] = c;
        if (r >= 2) {
            const int o = r - 2, gy = y0 + ty * STRIP + o;
            const float v = cn[o + 1];
            const float m8 = fmaxf(fmaxf(m3[o], m3[o + 2]), sd[o + 1]);
            const bool hit = xin && gy >= 1 && gy < h - 1 && v > thr && v > m8;
            const unsigned bits = __ballot_sync(0xffffffffu, hit);
            if (tx == 0 && gy < h && x0 < w) {
                mrow[(size_t)gy * wpr + (x0 >> 5)] = bits;
                if (bits) atomicAdd(&rc[gy], (unsigned)__popc(bits));
            }
        }
    }
}

// one launch per octave over the octave's tiles (tile table as k_deriv1_v3); dynamic shared memory det_smem_floats(max sigma)
__global__ void __launch_bounds__(NT, 4) k_detector_response(const float *__restrict__ Ls, const float *__restrict__ Lt0,
                                                             float *__restrict__ Lx, float *__restrict__ Ly, float *__restrict__ Ldet,
                                                             size_t bstride, EvoTable T, const unsigned char *__restrict__ tile_evo,
                                                             int tile_offset, MaskLayout ML, float thr, unsigned *__restrict__ mask,
                                                             unsigned *__restrict__ rowcount) {
    extern __shared__ float sm[];
    const int gtile = blockIdx.x + tile_offset;
    const int e = tile_evo[gtile];
    const EvoDev ev = T.e[e];
    int x0, y0;
    tile_origin_v3(ev, gtile, x0, y0);
    const size_t base = (size_t)blockIdx.z * bstride + ev.off;
    const float *src = (e == 0 ? Lt0 : Ls) + base;   // evolution 0: Lsmooth IS Lt (lib.rs:201)
    unsigned *mrow = mask + (size_t)blockIdx.z * ML.total_words + ML.wordbase[e];
    unsigned *rc = rowcount + (size_t)blockIdx.z * T.total_rows + ev.rowbase;
    switch (ev.sigma) {
    case 1: detector_response_body<1>(src, Lx + base, Ly + base, Ldet + base, ev, x0, y0, sm, thr, mrow, rc); break;
    case 2: detector_response_body<2>(src, Lx + base, Ly + base, Ldet + base, ev, x0, y0, sm, thr, mrow, rc); break;
    case 3: detector_response_body<3>(src, Lx + base, Ly + base, Ldet + base, ev, x0, y0, sm, thr, mrow, rc); break;
    case 4: detector_response_body<4>(src, Lx + base, Ly + base, Ldet + base, ev, x0, y0, sm, thr, mrow, rc); break;
    default: detector_response_body<5>(src, Lx + base, Ly + base, Ldet + base, ev, x0, y0, sm, thr, mrow, rc); break;
    }
}

// warp per row: expand the row's mask words into candidates at rowoff[row] (x ascending)
__global__ void __launch_bounds__(NT) k_extrema_emit(const float *__restrict__ Ldet, size_t bstride, EvoTable T, MaskLayout ML,
                                                     const unsigned *__restrict__ mask, const unsigned *__restrict__ rowcount,
                                                     const unsigned *__restrict__ rowoff, Cand *__restrict__ cand, unsigned cap,
                                                     unsigned *overflow) {
    const int warp = (blockIdx.x * NT + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= T.total_rows) return;
    const size_t ri = (size_t)blockIdx.z * T.total_rows + warp;
    if (rowcount[ri] == 0) return;
    int e = 0;
    while (e + 1 < T.n && warp >= T.e[e + 1].rowbase) e++;
    const int y = warp - T.e[e].rowbase, w = T.e[e].w;
    const int wpr = (w + 31) >> 5;
    const unsigned *mrow = mask + (size_t)blockIdx.z * ML.total_words + ML.wordbase[e] + (size_t)y * wpr;
    const float *D = Ldet + (size_t)blockIdx.z * bstride + T.e[e].off + (size_t)y * w;
    unsigned base = rowoff[ri];
    for (int wb = 0; wb < wpr; wb += 32) {
        unsigned word = (wb + lane < wpr) ? mrow[wb + lane] : 0u;
        const unsigned c = __popc(word);
        unsigned inc = c;
        for (int o = 1; o < 32; o <<= 1) { unsigned t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
        unsigned pos = base + inc - c;
        while (word) {
            const int b = __ffs(word) - 1;
            word &= word - 1;
            const int x = (wb + lane) * 32 + b;
            if (pos < cap) { Cand cd; cd.x = x; cd.y = y; cd.e = e; cd.v = D[x]; cand[(size_t)blockIdx.z * cap + pos] = cd; }
            else *overflow = 1u;
            pos++;
        }
        base += __shfl_sync(0xffffffffu, inc, 31);
    }
}

// exclusive scan of per-row counts; one CTA of 1024 threads per frame
__global__ void __launch_bounds__(1024) k_scan_rows(const unsigned *__restrict__ rowcount, unsigned *__restrict__ rowoff,
                                                    unsigned *__restrict__ total, int n) {
    __shared__ unsigned s_warp[32];
    __shared__ unsigned s_carry;
    const unsigned *in = rowcount + (size_t)blockIdx.x * n;
    unsigned *out = rowoff + (size_t)blockIdx.x * n;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (int base = 0; base < n; base += 1024) {
        int i = base + threadIdx.x;
        unsigned v = i < n ? in[i] : 0u, x = v;
        for (int o = 1; o < 32; o <<= 1) { unsigned t = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += t; }
        if (lane == 31) s_warp[wid] = x;
        __syncthreads();
        if (wid == 0) {
            unsigned y = s_warp[lane], z = y;
            for (int o = 1; o < 32; o <<= 1) { unsigned t = __shfl_up_sync(0xffffffffu, z, o); if (lane >= o) z += t; }
            s_warp[lane] = z - y;
        }
        __syncthreads();
        unsigned excl = s_carry + s_warp[wid] + x - v;
        if (i < n) out[i] = excl;
        __syncthreads();
        if (threadIdx.x == 1023) s_carry = excl + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) total[blockIdx.x] = s_carry;
}

// ---------------------------------------------------------------------------------------------
// Sequential-equivalent duplicate suppression (scale_space_extrema.rs:61-117).  One CTA per frame walks
// the candidates in reference order; for each one the whole CTA searches the keypoint cache in parallel
// for the FIRST (lowest slot) cached keypoint of the same or previous class within `size`, then thread 0
// applies the reference's replace / drop / append rule.  Candidates failing the border test never modify
// the cache (:95-116) and are skipped up front.
__global__ void __launch_bounds__(1024) k_suppress_seq(const Cand *__restrict__ cand, const unsigned *__restrict__ ncand,
                                                   unsigned capc, EvoTable T, cvb_keypoint *__restrict__ cache,
                                                   unsigned *__restrict__ ncache, unsigned *__restrict__ nneed, unsigned capk,
                                                   unsigned *overflow) {
    __shared__ unsigned s_min[32];
    __shared__ unsigned s_n, s_drop;
    const int b = blockIdx.x;
    const Cand *cd = cand + (size_t)b * capc;
    cvb_keypoint *kc = cache + (size_t)b * capk;
    const unsigned n = min(ncand[b], capc);
    const float smax = 10.0f * sqrtf(2.0f);
    if (threadIdx.x == 0) { s_n = 0; s_drop = 0; }
    __syncthreads();
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (unsigned ci = 0; ci < n; ci++) {
        const Cand c = cd[ci];
        const EvoDev ev = T.e[c.e];
        const float ratio = (float)(1 << ev.octave);
        const float size = ev.size;
        const float sigma_size = roundf(size / ratio);
        const float px = (float)c.x, py = (float)c.y;
        // border test (:97-104), evaluated first: a failing candidate has no effect on the cache
        const float left_x = roundf(px - smax * sigma_size) - 1.f, right_x = roundf(px + smax * sigma_size) + 1.f;
        const float up_y = roundf(py - smax * sigma_size) - 1.f, down_y = roundf(py + smax * sigma_size) + 1.f;
        const bool is_out = left_x < 0.f || right_x >= (float)ev.w || up_y < 0.f || down_y >= (float)ev.h;
        if (is_out) continue;   // uniform across the CTA
        const unsigned nc = s_n;
        const float fx = px * ratio, fy = py * ratio, s2 = size * size;
        unsigned kmin = 0xffffffffu;
        for (unsigned k = threadIdx.x; k < nc; k += 1024) {
            const cvb_keypoint p = kc[k];
            if ((unsigned)c.e == p.class_id || (c.e != 0 && (unsigned)(c.e - 1) == p.class_id)) {
                float dx = fx - p.x, dy = fy - p.y;
                float dist = dx * dx + dy * dy;
                if (dist <= s2) { kmin = k; break; }
            }
        }
        for (int o = 16; o; o >>= 1) kmin = min(kmin, __shfl_xor_sync(0xffffffffu, kmin, o));
        if (lane == 0) s_min[wid] = kmin;
        __syncthreads();
        if (wid == 0) {
            unsigned m = s_min[lane];
            for (int o = 16; o; o >>= 1) m = min(m, __shfl_xor_sync(0xffffffffu, m, o));
            if (lane == 0) {
                const float resp = fabsf(c.v);
                bool is_repeated = false, is_extremum = true;
                if (m != 0xffffffffu) {
                    if (resp > kc[m].response) is_repeated = true; else is_extremum = false;
                }
                if (is_extremum) {
                    cvb_keypoint kp;
                    kp.x = px * ratio + 0.5f * (ratio - 1.0f);
                    kp.y = py * ratio + 0.5f * (ratio - 1.0f);
                    kp.response = resp; kp.size = size; kp.angle = 0.f;
                    kp.octave = (uint32_t)ev.octave; kp.class_id = (uint32_t)c.e;
                    if (is_repeated) kc[m] = kp;
                    else if (nc < capk) { kc[nc] = kp; s_n = nc + 1; }
                    else { *overflow = 2u; s_drop++; }
                }
            }
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) { ncache[b] = s_n; nneed[b] = s_n + s_drop; }   // an upper bound on the need: a drop can hide a later match
}

// Parallel, provably sequential-equivalent duplicate suppression (scale_space_extrema.rs:61-117).
//
// The reference walks all candidates in order against a growing cache: first cached keypoint (lowest
// slot) of the same or previous class within `size` -> replace it if stronger, else drop; no hit ->
// append.  Observations that make it parallel without changing a single outcome:
//  * every cache slot is always occupied by a candidate, so the cache is a per-candidate state
//    (alive flag + slot key); a class-e candidate only ever matches occupants of class e or e-1;
//  * candidate c can be influenced by an earlier candidate c' only if c' is within `size` of c or of an
//    occupant within `size` of c, i.e. |F_c - F_c'| <= 2*size + 2*off (off = 0.5*(ratio-1) shift of the
//    stored point).  Classes are processed in order; inside a class, in rounds: a candidate is READY
//    when every earlier unresolved candidate of its class lies beyond that radius; all ready candidates
//    are mutually independent (they cannot touch a common occupant) and are resolved concurrently with
//    exactly the reference's comparisons.  The earliest unresolved candidate is always ready, so the
//    loop terminates; in the worst case (one long dependency chain) it degenerates to the serial order.
//  * "lowest slot" is decided on slot KEYS: real slot index for slots that existed before the class,
//    BASE + appender's candidate index for slots appended during the class (same relative order);
//    keys are turned into real indices by a prefix sum when the class is finished.
// One CTA per frame.  Uniform-grid bins (cell >= interaction radius) give O(neighbourhood) searches.
struct SupScratch {
    unsigned char *state;     // 0 unresolved, 1 resolved            [B][capc]
    unsigned char *alive;     // currently occupying a cache slot    [B][capc]
    unsigned char *rdy;       //                                      [B][capc]
    unsigned *key;            // slot key / final slot index          [B][capc]
    unsigned *rank;           // exclusive prefix of appended flags   [B][capc]
    int *next;                // bin linked lists                     [B][capc]
    int *binA, *binB;         // heads: class e-1 occupants / class e candidates   [B][nbmax]
    unsigned nbmax;
};

__device__ __forceinline__ unsigned block_excl_scan_1024(unsigned v, unsigned *s_warp, unsigned *total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    unsigned x = v;
    for (int o = 1; o < 32; o <<= 1) { unsigned t = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += t; }
    if (lane == 31) s_warp[wid] = x;
    __syncthreads();
    if (wid == 0) {
        unsigned y = s_warp[lane], z = y;
        for (int o = 1; o < 32; o <<= 1) { unsigned t = __shfl_up_sync(0xffffffffu, z, o); if (lane >= o) z += t; }
        s_warp[lane] = z - y;
        if (lane == 31) s_warp[32] = z;
    }
    __syncthreads();
    unsigned excl = s_warp[wid] + x - v;
    *total = s_warp[32];
    __syncthreads();
    return excl;
}

__global__ void __launch_bounds__(1024) k_suppress_par(const Cand *__restrict__ cand, const unsigned *__restrict__ ncand,
                                                       const unsigned *__restrict__ rowoff, unsigned capc, EvoTable T,
                                                       SupScratch S, cvb_keypoint *__restrict__ cache,
                                                       unsigned *__restrict__ ncache, unsigned *__restrict__ nneed, unsigned capk, unsigned *overflow,
                                                       const unsigned *__restrict__ fallback) {
    __shared__ unsigned s_warp[33];
    __shared__ int s_more;
    const unsigned BASE = 0x40000000u;
    const int b = blockIdx.x;
    if (fallback && !fallback[b]) return;   // already handled by k_suppress_smem
    const Cand *cd = cand + (size_t)b * capc;
    unsigned char *state = S.state + (size_t)b * capc, *alive = S.alive + (size_t)b * capc, *rdy = S.rdy + (size_t)b * capc;
    unsigned *key = S.key + (size_t)b * capc, *rank = S.rank + (size_t)b * capc;
    int *next = S.next + (size_t)b * capc;
    int *binA = S.binA + (size_t)b * S.nbmax, *binB = S.binB + (size_t)b * S.nbmax;
    const unsigned ntot = min(ncand[b], capc);
    const unsigned *ro = rowoff + (size_t)b * T.total_rows;
    const float smax = 10.0f * sqrtf(2.0f);
    const float W0 = (float)T.e[0].w, H0 = (float)T.e[0].h;
    unsigned N = 0;                       // slots so far
    unsigned prev_cs = 0, prev_ce = 0;    // candidate range of class e-1
    float prev_off = 0.f, prev_ratio = 1.f;
    for (int e = 0; e < T.n; e++) {
        const EvoDev ev = T.e[e];
        const unsigned cs = min(ro[ev.rowbase], ntot);
        const unsigned ce = (e + 1 < T.n) ? min(ro[T.e[e + 1].rowbase], ntot) : ntot;
        const float ratio = (float)(1 << ev.octave), off = 0.5f * (ratio - 1.0f), size = ev.size, s2 = size * size;
        const float sigma_size = roundf(size / ratio);
        const float Dr = 2.0f * size + 2.0f * off + 2.0f;
        const float cell = fmaxf(16.0f, ceilf(Dr));
        const float inv_cell = 1.0f / cell;
        const int nbx = (int)(W0 * inv_cell) + 2, nby = (int)(H0 * inv_cell) + 2;
        const int nb = nbx * nby;
        for (int t = threadIdx.x; t < nb; t += 1024) { binA[t] = -1; binB[t] = -1; }
        __syncthreads();
        // occupants of class e-1 (alive) binned by their stored point
        for (unsigned g = prev_cs + threadIdx.x; g < prev_ce; g += 1024) {
            if (!alive[g]) continue;
            const Cand c = cd[g];
            float sx = (float)c.x * prev_ratio + prev_off, sy = (float)c.y * prev_ratio + prev_off;
            int bx = min(max((int)(sx * inv_cell), 0), nbx - 1), by = min(max((int)(sy * inv_cell), 0), nby - 1);
            next[g] = atomicExch(&binA[by * nbx + bx], (int)g);
        }
        // candidates of class e: border test (:97-104); failing ones never touch the cache
        for (unsigned g = cs + threadIdx.x; g < ce; g += 1024) {
            const Cand c = cd[g];
            const float px = (float)c.x, py = (float)c.y;
            const float left_x = roundf(px - smax * sigma_size) - 1.f, right_x = roundf(px + smax * sigma_size) + 1.f;
            const float up_y = roundf(py - smax * sigma_size) - 1.f, down_y = roundf(py + smax * sigma_size) + 1.f;
            const bool is_out = left_x < 0.f || right_x >= (float)ev.w || up_y < 0.f || down_y >= (float)ev.h;
            alive[g] = 0; key[g] = 0xffffffffu; rank[g] = 0;
            if (is_out) { state[g] = 1; continue; }
            state[g] = 0;
            float fx = px * ratio, fy = py * ratio;
            int bx = min(max((int)(fx * inv_cell), 0), nbx - 1), by = min(max((int)(fy * inv_cell), 0), nby - 1);
            next[g] = atomicExch(&binB[by * nbx + bx], (int)g);
        }
        __syncthreads();
        // ---- rounds
        for (;;) {
            if (threadIdx.x == 0) s_more = 0;
            __syncthreads();
            // phase A: readiness against the state at the start of the round
            for (unsigned g = cs + threadIdx.x; g < ce; g += 1024) {
                if (state[g]) continue;
                const Cand c = cd[g];
                const float fx = (float)c.x * ratio, fy = (float)c.y * ratio;
                const int bx = min(max((int)(fx * inv_cell), 0), nbx - 1), by = min(max((int)(fy * inv_cell), 0), nby - 1);
                bool ready = true;
                for (int yy = max(by - 1, 0); yy <= min(by + 1, nby - 1) && ready; yy++)
                    for (int xx = max(bx - 1, 0); xx <= min(bx + 1, nbx - 1) && ready; xx++)
                        for (int j = binB[yy * nbx + xx]; j >= 0; j = next[j]) {
                            if ((unsigned)j >= g || state[j]) continue;
                            const Cand q = cd[j];
                            if (fabsf((float)q.x * ratio - fx) <= Dr && fabsf((float)q.y * ratio - fy) <= Dr) { ready = false; break; }
                        }
                rdy[g] = ready ? 1 : 0;
                if (!ready) s_more = 1;
            }
            __syncthreads();
            const int more = s_more;
            // phase B: resolve every ready candidate with the reference's own comparisons
            for (unsigned g = cs + threadIdx.x; g < ce; g += 1024) {
                if (state[g] || !rdy[g]) continue;
                const Cand c = cd[g];
                const float fx = (float)c.x * ratio, fy = (float)c.y * ratio;
                const float resp = fabsf(c.v);
                const int bx = min(max((int)(fx * inv_cell), 0), nbx - 1), by = min(max((int)(fy * inv_cell), 0), nby - 1);
                unsigned best_key = 0xffffffffu;
                int best = -1;
                for (int yy = max(by - 1, 0); yy <= min(by + 1, nby - 1); yy++)
                    for (int xx = max(bx - 1, 0); xx <= min(bx + 1, nbx - 1); xx++) {
                        const int bin = yy * nbx + xx;
                        for (int o = binA[bin]; o >= 0; o = next[o]) {        // occupants of class e-1
                            if (!alive[o]) continue;
                            const Cand q = cd[o];
                            float dx = fx - ((float)q.x * prev_ratio + prev_off), dy = fy - ((float)q.y * prev_ratio + prev_off);
                            float dist = dx * dx + dy * dy;
                            if (dist <= s2 && key[o] < best_key) { best_key = key[o]; best = o; }
                        }
                        for (int o = binB[bin]; o >= 0; o = next[o]) {        // occupants of class e (earlier candidates)
                            if ((unsigned)o >= g || !alive[o]) continue;
                            const Cand q = cd[o];
                            float dx = fx - ((float)q.x * ratio + off), dy = fy - ((float)q.y * ratio + off);
                            float dist = dx * dx + dy * dy;
                            if (dist <= s2 && key[o] < best_key) { best_key = key[o]; best = o; }
                        }
                    }
                if (best >= 0) {
                    if (resp > fabsf(cd[best].v)) { alive[best] = 0; key[g] = best_key; alive[g] = 1; }   // replace in place
                } else {
                    key[g] = BASE + (g - cs); alive[g] = 1; rank[g] = 1;                                   // append
                }
                state[g] = 1;
            }
            __syncthreads();
            if (!more) break;
        }
        // ---- slot keys -> real slot indices (appended slots keep candidate order)
        unsigned carry = 0;
        for (unsigned base = cs; base < ce; base += 1024) {
            const unsigned g = base + threadIdx.x;
            const unsigned v = g < ce ? rank[g] : 0u;
            unsigned tot;
            const unsigned ex = block_excl_scan_1024(v, s_warp, &tot);
            if (g < ce) rank[g] = carry + ex;
            carry += tot;
        }
        __syncthreads();
        for (unsigned g = cs + threadIdx.x; g < ce; g += 1024)
            if (alive[g] && key[g] >= BASE) key[g] = N + rank[cs + (key[g] - BASE)];
        N += carry;
        __syncthreads();
        prev_cs = cs; prev_ce = ce; prev_off = off; prev_ratio = ratio;
    }
    // ---- materialise the cache in slot order
    for (unsigned g = threadIdx.x; g < ntot; g += 1024) {
        if (!alive[g]) continue;
        const unsigned k = key[g];
        if (k >= capk) { *overflow = 2u; continue; }
        const Cand c = cd[g];
        const EvoDev ev = T.e[c.e];
        const float ratio = (float)(1 << ev.octave);
        cvb_keypoint kp;
        kp.x = (float)c.x * ratio + 0.5f * (ratio - 1.0f);
        kp.y = (float)c.y * ratio + 0.5f * (ratio - 1.0f);
        kp.response = fabsf(c.v); kp.size = ev.size; kp.angle = 0.f;
        kp.octave = (uint32_t)ev.octave; kp.class_id = (uint32_t)c.e;
        cache[(size_t)b * capk + k] = kp;
    }
    if (threadIdx.x == 0) { ncache[b] = min(N, capk); nneed[b] = N; }
}

// Shared-memory version of k_suppress_par (same algorithm, same outcomes): all mutable per-candidate state
// of the two live classes (e-1 and e) sits in a ring of SUP_CAPS entries in shared memory, so the bin walks
// cost shared-memory latency instead of L2 round trips.  Frames whose two consecutive classes exceed the
// ring, or whose bin grid exceeds SUP_NB, set fallback[b] and are handled by k_suppress_par.
constexpr unsigned SUP_CAPS = 8192, SUP_NB = 4096;
constexpr size_t SUP_SMEM = SUP_CAPS * (3 + 4 + 2 + 4 + 4 + 2) + SUP_NB * 2 * 4;

__global__ void __launch_bounds__(1024) k_suppress_smem(const Cand *__restrict__ cand, const unsigned *__restrict__ ncand,
                                                        const unsigned *__restrict__ rowoff, unsigned capc, EvoTable T,
                                                        SupScratch S, cvb_keypoint *__restrict__ cache,
                                                        unsigned *__restrict__ ncache, unsigned *__restrict__ nneed, unsigned capk, unsigned *overflow,
                                                        unsigned *__restrict__ fallback) {
    extern __shared__ __align__(16) unsigned char smraw[];
    unsigned *s_key = (unsigned *)smraw;                          // [CAPS]
    unsigned *s_pos = s_key + SUP_CAPS;                           // x | y << 16
    float *s_resp = (float *)(s_pos + SUP_CAPS);
    int *s_binA = (int *)(s_resp + SUP_CAPS);                     // [NB]
    int *s_binB = s_binA + SUP_NB;
    unsigned short *s_next = (unsigned short *)(s_binB + SUP_NB); // ring index or 0xffff
    unsigned short *s_rank = s_next + SUP_CAPS;
    unsigned char *s_state = (unsigned char *)(s_rank + SUP_CAPS);
    unsigned char *s_alive = s_state + SUP_CAPS;
    unsigned char *s_rdy = s_alive + SUP_CAPS;
    __shared__ unsigned s_warp[33];
    __shared__ int s_more;
    const unsigned BASE = 0x40000000u, M = SUP_CAPS - 1;
    const int b = blockIdx.x;
    const Cand *cd = cand + (size_t)b * capc;
    unsigned char *g_alive = S.alive + (size_t)b * capc;
    unsigned *g_key = S.key + (size_t)b * capc;
    const unsigned ntot = min(ncand[b], capc);
    const unsigned *ro = rowoff + (size_t)b * T.total_rows;
    const float smax = 10.0f * sqrtf(2.0f);
    const float W0 = (float)T.e[0].w, H0 = (float)T.e[0].h;
    // feasibility (uniform): ring capacity and bin grid
    {
        bool okk = true;
        unsigned pcs = 0;
        for (int e = 0; e < T.n; e++) {
            const unsigned cs = min(ro[T.e[e].rowbase], ntot);
            const unsigned ce = (e + 1 < T.n) ? min(ro[T.e[e + 1].rowbase], ntot) : ntot;
            if (ce - pcs > SUP_CAPS) okk = false;
            pcs = cs;
        }
        if (!okk) { if (threadIdx.x == 0) fallback[b] = 1; return; }
        if (threadIdx.x == 0) fallback[b] = 0;
    }
    unsigned N = 0, prev_cs = 0, prev_ce = 0;
    float prev_off = 0.f, prev_ratio = 1.f;
    for (int e = 0; e < T.n; e++) {
        const EvoDev ev = T.e[e];
        const unsigned cs = min(ro[ev.rowbase], ntot);
        const unsigned ce = (e + 1 < T.n) ? min(ro[T.e[e + 1].rowbase], ntot) : ntot;
        const float ratio = (float)(1 << ev.octave), off = 0.5f * (ratio - 1.0f), size = ev.size, s2 = size * size;
        const float sigma_size = roundf(size / ratio);
        const float Dr = 2.0f * size + 2.0f * off + 2.0f;
        float cell = fmaxf(32.0f, ceilf(Dr));
        while (((int)(W0 / cell) + 2) * ((int)(H0 / cell) + 2) > (int)SUP_NB) cell *= 2.0f;
        const float inv_cell = 1.0f / cell;
        const int nbx = (int)(W0 * inv_cell) + 2, nby = (int)(H0 * inv_cell) + 2;
        const int nb = min(nbx * nby, (int)SUP_NB);
        for (int t = threadIdx.x; t < nb; t += 1024) { s_binA[t] = -1; s_binB[t] = -1; }
        __syncthreads();
        for (unsigned g = prev_cs + threadIdx.x; g < prev_ce; g += 1024) {
            const unsigned r = g & M;
            if (!s_alive[r]) continue;
            const unsigned pp = s_pos[r];
            const float sx = (float)(pp & 0xffffu) * prev_ratio + prev_off, sy = (float)(pp >> 16) * prev_ratio + prev_off;
            const int bx = min(max((int)(sx * inv_cell), 0), nbx - 1), by = min(max((int)(sy * inv_cell), 0), nby - 1);
            s_next[r] = (unsigned short)atomicExch(&s_binA[min(by * nbx + bx, nb - 1)], (int)r);
        }
        for (unsigned g = cs + threadIdx.x; g < ce; g += 1024) {
            const unsigned r = g & M;
            const Cand c = cd[g];
            s_pos[r] = (unsigned)c.x | ((unsigned)c.y << 16);
            s_resp[r] = fabsf(c.v);
            const float px = (float)c.x, py = (float)c.y;
            const float left_x = roundf(px - smax * sigma_size) - 1.f, right_x = roundf(px + smax * sigma_size) + 1.f;
            const float up_y = roundf(py - smax * sigma_size) - 1.f, down_y = roundf(py + smax * sigma_size) + 1.f;
            const bool is_out = left_x < 0.f || right_x >= (float)ev.w || up_y < 0.f || down_y >= (float)ev.h;
            s_alive[r] = 0; s_key[r] = 0xffffffffu; s_rank[r] = 0;
            if (is_out) { s_state[r] = 1; continue; }
            s_state[r] = 0;
            const float fx = px * ratio, fy = py * ratio;
            const int bx = min(max((int)(fx * inv_cell), 0), nbx - 1), by = min(max((int)(fy * inv_cell), 0), nby - 1);
            s_next[r] = (unsigned short)atomicExch(&s_binB[min(by * nbx + bx, nb - 1)], (int)r);
        }
        __syncthreads();
        for (;;) {
            if (threadIdx.x == 0) s_more = 0;
            __syncthreads();
            for (unsigned g = cs + threadIdx.x; g < ce; g += 1024) {
                const unsigned r = g & M;
                if (s_state[r]) continue;
                const unsigned pp = s_pos[r];
                const float fx = (float)(pp & 0xffffu) * ratio, fy = (float)(pp >> 16) * ratio;
                const int bx = min(max((int)(fx * inv_cell), 0), nbx - 1), by = min(max((int)(fy * inv_cell), 0), nby - 1);
                bool ready = true;
                for (int yy = max(by - 1, 0); yy <= min(by + 1, nby - 1) && ready; yy++)
                    for (int xx = max(bx - 1, 0); xx <= min(bx + 1, nbx - 1) && ready; xx++)
                        for (int j = s_binB[min(yy * nbx + xx, nb - 1)]; j >= 0; j = (s_next[j] == 0xffffu ? -1 : (int)s_next[j])) {
                            // ring order == candidate order inside one class (the class fits the ring)
                            if (((unsigned)j - cs) % SUP_CAPS >= ((r - cs) % SUP_CAPS) || s_state[j]) continue;
                            const unsigned qq = s_pos[j];
                            if (fabsf((float)(qq & 0xffffu) * ratio - fx) <= Dr && fabsf((float)(qq >> 16) * ratio - fy) <= Dr) { ready = false; break; }
                        }
                s_rdy[r] = ready ? 1 : 0;
                if (!ready) s_more = 1;
            }
            __syncthreads();
            const int more = s_more;
            for (unsigned g = cs + threadIdx.x; g < ce; g += 1024) {
                const unsigned r = g & M;
                if (s_state[r] || !s_rdy[r]) continue;
                const unsigned pp = s_pos[r];
                const float fx = (float)(pp & 0xffffu) * ratio, fy = (float)(pp >> 16) * ratio;
                const float resp = s_resp[r];
                const int bx = min(max((int)(fx * inv_cell), 0), nbx - 1), by = min(max((int)(fy * inv_cell), 0), nby - 1);
                unsigned best_key = 0xffffffffu;
                int best = -1;
                const unsigned myord = (r - cs) % SUP_CAPS;
                for (int yy = max(by - 1, 0); yy <= min(by + 1, nby - 1); yy++)
                    for (int xx = max(bx - 1, 0); xx <= min(bx + 1, nbx - 1); xx++) {
                        const int bin = min(yy * nbx + xx, nb - 1);
                        for (int o = s_binA[bin]; o >= 0; o = (s_next[o] == 0xffffu ? -1 : (int)s_next[o])) {
                            if (!s_alive[o]) continue;
                            const unsigned qq = s_pos[o];
                            float dx = fx - ((float)(qq & 0xffffu) * prev_ratio + prev_off), dy = fy - ((float)(qq >> 16) * prev_ratio + prev_off);
                            float dist = dx * dx + dy * dy;
                            if (dist <= s2 && s_key[o] < best_key) { best_key = s_key[o]; best = o; }
                        }
                        for (int o = s_binB[bin]; o >= 0; o = (s_next[o] == 0xffffu ? -1 : (int)s_next[o])) {
                            if (((unsigned)o - cs) % SUP_CAPS >= myord || !s_alive[o]) continue;
                            const unsigned qq = s_pos[o];
                            float dx = fx - ((float)(qq & 0xffffu) * ratio + off), dy = fy - ((float)(qq >> 16) * ratio + off);
                            float dist = dx * dx + dy * dy;
                            if (dist <= s2 && s_key[o] < best_key) { best_key = s_key[o]; best = o; }
                        }
                    }
                if (best >= 0) {
                    if (resp > s_resp[best]) { s_alive[best] = 0; s_key[r] = best_key; s_alive[r] = 1; }
                } else {
                    s_key[r] = BASE + (g - cs); s_alive[r] = 1; s_rank[r] = 1;
                }
                s_state[r] = 1;
            }
            __syncthreads();
            if (!more) break;
        }
        // appended-slot prefix (ranks fit 16 bits: a class has at most SUP_CAPS candidates... store as u16 via two passes)
        unsigned carry = 0;
        for (unsigned base = cs; base < ce; base += 1024) {
            const unsigned g = base + threadIdx.x;
            const unsigned v = g < ce ? (unsigned)s_rank[g & M] : 0u;
            unsigned tot;
            const unsigned ex = block_excl_scan_1024(v, s_warp, &tot);
            if (g < ce) s_rank[g & M] = (unsigned short)(carry + ex);
            carry += tot;
        }
        __syncthreads();
        for (unsigned g = cs + threadIdx.x; g < ce; g += 1024) {
            const unsigned r = g & M;
            if (s_alive[r] && s_key[r] >= BASE) s_key[r] = N + (unsigned)s_rank[(cs + (s_key[r] - BASE)) & M];
        }
        N += carry;
        // class e-1 is final now: retire it to global memory
        for (unsigned g = prev_cs + threadIdx.x; g < prev_ce; g += 1024) { g_alive[g] = s_alive[g & M]; g_key[g] = s_key[g & M]; }
        __syncthreads();
        prev_cs = cs; prev_ce = ce; prev_off = off; prev_ratio = ratio;
    }
    for (unsigned g = prev_cs + threadIdx.x; g < prev_ce; g += 1024) { g_alive[g] = s_alive[g & M]; g_key[g] = s_key[g & M]; }
    __syncthreads();
    for (unsigned g = threadIdx.x; g < ntot; g += 1024) {
        if (!g_alive[g]) continue;
        const unsigned k = g_key[g];
        if (k >= capk) { *overflow = 2u; continue; }
        const Cand c = cd[g];
        const EvoDev ev = T.e[c.e];
        const float ratio = (float)(1 << ev.octave);
        cvb_keypoint kp;
        kp.x = (float)c.x * ratio + 0.5f * (ratio - 1.0f);
        kp.y = (float)c.y * ratio + 0.5f * (ratio - 1.0f);
        kp.response = fabsf(c.v); kp.size = ev.size; kp.angle = 0.f;
        kp.octave = (uint32_t)ev.octave; kp.class_id = (uint32_t)c.e;
        cache[(size_t)b * capk + k] = kp;
    }
    if (threadIdx.x == 0) { ncache[b] = min(N, capk); nneed[b] = N; }
}

// Upper-scale filter (:120-140): cache[i] is dropped when a LATER cache entry of class+1 lies within
// size_i and is at least as strong (any hit decides, so the scan order is irrelevant).
// grid = (i-chunks, j-chunks, B): each CTA tests 256 entries against one 256-entry tile of later entries
// and clears keep[i] on a hit (keep is preset to 1).
__global__ void __launch_bounds__(NT) k_filter_upper(const cvb_keypoint *__restrict__ cache,
                                                     const unsigned *__restrict__ ncache, unsigned capk,
                                                     unsigned char *__restrict__ keep) {
    __shared__ float s_x[NT], s_y[NT], s_r[NT];
    __shared__ unsigned s_c[NT];
    __shared__ unsigned s_lo[NT / 32], s_hi[NT / 32];
    const int b = blockIdx.z;
    const unsigned n = ncache[b];
    const cvb_keypoint *kc = cache + (size_t)b * capk;
    const unsigned nchunks = (n + NT - 1) / NT;
    for (unsigned ic = blockIdx.x; ic < nchunks; ic += gridDim.x) {
        const unsigned i = ic * NT + threadIdx.x;
        cvb_keypoint a = {};
        if (i < n) a = kc[i];
        // class range of this i-chunk: the cache is almost sorted by class, so most j-chunks hold no class this chunk's
        // keypoints compare against (class + 1) and are skipped after one vote
        unsigned lo = i < n ? a.class_id : 0xffffffffu, hi = i < n ? a.class_id : 0u;
        lo = __reduce_min_sync(0xffffffffu, lo); hi = __reduce_max_sync(0xffffffffu, hi);
        __syncthreads();
        if ((threadIdx.x & 31) == 0) { s_lo[threadIdx.x >> 5] = lo; s_hi[threadIdx.x >> 5] = hi; }
        __syncthreads();
        for (int k = 0; k < NT / 32; k++) { lo = min(lo, s_lo[k]); hi = max(hi, s_hi[k]); }
        const float s2 = a.size * a.size;
        bool rep = false;
        for (unsigned jc = ic + blockIdx.y; jc < nchunks; jc += gridDim.y) {
            const unsigned j = jc * NT + threadIdx.x;
            cvb_keypoint q = {};
            bool relevant = false;
            if (j < n) { q = kc[j]; relevant = q.class_id >= lo + 1 && q.class_id <= hi + 1; }
            if (!__syncthreads_or(relevant)) continue;          // also orders the previous round's reads before the stores below
            if (j < n) { s_x[threadIdx.x] = q.x; s_y[threadIdx.x] = q.y; s_r[threadIdx.x] = q.response; s_c[threadIdx.x] = q.class_id; }
            __syncthreads();
            if (i >= n) continue;
            const unsigned lim = min((unsigned)NT, n - jc * NT);
            for (unsigned u = 0; u < lim; u++) {
                if (jc * NT + u <= i || s_c[u] != a.class_id + 1) continue;
                float dx = a.x - s_x[u], dy = a.y - s_y[u];
                float dist = dx * dx + dy * dy;
                if (dist <= s2 && a.response <= s_r[u]) rep = true;
            }
        }
        if (rep) keep[(size_t)b * capk + i] = 0;
    }
}

// ---------------------------------------------------------------------------------------------
// Sub-pixel refinement + main orientation, one warp per keypoint (scale_space_extrema.rs:229-362).
struct OrientTables {
    int nwin;                 // number of sliding windows (ang1 = 0, += 0.15f while < 2pi)
    float ang1[64];
    float ang2[64];           // the window's upper end: ang1 + pi/3, or ang1 - 5pi/3 once that passes 2pi (scale_space_extrema.rs:262-266)
    int nn;                   // windows [0, nn) do not wrap (ang1 < ang2), windows [nn, nwin) do; both tables ascend inside each group
    signed char di[109], dj[109];
    float gw[109];            // GAUSS25[id[j+6]][id[i+6]]
};

__global__ void __launch_bounds__(NT) k_refine_orient(const cvb_keypoint *__restrict__ cache,
                                                      const unsigned *__restrict__ ncache, unsigned capk,
                                                      const unsigned char *__restrict__ keep, EvoTable T,
                                                      const float *__restrict__ Ldet, const float *__restrict__ Lx,
                                                      const float *__restrict__ Ly, size_t bstride,
                                                      const OrientTables *__restrict__ OT,
                                                      cvb_keypoint *__restrict__ refined,
                                                      unsigned char *__restrict__ valid) {
    // Window membership is decided once per SAMPLE instead of once per (window, sample): both window ends ascend with the window
    // index inside the non-wrapping and the wrapping group, so the windows that hold an angle are index ranges whose ends are
    // counts of table entries below the angle -- found from an arithmetic guess and corrected with the reference's own
    // comparisons (exact whatever the guess).  The 42 windows of a sample become one 64-bit mask; a lane then adds the samples
    // of its two windows in sample order, as before.
    __shared__ float2 s_r[NT / 32][112];
    __shared__ uint2 s_m[NT / 32][112];
    __shared__ float s_a1[64], s_a2[64];
    const int b = blockIdx.y;
    const unsigned n = ncache[b];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const float PI = 3.14159265358979323846f;
    const float two_pi = 2.0f * PI;
    const int nwin = OT->nwin, nn = OT->nn;
    if (threadIdx.x < 64) { s_a1[threadIdx.x] = OT->ang1[threadIdx.x]; s_a2[threadIdx.x] = OT->ang2[threadIdx.x]; }
    __syncthreads();
    auto count_lt = [](const float *A, int cnt, float v, int g) {        // #{i < cnt : A[i] < v}, A ascending
        g = min(max(g, 0), cnt);
        while (g < cnt && A[g] < v) g++;
        while (g > 0 && !(A[g - 1] < v)) g--;
        return g;
    };
    auto count_le = [](const float *A, int cnt, float v, int g) {        // #{i < cnt : A[i] <= v}
        g = min(max(g, 0), cnt);
        while (g < cnt && A[g] <= v) g++;
        while (g > 0 && !(A[g - 1] <= v)) g--;
        return g;
    };
    auto bits = [](int lo, int hi) -> unsigned long long { return hi > lo ? ((~0ull >> (64 - (hi - lo))) << lo) : 0ull; };
    for (unsigned q = blockIdx.x * (NT / 32) + wid; q < n; q += gridDim.x * (NT / 32)) {
        const size_t gi = (size_t)b * capk + q;
        if (!keep[gi]) { if (lane == 0) valid[gi] = 0; continue; }
        cvb_keypoint kp = cache[gi];
        const EvoDev ev = T.e[kp.class_id];
        const size_t poff = (size_t)b * bstride + ev.off;
        const float *D = Ldet + poff;
        const int w = ev.w;
        float ratio = (float)(1u << kp.octave);
        // `as usize` saturates negatives to 0
        float rxf = roundf(kp.x / ratio), ryf = roundf(kp.y / ratio);
        long long x = rxf > 0.f ? (long long)rxf : 0, y = ryf > 0.f ? (long long)ryf : 0;
        float x_i = D[y * w + x], x_p = D[y * w + x + 1], x_m = D[y * w + x - 1];
        float y_p = D[(y + 1) * w + x], y_m = D[(y - 1) * w + x];
        float x_p_y_p = D[(y + 1) * w + x + 1], x_p_y_m = D[(y - 1) * w + x + 1];
        float x_m_y_p = D[(y + 1) * w + x - 1], x_m_y_m = D[(y - 1) * w + x - 1];
        float d_x = 0.5f * (x_p - x_m), d_y = 0.5f * (y_p - y_m);
        float d_xx = x_p + x_m - 2.f * x_i;
        float d_yy = y_p + y_m - 2.f * x_i;
        float d_xy = 0.25f * (x_p_y_p + x_m_y_m) - 0.25f * (x_p_y_m + x_m_y_p);
        float inv_det = 1.0f / (d_xx * d_yy - d_xy * d_xy);
        float a0 = inv_det * d_yy, a1 = inv_det * -d_xy, a2 = inv_det * -d_xy, a3 = inv_det * d_xx;
        float dst0 = -d_x * a0 + -d_y * a1;
        float dst1 = -d_x * a2 + -d_y * a3;
        if (!(fabsf(dst0) <= 1.0f && fabsf(dst1) <= 1.0f)) { if (lane == 0) valid[gi] = 0; continue; }
        kp.x = (float)x + dst0; kp.y = (float)y + dst1;
        float power = (float)(1u << ev.octave);
        kp.x = kp.x * power + 0.5f * (power - 1.f);
        kp.y = kp.y * power + 0.5f * (power - 1.f);
        kp.size *= 2.f;
        // ---- compute_main_orientation (:229-288)
        const float *PX = Lx + poff, *PY = Ly + poff;
        ratio = (float)(1 << ev.octave);
        const float s = roundf(0.5f * kp.size / ratio);
        const float xf = kp.x / ratio, yf = kp.y / ratio;
        for (int idx = lane; idx < 109; idx += 32) {
            float fy = roundf(yf + (float)OT->dj[idx] * s), fx = roundf(xf + (float)OT->di[idx] * s);
            long long iy = fy > 0.f ? (long long)fy : 0, ix = fx > 0.f ? (long long)fx : 0;
            ix = ix > ev.w - 1 ? ev.w - 1 : ix;   // the reference would panic here; never taken after the border test
            iy = iy > ev.h - 1 ? ev.h - 1 : iy;
            float gwt = OT->gw[idx];
            float rx = gwt * PX[iy * w + ix], ry = gwt * PY[iy * w + ix];
            s_r[wid][idx] = make_float2(rx, ry);
            const float ang = dlm::fast_atan2_equiv(ry, rx);
            unsigned long long m = 0ull;
            if (ang == ang) {                        // (a NaN angle is in no window: every comparison of the reference is false)
                // scale_space_extrema.rs:268-271 per window w:  (a1 < a2 && a1 < ang && ang < a2) || (a2 < a1 && ((ang > 0 && ang < a2) || (ang > a1 && ang < 2pi)))
                const int g = (int)(ang * (1.0f / 0.15f));
                const int hi = count_lt(s_a1, nwin, ang, g + 1);                       // a1[w] < ang  <=>  w < hi
                const int c2 = count_le(s_a2, nn, ang, g - 6);                         // ang < a2[w]  <=>  w >= c2        (w < nn)
                m = bits(c2, min(hi, nn));
                if (ang > 0.f) m |= bits(nn + count_le(s_a2 + nn, nwin - nn, ang, g + 1), nwin);   // ang < a2[w], wrapping windows
                if (ang < two_pi) m |= bits(nn, hi);                                   // a1[w] < ang, wrapping windows
            }
            s_m[wid][idx] = make_uint2((unsigned)m, (unsigned)(m >> 32));
        }
        __syncwarp();
        float best_val = 0.f, best_sx = 0.f, best_sy = 0.f;
        int best_w = 0x7fffffff;
        // two consecutive windows per lane in ONE pass over the samples (42 windows -> lanes 0..20); each window adds its samples
        // in sample order.  (The tables hold at most 64 windows.)
        {
            const int wa = 2 * lane, wb = wa + 1;
            const unsigned *mw = reinterpret_cast<const unsigned *>(&s_m[wid][0]) + (lane >> 4);
            const int sh = wa & 31;
            float sxa = 0.f, sya = 0.f, sxb = 0.f, syb = 0.f;
#pragma unroll 4
            for (int k = 0; k < 109; k++) {
                const unsigned mb = mw[2 * k] >> sh;
                const float2 r = s_r[wid][k];
                if (mb & 1u) { sxa += r.x; sya += r.y; }
                if (mb & 2u) { sxb += r.x; syb += r.y; }
            }
            if (wa < nwin) {
                const float va = sxa * sxa + sya * sya;
                if (va > best_val) { best_val = va; best_sx = sxa; best_sy = sya; best_w = wa; }
            }
            if (wb < nwin) {
                const float vb = sxb * sxb + syb * syb;
                if (vb > best_val) { best_val = vb; best_sx = sxb; best_sy = syb; best_w = wb; }
            }
        }
        // sequential `if val > max` == first window attaining the maximum (when > 0)
        for (int o = 16; o; o >>= 1) {
            float ov = __shfl_xor_sync(0xffffffffu, best_val, o);
            float osx = __shfl_xor_sync(0xffffffffu, best_sx, o), osy = __shfl_xor_sync(0xffffffffu, best_sy, o);
            int ow = __shfl_xor_sync(0xffffffffu, best_w, o);
            if (ov > best_val || (ov == best_val && ow < best_w)) { best_val = ov; best_sx = osx; best_sy = osy; best_w = ow; }
        }
        if (lane == 0) {
            kp.angle = best_val > 0.f ? dlm::fast_atan2_equiv(best_sy, best_sx) : 0.f;
            refined[gi] = kp;
            valid[gi] = 1;
        }
        __syncwarp();
    }
}

// ---------------------------------------------------------------------------------------------
// Sort by descending response + truncate (lib.rs:326-327) as a rank sort over the valid refined
// keypoints: rank = #{ j valid : r_j > r_i  or (r_j == r_i and j < i) }.  (The reference sort is
// unstable; ties keep their original order here, the working definition (DESIGN.md section 2).)
// k_rank_count: grid = (i-chunks, j-chunks, B) partial ranks accumulated with atomics (rank preset to 0);
// k_rank_scatter writes sorted[rank] and the surviving count.
__global__ void __launch_bounds__(NT) k_rank_count(const cvb_keypoint *__restrict__ refined,
                                                   const unsigned char *__restrict__ valid,
                                                   const unsigned *__restrict__ ncache, unsigned capk,
                                                   unsigned *__restrict__ rank) {
    __shared__ float s_r[NT];
    const int b = blockIdx.z;
    const unsigned n = ncache[b];
    const cvb_keypoint *kp = refined + (size_t)b * capk;
    const unsigned char *vl = valid + (size_t)b * capk;
    const unsigned nchunks = (n + NT - 1) / NT;
    for (unsigned ic = blockIdx.x; ic < nchunks; ic += gridDim.x)
        for (unsigned jc = blockIdx.y; jc < nchunks; jc += gridDim.y) {
            const unsigned i = ic * NT + threadIdx.x, j = jc * NT + threadIdx.x;
            __syncthreads();
            s_r[threadIdx.x] = (j < n && vl[j]) ? kp[j].response : -1.0f;   // responses are |v| >= 0
            __syncthreads();
            if (i >= n || !vl[i]) continue;
            const float ri = kp[i].response;
            const unsigned lim = min((unsigned)NT, n - jc * NT);
            unsigned cnt = 0;
            for (unsigned u = 0; u < lim; u++) {
                const float rj = s_r[u];
                if (rj > ri || (rj == ri && (jc * NT + u) < i)) cnt++;
            }
            if (cnt) atomicAdd(&rank[(size_t)b * capk + i], cnt);
        }
}

__global__ void __launch_bounds__(NT) k_rank_scatter(const cvb_keypoint *__restrict__ refined,
                                                     const unsigned char *__restrict__ valid,
                                                     const unsigned *__restrict__ ncache, unsigned capk,
                                                     const unsigned *__restrict__ rank, long long max_features,
                                                     cvb_keypoint *__restrict__ sorted, unsigned *__restrict__ nvalid) {
    const int b = blockIdx.y;
    const unsigned n = ncache[b];
    unsigned cnt = 0;
    for (unsigned i = blockIdx.x * NT + threadIdx.x; i < n; i += gridDim.x * NT) {
        if (!valid[(size_t)b * capk + i]) continue;
        cnt++;
        const unsigned r = rank[(size_t)b * capk + i];
        if (max_features < 0 || (long long)r < max_features) sorted[(size_t)b * capk + r] = refined[(size_t)b * capk + i];
    }
    for (int o = 16; o; o >>= 1) cnt += __shfl_down_sync(0xffffffffu, cnt, o);
    if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(&nvalid[b], cnt);
}

__global__ void k_clamp_count(const unsigned *__restrict__ nvalid, long long max_features, unsigned *__restrict__ nsorted, int B) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    unsigned v = nvalid[b];
    if (max_features >= 0 && (long long)v > max_features) v = (unsigned)max_features;
    nsorted[b] = v;
}

// ---------------------------------------------------------------------------------------------
// M-LDB descriptor, one warp per keypoint, one lane per grid cell (descriptors.rs:55-202).
struct DescTables {
    // 29 cells: 2x2 (step 10), 3x3 (step ceil(10*2/3)=7), 4x4 (step 5) over [-pattern, pattern)
    int ncells;
    short ci[32], cj[32], cstep[32];
    int nbits;
    int nlat;                                   // lattice points per axis: k, l in [-pattern, -pattern + nlat)
    unsigned char ba[512], bb[512], bch[512];   // bit t = values[ba][ch] > values[bb][ch]
};

constexpr int DESC_WARPS = 4;      // warps (keypoints in flight) per CTA
constexpr int DESC_MAXLAT = 21;    // lattice points per axis: k, l in [-pattern, pattern]

// Every grid of the M-LDB pattern samples the same (k, l) lattice (descriptors.rs:117-130: the sample
// position depends on k and l only), so each lattice point is gathered ONCE per keypoint by the whole
// warp (Lt, Lx, Ly and the rotated derivatives), parked in shared memory, and the per-cell sums then
// read it back in the reference's k-outer / l-inner order -- same values, same order, 2.8x fewer gathers.
// Frame b's keypoints are kps[base, base + n): base = b * stride and n = counts[b] when offs is null (the extractor's
// per-frame slots); otherwise base = offs[b] and n = offs[b + 1] - base, both clamped to `stride` entries (caller keypoints
// in CSR layout).  A keypoint with class_id >= T.n or octave >= 32 (an out-of-bounds index or a shift overflow in the
// reference) gets ok = 0 and sets *flag = 4.
__global__ void __launch_bounds__(DESC_WARPS * 32) k_descriptors(const cvb_keypoint *__restrict__ kps,
                                                    const unsigned *__restrict__ counts, const unsigned *__restrict__ offs,
                                                    unsigned stride, EvoTable T,
                                                    const float *__restrict__ Lt, const float *__restrict__ Lx,
                                                    const float *__restrict__ Ly, size_t bstride,
                                                    const DescTables *__restrict__ DT, int nch, int pattern,
                                                    unsigned char *__restrict__ desc_tmp,
                                                    unsigned char *__restrict__ ok, unsigned *flag) {
    __shared__ float s_val[DESC_WARPS][32][3];
    __shared__ float s_lat[DESC_WARPS][3][DESC_MAXLAT * DESC_MAXLAT];
    const int b = blockIdx.y;
    size_t base;
    unsigned n;
    if (offs) {
        const unsigned lo = min(offs[b], stride), hi = min(max(offs[b + 1], lo), stride);
        base = lo; n = hi - lo;
    } else {
        base = (size_t)b * stride; n = counts[b];
    }
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int nl = DT->nlat;                   // lattice size per axis (<= DESC_MAXLAT)
    for (unsigned q = blockIdx.x * DESC_WARPS + wid; q < n; q += gridDim.x * DESC_WARPS) {
        const size_t gi = base + q;
        const cvb_keypoint kp = kps[gi];
        if (kp.class_id >= (unsigned)T.n || kp.octave >= 32u) {
            if (lane == 0) { ok[gi] = 0; *flag = 4u; }
            continue;
        }
        const EvoDev ev = T.e[kp.class_id];
        const size_t poff = (size_t)b * bstride + ev.off;
        const float *PT = Lt + poff, *PX = Lx + poff, *PY = Ly + poff;
        const int W = ev.w, H = ev.h;
        const float ratio = (float)(1u << kp.octave);
        const float scale = roundf(0.5f * kp.size / ratio);
        const float xf = kp.x / ratio, yf = kp.y / ratio;
        const float co = dlm::cosf_glibc(kp.angle), si = dlm::sinf_glibc(kp.angle);
        bool oob = false;
        const bool kmajor = fabsf(co) >= fabsf(si);
        // lattice gathers in batches: all addresses, then all loads, then the arithmetic (a rolled loop would pay one L2
        // round trip per iteration)
        constexpr int GB = 7;
        for (int p0 = lane; p0 < nl * nl; p0 += 32 * GB) {
            size_t g[GB];
            int slot[GB];
            float vt[GB], vx[GB], vy[GB];
#pragma unroll
            for (int u = 0; u < GB; u++) {
                const int p = p0 + 32 * u;
                g[u] = (size_t)-1;
                if (p < nl * nl) {
                    // consecutive lanes take consecutive lattice steps along the axis that advances mostly in x for this keypoint's
                    // rotation (k when |cos| >= |sin|, else l), so a warp-wide gather touches a few 32-byte sectors per image row
                    // instead of one per lane; every point still lands in its own slot ki * nl + lj
                    const int qa = p / nl, qb = p - qa * nl;
                    const int ki = kmajor ? qb : qa, lj = kmajor ? qa : qb;
                    const float kf = (float)(ki - pattern), lf = (float)(lj - pattern);
                    const float sample_y = yf + (lf * co * scale + kf * si * scale);
                    const float sample_x = xf + (-lf * si * scale + kf * co * scale);
                    // `f32::round(v) as isize` (descriptors.rs:129-130) saturates, and maps NaN to 0
                    float ry_ = roundf(sample_y), rx_ = roundf(sample_x);
                    if (ry_ != ry_) ry_ = 0.f;
                    if (rx_ != rx_) rx_ = 0.f;
                    if (!(rx_ >= 0.f && rx_ < (float)W) || !(ry_ >= 0.f && ry_ < (float)H)) oob = true;
                    else g[u] = (size_t)(int)ry_ * W + (int)rx_;
                    slot[u] = ki * nl + lj;
                }
            }
#pragma unroll
            for (int u = 0; u < GB; u++) {
                vt[u] = vx[u] = vy[u] = 0.f;
                if (g[u] != (size_t)-1) {
                    vt[u] = PT[g[u]];
                    if (nch > 1) { vx[u] = PX[g[u]]; vy[u] = PY[g[u]]; }
                }
            }
#pragma unroll
            for (int u = 0; u < GB; u++) {
                if (g[u] == (size_t)-1) continue;
                const int p = slot[u];
                s_lat[wid][0][p] = vt[u];
                if (nch > 1) {
                    const float rx = vx[u], ry = vy[u];
                    if (nch == 2) s_lat[wid][1][p] = sqrtf(rx * rx + ry * ry);
                    else {
                        s_lat[wid][2][p] = rx * co + ry * si;      // rry
                        s_lat[wid][1][p] = -rx * si + ry * co;     // rrx
                    }
                }
            }
        }
        // every lattice point belongs to a cell of the widest grid (it tiles [-pattern, -pattern+nlat) fully), so
        // "any sample out of bounds" (descriptors.rs:131-140) == "any lattice point out of bounds"
        const bool any_oob = __any_sync(0xffffffffu, oob);
        if (any_oob) {
            if (lane == 0) ok[gi] = 0;
            __syncwarp();
            continue;
        }
        __syncwarp();
        if (lane < DT->ncells) {
            const int i0 = DT->ci[lane] + pattern, j0 = DT->cj[lane] + pattern, step = DT->cstep[lane];
            float di = 0.f, dx = 0.f, dy = 0.f;
            for (int k = i0; k < i0 + step; k++) {
                const float *r0 = &s_lat[wid][0][k * nl + j0], *r1 = &s_lat[wid][1][k * nl + j0], *r2 = &s_lat[wid][2][k * nl + j0];
                for (int l = 0; l < step; l++) {
                    di += r0[l];
                    if (nch > 1) dx += r1[l];
                    if (nch > 2) dy += r2[l];
                }
            }
            const float ns = (float)(step * step);
            di /= ns; dx /= ns; dy /= ns;
            s_val[wid][lane][0] = di; s_val[wid][lane][1] = dx; s_val[wid][lane][2] = dy;
        }
        __syncwarp();
        // 512 output bits, 16 per lane
        unsigned bits = 0;
        for (int t = 0; t < 16; t++) {
            int bit = lane * 16 + t;
            if (bit < DT->nbits) {
                float a = s_val[wid][DT->ba[bit]][DT->bch[bit]], c = s_val[wid][DT->bb[bit]][DT->bch[bit]];
                bits |= (a > c ? 1u : 0u) << t;
            }
        }
        ((unsigned short *)(desc_tmp + gi * 64))[lane] = (unsigned short)bits;
        if (lane == 0) ok[gi] = 1;
        __syncwarp();
    }
}

// Ordered compaction of the surviving keypoints/descriptors into the caller's output arrays.
__global__ void __launch_bounds__(1024) k_compact_final(const cvb_keypoint *__restrict__ sorted,
                                                        const unsigned char *__restrict__ desc_tmp,
                                                        const unsigned char *__restrict__ ok,
                                                        const unsigned *__restrict__ nsorted, unsigned capk,
                                                        cvb_keypoint *__restrict__ kp_out,
                                                        unsigned char *__restrict__ desc_out, unsigned cap_out,
                                                        unsigned *__restrict__ n_out, unsigned *overflow) {
    __shared__ unsigned s_warp[32];
    __shared__ unsigned s_carry;
    const int b = blockIdx.x;
    const unsigned n = nsorted[b];
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (unsigned base = 0; base < n; base += 1024) {
        unsigned i = base + threadIdx.x;
        unsigned v = (i < n && ok[(size_t)b * capk + i]) ? 1u : 0u, x = v;
        for (int o = 1; o < 32; o <<= 1) { unsigned t = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += t; }
        if (lane == 31) s_warp[wid] = x;
        __syncthreads();
        if (wid == 0) {
            unsigned y = s_warp[lane], z = y;
            for (int o = 1; o < 32; o <<= 1) { unsigned t = __shfl_up_sync(0xffffffffu, z, o); if (lane >= o) z += t; }
            s_warp[lane] = z - y;
        }
        __syncthreads();
        unsigned pos = s_carry + s_warp[wid] + x - v;
        if (v) {
            if (pos < cap_out) {
                kp_out[(size_t)b * cap_out + pos] = sorted[(size_t)b * capk + i];
                const uint4 *s = (const uint4 *)(desc_tmp + ((size_t)b * capk + i) * 64);
                uint4 *d = (uint4 *)(desc_out + ((size_t)b * cap_out + pos) * 64);
                d[0] = s[0]; d[1] = s[1]; d[2] = s[2]; d[3] = s[3];
            } else *overflow = 3u;
        }
        __syncthreads();
        if (threadIdx.x == 1023) s_carry = pos + v;
        __syncthreads();
    }
    // the count never exceeds the capacity (the overflow flag reports the truncation): downstream kernels index by it
    if (threadIdx.x == 0) n_out[b] = min(s_carry, cap_out);
}

// Ordered compaction of caller-visible stage results, one block per frame.  Input entries in_base(b) + i for i < n(b) with
// keep[...] set go, in input order, to out[out_base(b) + pos] (with their 64-byte descriptors when desc_in is non-null).
//   find:     in_base = b * in_stride, n = counts[b]; out_base = b * cap; entries past cap are dropped and set *overflow = 3
//   describe: in_base = out_base = offs[b] and n = offs[b + 1] - offs[b], clamped to in_stride entries (never past the input)
// n_out[b] = the number kept (at most cap); need (optional) = the number that passed, capacity aside.
struct CompactArgs {
    const cvb_keypoint *kp_in;
    const unsigned char *desc_in, *keep;
    const unsigned *counts, *offs;
    unsigned in_stride, cap;
    cvb_keypoint *kp_out;
    unsigned char *desc_out;
    unsigned *n_out, *need, *overflow;
};
__global__ void __launch_bounds__(1024) k_compact_stage(CompactArgs A) {
    __shared__ unsigned s_warp[32];
    __shared__ unsigned s_carry;
    const int b = blockIdx.x;
    size_t in_base, out_base;
    unsigned n, cap;
    if (A.offs) {
        const unsigned lo = min(A.offs[b], A.in_stride), hi = min(max(A.offs[b + 1], lo), A.in_stride);
        in_base = out_base = lo; n = cap = hi - lo;
    } else {
        in_base = (size_t)b * A.in_stride; n = A.counts[b]; out_base = (size_t)b * A.cap; cap = A.cap;
    }
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (unsigned base = 0; base < n; base += 1024) {
        const unsigned i = base + threadIdx.x;
        const unsigned v = (i < n && A.keep[in_base + i]) ? 1u : 0u;
        unsigned x = v;
        for (int o = 1; o < 32; o <<= 1) { unsigned t = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += t; }
        if (lane == 31) s_warp[wid] = x;
        __syncthreads();
        if (wid == 0) {
            unsigned y = s_warp[lane], z = y;
            for (int o = 1; o < 32; o <<= 1) { unsigned t = __shfl_up_sync(0xffffffffu, z, o); if (lane >= o) z += t; }
            s_warp[lane] = z - y;
        }
        __syncthreads();
        const unsigned pos = s_carry + s_warp[wid] + x - v;
        if (v) {
            if (pos < cap) {
                A.kp_out[out_base + pos] = A.kp_in[in_base + i];
                if (A.desc_in) {
                    const uint4 *s = (const uint4 *)(A.desc_in + (in_base + i) * 64);
                    uint4 *d = (uint4 *)(A.desc_out + (out_base + pos) * 64);
                    d[0] = s[0]; d[1] = s[1]; d[2] = s[2]; d[3] = s[3];
                }
            } else *A.overflow = 3u;
        }
        __syncthreads();
        if (threadIdx.x == 1023) s_carry = pos + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        A.n_out[b] = min(s_carry, cap);
        if (A.need) A.need[b] = s_carry;
    }
}

}  // namespace akz
