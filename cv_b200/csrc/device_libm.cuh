// cv_b200/csrc/device_libm.cuh -- bit-exact device versions of the host libm routines the
// reference reaches through Rust std (f32::sin / cos / atan2 -> glibc 2.39 sinf/cosf/atan2f on
// x86-64 linux-gnu): akaze/src/descriptors.rs:70-71, akaze/src/scale_space_extrema.rs:242.
//
// CUDA's own sinf/cosf/atan2f are <=2 ulp but not bit-identical to glibc, and the angle feeds
// round(sample_x) and hence descriptor bits, so the glibc algorithms are restated here:
//   sinf/cosf     : Arm-optimized-routines double-precision polynomial, in the contraction pattern
//                   of glibc's -mfma ifunc variant (explicit fma()).
//   atanf/atan2f  : fdlibm single-precision code, no contraction.
// This translation unit MUST be compiled with -fmad=false so that no other multiply-add is fused.
// sinf_glibc / cosf_glibc are __host__ __device__ so that the same source can be checked against the host libm on a CPU
// (host code must then be compiled with -ffp-contract=off).
#pragma once
#include <stdint.h>
#include <string.h>

namespace dlm {

__host__ __device__ __forceinline__ uint32_t f32_bits(float x) {
#ifdef __CUDA_ARCH__
    return __float_as_uint(x);
#else
    uint32_t u;
    memcpy(&u, &x, 4);
    return u;
#endif
}

__host__ __device__ __forceinline__ float poly_sincos(double x, double x2, bool neg_cos, int n) {
    const double C0 = 0x1p0, C1 = -0x1.ffffffd0c621cp-2, C2 = 0x1.55553e1068f19p-5, C3 = -0x1.6c087e89a359dp-10,
                 C4 = 0x1.99343027bf8c3p-16;
    const double S1 = -0x1.555545995a603p-3, S2 = 0x1.1107605230bc4p-7, S3 = -0x1.994eb3774cf24p-13;
    if ((n & 1) == 0) {
        double x3 = x * x2;
        double s1 = fma(x2, S3, S2);
        double x7 = x3 * x2;
        double s = fma(x3, S1, x);
        return (float)fma(x7, s1, s);
    } else {
        double sg = neg_cos ? -1.0 : 1.0;
        double x4 = x2 * x2;
        double c2 = fma(x2, sg * C4, sg * C3);
        double c1 = fma(x2, sg * C1, sg * C0);
        double x6 = x4 * x2;
        double c = fma(x4, sg * C2, c1);
        return (float)fma(x6, c2, c);
    }
}

__host__ __device__ __forceinline__ uint32_t abstop12(float x) { return (f32_bits(x) >> 20) & 0x7ff; }

__host__ __device__ __forceinline__ double reduce_fast(double x, int *np) {
    const double HPI_INV = 0x1.45F306DC9C883p+23, HPI = 0x1.921FB54442D18p0;
    double r = x * HPI_INV;
    int n = ((int32_t)r + 0x800000) >> 24;
    *np = n;
    return fma(-(double)n, HPI, x);
}

// 4/pi in 8-bit steps: entry i holds bits 8i .. 8i + 31 of the fraction, so every exponent has an aligned word.  Constant memory
// on the device (a local array would be indexed from the stack), a plain table on the host.
#define DLM_INV_PIO4 {0xa2,       0xa2f9,     0xa2f983,   0xa2f9836e, 0xf9836e4e, 0x836e4e44, 0x6e4e4415, 0x4e441529, \
                      0x441529fc, 0x1529fc27, 0x29fc2757, 0xfc2757d1, 0x2757d1f5, 0x57d1f534, 0xd1f534dd, 0xf534ddc0, \
                      0x34ddc0db, 0xddc0db62, 0xc0db6295, 0xdb629599, 0x6295993c, 0x95993c43, 0x993c4390, 0x3c439041}
static __constant__ uint32_t inv_pio4_dev[24] = DLM_INV_PIO4;
static const uint32_t inv_pio4_host[24] = DLM_INV_PIO4;
#undef DLM_INV_PIO4

// glibc's reduce_large (sysdeps/ieee754/flt-32/s_sincosf.h) for 120 <= |y| < inf: x * 4/pi in 62-bit fixed point from the 24-bit
// mantissa times 96 bits of 4/pi chosen by the exponent; returns the remainder in [-pi/4, pi/4] and the quadrant in *np.
__host__ __device__ __forceinline__ double reduce_large(uint32_t xi, int *np) {
#ifdef __CUDA_ARCH__
    const uint32_t *arr = &inv_pio4_dev[(xi >> 26) & 15];
#else
    const uint32_t *arr = &inv_pio4_host[(xi >> 26) & 15];
#endif
    const double PI63 = 0x1.921FB54442D18p-62;   // pi * 2^-64
    const int shift = (xi >> 23) & 7;
    xi = (xi & 0xffffff) | 0x800000;
    xi <<= shift;
    uint64_t res0 = (uint32_t)(xi * arr[0]);
    const uint64_t res1 = (uint64_t)xi * arr[4];
    const uint64_t res2 = (uint64_t)xi * arr[8];
    res0 = (res2 >> 32) | (res0 << 32);
    res0 += res1;
    const uint64_t n = (res0 + (1ULL << 61)) >> 62;
    res0 -= n << 62;
    const double x = (double)(int64_t)res0;
    *np = (int)n;
    return x * PI63;
}

// glibc 2.39 sinf (s_sinf.c) over the whole float range: |y| < 120 reduces with reduce_fast, finite |y| >= 120 with reduce_large
// (the input's sign folded into the quadrant), and +-inf / NaN give NaN
__host__ __device__ __forceinline__ float sinf_glibc(float y) {
    double x = (double)y;
    if (abstop12(y) < abstop12(0x1.921FB6p-1f)) {
        if (abstop12(y) < abstop12(0x1p-12f)) return y;
        return poly_sincos(x, x * x, false, 0);
    }
    int n;
    if (abstop12(y) < abstop12(120.0f)) {
        x = reduce_fast(x, &n);
        double s = ((n & 3) == 1 || (n & 3) == 2) ? -1.0 : 1.0;
        return poly_sincos(x * s, x * x, (n & 2) != 0, n);
    }
    if (abstop12(y) < abstop12(__builtin_huge_valf())) {
        const uint32_t xi = f32_bits(y);
        x = reduce_large(xi, &n);
        const int q = n + (int)(xi >> 31);
        double s = ((q & 3) == 1 || (q & 3) == 2) ? -1.0 : 1.0;
        return poly_sincos(x * s, x * x, (q & 2) != 0, n);
    }
    return (y - y) / (y - y);
}

__host__ __device__ __forceinline__ float cosf_glibc(float y) {
    double x = (double)y;
    if (abstop12(y) < abstop12(0x1.921FB6p-1f)) {
        if (abstop12(y) < abstop12(0x1p-12f)) return 1.0f;
        return poly_sincos(x, x * x, false, 1);
    }
    int n;
    if (abstop12(y) < abstop12(120.0f)) {
        x = reduce_fast(x, &n);
        double s = ((n & 3) == 1 || (n & 3) == 2) ? -1.0 : 1.0;
        return poly_sincos(x * s, x * x, (n & 2) != 0, n ^ 1);
    }
    if (abstop12(y) < abstop12(__builtin_huge_valf())) {
        const uint32_t xi = f32_bits(y);
        x = reduce_large(xi, &n);
        const int q = n + (int)(xi >> 31);
        double s = ((q & 3) == 1 || (q & 3) == 2) ? -1.0 : 1.0;
        return poly_sincos(x * s, x * x, (q & 2) != 0, n ^ 1);
    }
    return (y - y) / (y - y);
}

__device__ __forceinline__ float atanf_glibc(float x) {
    const float atanhi[4] = {4.6364760399e-01f, 7.8539812565e-01f, 9.8279368877e-01f, 1.5707962513e+00f};
    const float atanlo[4] = {5.0121582440e-09f, 3.7748947079e-08f, 3.4473217170e-08f, 7.5497894159e-08f};
    const float aT0 = 3.3333334327e-01f, aT1 = -2.0000000298e-01f, aT2 = 1.4285714924e-01f, aT3 = -1.1111110449e-01f,
                aT4 = 9.0908870101e-02f, aT5 = -7.6918758452e-02f, aT6 = 6.6610731184e-02f, aT7 = -5.8335702866e-02f,
                aT8 = 4.9768779427e-02f, aT9 = -3.6531571299e-02f, aT10 = 1.6285819933e-02f;
    int32_t hx = (int32_t)__float_as_uint(x), ix = hx & 0x7fffffff, id;
    if (ix >= 0x4c000000) {
        if (ix > 0x7f800000) return x + x;
        if (hx > 0) return atanhi[3] + atanlo[3];
        return -atanhi[3] - atanlo[3];
    }
    if (ix < 0x3ee00000) {
        if (ix < 0x31000000) return x;
        id = -1;
    } else {
        x = fabsf(x);
        if (ix < 0x3f980000) {
            if (ix < 0x3f300000) { id = 0; x = (2.0f * x - 1.0f) / (2.0f + x); }
            else { id = 1; x = (x - 1.0f) / (x + 1.0f); }
        } else {
            if (ix < 0x401c0000) { id = 2; x = (x - 1.5f) / (1.0f + 1.5f * x); }
            else { id = 3; x = -1.0f / x; }
        }
    }
    float z = x * x;
    float w = z * z;
    float s1 = z * (aT0 + w * (aT2 + w * (aT4 + w * (aT6 + w * (aT8 + w * aT10)))));
    float s2 = w * (aT1 + w * (aT3 + w * (aT5 + w * (aT7 + w * aT9))));
    if (id < 0) return x - x * (s1 + s2);
    float hi = id == 0 ? atanhi[0] : id == 1 ? atanhi[1] : id == 2 ? atanhi[2] : atanhi[3];
    float lo = id == 0 ? atanlo[0] : id == 1 ? atanlo[1] : id == 2 ? atanlo[2] : atanlo[3];
    z = hi - ((x * (s1 + s2) - lo) - x);
    return (hx < 0) ? -z : z;
}

__device__ __forceinline__ float atan2f_glibc(float y, float x) {
    const float tiny = 1.0e-30f, pi_o_2 = 1.5707963705e+00f, pi_o_4 = 7.8539818525e-01f, pi = 3.1415927410e+00f,
                pi_lo = -8.7422776573e-08f;
    float z;
    int32_t hx = (int32_t)__float_as_uint(x), hy = (int32_t)__float_as_uint(y);
    int32_t ix = hx & 0x7fffffff, iy = hy & 0x7fffffff;
    if (ix > 0x7f800000 || iy > 0x7f800000) return x + y;
    if (hx == 0x3f800000) return atanf_glibc(y);
    int m = ((hy >> 31) & 1) | ((hx >> 30) & 2);
    if (iy == 0) {
        if (m < 2) return y;
        return m == 2 ? pi + tiny : -pi - tiny;
    }
    if (ix == 0) return (hy < 0) ? -pi_o_2 - tiny : pi_o_2 + tiny;
    if (ix == 0x7f800000) {
        if (iy == 0x7f800000) {
            switch (m) {
            case 0: return pi_o_4 + tiny;
            case 1: return -pi_o_4 - tiny;
            case 2: return 3.0f * pi_o_4 + tiny;
            default: return -3.0f * pi_o_4 - tiny;
            }
        } else {
            switch (m) {
            case 0: return 0.0f;
            case 1: return -0.0f;
            case 2: return pi + tiny;
            default: return -pi - tiny;
            }
        }
    }
    if (iy == 0x7f800000) return (hy < 0) ? -pi_o_2 - tiny : pi_o_2 + tiny;
    int k = (iy - ix) >> 23;
    if (k > 60) z = pi_o_2 + 0.5f * pi_lo;
    else if (hx < 0 && k < -60) z = 0.0f;
    else z = atanf_glibc(fabsf(y / x));
    switch (m) {
    case 0: return z;
    case 1: return __uint_as_float(__float_as_uint(z) ^ 0x80000000u);
    case 2: return pi - (z - pi_lo);
    default: return (z - pi_lo) - pi;
    }
}

// scale_space_extrema.rs:242  (y.atan2(x) + 2.*PI).rem_euclid(2.*PI); fmodf is exact on both sides.
__device__ __forceinline__ float fast_atan2_equiv(float y, float x) {
    const float two_pi = 2.0f * 3.14159265358979323846f;
    float v = atan2f_glibc(y, x) + two_pi;
    float r = fmodf(v, two_pi);
    if (r < 0.0f) r = r + fabsf(two_pi);
    return r;
}

}  // namespace dlm
