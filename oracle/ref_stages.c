/* oracle/ref_stages.c -- TEST INFRASTRUCTURE (CPU oracle), not product code.
 *
 * The oracle of include/cvb200_stages.h's describe call: akaze's extract_descriptors (akaze/src/descriptors.rs:16-202) at caller
 * keypoints, on the planes (Lt, multiscale Lx / Ly) of a scale space the extractor oracle (ref_akaze.c) built.  It differs from
 * ref_akaze.c's descriptor code exactly where caller keypoints reach cases the detector's own keypoints never do:
 *  - sin / cos over the whole float range: glibc 2.39 s_sinf.c / s_cosf.c take reduce_large (s_sincosf.h, 4/pi bit table) for
 *    120 <= |y| < inf and return NaN for +-inf / NaN; below 120 this is ref_libm.h's rl_sinf / rl_cosf unchanged;
 *  - `f32::round(v) as isize` (descriptors.rs:129-130) is a saturating cast: NaN becomes 0, +-inf and huge values saturate (so
 *    they stay out of bounds);
 *  - a keypoint with class_id >= the number of evolutions or octave >= 32 panics in the reference: the call returns -1 - index.
 * Built by oracle/stages.mk into _build/libcvb_oracle_stages.so; bound by oracle/pyoracle_stages.py. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "ref_akaze.h"
#include "ref_libm.h"

static const uint32_t rs_inv_pio4[24] = {
    0xa2,       0xa2f9,     0xa2f983,   0xa2f9836e, 0xf9836e4e, 0x836e4e44, 0x6e4e4415, 0x4e441529,
    0x441529fc, 0x1529fc27, 0x29fc2757, 0xfc2757d1, 0x2757d1f5, 0x57d1f534, 0xd1f534dd, 0xf534ddc0,
    0x34ddc0db, 0xddc0db62, 0xc0db6295, 0xdb629599, 0x6295993c, 0x95993c43, 0x993c4390, 0x3c439041};

/* s_sincosf.h reduce_large: |x| * 4/pi as a 2.62 fixed-point number from the 24-bit mantissa and 96 table bits */
static double rs_reduce_large(uint32_t xi, int *np) {
    const uint32_t *arr = &rs_inv_pio4[(xi >> 26) & 15];
    int shift = (xi >> 23) & 7;
    uint64_t n, res0, res1, res2;
    xi = (xi & 0xffffff) | 0x800000;
    xi <<= shift;
    res0 = (uint32_t)(xi * arr[0]);
    res1 = (uint64_t)xi * arr[4];
    res2 = (uint64_t)xi * arr[8];
    res0 = (res2 >> 32) | (res0 << 32);
    res0 += res1;
    n = (res0 + (1ULL << 61)) >> 62;
    res0 -= n << 62;
    *np = (int)n;
    return (double)(int64_t)res0 * 0x1.921FB54442D18p-62;
}

static float rs_sincos_large(float y, int cos) {
    if (rl_abstop12(y) >= rl_abstop12(INFINITY)) return (y - y) / (y - y);   /* __math_invalidf */
    uint32_t xi = rl_asuint(y);
    int n;
    double x = rs_reduce_large(xi, &n);
    int q = n + (int)(xi >> 31);
    double s = ((q & 3) == 1 || (q & 3) == 2) ? -1.0 : 1.0;
    return rl_sinf_poly(x * s, x * x, (q & 2) != 0, cos ? n ^ 1 : n);
}

float ref_full_sinf(float y) { return rl_abstop12(y) < rl_abstop12(120.0f) ? rl_sinf(y) : rs_sincos_large(y, 0); }
float ref_full_cosf(float y) { return rl_abstop12(y) < rl_abstop12(120.0f) ? rl_cosf(y) : rs_sincos_large(y, 1); }

/* Rust's `f32 as isize` after round(): NaN -> 0, saturating at the ends (a long holds isize on x86-64) */
static long rs_as_isize(float v) {
    if (v != v) return 0;
    if (v >= 9.2233720368547758e18f) return INT64_MAX;
    if (v <= -9.2233720368547758e18f) return INT64_MIN;
    return (long)v;
}

typedef struct { const float *Lt, *Lx, *Ly; int w, h; } rs_level;

/* descriptors.rs:102-177 mldb_fill_values; 1 when a sample falls outside the level */
static int rs_fill_values(const rs_level *e, int nch, int pattern, float *values, int sample_step, float xf, float yf, float co,
                          float si, float scale) {
    int vp = 0;
    for (int i = -pattern; i < pattern; i += sample_step)
        for (int j = -pattern; j < pattern; j += sample_step) {
            float di = 0.f, dx = 0.f, dy = 0.f;
            long ns = 0;
            for (int k = i; k < i + sample_step; k++)
                for (int l = j; l < j + sample_step; l++) {
                    float lf = (float)l, kf = (float)k;
                    float sample_y = yf + (lf * co * scale + kf * si * scale);
                    float sample_x = xf + (-lf * si * scale + kf * co * scale);
                    long y1 = rs_as_isize(roundf(sample_y)), x1 = rs_as_isize(roundf(sample_x));
                    if (x1 < 0 || y1 < 0 || x1 >= e->w || y1 >= e->h) return 1;
                    float ri = e->Lt[y1 * e->w + x1];
                    di += ri;
                    if (nch > 1) {
                        float rx = e->Lx[y1 * e->w + x1], ry = e->Ly[y1 * e->w + x1];
                        if (nch == 2) dx += sqrtf(rx * rx + ry * ry);
                        else {
                            float rry = rx * co + ry * si;
                            float rrx = -rx * si + ry * co;
                            dx += rrx; dy += rry;
                        }
                    }
                    ns++;
                }
            di /= (float)ns; dx /= (float)ns; dy /= (float)ns;
            values[vp] = di;
            if (nch > 1) values[vp + 1] = dx;
            if (nch > 2) values[vp + 2] = dy;
            vp += nch;
        }
    return 0;
}

/* descriptors.rs:55-98 get_mldb_descriptor + :181-202 mldb_binary_comparisons; 1 when dropped */
static int rs_descriptor(const rs_level *levels, int nch, int pattern, const ref_keypoint *kp, uint8_t *desc) {
    float values[16 * 3];
    memset(desc, 0, 64);
    memset(values, 0, sizeof(values));
    const float size_mult[3] = {1.0f, 2.0f / 3.0f, 1.0f / 2.0f};
    float ratio = (float)(1u << kp->octave);
    float scale = roundf(0.5f * kp->size / ratio);
    float xf = kp->x / ratio, yf = kp->y / ratio;
    float co = ref_full_cosf(kp->angle), si = ref_full_sinf(kp->angle);
    int dpos = 0;
    for (int lvl = 0; lvl < 3; lvl++) {
        int count = (lvl + 2) * (lvl + 2);
        int sample_size = (int)ceilf((float)pattern * size_mult[lvl]);
        if (rs_fill_values(&levels[kp->class_id], nch, pattern, values, sample_size, xf, yf, co, si, scale)) return 1;
        for (int pos = 0; pos < nch; pos++)
            for (int i = 0; i < count; i++) {
                float iv = values[nch * i + pos];
                for (int j = i + 1; j < count; j++) {
                    uint8_t res = iv > values[nch * j + pos] ? 1 : 0;
                    desc[dpos >> 3] |= (uint8_t)(res << (dpos & 7));
                    dpos++;
                }
            }
    }
    return 0;
}

/* descriptors.rs:16-45 extract_descriptors over E levels (Lt[i], Lx[i], Ly[i] of w[i] x h[i] floats): the kept keypoints in input
 * order to kp_out, their descriptors to desc_out, the count to *n_out.  Returns 0, or -1 - i for the first invalid keypoint i. */
int ref_describe(const float *const *Lt, const float *const *Lx, const float *const *Ly, const int *w, const int *h, int E, int nch,
                 int pattern, const ref_keypoint *kps, int n, ref_keypoint *kp_out, uint8_t *desc_out, int *n_out) {
    *n_out = 0;
    for (int i = 0; i < n; i++)
        if (kps[i].class_id >= (uint32_t)E || kps[i].octave >= 32) return -1 - i;
    rs_level *levels = (rs_level *)malloc(sizeof(rs_level) * (size_t)(E > 0 ? E : 1));
    for (int i = 0; i < E; i++) { levels[i].Lt = Lt[i]; levels[i].Lx = Lx[i]; levels[i].Ly = Ly[i]; levels[i].w = w[i]; levels[i].h = h[i]; }
    int m = 0;
    for (int i = 0; i < n; i++)
        if (!rs_descriptor(levels, nch, pattern, &kps[i], desc_out + (size_t)m * 64)) kp_out[m++] = kps[i];
    free(levels);
    *n_out = m;
    return 0;
}
