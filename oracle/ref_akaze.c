/* oracle/ref_akaze.c -- TEST INFRASTRUCTURE: CPU restatement of rust-cv `akaze` 0.7.0.
 *
 * This is the parity oracle (and the "port" CPU baseline) for the AKAZE extractor.  It is
 * NOT product code: only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs may load it.  Every function cites the reference lines it follows
 * (paths relative to the reference's akaze/src).
 *
 * Pinning: tests/test_oracle_akaze.py checks this file against the reference's own goldens
 * (akaze/tests/estimate_pose.rs:41-42,59 -> 399 / 343 descriptors, 11 Lowe matches;
 * akaze/src/image.rs:395-412 Gaussian kernel known answer).  Those goldens pin the algorithm
 * but not the f32 summation order of `wide::f32x4::reduce_add` (SURVEY.md Appendix A);
 * REF_REDUCE_ORDER selects it (default 0 = SSE2 path (l0+l2)+(l1+l3)).
 *
 * Build: gcc -O2 -ffp-contract=off (no -ffast-math): every f32 op rounds exactly once,
 * multiply-add is NOT fused (wide 0.7 `mul_add` without target_feature=fma is (a*b)+c).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <stdio.h>
#include "ref_libm.h"
#include "ref_akaze.h"

#ifndef REF_REDUCE_ORDER
#define REF_REDUCE_ORDER 0
#endif

/* ---------------------------------------------------------------- images */
typedef struct { int w, h; float *d; } img_t;

static img_t img_new(int w, int h) {
    img_t m; m.w = w; m.h = h;
    m.d = (float *)calloc((size_t)w * h > 0 ? (size_t)w * h : 1, sizeof(float));
    return m;
}
static void img_free(img_t *m) { free(m->d); m->d = NULL; m->w = m->h = 0; }
static img_t img_clone(const img_t *s) {
    img_t m = img_new(s->w, s->h);
    memcpy(m.d, s->d, (size_t)s->w * s->h * sizeof(float));
    return m;
}

/* wide::f32x4::reduce_add (external crate wide 0.7; call sites image.rs:247,325). */
static inline float reduce_add4(const float l[4]) {
#if REF_REDUCE_ORDER == 0
    return (l[0] + l[2]) + (l[1] + l[3]);
#elif REF_REDUCE_ORDER == 1
    return (l[0] + l[1]) + (l[2] + l[3]);
#else
    return ((l[0] + l[1]) + l[2]) + l[3];
#endif
}

/* image.rs:202-251 horizontal_filter: correlation (no flip), replicate border, taps chunked
 * by 4 into f32x4 lanes; lane j&3 accumulates taps j, j+4, ... as (w*k)+acc from 0.
 * The zero-padded kernel tail multiplies finite window values by 0.0 and adds +-0 to an
 * accumulator that is never -0, i.e. it is a no-op and is skipped here. */
void ref_horizontal_filter(const float *in, int w, int h, const float *k, int ks, float *out) {
    int half = ks / 2;
    for (int y = 0; y < h; y++) {
        const float *r = in + (size_t)y * w;
        float *o = out + (size_t)y * w;
        for (int x = 0; x < w; x++) {
            float l[4] = {0.f, 0.f, 0.f, 0.f};
            for (int j = 0; j < ks; j++) {
                int xx = x + j - half;
                xx = xx < 0 ? 0 : (xx > w - 1 ? w - 1 : xx);
                l[j & 3] = r[xx] * k[j] + l[j & 3];
            }
            o[x] = reduce_add4(l);
        }
    }
}

/* image.rs:253-331 vertical_filter (the 16-column scratch is a cache trick, no numeric effect). */
void ref_vertical_filter(const float *in, int w, int h, const float *k, int ks, float *out) {
    int half = ks / 2;
    for (int y = 0; y < h; y++) {
        float *o = out + (size_t)y * w;
        for (int x = 0; x < w; x++) {
            float l[4] = {0.f, 0.f, 0.f, 0.f};
            for (int j = 0; j < ks; j++) {
                int yy = y + j - half;
                yy = yy < 0 ? 0 : (yy > h - 1 ? h - 1 : yy);
                l[j & 3] = in[(size_t)yy * w + x] * k[j] + l[j & 3];
            }
            o[x] = reduce_add4(l);
        }
    }
}

/* image.rs:333-340 separable_filter: H then V, each into a fresh image. */
static img_t separable_filter(const img_t *s, const float *hk, int hks, const float *vk, int vks) {
    img_t t = img_new(s->w, s->h), o = img_new(s->w, s->h);
    ref_horizontal_filter(s->d, s->w, s->h, hk, hks, t.d);
    ref_vertical_filter(t.d, s->w, s->h, vk, vks, o.d);
    img_free(&t);
    return o;
}

/* image.rs:349-374 gaussian / gaussian_kernel (f32 throughout; expf is the host libm's, as
 * Rust's f32::exp is on linux-gnu). */
void ref_gaussian_kernel(float r, int ks, float *out) {
    int half = ks / 2;
    float sum = 0.f;
    for (int i = -half; i <= half; i++) {
        float x = (float)i;
        float val = (1.0f / (sqrtf(2.0f * 3.14159265358979323846f) * r)) * expf(-(x * x) / (2.0f * (r * r)));
        out[i + half] = val;
        sum += val;
    }
    for (int i = 0; i < ks; i++) out[i] /= sum;
}

/* image.rs:383-389 gaussian_blur */
static img_t gaussian_blur(const img_t *s, float r) {
    int radius = (int)ceilf(2.0f * r);
    int ks = radius * 2 + 1;
    float k[64];
    ref_gaussian_kernel(r, ks, k);
    return separable_filter(s, k, ks, k, ks);
}

/* image.rs:154-199 half_size.  ndarray `window.sum()` on a 2x2 strided view folds row by row:
 * (a00+a01)+(a10+a11) (ndarray 0.15 numeric_util::unrolled_fold per contiguous row). */
void ref_half_size(const float *in, int w, int h, float *out) {
    int hw = w / 2, hh = h / 2;
    for (int y = 0; y < hh; y++)
        for (int x = 0; x < hw; x++) {
            const float *p = in + (size_t)(2 * y) * w + 2 * x;
            out[(size_t)y * hw + x] = ((p[0] + p[1]) + (p[w] + p[w + 1])) * 0.25f;
        }
    if (hh * 2 != h && hh > 0) { /* bottom: last output row <- last input row, 1x2 windows */
        const float *p = in + (size_t)(h - 1) * w;
        for (int x = 0; x < hw; x++) out[(size_t)(hh - 1) * hw + x] = (p[2 * x] + p[2 * x + 1]) * 0.5f;
    }
    if (hw * 2 != w && hw > 0) { /* right: last output column <- last input column, 2x1 windows */
        for (int y = 0; y < hh; y++)
            out[(size_t)y * hw + hw - 1] = (in[(size_t)(2 * y) * w + w - 1] + in[(size_t)(2 * y + 1) * w + w - 1]) * 0.5f;
    }
    if (hw * 2 != w && hh * 2 != h && hw > 0 && hh > 0)
        out[(size_t)(hh - 1) * hw + hw - 1] = in[(size_t)(h - 1) * w + w - 1];
}

/* ---------------------------------------------------------------- derivatives.rs */
static img_t simple_scharr_horizontal(const img_t *s) { /* derivatives.rs:3-6 */
    const float a[3] = {-1.f, 0.f, 1.f}, b[3] = {3.f, 10.f, 3.f};
    return separable_filter(s, a, 3, b, 3);
}
static img_t simple_scharr_vertical(const img_t *s) { /* derivatives.rs:8-11 */
    const float a[3] = {-1.f, 0.f, 1.f}, b[3] = {3.f, 10.f, 3.f};
    return separable_filter(s, b, 3, a, 3);
}
/* derivatives.rs:54-79 computer_scharr_kernel */
static int scharr_kernel(uint32_t sigma, int main_order, float *k) {
    double w = 10.0 / 3.0;
    float norm = (float)(1.0 / (2.0 * (double)sigma * (w + 2.0)));
    float middle = norm * (float)w;
    int ks = (int)(3 + 2 * (sigma - 1));
    for (int i = 0; i < ks; i++) k[i] = 0.f;
    if (main_order) { k[0] = -1.f; k[ks - 1] = 1.f; }
    else { k[0] = norm; k[ks / 2] = middle; k[ks - 1] = norm; }
    return ks;
}
static img_t scharr_horizontal(const img_t *s, uint32_t sigma) { /* derivatives.rs:23-30 */
    if (sigma == 1) return simple_scharr_horizontal(s);
    float mk[512], ok[512];
    int ks = scharr_kernel(sigma, 1, mk); scharr_kernel(sigma, 0, ok);
    return separable_filter(s, mk, ks, ok, ks);
}
static img_t scharr_vertical(const img_t *s, uint32_t sigma) { /* derivatives.rs:42-49 */
    if (sigma == 1) return simple_scharr_vertical(s);
    float mk[512], ok[512];
    int ks = scharr_kernel(sigma, 1, mk); scharr_kernel(sigma, 0, ok);
    return separable_filter(s, ok, ks, mk, ks);
}

/* ---------------------------------------------------------------- fed_tau.rs */
static int is_prime_u64(uint64_t n) {
    if (n < 2) return 0;
    for (uint64_t d = 2; d * d <= n; d++) if (n % d == 0) return 0;
    return 1;
}
/* fed_tau.rs:26-93 fed_tau_by_process_time(T, 1, tau_max, reordering=true) */
int ref_fed_tau(double T, double tau_max, double *out, int cap) {
    double t = T / 1.0;
    long n = (long)(ceil(sqrt(3.0 * t / tau_max + 0.25) - 0.5 - 1.0e-8) + 0.5);
    if (n <= 0) return 0;
    if (n > cap) return -1;
    double scale = 3.0 * t / (tau_max * (double)(n * (n + 1)));
    double *tau = (double *)malloc(sizeof(double) * (size_t)n);
    for (long k = 0; k < n; k++) {
        double c = 1.0 / (4.0 * (double)n + 2.0);
        double d = scale * tau_max / 2.0;
        double hh = cos(3.14159265358979323846 * (2.0 * (double)k + 1.0) * c);
        tau[k] = d / (hh * hh);
    }
    long kappa = n / 2, prime = n + 1;
    while (!is_prime_u64((uint64_t)prime)) prime++;
    long k = 0;
    for (long i = 0; i < n; i++) {
        long index = ((k + 1) * kappa) % prime - 1;
        while (index >= n || index < 0) { /* index is usize in Rust: (..)%prime - 1 with 0 wraps to huge -> >= n */
            k++;
            index = ((k + 1) * kappa) % prime - 1;
        }
        k++;
        out[i] = tau[index];
    }
    free(tau);
    return (int)n;
}

/* ---------------------------------------------------------------- evolution.rs */
#define MAX_EVO 64
#define MAX_TAU 256
typedef struct {
    double etime, esigma;
    uint32_t octave, sublevel;
    img_t Lt, Lsmooth, Lx, Ly, Lxx, Lyy, Lxy, Lflow, Ldet;
    img_t Lflow_dbg;
    double tau[MAX_TAU];
    int ntau;
} evo_t;

struct ref_akaze {
    ref_akaze_cfg cfg;
    int w, h;
    int nevo;
    evo_t evo[MAX_EVO];
    double contrast_factor;
    /* stage outputs kept for the parity tests */
    ref_keypoint *cand; int ncand;        /* every thresholded 3x3 maximum, raster order */
    ref_keypoint *extrema; int nextrema;  /* after find_scale_space_extrema */
    ref_keypoint *refined; int nrefined;  /* after do_subpixel_refinement (+orientation) */
    ref_keypoint *sorted; int nsorted;    /* after sort + truncate */
    ref_keypoint *kps; uint8_t *desc; int nkp; /* final */
};

/* evolution.rs:46-58, 80-126 allocate_evolutions */
static void allocate_evolutions(struct ref_akaze *A) {
    const ref_akaze_cfg *c = &A->cfg;
    A->nevo = 0;
    for (uint32_t octave = 0; octave < c->max_octave_evolution; octave++) {
        double rfactor = pow(2.0, -(double)(int)octave); /* 2.0f64.powi(-octave): exact */
        uint32_t lh = (uint32_t)((double)A->h * rfactor);
        uint32_t lw = (uint32_t)((double)A->w * rfactor);
        uint32_t smallest = lw < lh ? lw : lh;
        if (smallest < 40) continue;
        uint32_t sub = smallest < 80 ? 1 : c->num_sublevels;
        for (uint32_t s = 0; s < sub && A->nevo < MAX_EVO; s++) {
            evo_t *e = &A->evo[A->nevo++];
            memset(e, 0, sizeof(*e));
            e->esigma = c->base_scale_offset * pow(2.0, (double)s / (double)c->num_sublevels + (double)octave);
            e->etime = 0.5 * (e->esigma * e->esigma);
            e->octave = octave; e->sublevel = s;
        }
    }
    for (int i = 1; i < A->nevo; i++) {
        double ttime = A->evo[i].etime - A->evo[i - 1].etime;
        A->evo[i].ntau = ref_fed_tau(ttime, 0.25, A->evo[i].tau, MAX_TAU);
    }
}

/* ---------------------------------------------------------------- contrast_factor.rs:16-64 */
static double compute_contrast_factor(const img_t *image, double percentile, double gscale, int nbins) {
    img_t g = gaussian_blur(image, (float)gscale);
    img_t Lx = simple_scharr_horizontal(&g), Ly = simple_scharr_vertical(&g);
    int w = g.w, h = g.h;
    double maxv = -1.0; /* FloatOrd max over interior; values are >= 0 */
    for (int y = 1; y < h - 1; y++)
        for (int x = 1; x < w - 1; x++) {
            float lx = Lx.d[(size_t)y * w + x], ly = Ly.d[(size_t)y * w + x];
            double v = (double)(lx * lx) + (double)(ly * ly);
            if (v > maxv) maxv = v;
        }
    double hmax = sqrt(maxv);
    long *hist = (long *)calloc((size_t)nbins, sizeof(long));
    double num_points = 0.0;
    for (int y = 1; y < h - 1; y++)
        for (int x = 1; x < w - 1; x++) {
            float lx = Lx.d[(size_t)y * w + x], ly = Ly.d[(size_t)y * w + x];
            double modg = sqrt((double)(lx * lx) + (double)(ly * ly));
            if (modg != 0.0) {
                double b = floor((double)nbins * (modg / hmax));
                long bin = (long)b;
                if (bin == nbins) bin -= 1;
                if (bin >= 0 && bin < nbins) hist[bin] += 1;
                num_points += 1.0;
            }
        }
    long threshold = (long)(num_points * percentile);
    long k = 0, nel = 0;
    while (nel < threshold && k < nbins) { nel += hist[k]; k++; }
    free(hist);
    img_free(&g); img_free(&Lx); img_free(&Ly);
    if (nel >= threshold) return hmax * (double)k / (double)nbins;
    return 0.03;
}

/* ---------------------------------------------------------------- nonlinear_diffusion.rs */
/* :70-83 pm_g2 */
static img_t pm_g2(const img_t *Lx, const img_t *Ly, double k) {
    float inverse_k = (float)(1.0 / (k * k));
    img_t c = img_new(Lx->w, Lx->h);
    size_t n = (size_t)Lx->w * Lx->h;
    for (size_t i = 0; i < n; i++) {
        float x = Lx->d[i], y = Ly->d[i];
        c.d[i] = 1.0f / (1.0f + inverse_k * (x * x + y * y));
    }
    return c;
}
/* :14-58 calculate_step: flows from the OLD image, then +hflow[x], -hflow[x-1], +vflow[y],
 * -vflow[y-1] in that order; borders by omission. */
static void calculate_step(img_t *L, const img_t *C, float step) {
    int w = L->w, h = L->h;
    float *o = (float *)malloc(sizeof(float) * (size_t)w * h);
    const float *l = L->d, *c = C->d;
    float hs = 0.5f * step;
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            size_t i = (size_t)y * w + x;
            float v = l[i];
            if (x < w - 1) v += (hs * (c[i] + c[i + 1])) * (l[i + 1] - l[i]);
            if (x > 0) v -= (hs * (c[i - 1] + c[i])) * (l[i] - l[i - 1]);
            if (y < h - 1) v += (hs * (c[i] + c[i + w])) * (l[i + w] - l[i]);
            if (y > 0) v -= (hs * (c[i - w] + c[i])) * (l[i] - l[i - w]);
            o[i] = v;
        }
    memcpy(L->d, o, sizeof(float) * (size_t)w * h);
    free(o);
}

/* ---------------------------------------------------------------- lib.rs:193-258 */
static void create_nonlinear_scale_space(struct ref_akaze *A, const img_t *image) {
    const ref_akaze_cfg *c = &A->cfg;
    evo_t *E = A->evo;
    E[0].Lt = gaussian_blur(image, (float)c->base_scale_offset);
    E[0].Lsmooth = img_clone(&E[0].Lt);
    double contrast = compute_contrast_factor(image, c->contrast_percentile, 1.0, (int)c->contrast_factor_num_bins);
    A->contrast_factor = contrast;
    for (int i = 1; i < A->nevo; i++) {
        if (E[i].octave > E[i - 1].octave) {
            E[i].Lt = img_new(E[i - 1].Lt.w / 2, E[i - 1].Lt.h / 2);
            ref_half_size(E[i - 1].Lt.d, E[i - 1].Lt.w, E[i - 1].Lt.h, E[i].Lt.d);
            contrast *= 0.75;
        } else {
            E[i].Lt = img_clone(&E[i - 1].Lt);
        }
        E[i].Lsmooth = gaussian_blur(&E[i].Lt, 1.0f);
        E[i].Lx = simple_scharr_horizontal(&E[i].Lsmooth);
        E[i].Ly = simple_scharr_vertical(&E[i].Lsmooth);
        E[i].Lflow = pm_g2(&E[i].Lx, &E[i].Ly, contrast);
        for (int j = 0; j < E[i].ntau; j++) calculate_step(&E[i].Lt, &E[i].Lflow, (float)E[i].tau[j]);
    }
}

static double round_half_away(double v) { return round(v); }

/* detector_response.rs:8-85 */
static void detector_response(struct ref_akaze *A) {
    const ref_akaze_cfg *c = &A->cfg;
#pragma omp parallel for schedule(dynamic, 1)
    for (int i = 0; i < A->nevo; i++) {
        evo_t *e = &A->evo[i];
        double ratio = pow(2.0, (double)(int)e->octave);
        uint32_t sigma = (uint32_t)round_half_away(e->esigma * c->derivative_factor / ratio);
        img_free(&e->Lx); img_free(&e->Ly);
        e->Lx = scharr_horizontal(&e->Lsmooth, sigma);
        e->Ly = scharr_vertical(&e->Lsmooth, sigma);
        e->Lxx = scharr_horizontal(&e->Lx, sigma);
        e->Lyy = scharr_vertical(&e->Ly, sigma);
        e->Lxy = scharr_vertical(&e->Lx, sigma);
        double ss = round_half_away(e->esigma * c->derivative_factor / ratio);
        float quat = (float)(ss * ss * ss * ss); /* f64 powi(4) == ((s*s)*s)*s; s is a small integer: exact */
        e->Ldet = img_new(e->Lxx.w, e->Lxx.h);
        size_t n = (size_t)e->Lxx.w * e->Lxx.h;
        for (size_t p = 0; p < n; p++)
            e->Ldet.d[p] = (e->Lxx.d[p] * e->Lyy.d[p] - e->Lxy.d[p] * e->Lxy.d[p]) * quat;
    }
}

/* ---------------------------------------------------------------- scale_space_extrema.rs */
static void kp_push(ref_keypoint **v, int *n, int *cap, ref_keypoint k) {
    if (*n == *cap) { *cap = *cap ? *cap * 2 : 1024; *v = (ref_keypoint *)realloc(*v, sizeof(ref_keypoint) * (size_t)*cap); }
    (*v)[(*n)++] = k;
}

/* :14-143 find_scale_space_extrema */
static void find_scale_space_extrema(struct ref_akaze *A) {
    const ref_akaze_cfg *c = &A->cfg;
    ref_keypoint *cache = NULL; int ncache = 0, capcache = 0;
    int capcand = 0; A->ncand = 0; free(A->cand); A->cand = NULL;
    float smax = 10.0f * sqrtf(2.0f);
    float thr = (float)c->detector_threshold;
    for (int e_id = 0; e_id < A->nevo; e_id++) {
        evo_t *e = &A->evo[e_id];
        int w = e->Ldet.w, h = e->Ldet.h;
        const float *D = e->Ldet.d;
        for (int y = 1; y < h - 1; y++)
            for (int x = 1; x < w - 1; x++) {
                const float *p = D + (size_t)y * w + x;
                float v = *p;
                if (!(v > thr && v > p[-w - 1] && v > p[-w] && v > p[-w + 1] && v > p[-1] && v > p[1] &&
                      v > p[w - 1] && v > p[w] && v > p[w + 1]))
                    continue;
                ref_keypoint kp;
                kp.response = fabsf(v);
                kp.size = (float)(e->esigma * c->derivative_factor);
                kp.octave = e->octave; kp.class_id = (uint32_t)e_id;
                kp.x = (float)x; kp.y = (float)y; kp.angle = 0.f;
                kp_push(&A->cand, &A->ncand, &capcand, kp);
                float ratio = (float)(1u << e->octave); /* powf(2, octave): exact */
                float sigma_size = roundf(kp.size / ratio);
                int id_repeated = 0, is_repeated = 0, is_extremum = 1;
                for (int k = 0; k < ncache; k++) {
                    const ref_keypoint *pk = &cache[k];
                    if (kp.class_id == pk->class_id || (kp.class_id != 0 && kp.class_id - 1 == pk->class_id)) {
                        float dx = kp.x * ratio - pk->x;
                        float dy = kp.y * ratio - pk->y;
                        float dist = dx * dx + dy * dy;
                        if (dist <= kp.size * kp.size) {
                            if (kp.response > pk->response) { id_repeated = k; is_repeated = 1; }
                            else is_extremum = 0;
                            break;
                        }
                    }
                }
                if (is_extremum) {
                    float left_x = roundf(kp.x - smax * sigma_size) - 1.f;
                    float right_x = roundf(kp.x + smax * sigma_size) + 1.f;
                    float up_y = roundf(kp.y - smax * sigma_size) - 1.f;
                    float down_y = roundf(kp.y + smax * sigma_size) + 1.f;
                    int is_out = left_x < 0.f || right_x >= (float)w || up_y < 0.f || down_y >= (float)h;
                    if (!is_out) {
                        kp.x = kp.x * ratio + 0.5f * (ratio - 1.0f);
                        kp.y = kp.y * ratio + 0.5f * (ratio - 1.0f);
                        if (!is_repeated) kp_push(&cache, &ncache, &capcache, kp);
                        else cache[id_repeated] = kp;
                    }
                }
            }
    }
    /* :120-140 filter against the upper scale level */
    free(A->extrema); A->extrema = NULL; A->nextrema = 0; int capx = 0;
    for (int i = 0; i < ncache; i++) {
        int rep = 0;
        ref_keypoint a = cache[i];
        for (int j = i + 1; j < ncache; j++) {
            const ref_keypoint *b = &cache[j];
            if (a.class_id + 1 == b->class_id) {
                float dx = a.x - b->x, dy = a.y - b->y;
                float dist = dx * dx + dy * dy;
                if (dist <= a.size * a.size && a.response <= b->response) { rep = 1; break; }
            }
        }
        if (!rep) kp_push(&A->extrema, &A->nextrema, &capx, a);
    }
    free(cache);
}

/* :162-226 GAUSS25 */
static const float GAUSS25[7][7] = {
    {0.02546481f, 0.02350698f, 0.01849125f, 0.01239505f, 0.00708017f, 0.00344629f, 0.00142946f},
    {0.02350698f, 0.02169968f, 0.01706957f, 0.01144208f, 0.00653582f, 0.00318132f, 0.00131956f},
    {0.01849125f, 0.01706957f, 0.01342740f, 0.00900066f, 0.00514126f, 0.00250252f, 0.00103800f},
    {0.01239505f, 0.01144208f, 0.00900066f, 0.00603332f, 0.00344629f, 0.00167749f, 0.00069579f},
    {0.00708017f, 0.00653582f, 0.00514126f, 0.00344629f, 0.00196855f, 0.00095820f, 0.00039744f},
    {0.00344629f, 0.00318132f, 0.00250252f, 0.00167749f, 0.00095820f, 0.00046640f, 0.00019346f},
    {0.00142946f, 0.00131956f, 0.00103800f, 0.00069579f, 0.00039744f, 0.00019346f, 0.00008024f},
};

#define PI_F 3.14159265358979323846f

/* Rust `f32 as usize` saturates: negative / NaN -> 0. */
static inline long f32_as_usize(float v) { if (!(v > 0.f)) return 0; if (v > 9.0e18f) return (long)9.0e18; return (long)v; }

/* :242 cv_fast_atan2_equiv: (y.atan2(x) + 2pi).rem_euclid(2pi); rem_euclid = fmodf (+|rhs| if <0) */
static inline float fast_atan2_equiv(float y, float x) {
    float two_pi = 2.f * PI_F;
    float v = rl_atan2f(y, x) + two_pi;
    float r = fmodf(v, two_pi);
    if (r < 0.0f) r = r + fabsf(two_pi);
    return r;
}

/* :229-288 compute_main_orientation */
static int compute_main_orientation(ref_keypoint *kp, const struct ref_akaze *A) {
    float res_x[109], res_y[109], angs[109];
    static const int id[13] = {6, 5, 4, 3, 2, 1, 0, 1, 2, 3, 4, 5, 6};
    const evo_t *e = &A->evo[kp->class_id];
    float ratio = (float)(1 << e->octave);
    float s = roundf(0.5f * kp->size / ratio);
    float xf = kp->x / ratio, yf = kp->y / ratio;
    int idx = 0, oob = 0;
    for (int j = -6; j <= 6; j++)
        for (int i = -6; i <= 6; i++)
            if (i * i + j * j < 36) {
                long iy = f32_as_usize(roundf(yf + (float)j * s));
                long ix = f32_as_usize(roundf(xf + (float)i * s));
                if (ix >= e->Lx.w || iy >= e->Lx.h) { oob = 1; ix = ix >= e->Lx.w ? e->Lx.w - 1 : ix; iy = iy >= e->Lx.h ? e->Lx.h - 1 : iy; }
                float gw = GAUSS25[id[j + 6]][id[i + 6]];
                res_x[idx] = gw * e->Lx.d[(size_t)iy * e->Lx.w + ix];
                res_y[idx] = gw * e->Ly.d[(size_t)iy * e->Ly.w + ix];
                angs[idx] = fast_atan2_equiv(res_y[idx], res_x[idx]);
                idx++;
            }
    float ang1 = 0.f, maxv = 0.f;
    while (ang1 < 2.0f * PI_F) {
        float sum_x = 0.f, sum_y = 0.f;
        float ang2 = (ang1 + PI_F / 3.0f > 2.0f * PI_F) ? ang1 - 5.0f * PI_F / 3.0f : ang1 + PI_F / 3.0f;
        for (int k = 0; k < 109; k++) {
            float ang = angs[k];
            if ((ang1 < ang2 && ang1 < ang && ang < ang2) ||
                (ang2 < ang1 && ((ang > 0.f && ang < ang2) || (ang > ang1 && ang < 2.0f * PI_F)))) {
                sum_x += res_x[k];
                sum_y += res_y[k];
            }
        }
        float val = sum_x * sum_x + sum_y * sum_y;
        if (val > maxv) { maxv = val; kp->angle = fast_atan2_equiv(sum_y, sum_x); }
        ang1 += 0.15f;
    }
    return oob;
}

/* :297-362 do_subpixel_refinement */
static void do_subpixel_refinement(struct ref_akaze *A) {
    int n = A->nextrema;
    ref_keypoint *out = (ref_keypoint *)malloc(sizeof(ref_keypoint) * (size_t)(n > 0 ? n : 1));
    char *keep = (char *)calloc((size_t)(n > 0 ? n : 1), 1);
#pragma omp parallel for schedule(dynamic, 64)
    for (int q = 0; q < n; q++) {
        ref_keypoint kp = A->extrema[q];
        const evo_t *e = &A->evo[kp.class_id];
        const float *D = e->Ldet.d; int w = e->Ldet.w;
        float ratio = (float)(1u << kp.octave);
        long x = f32_as_usize(roundf(kp.x / ratio)), y = f32_as_usize(roundf(kp.y / ratio));
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
        if (fabsf(dst0) <= 1.0f && fabsf(dst1) <= 1.0f) {
            kp.x = (float)x + dst0; kp.y = (float)y + dst1;
            float power = (float)(1u << e->octave);
            kp.x = kp.x * power + 0.5f * (power - 1.f);
            kp.y = kp.y * power + 0.5f * (power - 1.f);
            kp.size *= 2.f;
            compute_main_orientation(&kp, A);
            out[q] = kp; keep[q] = 1;
        }
    }
    free(A->refined); A->refined = (ref_keypoint *)malloc(sizeof(ref_keypoint) * (size_t)(n > 0 ? n : 1));
    A->nrefined = 0;
    for (int q = 0; q < n; q++) if (keep[q]) A->refined[A->nrefined++] = out[q];
    free(out); free(keep);
}

/* lib.rs:326-327: sort_unstable_by_key(Reverse(FloatOrd(response))) + truncate.  The Rust sort is
 * unstable (tie order unspecified / rustc-version dependent); the oracle's working definition is
 * descending response, ties in original order (SURVEY.md hard part 6). */
typedef struct { ref_keypoint k; int idx; } sort_item;
static int cmp_desc(const void *a, const void *b) {
    const sort_item *p = (const sort_item *)a, *q = (const sort_item *)b;
    if (p->k.response > q->k.response) return -1;
    if (p->k.response < q->k.response) return 1;
    return p->idx - q->idx;
}
static void sort_truncate(struct ref_akaze *A) {
    int n = A->nrefined;
    sort_item *it = (sort_item *)malloc(sizeof(sort_item) * (size_t)(n > 0 ? n : 1));
    for (int i = 0; i < n; i++) { it[i].k = A->refined[i]; it[i].idx = i; }
    qsort(it, (size_t)n, sizeof(sort_item), cmp_desc);
    int64_t m = A->cfg.maximum_features;
    int keep = (m >= 0 && m < n) ? (int)m : n;
    free(A->sorted); A->sorted = (ref_keypoint *)malloc(sizeof(ref_keypoint) * (size_t)(keep > 0 ? keep : 1));
    for (int i = 0; i < keep; i++) A->sorted[i] = it[i].k;
    A->nsorted = keep;
    free(it);
}

/* ---------------------------------------------------------------- descriptors.rs */
/* :102-177 mldb_fill_values ; returns 0 ok, 1 sample out of bounds */
static int mldb_fill_values(const struct ref_akaze *A, float *values, int sample_step, int level, float xf, float yf,
                            float co, float si, float scale) {
    int pattern = (int)A->cfg.descriptor_pattern_size, nch = (int)A->cfg.descriptor_channels;
    const evo_t *e = &A->evo[level];
    int W = e->Lt.w, H = e->Lt.h;
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
                    float ry_ = roundf(sample_y), rx_ = roundf(sample_x);
                    /* `as isize` saturating cast, then range check */
                    if (!(rx_ >= 0.f && rx_ < (float)W) || !(ry_ >= 0.f && ry_ < (float)H)) return 1;
                    long y1 = (long)ry_, x1 = (long)rx_;
                    float ri = e->Lt.d[y1 * W + x1];
                    di += ri;
                    if (nch > 1) {
                        float rx = e->Lx.d[y1 * W + x1], ry = e->Ly.d[y1 * W + x1];
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
/* :181-202 mldb_binary_comparisons */
static void mldb_binary_comparisons(const float *values, uint8_t *desc, int count, int *dpos, int nch) {
    for (int pos = 0; pos < nch; pos++)
        for (int i = 0; i < count; i++) {
            float iv = values[nch * i + pos];
            for (int j = i + 1; j < count; j++) {
                uint8_t res = iv > values[nch * j + pos] ? 1 : 0;
                desc[*dpos >> 3] |= (uint8_t)(res << (*dpos & 7));
                (*dpos)++;
            }
        }
}
/* :55-98 get_mldb_descriptor */
static int get_mldb_descriptor(const struct ref_akaze *A, const ref_keypoint *kp, uint8_t *desc) {
    float values[16 * 3];
    memset(desc, 0, 64);
    memset(values, 0, sizeof(values));
    const float size_mult[3] = {1.0f, 2.0f / 3.0f, 1.0f / 2.0f};
    float ratio = (float)(1u << kp->octave);
    float scale = roundf(0.5f * kp->size / ratio);
    float xf = kp->x / ratio, yf = kp->y / ratio;
    float co = rl_cosf(kp->angle), si = rl_sinf(kp->angle);
    float pattern = (float)A->cfg.descriptor_pattern_size;
    int dpos = 0;
    for (int lvl = 0; lvl < 3; lvl++) {
        int val_count = (lvl + 2) * (lvl + 2);
        int sample_size = (int)ceilf(pattern * size_mult[lvl]);
        if (mldb_fill_values(A, values, sample_size, (int)kp->class_id, xf, yf, co, si, scale)) return 1;
        mldb_binary_comparisons(values, desc, val_count, &dpos, (int)A->cfg.descriptor_channels);
    }
    return 0;
}
/* :16-45 extract_descriptors: keypoints whose patch leaves the image are dropped */
static void extract_descriptors(struct ref_akaze *A) {
    int n = A->nsorted;
    uint8_t *d = (uint8_t *)malloc((size_t)(n > 0 ? n : 1) * 64);
    char *ok = (char *)calloc((size_t)(n > 0 ? n : 1), 1);
#pragma omp parallel for schedule(dynamic, 64)
    for (int i = 0; i < n; i++) ok[i] = !get_mldb_descriptor(A, &A->sorted[i], d + (size_t)i * 64);
    free(A->kps); free(A->desc);
    A->kps = (ref_keypoint *)malloc(sizeof(ref_keypoint) * (size_t)(n > 0 ? n : 1));
    A->desc = (uint8_t *)malloc((size_t)(n > 0 ? n : 1) * 64);
    A->nkp = 0;
    for (int i = 0; i < n; i++)
        if (ok[i]) { A->kps[A->nkp] = A->sorted[i]; memcpy(A->desc + (size_t)A->nkp * 64, d + (size_t)i * 64, 64); A->nkp++; }
    free(d); free(ok);
}

/* ---------------------------------------------------------------- public API */
void ref_akaze_default_cfg(ref_akaze_cfg *c) { /* lib.rs:169-185 */
    c->maximum_features = -1; /* usize::MAX */
    c->num_sublevels = 4; c->max_octave_evolution = 4;
    c->base_scale_offset = 1.6; c->initial_contrast = 0.001; c->contrast_percentile = 0.7;
    c->contrast_factor_num_bins = 300; c->derivative_factor = 1.5; c->detector_threshold = 0.001;
    c->descriptor_channels = 3; c->descriptor_pattern_size = 10;
}

static void evo_free(evo_t *e) {
    img_free(&e->Lt); img_free(&e->Lsmooth); img_free(&e->Lx); img_free(&e->Ly); img_free(&e->Lxx);
    img_free(&e->Lyy); img_free(&e->Lxy); img_free(&e->Lflow); img_free(&e->Ldet); img_free(&e->Lflow_dbg);
}

struct ref_akaze *ref_akaze_create(const ref_akaze_cfg *cfg) {
    struct ref_akaze *A = (struct ref_akaze *)calloc(1, sizeof(struct ref_akaze));
    A->cfg = *cfg;
    return A;
}
void ref_akaze_destroy(struct ref_akaze *A) {
    if (!A) return;
    for (int i = 0; i < MAX_EVO; i++) evo_free(&A->evo[i]);
    free(A->cand); free(A->extrema); free(A->refined); free(A->sorted); free(A->kps); free(A->desc);
    free(A);
}

/* lib.rs:309-339 extract_from_gray_float_image */
int ref_akaze_extract(struct ref_akaze *A, const float *image, int w, int h) {
    for (int i = 0; i < MAX_EVO; i++) evo_free(&A->evo[i]);
    A->w = w; A->h = h;
    allocate_evolutions(A);
    if (A->nevo == 0) { A->nkp = 0; return 0; }
    img_t im; im.w = w; im.h = h; im.d = (float *)image;
    create_nonlinear_scale_space(A, &im);
    detector_response(A);
    find_scale_space_extrema(A);
    do_subpixel_refinement(A);
    sort_truncate(A);
    extract_descriptors(A);
    return A->nkp;
}

int ref_akaze_num_evolutions(const struct ref_akaze *A) { return A->nevo; }
int ref_akaze_evolution_info(const struct ref_akaze *A, int i, int *w, int *h, uint32_t *octave, double *esigma, int *ntau, double *tau) {
    if (i < 0 || i >= A->nevo) return -1;
    const evo_t *e = &A->evo[i];
    *w = e->Lt.w; *h = e->Lt.h; *octave = e->octave; *esigma = e->esigma; *ntau = e->ntau;
    if (tau) memcpy(tau, e->tau, sizeof(double) * (size_t)e->ntau);
    return 0;
}
double ref_akaze_contrast_factor(const struct ref_akaze *A) { return A->contrast_factor; }
/* plane ids: 0 Lt, 1 Lsmooth, 2 Lx, 3 Ly, 4 Lflow, 5 Ldet, 6 Lxx, 7 Lyy, 8 Lxy */
const float *ref_akaze_plane(const struct ref_akaze *A, int i, int plane) {
    if (i < 0 || i >= A->nevo) return NULL;
    const evo_t *e = &A->evo[i];
    switch (plane) {
    case 0: return e->Lt.d; case 1: return e->Lsmooth.d; case 2: return e->Lx.d; case 3: return e->Ly.d;
    case 4: return e->Lflow.d; case 5: return e->Ldet.d; case 6: return e->Lxx.d; case 7: return e->Lyy.d;
    case 8: return e->Lxy.d; default: return NULL;
    }
}
/* stage ids: 0 candidates, 1 extrema, 2 refined, 3 sorted, 4 final */
int ref_akaze_stage(const struct ref_akaze *A, int stage, const ref_keypoint **out) {
    switch (stage) {
    case 0: *out = A->cand; return A->ncand;
    case 1: *out = A->extrema; return A->nextrema;
    case 2: *out = A->refined; return A->nrefined;
    case 3: *out = A->sorted; return A->nsorted;
    case 4: *out = A->kps; return A->nkp;
    default: *out = NULL; return -1;
    }
}
const uint8_t *ref_akaze_descriptors(const struct ref_akaze *A) { return A->desc; }

#ifdef _OPENMP
#include <omp.h>
#endif
/* number of OpenMP threads used at the reference's rayon sites (bench.py's CPU arm) */
void ref_set_num_threads(int n) {
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}

/* scalar helpers exported so tests can pin the restated libm against the host libm */
float ref_sinf(float x) { return rl_sinf(x); }
float ref_cosf(float x) { return rl_cosf(x); }
float ref_atan2f(float y, float x) { return rl_atan2f(y, x); }
float ref_fast_atan2_equiv(float y, float x) { return fast_atan2_equiv(y, x); }
