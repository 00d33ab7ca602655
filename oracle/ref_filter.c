/* oracle/ref_filter.c -- TEST INFRASTRUCTURE: CPU restatement of akaze::image's public filters (akaze 0.7.0, image.rs:202-331) as
 * include/cvb200_filter.h exposes them, zero-weighted tail taps included.
 *
 * The reference pads the kernel with zeros into f32x4 chunks (kernel.chunks(4)), builds a scratch line
 * [half x first][line][half x last][3 x 0.0] (kernel_simd_size = 4 * (ks + 3) / 4 = ks + 3, so 3 extra elements) and takes, for each
 * output, the window of ks + 3 scratch elements starting at the output's index, split by chunks_exact(4) (the window's last ks + 3 mod 4
 * elements are dropped) and zipped with the kernel's chunks.  So every output evaluates 4 * ceil(ks / 4) taps; the tail taps multiply
 * 0.0 by whatever the scratch holds there.  On finite data that adds +-0 to a lane that is never -0, a no-op (oracle/ref_akaze.c, the
 * extractor's oracle, skips them); a NaN or +-inf under a tail tap makes the output NaN, and this file keeps that.
 *
 * Lane j & 3 accumulates tap j as (pixel * k[j]) + acc from +0 (wide 0.7 mul_add without the fma target feature), and reduce_add is
 * (l0 + l2) + (l1 + l3) (the SSE2 path, the default of oracle/ref_akaze.c's REF_REDUCE_ORDER).  The vertical filter's 16-column scratch
 * (image.rs:283-300) is a cache layout with no numeric effect: a column is filtered exactly like a row.
 *
 * Build: oracle/filter.mk, gcc -ffp-contract=off -fno-fast-math (no fused multiply-add). */
#include <stdlib.h>
#include <string.h>

/* one line of n pixels, element i at line[i * stride] -> out[i * ostride]; kpad: the kernel zero-padded to 4 * ceil(ks / 4) taps */
static void filter_line(const float *line, size_t stride, int n, int ks, const float *kpad, float *out, size_t ostride, float *scratch) {
    const int half = ks / 2, chunks = (ks + 3) / 4;
    for (int i = 0; i < half; i++) scratch[i] = line[0];
    for (int i = 0; i < n; i++) scratch[half + i] = line[(size_t)i * stride];
    for (int i = 0; i < half; i++) scratch[half + n + i] = line[(size_t)(n - 1) * stride];
    for (int i = 0; i < 3; i++) scratch[2 * half + n + i] = 0.0f;
    for (int x = 0; x < n; x++) {
        const float *win = scratch + x;
        float l[4] = {0.0f, 0.0f, 0.0f, 0.0f};
        for (int c = 0; c < chunks; c++)
            for (int u = 0; u < 4; u++) l[u] = win[4 * c + u] * kpad[4 * c + u] + l[u];
        out[(size_t)x * ostride] = (l[0] + l[2]) + (l[1] + l[3]);
    }
}

/* 0, or -1 for an even kernel size or a failed allocation */
static int filter(const float *in, int w, int h, const float *k, int ks, float *out, int vertical) {
    if (ks % 2 == 0 || w <= 0 || h <= 0) return -1;
    const int n = vertical ? h : w, lines = vertical ? w : h, chunks = (ks + 3) / 4;
    float *scratch = malloc(sizeof(float) * (size_t)(n + ks + 2)), *kpad = calloc((size_t)chunks * 4, sizeof(float));
    if (!scratch || !kpad) { free(scratch); free(kpad); return -1; }
    memcpy(kpad, k, sizeof(float) * (size_t)ks);
    for (int i = 0; i < lines; i++) {
        if (vertical) filter_line(in + i, (size_t)w, h, ks, kpad, out + i, (size_t)w, scratch);
        else filter_line(in + (size_t)i * w, 1, w, ks, kpad, out + (size_t)i * w, 1, scratch);
    }
    free(scratch);
    free(kpad);
    return 0;
}

/* image.rs:202-251 horizontal_filter */
int ref_filter_horizontal(const float *in, int w, int h, const float *k, int ks, float *out) { return filter(in, w, h, k, ks, out, 0); }

/* image.rs:253-331 vertical_filter */
int ref_filter_vertical(const float *in, int w, int h, const float *k, int ks, float *out) { return filter(in, w, h, k, ks, out, 1); }
