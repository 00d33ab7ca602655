/* Test infrastructure: a plain C translation unit against include/cvb200_filter.h that calls EVERY entry point that header declares, so
 * that the prototypes a Rust / cgo / JNI binding transcribes are checked by a C compiler (ctypes never sees the header).
 *   mode 0 (no GPU): context creation reports no device; every entry point rejects a null context; gaussian_kernel (host arithmetic)
 *                    meets the reference's known answer and rejects an even size.
 *   mode 1 (GPU):    bad sizes, sigmas and overlapping buffers are rejected by the host and _dev forms; on a small plane a 1-tap kernel
 *                    of 1.0 is the identity, separable_filter is the two passes, gaussian_blur is separable_filter with gaussian_kernel,
 *                    and half_size averages 2x2 boxes.  (tests/test_gpu_filter.py runs the _dev forms on device buffers.)
 * Build: gcc -std=c11 -Wall -Wextra -Werror abi_smoke_filter.c -I../../include -L../../cv_b200 -lcvb200_filter -lcvb200 -lm */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "cvb200_filter.h"

#define CHECK(cond) do { if (!(cond)) { fprintf(stderr, "abi_smoke_filter: %s:%d: %s\n", __FILE__, __LINE__, #cond); return 1; } } while (0)

static int host_checks(void) {
    /* image.rs:395-412 known answer */
    static const float known[7] = {0.10628852f, 0.14032133f, 0.16577007f, 0.17524014f, 0.16577007f, 0.14032133f, 0.10628852f};
    float k[7];
    CHECK(cvb_gaussian_kernel(3.0f, 7, k) == CVB_OK);
    for (int i = 0; i < 7; i++) CHECK(fabsf(k[i] - known[i]) < 1e-4f);
    CHECK(cvb_gaussian_kernel(3.0f, 6, k) == CVB_EINVAL);
    CHECK(cvb_gaussian_kernel(3.0f, 0, k) == CVB_EINVAL);
    CHECK(cvb_gaussian_kernel(3.0f, 7, NULL) == CVB_EINVAL);
    return 0;
}

static int no_gpu_checks(void) {
    cvb_ctx *ctx = NULL;
    const int rc = cvb_ctx_create(0, &ctx);
    if (rc == CVB_OK) { cvb_ctx_destroy(ctx); return -1; }      /* a GPU is present: the caller runs mode 1 */
    CHECK(rc == CVB_ENODEV && ctx == NULL);                     /* no CPU fallback */
    float in[64] = {0}, out[64], k[3] = {0.25f, 0.5f, 0.25f};
    CHECK(cvb_horizontal_filter(NULL, in, 1, 8, 8, k, 3, out) == CVB_EINVAL);
    CHECK(cvb_horizontal_filter_dev(NULL, in, 1, 8, 8, k, 3, out) == CVB_EINVAL);
    CHECK(cvb_vertical_filter(NULL, in, 1, 8, 8, k, 3, out) == CVB_EINVAL);
    CHECK(cvb_vertical_filter_dev(NULL, in, 1, 8, 8, k, 3, out) == CVB_EINVAL);
    CHECK(cvb_separable_filter(NULL, in, 1, 8, 8, k, 3, k, 3, out) == CVB_EINVAL);
    CHECK(cvb_separable_filter_dev(NULL, in, 1, 8, 8, k, 3, k, 3, out) == CVB_EINVAL);
    CHECK(cvb_gaussian_blur(NULL, in, 1, 8, 8, 1.0f, out) == CVB_EINVAL);
    CHECK(cvb_gaussian_blur_dev(NULL, in, 1, 8, 8, 1.0f, out) == CVB_EINVAL);
    CHECK(cvb_half_size(NULL, in, 1, 8, 8, out) == CVB_EINVAL);
    CHECK(cvb_half_size_dev(NULL, in, 1, 8, 8, out) == CVB_EINVAL);
    return 0;
}

static int gpu_workflow(void) {
    cvb_ctx *ctx = NULL;
    CHECK(cvb_ctx_create(0, &ctx) == CVB_OK);
    enum { W = 37, H = 23, N = W * H };
    float *in = malloc(sizeof(float) * N), *a = malloc(sizeof(float) * N), *b = malloc(sizeof(float) * N), *c = malloc(sizeof(float) * N);
    for (int i = 0; i < N; i++) in[i] = (float)((i * 7919) % 101) / 101.0f - 0.5f;
    const float one = 1.0f, k5[5] = {-0.5f, 0.25f, 1.0f, 0.125f, -0.0625f};
    /* argument errors */
    CHECK(cvb_horizontal_filter(ctx, in, 1, W, H, k5, 4, a) == CVB_EINVAL);
    CHECK(strlen(cvb_last_error(ctx)) > 0);
    CHECK(cvb_vertical_filter(ctx, in, 1, W, H, k5, CVB_FILTER_MAX_TAPS + 2, a) == CVB_EUNSUPPORTED);
    CHECK(cvb_separable_filter(ctx, in, 0, W, H, k5, 5, k5, 5, a) == CVB_EINVAL);
    CHECK(cvb_gaussian_blur(ctx, in, 1, W, H, 0.0f, a) == CVB_EINVAL);
    CHECK(cvb_gaussian_blur(ctx, in, 1, W, H, NAN, a) == CVB_EINVAL);
    CHECK(cvb_gaussian_blur(ctx, in, 1, W, H, 1000.0f, a) == CVB_EUNSUPPORTED);
    CHECK(cvb_half_size(ctx, in, 1, W, 0, a) == CVB_EINVAL);
    CHECK(cvb_horizontal_filter(ctx, in, 1, W, H, k5, 5, in + 1) == CVB_EINVAL);
    /* a 1-tap kernel of 1.0 is the identity; separable_filter is the two passes */
    CHECK(cvb_horizontal_filter(ctx, in, 1, W, H, &one, 1, a) == CVB_OK);
    CHECK(!memcmp(a, in, sizeof(float) * N));
    CHECK(cvb_horizontal_filter(ctx, in, 1, W, H, k5, 5, a) == CVB_OK);
    CHECK(cvb_vertical_filter(ctx, a, 1, W, H, k5, 5, b) == CVB_OK);
    CHECK(cvb_separable_filter(ctx, in, 1, W, H, k5, 5, k5, 5, c) == CVB_OK && !memcmp(b, c, sizeof(float) * N));
    /* the _dev forms check their arguments before touching a buffer */
    CHECK(cvb_horizontal_filter_dev(ctx, in, 1, W, H, k5, 6, a) == CVB_EINVAL);
    CHECK(cvb_vertical_filter_dev(ctx, in, 1, W, H, k5, 5, in) == CVB_EINVAL);
    CHECK(cvb_separable_filter_dev(ctx, in, 1, W, H, k5, 5, k5, 5, NULL) == CVB_EINVAL);
    CHECK(cvb_gaussian_blur_dev(ctx, in, 1, W, H, -1.0f, a) == CVB_EINVAL);
    CHECK(cvb_half_size_dev(ctx, in, 0, W, H, a) == CVB_EINVAL);
    /* gaussian_blur(1.6) = separable_filter with gaussian_kernel(1.6, 9) */
    float g[9];
    CHECK(cvb_gaussian_kernel(1.6f, 9, g) == CVB_OK);
    CHECK(cvb_separable_filter(ctx, in, 1, W, H, g, 9, g, 9, a) == CVB_OK);
    CHECK(cvb_gaussian_blur(ctx, in, 1, W, H, 1.6f, b) == CVB_OK && !memcmp(a, b, sizeof(float) * N));
    /* half_size: interior 2x2 boxes */
    enum { HW = W / 2, HH = H / 2 };
    CHECK(cvb_half_size(ctx, in, 1, W, H, a) == CVB_OK);
    for (int y = 0; y + 1 < HH; y++)
        for (int x = 0; x + 1 < HW; x++) {
            const float *p = in + 2 * y * W + 2 * x;
            CHECK(a[y * HW + x] == ((p[0] + p[1]) + (p[W] + p[W + 1])) * 0.25f);
        }
    CHECK(a[HH * HW - 1] == in[N - 1]);   /* odd by odd: the corner is copied */
    free(in); free(a); free(b); free(c);
    cvb_ctx_destroy(ctx);
    printf("GPU workflow ok\n");
    return 0;
}

int main(int argc, char **argv) {
    const int mode = argc > 1 ? atoi(argv[1]) : 0;
    if (host_checks()) return 1;
    if (mode == 0) {
        const int r = no_gpu_checks();
        if (r > 0) return 1;
        printf(r < 0 ? "GPU present: mode 0 skipped\n" : "no-GPU checks ok\n");
        return 0;
    }
    return gpu_workflow();
}
