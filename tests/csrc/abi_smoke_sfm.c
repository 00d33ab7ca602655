/* Test infrastructure: a plain C translation unit against include/cvb200_sfm.h that calls EVERY entry point that header declares, so
 * that the prototypes a Rust / cgo / JNI binding transcribes are checked by a C compiler (ctypes never sees the header).
 *   mode 0 (no GPU): context creation reports no device; every entry point rejects a null context.
 *   mode 1 (GPU):    the K1 entry points with k1 = 0 equal the undistorted ones; frame ingestion on two synthetic frames.
 * Build: gcc -std=c11 -Wall -Wextra -Werror abi_smoke_sfm.c -I../../include -L../../cv_b200 -lcvb200 -lm */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "cvb200_sfm.h"

#define CHECK(cond) do { if (!(cond)) { fprintf(stderr, "abi_smoke_sfm: %s:%d: %s\n", __FILE__, __LINE__, #cond); return 1; } } while (0)

static int no_gpu_checks(void) {
    cvb_ctx *ctx = NULL;
    const int rc = cvb_ctx_create(0, &ctx);
    if (rc == CVB_OK) { cvb_ctx_destroy(ctx); return -1; }      /* a GPU is present: the caller runs mode 1 */
    CHECK(rc == CVB_ENODEV && ctx == NULL);                     /* no CPU fallback */
    cvb_akaze_cfg ac;
    cvb_akaze_default_cfg(&ac);
    cvb_arrsac_cfg rc_;
    cvb_arrsac_default_cfg(&rc_, 1e-7);
    cvb_rng rng;
    cvb_rng_seed_xoshiro256pp(&rng, 0);
    float img[16] = {0};
    uint8_t rgb[48] = {0}, desc[4 * 64];
    cvb_keypoint kp[4];
    uint32_t n = 0, u[16];
    double d[64] = {0};
    cvb_pose pose;
    int32_t found;
    const cvb_intrinsics_k1 K1 = {1000.0, 1000.0, 960.0, 540.0, 0.0, -0.28};
    CHECK(cvb_pair_bearings_k1_dev(NULL, kp, kp, u, &n, 4, &K1, d, d) == CVB_EINVAL);
    CHECK(cvb_two_view_pair_k1_dev(NULL, kp, desc, &n, kp, desc, &n, 4, 24, &K1, &rc_, &rng, u, 4, &n, &pose, u, &n, &found) == CVB_EINVAL);
    CHECK(cvb_two_view_frames_k1(NULL, &ac, img, 4, 4, 24, &K1, &rc_, &rng, kp, desc, 4, u, u, &n, &pose, u, &n, &found) == CVB_EINVAL);
    CHECK(cvb_frame_features_batch(NULL, &ac, img, rgb, 1, 4, 4, &K1, kp, desc, d, rgb, 4, &n) == CVB_EINVAL);
    CHECK(cvb_frame_features_batch_dev(NULL, kp, &n, 1, 4, rgb, 4, 4, &K1, d, rgb) == CVB_EINVAL);
    return 0;
}

/* deterministic pseudo-random image: value noise + blobs, enough structure for a few hundred keypoints */
static void make_image(float *img, int w, int h, float dx) {
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            float xf = (float)x + dx, v = 0.5f;
            v += 0.20f * sinf(0.11f * xf) * cosf(0.07f * (float)y) + 0.15f * sinf(0.31f * xf + 0.23f * (float)y);
            v += 0.10f * cosf(0.53f * xf - 0.41f * (float)y) + 0.05f * sinf(1.3f * xf) * sinf(1.1f * (float)y);
            img[(size_t)y * w + x] = v < 0.f ? 0.f : (v > 1.f ? 1.f : v);
        }
}

static int gpu_workflow(void) {
    cvb_ctx *ctx = NULL;
    CHECK(cvb_ctx_create(0, &ctx) == CVB_OK && ctx != NULL);
    const int w = 320, h = 240;
    const uint32_t cap = 4096;
    float *frames = (float *)malloc(sizeof(float) * 2 * w * h);
    make_image(frames, w, h, 0.f);
    make_image(frames + w * h, w, h, 2.5f);
    cvb_akaze_cfg ac;
    cvb_akaze_default_cfg(&ac);
    cvb_arrsac_cfg rc_;
    cvb_arrsac_default_cfg(&rc_, 1e-6);
    cvb_keypoint *kp = (cvb_keypoint *)malloc(sizeof(cvb_keypoint) * 2 * cap), *kp1 = (cvb_keypoint *)malloc(sizeof(cvb_keypoint) * 2 * cap);
    uint8_t *desc = (uint8_t *)malloc((size_t)2 * cap * 64), *desc1 = (uint8_t *)malloc((size_t)2 * cap * 64);
    uint32_t *pairs = (uint32_t *)malloc(sizeof(uint32_t) * 2 * cap), *pairs1 = (uint32_t *)malloc(sizeof(uint32_t) * 2 * cap);
    uint32_t *inl = (uint32_t *)malloc(sizeof(uint32_t) * cap), *inl1 = (uint32_t *)malloc(sizeof(uint32_t) * cap);
    uint32_t n[2], n1[2], npairs = 0, npairs1 = 0, ninl = 0, ninl1 = 0;
    int32_t found = 0, found1 = 0;
    cvb_pose model, model1;
    /* the K1 entry point with k1 = 0 is the undistorted one, result for result */
    const cvb_intrinsics K = {300.0, 300.0, 160.0, 120.0, 0.0};
    const cvb_intrinsics_k1 K1 = {300.0, 300.0, 160.0, 120.0, 0.0, 0.0};
    cvb_rng rng, rng1;
    cvb_rng_seed_xoshiro256pp(&rng, 0);
    cvb_rng_seed_xoshiro256pp(&rng1, 0);
    CHECK(cvb_two_view_frames(ctx, &ac, frames, (uint32_t)w, (uint32_t)h, 24, &K, &rc_, &rng, kp, desc, cap, n, pairs, &npairs, &model, inl,
                              &ninl, &found) == CVB_OK);
    CHECK(cvb_two_view_frames_k1(ctx, &ac, frames, (uint32_t)w, (uint32_t)h, 24, &K1, &rc_, &rng1, kp1, desc1, cap, n1, pairs1, &npairs1,
                                 &model1, inl1, &ninl1, &found1) == CVB_OK);
    CHECK(n[0] > 20 && n1[0] == n[0] && n1[1] == n[1] && npairs1 == npairs && ninl1 == ninl && found1 == found);
    CHECK(memcmp(pairs, pairs1, sizeof(uint32_t) * 2 * npairs) == 0 && memcmp(inl, inl1, sizeof(uint32_t) * ninl) == 0);
    CHECK(!found || memcmp(&model, &model1, sizeof model) == 0);
    CHECK(rng.kind == rng1.kind && memcmp(rng.s, rng1.s, sizeof rng.s) == 0);   /* the same draws consumed (fields: the struct has padding) */
    /* frame ingestion: the extractor's own keypoints, unit bearings, the colour of a constant grey frame (or black at the border) */
    uint8_t *rgb = (uint8_t *)malloc((size_t)2 * w * h * 3);
    memset(rgb, 77, (size_t)2 * w * h * 3);
    double *bear = (double *)malloc(sizeof(double) * 2 * cap * 3);
    uint8_t *col = (uint8_t *)malloc((size_t)2 * cap * 3);
    uint32_t n2[2] = {0, 0};
    const cvb_intrinsics_k1 Kd = {300.0, 300.0, 160.0, 120.0, 0.0, -0.28};
    CHECK(cvb_frame_features_batch(ctx, &ac, frames, rgb, 2, (uint32_t)w, (uint32_t)h, &Kd, kp1, desc1, bear, col, cap, n2) == CVB_OK);
    CHECK(n2[0] == n[0] && n2[1] == n[1] && memcmp(desc, desc1, (size_t)n[0] * 64) == 0);
    for (uint32_t i = 0; i < n2[0]; i++) {
        const double *v = bear + 3 * i;
        const uint8_t *c = col + 3 * i;
        CHECK(fabs(v[0] * v[0] + v[1] * v[1] + v[2] * v[2] - 1.0) < 1e-12 && v[2] > 0.0);
        CHECK((c[0] == 77 && c[1] == 77 && c[2] == 77) || (c[0] == 0 && c[1] == 0 && c[2] == 0));
    }
    CHECK(cvb_ctx_sync(ctx) == CVB_OK);
    cvb_ctx_destroy(ctx);
    free(frames); free(kp); free(kp1); free(desc); free(desc1); free(pairs); free(pairs1); free(inl); free(inl1);
    free(rgb); free(bear); free(col);
    return 0;
}

int main(int argc, char **argv) {
    const int mode = argc > 1 ? atoi(argv[1]) : 0;
    if (mode == 0) {
        const int r = no_gpu_checks();
        if (r < 0) { printf("abi_smoke_sfm: GPU present, skipping the no-GPU checks\n"); return 0; }
        if (r == 0) printf("abi_smoke_sfm: no device reported; every entry point rejects a null context\n");
        return r;
    }
    const int r = gpu_workflow();
    if (r == 0) printf("abi_smoke_sfm: GPU workflow ok\n");
    return r;
}
