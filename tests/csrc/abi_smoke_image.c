/* Test infrastructure: a plain C translation unit against include/cvb200_image.h that calls EVERY entry point that header declares, so
 * that the prototypes a Rust / cgo / JNI binding transcribes are checked by a C compiler (ctypes never sees the header).
 *   mode 0 (no GPU): context creation reports no device; every entry point rejects a null context.
 *   mode 1 (GPU):    bad formats and sizes are rejected, float formats and 16-bit frame ingestion are unsupported, a Luma8 frame gives
 *                    the same keypoints through the pixel-format entry as through the f32 entry, and the conversion alone is exact.
 * Build: gcc -std=c11 -Wall -Wextra -Werror abi_smoke_image.c -I../../include -L../../cv_b200 -lcvb200_image -lcvb200 -lcudart */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "cvb200_image.h"

#define CHECK(cond) do { if (!(cond)) { fprintf(stderr, "abi_smoke_image: %s:%d: %s\n", __FILE__, __LINE__, #cond); return 1; } } while (0)

static int no_gpu_checks(void) {
    cvb_ctx *ctx = NULL;
    const int rc = cvb_ctx_create(0, &ctx);
    if (rc == CVB_OK) { cvb_ctx_destroy(ctx); return -1; }      /* a GPU is present: the caller runs mode 1 */
    CHECK(rc == CVB_ENODEV && ctx == NULL);                     /* no CPU fallback */
    cvb_akaze_cfg cfg;
    cvb_akaze_default_cfg(&cfg);
    cvb_arrsac_cfg acfg;
    cvb_arrsac_default_cfg(&acfg, 1e-7);
    cvb_intrinsics_k1 K = {1000, 1000, 16, 16, 0, 0};
    cvb_rng rng;
    cvb_rng_seed_xoshiro256pp(&rng, 0);
    cvb_pose pose;
    uint8_t px[64] = {0}, desc[64];
    float gray[64];
    cvb_keypoint kp[1];
    double bear[3];
    uint32_t n[2], pairs[2], np = 0, ni = 0, inl[1];
    int32_t found = 0;
    CHECK(cvb_gray_float_from_dynamic_dev(NULL, CVB_PIXEL_LUMA8, px, 1, 8, 8, gray, NULL) == CVB_EINVAL);
    CHECK(cvb_akaze_extract_dynamic_batch(NULL, &cfg, CVB_PIXEL_LUMA8, px, 1, 8, 8, kp, desc, 1, n) == CVB_EINVAL);
    CHECK(cvb_akaze_extract_dynamic_batch_dev(NULL, &cfg, CVB_PIXEL_LUMA8, px, 1, 8, 8, kp, desc, 1, n) == CVB_EINVAL);
    CHECK(cvb_frame_features_dynamic_batch(NULL, &cfg, CVB_PIXEL_RGB8, px, 1, 4, 4, &K, kp, desc, bear, px, 1, n) == CVB_EINVAL);
    CHECK(cvb_two_view_frames_dynamic_k1(NULL, &cfg, CVB_PIXEL_LUMA8, px, 4, 4, 25, &K, &acfg, &rng, kp, desc, 1, n, pairs, &np, &pose, inl,
                                         &ni, &found) == CVB_EINVAL);
    return 0;
}

static int gpu_workflow(void) {
    cvb_ctx *ctx = NULL;
    CHECK(cvb_ctx_create(0, &ctx) == CVB_OK);
    cvb_akaze_cfg cfg;
    cvb_akaze_default_cfg(&cfg);
    enum { W = 160, H = 120, CAP = 4096 };
    uint8_t *img = malloc(W * H);
    float *f = malloc(sizeof(float) * W * H);
    for (int y = 0; y < H; y++)
        for (int x = 0; x < W; x++) img[y * W + x] = (uint8_t)((((x / 9) ^ (y / 7)) & 1) ? 200 : 30) + (uint8_t)((x * 7 + y * 13) % 17);
    for (int i = 0; i < W * H; i++) f[i] = (float)img[i] / 255.0f;
    cvb_keypoint *kp_a = malloc(sizeof(cvb_keypoint) * CAP), *kp_b = malloc(sizeof(cvb_keypoint) * CAP);
    uint8_t *d_a = malloc(64 * CAP), *d_b = malloc(64 * CAP);
    uint32_t na = 0, nb = 0;
    CHECK(cvb_akaze_extract_batch(ctx, &cfg, f, 1, W, H, kp_a, d_a, CAP, &na) == CVB_OK);
    CHECK(cvb_akaze_extract_dynamic_batch(ctx, &cfg, CVB_PIXEL_LUMA8, img, 1, W, H, kp_b, d_b, CAP, &nb) == CVB_OK);
    CHECK(na == nb && na > 0 && !memcmp(kp_a, kp_b, sizeof(cvb_keypoint) * na) && !memcmp(d_a, d_b, 64 * (size_t)na));
    /* argument errors */
    CHECK(cvb_akaze_extract_dynamic_batch(ctx, &cfg, 10, img, 1, W, H, kp_b, d_b, CAP, &nb) == CVB_EINVAL);
    CHECK(strlen(cvb_last_error(ctx)) > 0);
    CHECK(cvb_akaze_extract_dynamic_batch(ctx, &cfg, CVB_PIXEL_LUMA8, img, 1, 0, H, kp_b, d_b, CAP, &nb) == CVB_EINVAL);
    CHECK(cvb_akaze_extract_dynamic_batch(ctx, &cfg, CVB_PIXEL_LUMA8, NULL, 1, W, H, kp_b, d_b, CAP, &nb) == CVB_EINVAL);
    CHECK(cvb_akaze_extract_dynamic_batch(ctx, &cfg, CVB_PIXEL_RGB32F, img, 1, W, H, kp_b, d_b, CAP, &nb) == CVB_EUNSUPPORTED);
    CHECK(cvb_akaze_extract_dynamic_batch_dev(ctx, &cfg, CVB_PIXEL_RGBA32F, img, 1, W, H, kp_b, d_b, CAP, &nb) == CVB_EUNSUPPORTED);
    CHECK(cvb_akaze_extract_dynamic_batch_dev(ctx, &cfg, CVB_PIXEL_LUMA8, img, 1, W, H, NULL, d_b, CAP, &nb) == CVB_EINVAL);
    CHECK(cvb_gray_float_from_dynamic_dev(ctx, CVB_PIXEL_LUMA16, img, 1, W, H, NULL, NULL) == CVB_EINVAL);
    CHECK(cvb_gray_float_from_dynamic_dev(ctx, CVB_PIXEL_LUMA16, img, 1, W, H, f, (uint8_t *)f) == CVB_EUNSUPPORTED);
    cvb_intrinsics_k1 K = {1000, 1000, 80, 60, 0, -0.1};
    double *bear = malloc(sizeof(double) * 3 * CAP);
    uint8_t *col = malloc(3 * CAP);
    CHECK(cvb_frame_features_dynamic_batch(ctx, &cfg, CVB_PIXEL_LUMA16, img, 1, W / 2, H, &K, kp_b, d_b, bear, col, CAP, &nb) ==
          CVB_EUNSUPPORTED);
    CHECK(cvb_frame_features_dynamic_batch(ctx, &cfg, CVB_PIXEL_LUMA8, img, 1, W, H, &K, kp_b, d_b, bear, col, CAP, &nb) == CVB_OK);
    CHECK(nb == na && !memcmp(kp_a, kp_b, sizeof(cvb_keypoint) * na));
    cvb_arrsac_cfg acfg;
    cvb_arrsac_default_cfg(&acfg, 1e-7);
    cvb_rng rng;
    cvb_rng_seed_xoshiro256pp(&rng, 0);
    cvb_pose pose;
    uint8_t *two = malloc(2 * W * H);
    memcpy(two, img, W * H); memcpy(two + W * H, img, W * H);
    cvb_keypoint *kp2 = malloc(sizeof(cvb_keypoint) * 2 * CAP);
    uint8_t *d2 = malloc(2 * 64 * CAP);
    uint32_t n2[2], *pairs = malloc(sizeof(uint32_t) * 2 * CAP), *inl = malloc(sizeof(uint32_t) * CAP), np = 0, ni = 0;
    int32_t found = 0;
    CHECK(cvb_two_view_frames_dynamic_k1(ctx, &cfg, CVB_PIXEL_LUMA8, two, W, H, 25, &K, &acfg, &rng, kp2, d2, CAP, n2, pairs, &np, &pose,
                                         inl, &ni, &found) == CVB_OK);
    CHECK(n2[0] == na && n2[1] == na && np > 0 && np <= na);   /* a frame matched with itself */
    CHECK(cvb_two_view_frames_dynamic_k1(ctx, &cfg, 11, two, W, H, 25, &K, &acfg, &rng, kp2, d2, CAP, n2, pairs, &np, &pose, inl, &ni,
                                         &found) == CVB_EINVAL);
    free(img); free(f); free(kp_a); free(kp_b); free(d_a); free(d_b); free(bear); free(col); free(two); free(kp2); free(d2); free(pairs);
    free(inl);
    cvb_ctx_destroy(ctx);
    printf("GPU workflow ok\n");
    return 0;
}

int main(int argc, char **argv) {
    const int mode = argc > 1 ? atoi(argv[1]) : 0;
    if (mode == 0) {
        const int r = no_gpu_checks();
        if (r > 0) return 1;
        printf(r < 0 ? "GPU present: mode 0 skipped\n" : "no-GPU checks ok\n");
        return 0;
    }
    return gpu_workflow();
}
