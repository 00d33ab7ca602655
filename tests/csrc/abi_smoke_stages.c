/* Test infrastructure: a plain C translation unit against include/cvb200_stages.h that calls EVERY entry point that header declares, so
 * that the prototypes a Rust / cgo / JNI binding transcribes are checked by a C compiler (ctypes never sees the header).
 *   mode 0 (no GPU): context creation reports no device, and every entry point returns CVB_EINVAL for the missing context.
 *   mode 1 (GPU):    a scale space of a synthetic frame; its evolution table; find; describe of the found keypoints equals find's
 *                    keypoints that stay inside their level; a NULL keypoint array, an invalid keypoint and a stale ticket
 *                    give CVB_EINVAL.
 *                    (tests/test_gpu_stages.py holds every result to the oracle and runs the _dev forms on device buffers.)
 * Build: gcc -std=c11 -Wall -Wextra -Werror abi_smoke_stages.c -I../../include -L../../cv_b200 -lcvb200_stages -lcvb200 -lm */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "cvb200_stages.h"

#define CHECK(cond) do { if (!(cond)) { fprintf(stderr, "abi_smoke_stages: %s:%d: %s\n", __FILE__, __LINE__, #cond); return 1; } } while (0)

enum { W = 320, H = 240, CAP = 8192 };
static float img[W * H];
static cvb_keypoint kps[CAP], kout[CAP];
static uint8_t desc[CAP * 64];
static cvb_akaze_evolution evo[64];

static int no_context(void) {
    cvb_akaze_cfg cfg;
    cvb_akaze_default_cfg(&cfg);
    uint64_t t = 0;
    uint32_t n = 0, offs[2] = {0, 0};
    CHECK(cvb_akaze_scale_space(NULL, &cfg, img, 1, W, H, &t) == CVB_EINVAL);
    CHECK(cvb_akaze_scale_space_dev(NULL, &cfg, img, 1, W, H, &t) == CVB_EINVAL);
    CHECK(cvb_akaze_evolutions(NULL, 1, evo, 64, &n) == CVB_EINVAL);
    CHECK(cvb_akaze_find_image_keypoints(NULL, 1, kps, CAP, &n) == CVB_EINVAL);
    CHECK(cvb_akaze_find_image_keypoints_dev(NULL, 1, kps, CAP, &n) == CVB_EINVAL);
    CHECK(cvb_akaze_extract_descriptors(NULL, &cfg, 1, kps, offs, kout, desc, &n) == CVB_EINVAL);
    CHECK(cvb_akaze_extract_descriptors_dev(NULL, &cfg, 1, kps, offs, 0, kout, desc, &n) == CVB_EINVAL);
    return 0;
}

int main(int argc, char **argv) {
    const int gpu = argc > 1 && atoi(argv[1]) == 1;
    for (int y = 0; y < H; y++)
        for (int x = 0; x < W; x++) img[y * W + x] = 0.5f + 0.25f * sinf(0.11f * x) * cosf(0.07f * y) + ((x / 16 + y / 16) & 1 ? 0.2f : 0.f);
    if (no_context()) return 1;
    cvb_ctx *ctx = NULL;
    int rc = cvb_ctx_create(0, &ctx);
    if (!gpu) {
        CHECK(rc == CVB_ENODEV && ctx == NULL);
        printf("no-device checks ok\n");
        return 0;
    }
    CHECK(rc == 0 && ctx);
    cvb_akaze_cfg cfg;
    cvb_akaze_default_cfg(&cfg);
    uint64_t t = 0;
    uint32_t ne = 0, n = 0, m = 0;
    CHECK(cvb_akaze_scale_space(ctx, &cfg, img, 1, W, H, &t) == 0 && t != 0);
    CHECK(cvb_akaze_evolutions(ctx, t, evo, 64, &ne) == 0 && ne > 0 && evo[0].width == W && evo[0].height == H);
    CHECK(cvb_akaze_find_image_keypoints(ctx, t, kps, CAP, &n) == 0 && n > 0);
    uint32_t offs[2] = {0, n};
    CHECK(cvb_akaze_extract_descriptors(ctx, &cfg, t, kps, offs, kout, desc, &m) == 0 && m > 0 && m <= n);
    for (uint32_t i = 0, j = 0; i < m; i++, j++) {   /* the kept keypoints are a subsequence of the input, bit for bit */
        while (j < n && memcmp(&kps[j], &kout[i], sizeof(cvb_keypoint))) j++;
        CHECK(j < n);
    }
    CHECK(cvb_akaze_extract_descriptors(ctx, &cfg, t, NULL, offs, kout, desc, &m) == CVB_EINVAL);
    kps[0].class_id = ne;
    CHECK(cvb_akaze_extract_descriptors(ctx, &cfg, t, kps, offs, kout, desc, &m) == CVB_EINVAL && strstr(cvb_last_error(ctx), "keypoint 0"));
    uint32_t n_ex = 0;
    CHECK(cvb_akaze_extract(ctx, &cfg, img, W, H, kout, desc, CAP, &n_ex) == 0);
    CHECK(cvb_akaze_find_image_keypoints(ctx, t, kps, CAP, &n) == CVB_EINVAL && strstr(cvb_last_error(ctx), "scale space replaced"));
    cvb_ctx_destroy(ctx);
    printf("GPU workflow ok: %u evolutions, %u keypoints found\n", ne, offs[1]);
    return 0;
}
