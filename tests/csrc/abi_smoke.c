/* Test infrastructure: a plain C translation unit against include/cvb200.h that calls EVERY entry point the header declares, so that
 * the prototypes a Rust / cgo / JNI binding transcribes are checked by a C compiler (ctypes never sees the header).
 *   mode 0 (no GPU): argument validation only -- every call must return an error code or a defined value, never crash.
 *   mode 1 (GPU):    a small real workflow (extract -> match -> consensus -> triangulate) with sanity checks on the results.
 * Build: gcc -std=c11 -Wall -Wextra -Werror abi_smoke.c -I../../include -L../../cv_b200 -lcvb200 -lm */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "cvb200.h"

#define CHECK(cond) do { if (!(cond)) { fprintf(stderr, "abi_smoke: %s:%d: %s\n", __FILE__, __LINE__, #cond); return 1; } } while (0)

static int no_gpu_checks(void) {
    cvb_ctx *ctx = NULL;
    int rc = cvb_ctx_create(0, &ctx);
    if (rc == CVB_OK) { cvb_ctx_destroy(ctx); return -1; }      /* a GPU is present: the caller runs mode 1 */
    CHECK(rc == CVB_ENODEV && ctx == NULL);                     /* no CPU fallback */
    CHECK(cvb_ctx_create_on_stream(0, NULL, &ctx) == CVB_ENODEV);
    cvb_ctx_destroy(NULL);
    CHECK(cvb_ctx_sync(NULL) == CVB_EINVAL);
    CHECK(cvb_last_error(NULL) != NULL && strstr(cvb_version(), "sm_90a") != NULL);
    CHECK(cvb_ctx_launch_count(NULL) == 0);
    float ms;
    CHECK(cvb_ctx_timer_begin(NULL) == CVB_EINVAL && cvb_ctx_timer_end(NULL, &ms) == CVB_EINVAL);
    char buf[16];
    CHECK(cvb_ctx_profile(NULL, 1) == CVB_EINVAL && cvb_ctx_profile_report(NULL, buf, sizeof buf) == CVB_EINVAL);
    cvb_akaze_cfg ac;
    cvb_akaze_default_cfg(&ac);
    CHECK(ac.num_sublevels == 4 && ac.detector_threshold == 0.001 && ac.descriptor_pattern_size == 10);
    float img[16] = {0};
    cvb_keypoint kp[4];
    uint8_t desc[4 * 64];
    uint32_t n = 0, u[16];
    CHECK(cvb_akaze_extract(NULL, &ac, img, 4, 4, kp, desc, 4, &n) == CVB_EINVAL);
    CHECK(cvb_akaze_extract_batch(NULL, &ac, img, 1, 4, 4, kp, desc, 4, &n) == CVB_EINVAL);
    CHECK(cvb_akaze_extract_batch_dev(NULL, &ac, img, 1, 4, 4, kp, desc, 4, &n) == CVB_EINVAL);
    CHECK(cvb_akaze_dev_overflow(NULL, &n) == CVB_EINVAL);
    CHECK(cvb_akaze_debug_num_evolutions(NULL, &n) == CVB_EINVAL);
    CHECK(cvb_akaze_debug_evolution(NULL, 0, u, u + 1, u + 2, u + 3, u + 4) == CVB_EINVAL);
    CHECK(cvb_akaze_debug_plane(NULL, 0, 0, 0, img) == CVB_EINVAL);
    double d[64] = {0};
    CHECK(cvb_akaze_debug_contrast(NULL, 0, d) == CVB_EINVAL);
    CHECK(cvb_akaze_debug_stage(NULL, 0, 0, kp, 4, &n) == CVB_EINVAL);
    CHECK(cvb_hamming_knn(NULL, desc, 1, desc, 1, 1, u, u + 1) == CVB_EINVAL);
    CHECK(cvb_hamming_knn_dev(NULL, desc, 1, desc, 1, 1, u, u + 1) == CVB_EINVAL);
    CHECK(cvb_hamming_knn_dev_counts(NULL, desc, &n, 1, desc, &n, 1, 1, u, u + 1) == CVB_EINVAL);
    CHECK(cvb_match_symmetric(NULL, desc, 2, desc, 2, 24, u, 2, &n) == CVB_EINVAL);
    CHECK(cvb_match_symmetric_dev(NULL, desc, 2, desc, 2, 24, u) == CVB_EINVAL);
    CHECK(cvb_hash_bag(NULL, desc, 1, desc, 32, desc) == CVB_EINVAL && cvb_hash_bag_dev(NULL, desc, &n, 1, desc, 32, desc) == CVB_EINVAL);
    CHECK(cvb_match_symmetric_pairs_dev(NULL, desc, &n, 2, desc, &n, 2, 24, u, 2, &n) == CVB_EINVAL);
    cvb_arrsac_cfg rc_;
    cvb_arrsac_default_cfg(&rc_, 1e-7);
    CHECK(rc_.initialization_hypotheses == 256 && rc_.block_size == 64 && rc_.inlier_threshold == 1e-7);
    cvb_rng rng, rng2;
    cvb_rng_seed_xoshiro256pp(&rng, 0);
    const uint32_t first = cvb_rng_next_u32(&rng);
    cvb_rng_seed_xoshiro256pp(&rng2, 0);
    CHECK(cvb_rng_next_u32(&rng2) == first);                    /* deterministic */
    uint8_t seed[32];
    memset(seed, 1, sizeof seed);
    cvb_rng_seed_pcg64(&rng2, seed);
    (void)cvb_rng_next_u32(&rng2);
    cvb_pose pose;
    uint8_t np8;
    int32_t found;
    CHECK(cvb_eight_point_batch(NULL, d, d, 8, u, 1, &pose, &np8) == CVB_EINVAL);
    CHECK(cvb_p3p_batch(NULL, d, d, 3, u, 1, &pose, &np8) == CVB_EINVAL);
    CHECK(cvb_five_point_batch(NULL, d, d, 5, u, 1, 5, &pose, &np8) == CVB_EINVAL);
    CHECK(cvb_residuals_camera_to_camera(NULL, &pose, 1, d, d, 1, d) == CVB_EINVAL);
    CHECK(cvb_residuals_world_to_camera(NULL, &pose, 1, d, d, 1, d) == CVB_EINVAL);
    CHECK(cvb_triangulate_linear_eigen(NULL, &pose, d, u, 1, d, &np8) == CVB_EINVAL);
    CHECK(cvb_arrsac_eight_point(NULL, &rc_, d, d, 8, &rng, &pose, u, 8, &n, &found) == CVB_EINVAL);
    CHECK(cvb_arrsac_five_point(NULL, &rc_, d, d, 8, &rng, 5, &pose, u, 8, &n, &found) == CVB_EINVAL);
    CHECK(cvb_arrsac_p3p(NULL, &rc_, d, d, 8, &rng, &pose, u, 8, &n, &found) == CVB_EINVAL);
    cvb_intrinsics K = {1000.0, 1000.0, 960.0, 540.0, 0.0};
    CHECK(cvb_pair_bearings_dev(NULL, kp, kp, u, &n, 4, &K, d, d) == CVB_EINVAL);
    CHECK(cvb_arrsac_eight_point_dev(NULL, &rc_, d, d, &n, 8, &rng, &pose, u, 8, &n, &found) == CVB_EINVAL);
    CHECK(cvb_arrsac_p3p_dev(NULL, &rc_, d, d, &n, 8, &rng, &pose, u, 8, &n, &found) == CVB_EINVAL);
    CHECK(cvb_arrsac_commit_rng(NULL, &rng, u) == CVB_EINVAL);
    CHECK(cvb_two_view_pair_dev(NULL, kp, desc, &n, kp, desc, &n, 4, 24, &K, &rc_, &rng, u, 4, &n, &pose, u, &n, &found) == CVB_EINVAL);
    CHECK(cvb_two_view_frames(NULL, &ac, img, 4, 4, 24, &K, &rc_, &rng, kp, desc, 4, u, u, &n, &pose, u, &n, &found) == CVB_EINVAL);
    CHECK(cvb_single_view_optimize_l2(NULL, &pose, 1, 0.1, 10, d, d, u, &pose, u) == CVB_EINVAL);
    CHECK(cvb_three_view_optimize_l2(NULL, &pose, 1, 0, 0.1, 10, d, u, &pose, u) == CVB_EINVAL);
    CHECK(cvb_observation_losses(NULL, &pose, d, u, 1, d) == CVB_EINVAL);
    CHECK(cvb_tri_landmarks_robust(NULL, &pose, &pose, d, 1, 1e-5, 1e-3, &np8) == CVB_EINVAL);
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
    cvb_keypoint *kp = (cvb_keypoint *)malloc(sizeof(cvb_keypoint) * 2 * cap);
    uint8_t *desc = (uint8_t *)malloc((size_t)2 * cap * 64);
    uint32_t n[2] = {0, 0};
    CHECK(cvb_akaze_extract_batch(ctx, &ac, frames, 2, (uint32_t)w, (uint32_t)h, kp, desc, cap, n) == CVB_OK);
    CHECK(n[0] > 20 && n[1] > 20 && n[0] <= cap);
    uint32_t n1 = 0;
    CHECK(cvb_akaze_extract(ctx, &ac, frames, (uint32_t)w, (uint32_t)h, kp, desc, cap, &n1) == CVB_OK && n1 == n[0]);
    uint32_t *pairs = (uint32_t *)malloc(sizeof(uint32_t) * 2 * cap), npairs = 0;
    CHECK(cvb_match_symmetric(ctx, desc, n[0], desc + (size_t)cap * 64, n[1], 24, pairs, cap, &npairs) == CVB_OK);
    uint32_t idx[2], dist[2];
    CHECK(cvb_hamming_knn(ctx, desc, 1, desc, n[0], 2, idx, dist) == CVB_OK && idx[0] == 0 && dist[0] == 0 && dist[1] >= dist[0]);
    /* the fused entry point returns the same features and matches */
    cvb_intrinsics K = {300.0, 300.0, 160.0, 120.0, 0.0};
    cvb_arrsac_cfg rc_;
    cvb_arrsac_default_cfg(&rc_, 1e-6);
    cvb_rng rng;
    cvb_rng_seed_xoshiro256pp(&rng, 0);
    cvb_keypoint *kp2 = (cvb_keypoint *)malloc(sizeof(cvb_keypoint) * 2 * cap);
    uint8_t *desc2 = (uint8_t *)malloc((size_t)2 * cap * 64);
    uint32_t *pairs2 = (uint32_t *)malloc(sizeof(uint32_t) * 2 * cap), *inl = (uint32_t *)malloc(sizeof(uint32_t) * cap);
    uint32_t n2[2], npairs2 = 0, ninl = 0;
    int32_t found = 0;
    cvb_pose model;
    CHECK(cvb_two_view_frames(ctx, &ac, frames, (uint32_t)w, (uint32_t)h, 24, &K, &rc_, &rng, kp2, desc2, cap, n2, pairs2, &npairs2, &model,
                              inl, &ninl, &found) == CVB_OK);
    CHECK(n2[0] == n[0] && n2[1] == n[1] && npairs2 == npairs);
    CHECK(memcmp(pairs, pairs2, sizeof(uint32_t) * 2 * npairs) == 0 && memcmp(desc, desc2, (size_t)n[0] * 64) == 0);
    CHECK(ninl <= npairs && (found == 0 || found == 1));
    /* a synthetic two-view scene through the consensus entry point: the identity rotation + x translation */
    enum { N = 200 };
    double a[3 * N], b[3 * N];
    for (int i = 0; i < N; i++) {
        double X = -2.0 + 4.0 * ((i * 37) % N) / N, Y = -1.5 + 3.0 * ((i * 91) % N) / N, Z = 4.0 + 3.0 * ((i * 53) % N) / N;
        double na = sqrt(X * X + Y * Y + Z * Z), Xb = X + 0.5, nb = sqrt(Xb * Xb + Y * Y + Z * Z);
        a[3 * i] = X / na; a[3 * i + 1] = Y / na; a[3 * i + 2] = Z / na;
        b[3 * i] = Xb / nb; b[3 * i + 1] = Y / nb; b[3 * i + 2] = Z / nb;
    }
    uint32_t inl2[N], cnt = 0;
    cvb_rng_seed_xoshiro256pp(&rng, 1);
    CHECK(cvb_arrsac_eight_point(ctx, &rc_, a, b, N, &rng, &model, inl2, N, &cnt, &found) == CVB_OK);
    CHECK(found == 1 && cnt > N / 2);
    CHECK(fabs(fabs(model.t[0]) - 1.0) < 1e-6 && fabs(model.r[0] - 1.0) < 1e-6);      /* unit translation along x, identity rotation */
    double res[N];
    CHECK(cvb_residuals_camera_to_camera(ctx, &model, 1, a, b, N, res) == CVB_OK);
    for (uint32_t i = 0; i < cnt; i++) CHECK(res[inl2[i]] < 1e-6);
    /* triangulate landmark 0 from the two views */
    cvb_pose views[2] = {{{1, 0, 0, 0, 1, 0, 0, 0, 1}, {0, 0, 0}}, model};
    double bear[6] = {a[0], a[1], a[2], b[0], b[1], b[2]}, xyzw[4];
    uint32_t off[2] = {0, 2};
    uint8_t ok = 0;
    CHECK(cvb_triangulate_linear_eigen(ctx, views, bear, off, 1, xyzw, &ok) == CVB_OK);
    CHECK(cvb_ctx_sync(ctx) == CVB_OK && cvb_ctx_launch_count(ctx) > 0);
    cvb_ctx_destroy(ctx);
    free(frames); free(kp); free(desc); free(pairs); free(kp2); free(desc2); free(pairs2); free(inl);
    return 0;
}

int main(int argc, char **argv) {
    const int mode = argc > 1 ? atoi(argv[1]) : 0;
    if (mode == 0) {
        const int r = no_gpu_checks();
        if (r < 0) { printf("abi_smoke: GPU present, skipping the no-GPU checks\n"); return 0; }
        if (r == 0) printf("abi_smoke: every entry point rejects a null context / reports no device\n");
        return r;
    }
    const int r = gpu_workflow();
    if (r == 0) printf("abi_smoke: GPU workflow ok\n");
    return r;
}
