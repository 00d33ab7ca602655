/* Test infrastructure: a plain C translation unit against include/cvb200_lsh.h that calls EVERY entry point that header declares, so
 * that the prototypes a Rust / cgo / JNI binding transcribes are checked by a C compiler (ctypes never sees the header).
 *   mode 0 (no GPU): context creation reports no device; every entry point returns CVB_EINVAL for words 0 and 129, k 0 and 1025, NULL
 *                    arrays, misaligned device arrays (and for the missing context).
 *   mode 1 (GPU):    the same argument errors on a live context, with a message; then a small search equals a brute force written
 *                    here (ascending distance, lower index first, 0xffffffff past m), and m = 0 fills every slot with 0xffffffff.
 *                    (tests/test_gpu_lsh.py runs the _dev form on device buffers.)
 * Build: gcc -std=c11 -Wall -Wextra -Werror abi_smoke_lsh.c -I../../include -L../../cv_b200 -lcvb200_lsh -lcvb200 */
#include <stdalign.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "cvb200_lsh.h"

#define CHECK(cond) do { if (!(cond)) { fprintf(stderr, "abi_smoke_lsh: %s:%d: %s\n", __FILE__, __LINE__, #cond); return 1; } } while (0)

enum { WORDS = 3, N = 3, M = 100, KMAX = 130 };
static alignas(16) uint32_t q[N * WORDS], db[M * WORDS], idx[N * KMAX + 4], dist[N * KMAX + 4];

/* every argument error, on ctx (NULL in mode 0) */
static int argument_errors(cvb_ctx *ctx) {
    const uint8_t *qb = (const uint8_t *)q, *dbb = (const uint8_t *)db;
    CHECK(cvb_hash_knn(ctx, 0, qb, N, dbb, M, 4, idx, dist) == CVB_EINVAL);
    CHECK(cvb_hash_knn(ctx, CVB_LSH_MAX_WORDS + 1, qb, N, dbb, M, 4, idx, dist) == CVB_EINVAL);
    CHECK(cvb_hash_knn(ctx, WORDS, qb, N, dbb, M, 0, idx, dist) == CVB_EINVAL);
    CHECK(cvb_hash_knn(ctx, WORDS, qb, N, dbb, M, CVB_LSH_MAX_K + 1, idx, dist) == CVB_EINVAL);
    CHECK(cvb_hash_knn(ctx, WORDS, NULL, N, dbb, M, 4, idx, dist) == CVB_EINVAL);
    CHECK(cvb_hash_knn(ctx, WORDS, qb, N, NULL, M, 4, idx, dist) == CVB_EINVAL);
    CHECK(cvb_hash_knn(ctx, WORDS, qb, N, dbb, M, 4, NULL, dist) == CVB_EINVAL);
    CHECK(cvb_hash_knn(ctx, WORDS, qb, N, dbb, M, 4, idx, NULL) == CVB_EINVAL);
    CHECK(cvb_hash_knn(ctx, WORDS, qb, N, dbb, 0xffffffffu, 4, idx, dist) == CVB_EINVAL);
    CHECK(cvb_hash_knn_dev(ctx, 0, qb, NULL, N, dbb, NULL, M, 4, idx, dist) == CVB_EINVAL);
    CHECK(cvb_hash_knn_dev(ctx, CVB_LSH_MAX_WORDS + 1, qb, NULL, N, dbb, NULL, M, 4, idx, dist) == CVB_EINVAL);
    CHECK(cvb_hash_knn_dev(ctx, WORDS, qb, NULL, N, dbb, NULL, M, 0, idx, dist) == CVB_EINVAL);
    CHECK(cvb_hash_knn_dev(ctx, WORDS, qb, NULL, N, dbb, NULL, M, CVB_LSH_MAX_K + 1, idx, dist) == CVB_EINVAL);
    CHECK(cvb_hash_knn_dev(ctx, WORDS, NULL, NULL, N, dbb, NULL, M, 4, idx, dist) == CVB_EINVAL);
    CHECK(cvb_hash_knn_dev(ctx, WORDS, qb, NULL, N, NULL, NULL, M, 4, idx, dist) == CVB_EINVAL);
    CHECK(cvb_hash_knn_dev(ctx, WORDS, qb, NULL, N, dbb, NULL, M, 4, NULL, dist) == CVB_EINVAL);
    CHECK(cvb_hash_knn_dev(ctx, WORDS, qb, NULL, N, dbb, NULL, M, 4, idx, NULL) == CVB_EINVAL);
    CHECK(cvb_hash_knn_dev(ctx, WORDS, qb + 8, NULL, N, dbb, NULL, M, 4, idx, dist) == CVB_EINVAL);
    CHECK(cvb_hash_knn_dev(ctx, WORDS, qb, NULL, N, dbb + 12, NULL, M, 4, idx, dist) == CVB_EINVAL);
    CHECK(cvb_hash_knn_dev(ctx, WORDS, qb, NULL, N, dbb, NULL, M, 4, idx, dist + 2) == CVB_EINVAL);
    if (ctx) CHECK(strlen(cvb_last_error(ctx)) > 0);
    return 0;
}

static int no_gpu_checks(void) {
    cvb_ctx *ctx = NULL;
    const int rc = cvb_ctx_create(0, &ctx);
    if (rc == CVB_OK) { cvb_ctx_destroy(ctx); return -1; }      /* a GPU is present: the caller runs mode 1 */
    CHECK(rc == CVB_ENODEV && ctx == NULL);                     /* no CPU fallback */
    return argument_errors(NULL);
}

static uint32_t hamming(const uint32_t *a, const uint32_t *b) {
    uint32_t d = 0;
    for (int w = 0; w < WORDS; w++) d += (uint32_t)__builtin_popcount(a[w] ^ b[w]);
    return d;
}

/* row i of (idx, dist) for k: insertion at the partition point, so equal distances keep ascending index */
static int check_row(int i, uint32_t k) {
    uint32_t bi[KMAX], bd[KMAX], cnt = 0;
    for (uint32_t j = 0; j < M; j++) {
        const uint32_t d = hamming(q + i * WORDS, db + j * WORDS);
        uint32_t pos = cnt;
        while (pos > 0 && bd[pos - 1] > d) pos--;
        if (pos >= k) continue;
        for (uint32_t s = (cnt < k ? cnt : k - 1); s > pos; s--) { bi[s] = bi[s - 1]; bd[s] = bd[s - 1]; }
        bi[pos] = j; bd[pos] = d;
        if (cnt < k) cnt++;
    }
    for (uint32_t s = 0; s < k; s++) {
        CHECK(idx[i * k + s] == (s < cnt ? bi[s] : 0xffffffffu));
        CHECK(dist[i * k + s] == (s < cnt ? bd[s] : 0xffffffffu));
    }
    return 0;
}

static int gpu_workflow(void) {
    cvb_ctx *ctx = NULL;
    CHECK(cvb_ctx_create(0, &ctx) == CVB_OK);
    if (argument_errors(ctx)) return 1;
    uint32_t s = 12345u;
    for (int i = 0; i < M * WORDS; i++) { s = s * 1664525u + 1013904223u; db[i] = s & 0x0f0f0f0fu; }   /* few distinct distances: ties */
    for (int i = 0; i < N * WORDS; i++) { s = s * 1664525u + 1013904223u; q[i] = s & 0x0f0f0f0fu; }
    memcpy(db + 7 * WORDS, q, sizeof(uint32_t) * WORDS);                                             /* query 0 is row 7: distance 0 */
    const uint32_t ks[3] = {1, 8, KMAX};
    for (int t = 0; t < 3; t++) {
        CHECK(cvb_hash_knn(ctx, WORDS, (const uint8_t *)q, N, (const uint8_t *)db, M, ks[t], idx, dist) == CVB_OK);
        for (int i = 0; i < N; i++)
            if (check_row(i, ks[t])) return 1;
        CHECK(idx[0] == 7 && dist[0] == 0);
    }
    CHECK(cvb_hash_knn(ctx, WORDS, (const uint8_t *)q, N, (const uint8_t *)db, 0, 4, idx, dist) == CVB_OK);
    for (int i = 0; i < N * 4; i++) CHECK(idx[i] == 0xffffffffu && dist[i] == 0xffffffffu);
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
