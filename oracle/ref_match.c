/* oracle/ref_match.c -- TEST INFRASTRUCTURE: CPU restatement of the brute-force matcher.
 *
 * Follows `space::LinearKnn{metric: Hamming, iter}.knn(query, k)` (external crate space 0.17.0)
 * with `bitarray::Hamming` over `BitArray<64>` (external crate bitarray 0.9.0), as called at
 * akaze/tests/estimate_pose.rs:78-97 and tutorial-code/chapter4-feature-matching/
 * src/main.rs:91-106.  Neither crate's source is in the reference checkout; the published algorithm is:
 * distance = sum popcount(a[i]^b[i]) over 64 bytes (u32); knn keeps the k smallest in ascending
 * distance, and among equal distances the EARLIER database index stays first (insert position =
 * partition_point(|n| n.distance <= d)).  Pinned by the reference's own golden: 11 Lowe-ratio
 * matches between res/0000000000.png and res/0000000014.png (estimate_pose.rs:59).
 * Not product code.
 */
#include <stdint.h>
#include <string.h>
#include "ref_akaze.h"

static inline uint32_t hamming64(const uint8_t *a, const uint8_t *b) {
    uint32_t d = 0;
    for (int i = 0; i < 8; i++) {
        uint64_t x, y;
        memcpy(&x, a + 8 * i, 8); memcpy(&y, b + 8 * i, 8);
        d += (uint32_t)__builtin_popcountll(x ^ y);
    }
    return d;
}

/* out[n][k]; when m < k the missing slots hold idx = 0xffffffff, dist = 0xffffffff */
void ref_hamming_knn(const uint8_t *q, uint32_t n, const uint8_t *db, uint32_t m, uint32_t k, uint32_t *idx_out,
                     uint32_t *dist_out) {
#pragma omp parallel for schedule(static)
    for (uint32_t i = 0; i < n; i++) {
        uint32_t *bi = idx_out + (size_t)i * k, *bd = dist_out + (size_t)i * k;
        uint32_t cnt = 0;
        for (uint32_t s = 0; s < k; s++) { bi[s] = 0xffffffffu; bd[s] = 0xffffffffu; }
        for (uint32_t j = 0; j < m; j++) {
            uint32_t d = hamming64(q + (size_t)i * 64, db + (size_t)j * 64);
            /* position after all entries with distance <= d (earlier index wins ties) */
            uint32_t pos = cnt;
            while (pos > 0 && bd[pos - 1] > d) pos--;
            if (pos >= k) continue;
            uint32_t last = cnt < k ? cnt : k - 1;
            for (uint32_t s = last; s > pos; s--) { bi[s] = bi[s - 1]; bd[s] = bd[s - 1]; }
            bi[pos] = j; bd[pos] = d;
            if (cnt < k) cnt++;
        }
    }
}
