/* oracle/ref_lsh.c -- TEST INFRASTRUCTURE: CPU restatement of include/cvb200_lsh.h's search, the exact form of cv-sfm's
 * `lsh_to_frame.knn_values(&lsh, num)` (cv-sfm/src/lib.rs:597-668) over frame hashes of 32 * words bits.
 *
 * Follows `space::LinearKnn{metric: Hamming, iter}.knn(query, k)` (external crate space 0.17.0) over `BitArray<4 * words>` (external
 * crate bitarray 0.9.0): distance = sum popcount(a[i] ^ b[i]) over the code's 32-bit words; the database is walked in index order and
 * each item is inserted at partition_point(|n| n.distance <= d), so among equal distances the EARLIER index stays first, and the list
 * is cut to k.  Parity with the reference is unpinned: LinearKnn sorts its first k items with sort_unstable_by_key, which leaves tied
 * items beyond k = 20 in pdqsort's order; this restatement orders them by index, and defines the result.  Not product code.
 */
#include <stdint.h>
#include <string.h>

static inline uint32_t hamming_words(const uint8_t *a, const uint8_t *b, uint32_t words) {
    uint32_t d = 0;
    for (uint32_t i = 0; i < words; i++) {
        uint32_t x, y;
        memcpy(&x, a + 4 * (size_t)i, 4); memcpy(&y, b + 4 * (size_t)i, 4);
        d += (uint32_t)__builtin_popcount(x ^ y);
    }
    return d;
}

/* codes are 4 * words bytes; out[n][k]; when m < k the missing slots hold idx = dist = 0xffffffff */
void ref_hash_knn(uint32_t words, const uint8_t *q, uint32_t n, const uint8_t *db, uint32_t m, uint32_t k, uint32_t *idx_out,
                  uint32_t *dist_out) {
    const size_t row = 4 * (size_t)words;
#pragma omp parallel for schedule(dynamic, 1)
    for (uint32_t i = 0; i < n; i++) {
        uint32_t *bi = idx_out + (size_t)i * k, *bd = dist_out + (size_t)i * k;
        uint32_t cnt = 0;
        for (uint32_t s = 0; s < k; s++) { bi[s] = 0xffffffffu; bd[s] = 0xffffffffu; }
        for (uint32_t j = 0; j < m; j++) {
            const uint32_t d = hamming_words(q + (size_t)i * row, db + (size_t)j * row, words);
            uint32_t pos = cnt;   /* partition_point(|n| n.distance <= d) */
            while (pos > 0 && bd[pos - 1] > d) pos--;
            if (pos >= k) continue;
            const uint32_t last = cnt < k ? cnt : k - 1;
            for (uint32_t s = last; s > pos; s--) { bi[s] = bi[s - 1]; bd[s] = bd[s - 1]; }
            bi[pos] = j; bd[pos] = d;
            if (cnt < k) cnt++;
        }
    }
}
