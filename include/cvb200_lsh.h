/* include/cvb200_lsh.h -- C ABI of the similar-frame search on the device: exact Hamming k-NN over wide binary codes, such as the
 * bag-of-words frame hashes cvb_hash_bag(_dev) makes.
 *
 *   cvb_hash_knn(_dev)   <- `lsh_to_frame.knn_values(&lsh, num)` in cv-sfm's find_visually_similar_and_recent_frames
 *                           (cv-sfm/src/lib.rs:597-668; lsh_to_frame is HggLite<Hamming, BitArray<512>, FrameKey>, lib.rs:207),
 *                           answered exactly, as space::LinearKnn { metric: Hamming, iter } on BitArray<4 * words> would
 *
 * Library: libcvb200_lsh.so, a module over libcvb200.so that takes its contexts (link with -lcvb200_lsh -lcvb200).  The conventions of
 * include/cvb200.h hold: return codes, HOST pointers unless the name ends in _dev, asynchronous _dev variants on the context's stream,
 * no CPU fallback (no device: no context, CVB_ENODEV).  The calls are stateless: the caller owns the database buffer.
 *
 * Codes: row r of an array of codes is 4 * words bytes at r * 4 * words, little-endian 32-bit words (the byte layout cvb_hash_bag
 * writes: bit i of the code is bit i & 7 of byte i >> 3).
 *
 * Semantics:
 *   - distance = popcount(q XOR d) over all 32 * words bits;
 *   - row q of the output lists the k nearest database rows in ascending distance, and among equal distances the LOWER database index
 *     first (the rule of cvb_hamming_knn); exact and deterministic for any number of ties;
 *   - when the database holds m < k codes, slots m .. k - 1 hold 0xffffffff in both idx and dist.
 *   Parity with the reference is UNPINNED: cv-sfm searches an approximate HGG, and LinearKnn orders its first k items with
 *   sort_unstable_by_key, which leaves the order of tied items beyond k = 20 to pdqsort.  The CPU restatement oracle/ref_lsh.c, with
 *   index-ordered ties, defines the result.
 *
 * Limits: 1 <= words <= CVB_LSH_MAX_WORDS (cvb_hash_bag's ncode / 32: every hash it makes can be searched; cv-sfm's 4096-codeword
 * table gives words = 128), 1 <= k <= CVB_LSH_MAX_K, m < 2^32 - 1, no NULL array, and every device array 16-byte aligned (host
 * arrays are copied and may have any alignment).  Anything else is CVB_EINVAL.  n = 0 writes nothing; m = 0 fills the n rows with 0xffffffff.
 *
 * Device counts (cvb_hash_knn_dev): n_dev / m_dev point to device u32 counts; the call searches min(*n_dev, n_max) queries against
 * min(*m_dev, m_max) codes.  NULL means n_max / m_max.  Output rows at or beyond the query count are left untouched; idx_out_dev and
 * dist_out_dev hold n_max x k u32 each.  The buffers are sized (and the work planned) from n_max and m_max.
 *
 * A device-resident add-frame, as cv-sfm's VSlam::add_frame does it (insert, then search, so the frame finds itself at distance 0),
 * composes two existing calls over a database buffer of capacity x 4 * words bytes and a device count m:
 *   1. cvb_hash_bag_dev(ctx, desc_dev, n_desc_dev, n_max, codewords_dev, 32 * words, database_dev + m * 4 * words);
 *   2. cvb_hash_knn_dev(ctx, words, database_dev + m * 4 * words, NULL, 1, database_dev, m_dev, capacity, k, idx_dev, dist_dev)
 *      with *m_dev = m + 1 (the caller advances its count on the device or the host).
 * Both run on the context's stream, so no host synchronisation is needed between them. */
#ifndef CVB200_LSH_H
#define CVB200_LSH_H
#include "cvb200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* the widest code: 128 words = 4096 bits, cv-sfm's frame hash */
#define CVB_LSH_MAX_WORDS 128
/* the most neighbours per query (cv-sfm's default tracking_similar_frame_search_num is 512) */
#define CVB_LSH_MAX_K 1024

/* host buffers: queries [n][4 * words] bytes, database [m][4 * words] bytes, idx_out / dist_out [n][k] */
int cvb_hash_knn(cvb_ctx *ctx, uint32_t words, const uint8_t *queries, uint32_t n, const uint8_t *database, uint32_t m, uint32_t k,
                 uint32_t *idx_out, uint32_t *dist_out);

/* device buffers; n_dev / m_dev may be NULL (use n_max / m_max) */
int cvb_hash_knn_dev(cvb_ctx *ctx, uint32_t words, const uint8_t *queries_dev, const uint32_t *n_dev, uint32_t n_max,
                     const uint8_t *database_dev, const uint32_t *m_dev, uint32_t m_max, uint32_t k, uint32_t *idx_out_dev,
                     uint32_t *dist_out_dev);

#ifdef __cplusplus
}
#endif
#endif /* CVB200_LSH_H */
