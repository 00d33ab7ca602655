// cv_b200/csrc/lsh_abi.cu -- libcvb200_lsh.so, the module that exports the C ABI of include/cvb200_lsh.h (exact Hamming k-NN over wide
// codes: cv-sfm's similar-frame search).  The kernels and their host code live in lsh.cu inside libcvb200.so; this module only gives
// them their C names, so that libcvb200.so's own exports stay exactly those of cvb200.h, cvb200_sfm.h and cvb200_tri.h.  It links
// libcvb200.so (rpath $ORIGIN) and takes that library's contexts.
#include "../../include/cvb200_lsh.h"

int lsh_hash_knn(cvb_ctx *ctx, uint32_t words, const uint8_t *queries, uint32_t n, const uint8_t *database, uint32_t m, uint32_t k,
                 uint32_t *idx_out, uint32_t *dist_out);
int lsh_hash_knn_dev(cvb_ctx *ctx, uint32_t words, const uint8_t *queries_dev, const uint32_t *n_dev, uint32_t n_max,
                     const uint8_t *database_dev, const uint32_t *m_dev, uint32_t m_max, uint32_t k, uint32_t *idx_out_dev,
                     uint32_t *dist_out_dev);

extern "C" {

int cvb_hash_knn(cvb_ctx *ctx, uint32_t words, const uint8_t *queries, uint32_t n, const uint8_t *database, uint32_t m, uint32_t k,
                 uint32_t *idx_out, uint32_t *dist_out) {
    return lsh_hash_knn(ctx, words, queries, n, database, m, k, idx_out, dist_out);
}

int cvb_hash_knn_dev(cvb_ctx *ctx, uint32_t words, const uint8_t *queries_dev, const uint32_t *n_dev, uint32_t n_max,
                     const uint8_t *database_dev, const uint32_t *m_dev, uint32_t m_max, uint32_t k, uint32_t *idx_out_dev,
                     uint32_t *dist_out_dev) {
    return lsh_hash_knn_dev(ctx, words, queries_dev, n_dev, n_max, database_dev, m_dev, m_max, k, idx_out_dev, dist_out_dev);
}

}  // extern "C"
