// cv_b200/csrc/match.cu -- brute-force Hamming k-NN over 64-byte descriptors (sm_90a).
//
// Replaces `space::LinearKnn{metric: bitarray::Hamming, iter}.knn(query, k)` (external crates space 0.17 /
// bitarray 0.9; call sites akaze/tests/estimate_pose.rs:78-97, tutorial-code/
// chapter4-feature-matching/src/main.rs:91-106, cv-sfm/src/lib.rs:3097-3114) for ALL queries at once.
// Semantics kept bit-exact: distance = popcount(a ^ b) over 512 bits; the k smallest in ascending
// distance; among equal distances the lower database index comes first.
//
// Kernel: one query per thread held in registers (8 x u64); the database streams through shared memory
// in 8 KB tiles fetched by the TMA engine (cp.async.bulk + mbarrier, double buffered) and is read by all
// threads at the same address (broadcast).  (distance, index) is packed into one 32-bit key
// (distance << 22 | local index) so the running best-k is maintained with integer min/max only.  The
// database is split across gridDim.y so that the grid covers all SMs; a second small kernel merges the
// per-split lists in index order.  The bound is the integer popc pipe, not HBM (working set is L2 resident).
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <vector>
#include "common.cuh"

namespace {

constexpr int QT = 128;          // queries per CTA (1 per thread)
constexpr int DTILE = 128;       // database descriptors per shared-memory tile (8 KB)
constexpr int MAXKNN = 8;
#ifndef CVB_KNN_DEFAULT_MODE
#define CVB_KNN_DEFAULT_MODE 2     // 1: mma.sync int8, 2: wgmma (CVB_KNN_WGMMA=1 / =0 override at run time)
#endif
constexpr unsigned IDX_BITS = 22;
constexpr unsigned IDX_MASK = (1u << IDX_BITS) - 1u;

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, unsigned phase) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(phase) : "memory");
}
// 1-D bulk copy global -> shared through the TMA unit, completion signalled on an mbarrier
__device__ __forceinline__ void tma_load_1d(void *dst, const void *src, unsigned bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

template <int K>
__device__ __forceinline__ void insert_key(uint32_t (&best)[K], uint32_t key) {
#pragma unroll
    for (int i = 0; i < K; i++) {
        uint32_t lo = min(best[i], key);
        key = max(best[i], key);
        best[i] = lo;
    }
}

// grid = (ceil(n_max/QT), splits); partial[(q * splits + s) * K + i] = key with split-local index
template <int K>
__global__ void __launch_bounds__(QT) k_hamming_knn(const uint8_t *__restrict__ queries, const uint32_t *__restrict__ n_dev,
                                                    uint32_t n_host, const uint8_t *__restrict__ db,
                                                    const uint32_t *__restrict__ m_dev, uint32_t m_host, uint32_t chunk,
                                                    uint32_t *__restrict__ partial) {
    __shared__ __align__(128) uint8_t s_db[2][DTILE * 64];
    __shared__ __align__(8) uint64_t s_bar[2];
    const uint32_t n = n_dev ? min(*n_dev, n_host) : n_host, m = m_dev ? min(*m_dev, m_host) : m_host;
    const uint32_t q = blockIdx.x * QT + threadIdx.x;
    if (blockIdx.x * QT >= n) return;
    const uint32_t lo = min(blockIdx.y * chunk, m), hi = min(lo + chunk, m);
    const uint32_t cnt = hi - lo;
    uint64_t qa[8];
    {
        const uint4 *p = (const uint4 *)(queries + (size_t)min(q, n - 1) * 64);
#pragma unroll
        for (int i = 0; i < 4; i++) {
            uint4 v = p[i];
            qa[2 * i] = ((uint64_t)v.y << 32) | v.x;
            qa[2 * i + 1] = ((uint64_t)v.w << 32) | v.z;
        }
    }
    uint32_t best[K];
#pragma unroll
    for (int i = 0; i < K; i++) best[i] = 0xffffffffu;
    const uint32_t ntiles = (cnt + DTILE - 1) / DTILE;
    if (threadIdx.x == 0) {
        mbar_init(&s_bar[0], 1);
        mbar_init(&s_bar[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    auto issue = [&](uint32_t t) {
        const uint32_t first = t * DTILE, rows = min((uint32_t)DTILE, cnt - first), bytes = rows * 64u;
        mbar_expect_tx(&s_bar[t & 1], bytes);
        tma_load_1d(s_db[t & 1], db + (size_t)(lo + first) * 64, bytes, &s_bar[t & 1]);
    };
    if (threadIdx.x == 0) {
        if (ntiles > 0) issue(0);
        if (ntiles > 1) issue(1);
    }
    for (uint32_t t = 0; t < ntiles; t++) {
        mbar_wait(&s_bar[t & 1], (t >> 1) & 1);
        const uint32_t first = t * DTILE, rows = min((uint32_t)DTILE, cnt - first);
        const uint64_t *tile = (const uint64_t *)s_db[t & 1];
#pragma unroll 4
        for (uint32_t r = 0; r < rows; r++) {
            const ulonglong2 *d = (const ulonglong2 *)(tile + r * 8);
            uint32_t dist = 0;
#pragma unroll
            for (int i = 0; i < 4; i++) {
                ulonglong2 v = d[i];   // same address for every thread: shared-memory broadcast
                dist += __popcll(qa[2 * i] ^ v.x) + __popcll(qa[2 * i + 1] ^ v.y);
            }
            insert_key<K>(best, (dist << IDX_BITS) | (first + r));
        }
        __syncthreads();   // everyone is done with buffer t&1
        if (threadIdx.x == 0 && t + 2 < ntiles) issue(t + 2);
    }
    if (q < n) {
        uint32_t *out = partial + ((size_t)q * gridDim.y + blockIdx.y) * K;
#pragma unroll
        for (int i = 0; i < K; i++) out[i] = best[i];
    }
}

// ---------------------------------------------------------------------------------------------------
// Tensor-core formulation (BASELINE north_star: "tensor cores only if the distance matrix is reformulated as
// a dense int8 contraction").  Each descriptor is unpacked to 512 int8 values in {0,1}; then
//     hamming(a, b) = |a| + |b| - 2 <a, b>           (exact in s32)
// and <a, b> for a 16 x 8 block of (query, database) pairs is 16 `mma.sync.m16n8k32.u8.u8.s32` (IMMA.16832)
// instructions.  A warp keeps its 16 query rows (16 x 512 B) in registers for the whole kernel; database
// tiles of 64 unpacked descriptors are staged in shared memory with cp.async (double buffered, row stride
// 576 B so that the 128-bit fragment loads are bank-conflict free).  The (distance, index) key logic and the
// split / merge structure are shared with the popcount kernel, so results are identical by construction.
constexpr int IM_WARPS = 4, IM_QT = 16 * IM_WARPS, IM_DT = 32, IM_ROWB = 576;
constexpr size_t IM_SMEM = 2 * (size_t)IM_DT * IM_ROWB + 2 * IM_DT * sizeof(uint16_t);

// one warp per descriptor: 512 bits -> 512 bytes (0/1) + population count
__global__ void __launch_bounds__(256) k_unpack_bits(const uint8_t *__restrict__ desc, const uint32_t *__restrict__ n_dev,
                                                     uint32_t n_host, uint8_t *__restrict__ U, uint16_t *__restrict__ pc) {
    const uint32_t n = n_dev ? min(*n_dev, n_host) : n_host;
    const uint32_t row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (row >= n) return;
    const uint32_t bits = ((const uint16_t *)(desc + (size_t)row * 64))[lane];   // bits 16*lane .. 16*lane+15
    uint32_t w[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const uint32_t nib = (bits >> (4 * k)) & 0xfu;
        w[k] = (nib & 1u) | ((nib & 2u) << 7) | ((nib & 4u) << 14) | ((nib & 8u) << 21);
    }
    *(uint4 *)(U + (size_t)row * 512 + 16 * lane) = make_uint4(w[0], w[1], w[2], w[3]);
    uint32_t c = __popc(bits);
    for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (lane == 0) pc[row] = (uint16_t)c;
}

__device__ __forceinline__ void imma_16832(int (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void cp_async16(void *dst, const void *src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}

template <int K>
__global__ void __launch_bounds__(IM_WARPS * 32) k_hamming_imma(const uint8_t *__restrict__ Uq, const uint16_t *__restrict__ pq,
                                                                const uint32_t *__restrict__ n_dev, uint32_t n_host,
                                                                const uint8_t *__restrict__ Udb, const uint16_t *__restrict__ pdb,
                                                                const uint32_t *__restrict__ m_dev, uint32_t m_host, uint32_t chunk,
                                                                uint32_t *__restrict__ partial) {
    extern __shared__ __align__(128) uint8_t smraw[];
    uint8_t *s_db = smraw;                                              // [2][IM_DT][IM_ROWB]
    uint16_t *s_pb = (uint16_t *)(smraw + 2 * (size_t)IM_DT * IM_ROWB);   // [2][IM_DT]
    const uint32_t n = n_dev ? min(*n_dev, n_host) : n_host, m = m_dev ? min(*m_dev, m_host) : m_host;
    if (blockIdx.x * IM_QT >= n) return;
    const uint32_t lo = min(blockIdx.y * chunk, m), hi = min(lo + chunk, m), cnt = hi - lo;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    const uint32_t q0 = blockIdx.x * IM_QT + wid * 16;
    const uint32_t rA = min(q0 + g, n - 1), rB = min(q0 + g + 8, n - 1);
    // A fragments for all 16 k-steps: 8 x 16 B per row
    uint4 fa[8], fb[8];
#pragma unroll
    for (int u = 0; u < 8; u++) {
        fa[u] = *(const uint4 *)(Uq + (size_t)rA * 512 + 64 * u + 16 * t);
        fb[u] = *(const uint4 *)(Uq + (size_t)rB * 512 + 64 * u + 16 * t);
    }
    const int pa0 = pq[rA], pa1 = pq[rB];
    uint32_t best0[K], best1[K];
#pragma unroll
    for (int i = 0; i < K; i++) { best0[i] = 0xffffffffu; best1[i] = 0xffffffffu; }
    const uint32_t ntiles = (cnt + IM_DT - 1) / IM_DT;
    auto stage = [&](uint32_t tile) {
        uint8_t *dst = s_db + (size_t)(tile & 1) * IM_DT * IM_ROWB;
        const uint32_t first = tile * IM_DT;
        for (int c = threadIdx.x; c < IM_DT * 32; c += IM_WARPS * 32) {    // 32 chunks of 16 B per row
            const int r = c >> 5, col = c & 31;
            const uint32_t src_row = lo + min(first + (uint32_t)r, cnt - 1);
            cp_async16(dst + r * IM_ROWB + col * 16, Udb + (size_t)src_row * 512 + col * 16);
        }
        if (threadIdx.x < IM_DT) s_pb[(tile & 1) * IM_DT + threadIdx.x] = pdb[lo + min(first + threadIdx.x, cnt - 1)];
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    if (ntiles > 0) stage(0);
    for (uint32_t tile = 0; tile < ntiles; tile++) {
        if (tile + 1 < ntiles) { stage(tile + 1); asm volatile("cp.async.wait_group 1;" ::: "memory"); }
        else asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncthreads();
        const uint8_t *tb = s_db + (size_t)(tile & 1) * IM_DT * IM_ROWB;
        const uint16_t *tp = s_pb + (tile & 1) * IM_DT;
        const uint32_t first = tile * IM_DT;
#pragma unroll 2
        for (int j = 0; j < IM_DT / 8; j++) {
            int c[4] = {0, 0, 0, 0};
            const uint8_t *brow = tb + (8 * j + g) * IM_ROWB + 16 * t;
#pragma unroll
            for (int u = 0; u < 8; u++) {
                const uint4 b = *(const uint4 *)(brow + 64 * u);
                imma_16832(c, fa[u].x, fb[u].x, fa[u].y, fb[u].y, b.x, b.y);
                imma_16832(c, fa[u].z, fb[u].z, fa[u].w, fb[u].w, b.z, b.w);
            }
            const uint32_t col = first + 8 * j + 2 * t;       // split-local database index of c[0] / c[2]
            const int pb0 = tp[8 * j + 2 * t], pb1 = tp[8 * j + 2 * t + 1];
            if (col < cnt) {
                insert_key<K>(best0, ((uint32_t)(pa0 + pb0 - 2 * c[0]) << IDX_BITS) | col);
                insert_key<K>(best1, ((uint32_t)(pa1 + pb0 - 2 * c[2]) << IDX_BITS) | col);
            }
            if (col + 1 < cnt) {
                insert_key<K>(best0, ((uint32_t)(pa0 + pb1 - 2 * c[1]) << IDX_BITS) | (col + 1));
                insert_key<K>(best1, ((uint32_t)(pa1 + pb1 - 2 * c[3]) << IDX_BITS) | (col + 1));
            }
        }
        __syncthreads();   // buffer (tile & 1) may be overwritten by stage(tile + 2)
    }
    // merge the four lanes that share a row
#pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {
        uint32_t o0[K], o1[K];
#pragma unroll
        for (int i = 0; i < K; i++) { o0[i] = __shfl_xor_sync(0xffffffffu, best0[i], o); o1[i] = __shfl_xor_sync(0xffffffffu, best1[i], o); }
#pragma unroll
        for (int i = 0; i < K; i++) { insert_key<K>(best0, o0[i]); insert_key<K>(best1, o1[i]); }
    }
    if (t == 0) {
        if (q0 + g < n) {
            uint32_t *out = partial + ((size_t)(q0 + g) * gridDim.y + blockIdx.y) * K;
#pragma unroll
            for (int i = 0; i < K; i++) out[i] = best0[i];
        }
        if (q0 + g + 8 < n) {
            uint32_t *out = partial + ((size_t)(q0 + g + 8) * gridDim.y + blockIdx.y) * K;
#pragma unroll
            for (int i = 0; i < K; i++) out[i] = best1[i];
        }
    }
}

#include "match_wgmma.cuh"

// merge the per-split lists (split order == index order) into global (idx, dist)
template <int K>
__global__ void k_knn_merge(const uint32_t *__restrict__ partial, const uint32_t *__restrict__ n_dev, uint32_t n_host,
                            uint32_t splits, uint32_t chunk, uint32_t *__restrict__ idx_out, uint32_t *__restrict__ dist_out) {
    const uint32_t n = n_dev ? min(*n_dev, n_host) : n_host;
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n) return;
    uint64_t best[K];
#pragma unroll
    for (int i = 0; i < K; i++) best[i] = ~0ull;
    for (uint32_t s = 0; s < splits; s++) {
        const uint32_t *p = partial + ((size_t)q * splits + s) * K;
#pragma unroll
        for (int i = 0; i < K; i++) {
            uint32_t key = p[i];
            if (key == 0xffffffffu) continue;
            uint64_t g = ((uint64_t)(key >> IDX_BITS) << 32) | (uint64_t)((key & IDX_MASK) + s * chunk);
#pragma unroll
            for (int j = 0; j < K; j++) {
                uint64_t lo = min(best[j], g);
                g = max(best[j], g);
                best[j] = lo;
            }
        }
    }
#pragma unroll
    for (int i = 0; i < K; i++) {
        idx_out[(size_t)q * K + i] = best[i] == ~0ull ? 0xffffffffu : (uint32_t)(best[i] & 0xffffffffu);
        dist_out[(size_t)q * K + i] = best[i] == ~0ull ? 0xffffffffu : (uint32_t)(best[i] >> 32);
    }
}

// cv-sfm symmetric_matching (cv-sfm/src/lib.rs:3097-3133) on the two 2-NN tables
__global__ void k_symmetric(const uint32_t *__restrict__ fidx, const uint32_t *__restrict__ fdist,
                            const uint32_t *__restrict__ ridx, const uint32_t *__restrict__ rdist, uint32_t n, uint32_t m,
                            uint32_t better_by, uint32_t *__restrict__ flag) {
    const uint32_t a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= n) return;
    uint32_t f = 0xffffffffu;
    if (n >= 2 && m >= 2) {
        if (fdist[2 * a] + better_by <= fdist[2 * a + 1]) {
            uint32_t bix = fidx[2 * a];
            if (rdist[2 * bix] + better_by <= rdist[2 * bix + 1] && ridx[2 * bix] == a) f = bix;
        }
    }
    flag[a] = f;
}


// symmetric rule with device-resident counts, followed by an ordered compaction into (a, b) index pairs (ascending a):
// one CTA walks the n <= n_max queries in chunks of 1024 (cv-sfm/src/lib.rs:3097-3133)
__global__ void __launch_bounds__(1024) k_symmetric_pairs(const uint32_t *__restrict__ fidx, const uint32_t *__restrict__ fdist,
                                                          const uint32_t *__restrict__ ridx, const uint32_t *__restrict__ rdist,
                                                          const uint32_t *__restrict__ n_dev, uint32_t n_max,
                                                          const uint32_t *__restrict__ m_dev, uint32_t m_max, uint32_t better_by,
                                                          uint32_t *__restrict__ pairs, uint32_t cap, uint32_t *__restrict__ npairs,
                                                          uint32_t *__restrict__ overflow) {
    __shared__ uint32_t s_warp[32];
    __shared__ uint32_t s_carry;
    const uint32_t n = min(*n_dev, n_max), m = min(*m_dev, m_max);
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (uint32_t base = 0; base < n; base += 1024) {
        const uint32_t a = base + threadIdx.x;
        uint32_t f = 0xffffffffu;
        if (a < n && n >= 2 && m >= 2 && fdist[2 * a] + better_by <= fdist[2 * a + 1]) {
            const uint32_t bix = fidx[2 * a];
            if (rdist[2 * bix] + better_by <= rdist[2 * bix + 1] && ridx[2 * bix] == a) f = bix;
        }
        const uint32_t v = f != 0xffffffffu ? 1u : 0u;
        uint32_t x = v;
        for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, x, o); if ((int)lane >= o) x += t; }
        if (lane == 31) s_warp[wid] = x;
        __syncthreads();
        if (wid == 0) {
            const uint32_t y = s_warp[lane];
            uint32_t z = y;
            for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, z, o); if ((int)lane >= o) z += t; }
            s_warp[lane] = z - y;
        }
        __syncthreads();
        const uint32_t pos = s_carry + s_warp[wid] + x - v;
        if (v) {
            if (pos < cap) { pairs[2 * pos] = a; pairs[2 * pos + 1] = f; }
            else if (overflow) *overflow = 1u;
        }
        __syncthreads();
        if (threadIdx.x == 1023) s_carry = pos + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) *npairs = min(s_carry, cap);
}


// HammingHasher::hash_bag (external crate hamming-lsh 0.3.2; call site cv-sfm/src/lib.rs:672 with the 4 096-codeword table of
// cv-sfm/src/codewords.rs): every feature sets the bit of its nearest codeword (first minimum on ties, like Iterator::min_by_key).
// The nearest codeword IS a 1-NN query of the matcher above; this kernel ORs the winners' bits into the hash.
__global__ void __launch_bounds__(256) k_hash_set_bits(const uint32_t *__restrict__ nearest, const uint32_t *__restrict__ n_dev, uint32_t n_host,
                                                       uint32_t ncode, uint32_t *__restrict__ hash_words) {
    const uint32_t n = n_dev ? min(*n_dev, n_host) : n_host;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t ix = nearest[i];
    if (ix < ncode) atomicOr(&hash_words[ix >> 5], 1u << (ix & 31));      // little-endian words: bit ix & 7 of byte ix >> 3
}

}  // namespace

struct MatchWorkspace {
    uint32_t *partial = nullptr;
    size_t partial_elems = 0;
    uint8_t *q = nullptr, *db = nullptr;
    size_t q_bytes = 0, db_bytes = 0;
    uint32_t *idx = nullptr, *dist = nullptr, *idx2 = nullptr, *dist2 = nullptr, *flag = nullptr;
    size_t idx_elems = 0, dist_elems = 0, idx2_elems = 0, dist2_elems = 0, flag_elems = 0;
    uint8_t *uq = nullptr, *udb = nullptr;         // unpacked (int8 0/1) descriptors for the tensor-core path
    uint16_t *pq = nullptr, *pdb = nullptr;
    size_t uq_bytes = 0, udb_bytes = 0, pq_elems = 0, pdb_elems = 0;
    int use_imma = -1;                              // 2 wgmma (default), 1 mma.sync (CVB_KNN_IMMA=1), 0 popcount (CVB_KNN_POPC=1)
};

void match_workspace_free(MatchWorkspace *ws) {
    if (!ws) return;
    cudaFree(ws->partial); cudaFree(ws->q); cudaFree(ws->db); cudaFree(ws->idx); cudaFree(ws->dist);
    cudaFree(ws->idx2); cudaFree(ws->dist2); cudaFree(ws->flag);
    cudaFree(ws->uq); cudaFree(ws->udb); cudaFree(ws->pq); cudaFree(ws->pdb);
    delete ws;
}

namespace {

template <typename T>
int grow(cvb_ctx *ctx, T **p, size_t *have, size_t need) {
    if (*have >= need && *p) return 0;
    if (*p) { cvb_wait(ctx, ctx->stream); cudaFree(*p); *p = nullptr; }
    size_t n = std::max<size_t>(need, 1);
    cudaError_t e = cudaMalloc((void **)p, n * sizeof(T));
    if (e != cudaSuccess) { *have = 0; return cvb_set_error(ctx, CVB_ENOMEM, "cudaMalloc(%zu): %s", n * sizeof(T), cudaGetErrorString(e)); }
    *have = n;
    return 0;
}

template <int K>
int launch_knn(cvb_ctx *ctx, const uint8_t *q, const uint32_t *n_dev, uint32_t n, const uint8_t *db, const uint32_t *m_dev,
               uint32_t m, uint32_t splits, uint32_t chunk, uint32_t *partial, uint32_t *idx, uint32_t *dist) {
    dim3 grid(cdiv(n, QT), splits);
    CVB_PROF(ctx, "k_hamming_knn", 64.0 * (double)n * (double)m);
    k_hamming_knn<K><<<grid, QT, 0, ctx->stream>>>(q, n_dev, n, db, m_dev, m, chunk, partial);
    CVB_LAUNCH_CHECK(ctx);
    k_knn_merge<K><<<cdiv(n, 128), 128, 0, ctx->stream>>>(partial, n_dev, n, splits, chunk, idx, dist);
    CVB_LAUNCH_CHECK(ctx);
    return 0;
}

template <int K>
int launch_knn_imma(cvb_ctx *ctx, MatchWorkspace *ws, const uint8_t *q, const uint32_t *n_dev, uint32_t n, const uint8_t *db,
                    const uint32_t *m_dev, uint32_t m, uint32_t splits, uint32_t chunk, uint32_t *idx, uint32_t *dist) {
    {
        CVB_PROF(ctx, "k_unpack_bits", 0);
        k_unpack_bits<<<cdiv(n * 32, 256), 256, 0, ctx->stream>>>(q, n_dev, n, ws->uq, ws->pq);
        CVB_LAUNCH_CHECK(ctx);
        k_unpack_bits<<<cdiv(m * 32, 256), 256, 0, ctx->stream>>>(db, m_dev, m, ws->udb, ws->pdb);
        CVB_LAUNCH_CHECK(ctx);
    }
    {
        static bool attr_set = false;   // per template instance, once per process
        if (!attr_set) { cudaFuncSetAttribute(k_hamming_imma<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)IM_SMEM); attr_set = true; }
        dim3 grid(cdiv(n, IM_QT), splits);
        CVB_PROF(ctx, "k_hamming_knn", 64.0 * (double)n * (double)m);
        k_hamming_imma<K><<<grid, IM_WARPS * 32, IM_SMEM, ctx->stream>>>(ws->uq, ws->pq, n_dev, n, ws->udb, ws->pdb, m_dev, m, chunk, ws->partial);
        CVB_LAUNCH_CHECK(ctx);
    }
    k_knn_merge<K><<<cdiv(n, 128), 128, 0, ctx->stream>>>(ws->partial, n_dev, n, splits, chunk, idx, dist);
    CVB_LAUNCH_CHECK(ctx);
    return 0;
}

template <int K>
int launch_knn_wgmma(cvb_ctx *ctx, MatchWorkspace *ws, const uint8_t *q, const uint32_t *n_dev, uint32_t n, const uint8_t *db,
                     const uint32_t *m_dev, uint32_t m, uint32_t splits, uint32_t chunk, uint32_t *idx, uint32_t *dist) {
    {
        static bool attr_set = false;   // per template instance, once per process
        if (!attr_set) { cudaFuncSetAttribute(wg::k_hamming_wgmma<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wg::SMEM); attr_set = true; }
        dim3 grid(cdiv(n, wg::QT), splits);
        CVB_PROF(ctx, "k_hamming_knn", 64.0 * (double)n * (double)m);
        wg::k_hamming_wgmma<K><<<grid, wg::THREADS, wg::SMEM, ctx->stream>>>(q, n_dev, n, db, m_dev, m, chunk, ws->partial);
        CVB_LAUNCH_CHECK(ctx);
    }
    k_knn_merge<K><<<cdiv(n, 128), 128, 0, ctx->stream>>>(ws->partial, n_dev, n, splits, chunk, idx, dist);
    CVB_LAUNCH_CHECK(ctx);
    return 0;
}

int knn_dev(cvb_ctx *ctx, const uint8_t *q, const uint32_t *n_dev, uint32_t n, const uint8_t *db, const uint32_t *m_dev,
            uint32_t m, uint32_t k, uint32_t *idx, uint32_t *dist) {
    if (k < 1 || k > MAXKNN) return cvb_set_error(ctx, CVB_EINVAL, "k must be 1..%d", MAXKNN);
    if (n == 0) return 0;
    if (((uintptr_t)q & 15) || ((uintptr_t)db & 15)) return cvb_set_error(ctx, CVB_EINVAL, "descriptor arrays must be 16-byte aligned");
    if (!ctx->match) ctx->match = new MatchWorkspace();
    MatchWorkspace *ws = ctx->match;
    if (ws->use_imma < 0) {     // 2: wgmma (default), 1: legacy mma.sync int8 (CVB_KNN_IMMA=1), 0: popcount (CVB_KNN_POPC=1)
        const char *env = getenv("CVB_KNN_POPC"), *env2 = getenv("CVB_KNN_IMMA"), *env3 = getenv("CVB_KNN_WGMMA");
        ws->use_imma = (env && env[0] == '1') ? 0 : ((env2 && env2[0] == '1') ? 1 : ((env3 && env3[0] == '0') ? 1 : (env3 && env3[0] == '1') ? 2 : CVB_KNN_DEFAULT_MODE));
    }
    if (ws->use_imma == 2 && m > 0) {
        // wgmma path: 128-query CTAs (one per SM: 145 KB of shared memory); the database is split so that the grid is one wave
        const uint32_t qblocks = cdiv(n, wg::QT);
        uint32_t splits = std::max<uint32_t>(1, (uint32_t)ctx->num_sms / qblocks);
        splits = std::min<uint32_t>(splits, std::max<uint32_t>(1, cdiv(m, wg::DT)));
        uint32_t chunk = cdiv(cdiv(m, splits), wg::DT) * wg::DT;
        while (chunk > IDX_MASK) { splits *= 2; chunk = cdiv(cdiv(m, splits), wg::DT) * wg::DT; }
        splits = cdiv(m, chunk);
        int rc;
        if ((rc = grow(ctx, &ws->partial, &ws->partial_elems, (size_t)n * splits * k))) return rc;
        switch (k) {
        case 1: return launch_knn_wgmma<1>(ctx, ws, q, n_dev, n, db, m_dev, m, splits, chunk, idx, dist);
        case 2: return launch_knn_wgmma<2>(ctx, ws, q, n_dev, n, db, m_dev, m, splits, chunk, idx, dist);
        case 3: return launch_knn_wgmma<3>(ctx, ws, q, n_dev, n, db, m_dev, m, splits, chunk, idx, dist);
        case 4: return launch_knn_wgmma<4>(ctx, ws, q, n_dev, n, db, m_dev, m, splits, chunk, idx, dist);
        case 5: return launch_knn_wgmma<5>(ctx, ws, q, n_dev, n, db, m_dev, m, splits, chunk, idx, dist);
        case 6: return launch_knn_wgmma<6>(ctx, ws, q, n_dev, n, db, m_dev, m, splits, chunk, idx, dist);
        case 7: return launch_knn_wgmma<7>(ctx, ws, q, n_dev, n, db, m_dev, m, splits, chunk, idx, dist);
        default: return launch_knn_wgmma<8>(ctx, ws, q, n_dev, n, db, m_dev, m, splits, chunk, idx, dist);
        }
    }
    if (ws->use_imma == 1 && m > 0) {
        // legacy tensor-core path (mma.sync): 64-query CTAs; the database is split so that the grid is ONE full wave
        // (4 CTAs of 128 threads fit per SM: 105 registers, 37 KB shared memory)
        uint32_t qblocks = cdiv(n, IM_QT);
        uint32_t splits = std::max<uint32_t>(1, ((uint32_t)ctx->num_sms * 4u) / qblocks);
        splits = std::min<uint32_t>(splits, std::max<uint32_t>(1, cdiv(m, IM_DT * 2)));
        uint32_t chunk = cdiv(cdiv(m, splits), IM_DT) * IM_DT;
        while (chunk > IDX_MASK) { splits *= 2; chunk = cdiv(cdiv(m, splits), IM_DT) * IM_DT; }
        splits = cdiv(m, chunk);
        int rc;
        if ((rc = grow(ctx, &ws->partial, &ws->partial_elems, (size_t)n * splits * k))) return rc;
        if ((rc = grow(ctx, &ws->uq, &ws->uq_bytes, (size_t)n * 512))) return rc;
        if ((rc = grow(ctx, &ws->udb, &ws->udb_bytes, (size_t)m * 512))) return rc;
        if ((rc = grow(ctx, &ws->pq, &ws->pq_elems, (size_t)n))) return rc;
        if ((rc = grow(ctx, &ws->pdb, &ws->pdb_elems, (size_t)m))) return rc;
        switch (k) {
        case 1: return launch_knn_imma<1>(ctx, ws, q, n_dev, n, db, m_dev, m, splits, chunk, idx, dist);
        case 2: return launch_knn_imma<2>(ctx, ws, q, n_dev, n, db, m_dev, m, splits, chunk, idx, dist);
        case 3: return launch_knn_imma<3>(ctx, ws, q, n_dev, n, db, m_dev, m, splits, chunk, idx, dist);
        case 4: return launch_knn_imma<4>(ctx, ws, q, n_dev, n, db, m_dev, m, splits, chunk, idx, dist);
        case 5: return launch_knn_imma<5>(ctx, ws, q, n_dev, n, db, m_dev, m, splits, chunk, idx, dist);
        case 6: return launch_knn_imma<6>(ctx, ws, q, n_dev, n, db, m_dev, m, splits, chunk, idx, dist);
        case 7: return launch_knn_imma<7>(ctx, ws, q, n_dev, n, db, m_dev, m, splits, chunk, idx, dist);
        default: return launch_knn_imma<8>(ctx, ws, q, n_dev, n, db, m_dev, m, splits, chunk, idx, dist);
        }
    }
    // split the database so that the grid covers the machine (>= 2 CTAs per SM) and chunks fit IDX_BITS
    uint32_t qblocks = cdiv(n, QT);
    uint32_t splits = std::max<uint32_t>(1, cdiv((uint32_t)ctx->num_sms * 4u, qblocks));
    splits = std::min<uint32_t>(splits, std::max<uint32_t>(1, cdiv(std::max<uint32_t>(m, 1), DTILE * 2)));
    uint32_t chunk = cdiv(std::max<uint32_t>(m, 1), splits);
    chunk = cdiv(chunk, DTILE) * DTILE;
    while (chunk > IDX_MASK) { splits *= 2; chunk = cdiv(cdiv(m, splits), DTILE) * DTILE; }
    splits = cdiv(std::max<uint32_t>(m, 1), chunk);
    int rc = grow(ctx, &ws->partial, &ws->partial_elems, (size_t)n * splits * k);
    if (rc) return rc;
    switch (k) {
    case 1: return launch_knn<1>(ctx, q, n_dev, n, db, m_dev, m, splits, chunk, ws->partial, idx, dist);
    case 2: return launch_knn<2>(ctx, q, n_dev, n, db, m_dev, m, splits, chunk, ws->partial, idx, dist);
    case 3: return launch_knn<3>(ctx, q, n_dev, n, db, m_dev, m, splits, chunk, ws->partial, idx, dist);
    case 4: return launch_knn<4>(ctx, q, n_dev, n, db, m_dev, m, splits, chunk, ws->partial, idx, dist);
    case 5: return launch_knn<5>(ctx, q, n_dev, n, db, m_dev, m, splits, chunk, ws->partial, idx, dist);
    case 6: return launch_knn<6>(ctx, q, n_dev, n, db, m_dev, m, splits, chunk, ws->partial, idx, dist);
    case 7: return launch_knn<7>(ctx, q, n_dev, n, db, m_dev, m, splits, chunk, ws->partial, idx, dist);
    default: return launch_knn<8>(ctx, q, n_dev, n, db, m_dev, m, splits, chunk, ws->partial, idx, dist);
    }
}

}  // namespace

extern "C" {

int cvb_hamming_knn_dev(cvb_ctx *ctx, const uint8_t *q, uint32_t n, const uint8_t *db, uint32_t m, uint32_t k, uint32_t *idx,
                        uint32_t *dist) {
    if (!ctx) return CVB_EINVAL;
    if ((n && !q) || (m && !db) || (n && (!idx || !dist))) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    return knn_dev(ctx, q, nullptr, n, db, nullptr, m, k, idx, dist);
}

int cvb_hamming_knn_dev_counts(cvb_ctx *ctx, const uint8_t *q, const uint32_t *n_dev, uint32_t n_max, const uint8_t *db,
                               const uint32_t *m_dev, uint32_t m_max, uint32_t k, uint32_t *idx, uint32_t *dist) {
    if (!ctx) return CVB_EINVAL;
    if (!q || !db || !idx || !dist || !n_dev || !m_dev) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    return knn_dev(ctx, q, n_dev, n_max, db, m_dev, m_max, k, idx, dist);
}

int cvb_hamming_knn(cvb_ctx *ctx, const uint8_t *q, uint32_t n, const uint8_t *db, uint32_t m, uint32_t k, uint32_t *idx,
                    uint32_t *dist) {
    if (!ctx) return CVB_EINVAL;
    if ((n && !q) || (m && !db) || (n && (!idx || !dist))) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (k < 1 || k > MAXKNN) return cvb_set_error(ctx, CVB_EINVAL, "k must be 1..%d", MAXKNN);
    if (n == 0) return 0;
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    if (!ctx->match) ctx->match = new MatchWorkspace();
    MatchWorkspace *ws = ctx->match;
    int rc;
    if ((rc = grow(ctx, &ws->q, &ws->q_bytes, (size_t)n * 64))) return rc;
    if ((rc = grow(ctx, &ws->db, &ws->db_bytes, (size_t)std::max<uint32_t>(m, 1) * 64))) return rc;
    if ((rc = grow(ctx, &ws->idx, &ws->idx_elems, (size_t)n * k))) return rc;
    if ((rc = grow(ctx, &ws->dist, &ws->dist_elems, (size_t)n * k))) return rc;
    cudaStream_t st = ctx->stream;
    CVB_CUDA(ctx, cudaMemcpyAsync(ws->q, q, (size_t)n * 64, cudaMemcpyHostToDevice, st));
    if (m) CVB_CUDA(ctx, cudaMemcpyAsync(ws->db, db, (size_t)m * 64, cudaMemcpyHostToDevice, st));
    rc = knn_dev(ctx, ws->q, nullptr, n, ws->db, nullptr, m, k, ws->idx, ws->dist);
    if (rc) return rc;
    CVB_CUDA(ctx, cudaMemcpyAsync(idx, ws->idx, sizeof(uint32_t) * (size_t)n * k, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(dist, ws->dist, sizeof(uint32_t) * (size_t)n * k, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    return 0;
}

int cvb_match_symmetric_dev(cvb_ctx *ctx, const uint8_t *a_dev, uint32_t n, const uint8_t *b_dev, uint32_t m, uint32_t better_by,
                            uint32_t *match_out_dev) {
    if (!ctx) return CVB_EINVAL;
    if (n == 0) return 0;
    if (!a_dev || !match_out_dev || (m && !b_dev)) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    if (!ctx->match) ctx->match = new MatchWorkspace();
    MatchWorkspace *ws = ctx->match;
    if (n < 2 || m < 2) {   // cv-sfm/src/lib.rs:3099-3101: no matches at all
        CVB_CUDA(ctx, cudaMemsetAsync(match_out_dev, 0xff, sizeof(uint32_t) * n, ctx->stream));
        return 0;
    }
    int rc;
    if ((rc = grow(ctx, &ws->idx, &ws->idx_elems, (size_t)n * 2))) return rc;
    if ((rc = grow(ctx, &ws->dist, &ws->dist_elems, (size_t)n * 2))) return rc;
    if ((rc = grow(ctx, &ws->idx2, &ws->idx2_elems, (size_t)m * 2))) return rc;
    if ((rc = grow(ctx, &ws->dist2, &ws->dist2_elems, (size_t)m * 2))) return rc;
    if ((rc = knn_dev(ctx, a_dev, nullptr, n, b_dev, nullptr, m, 2, ws->idx, ws->dist))) return rc;
    if ((rc = knn_dev(ctx, b_dev, nullptr, m, a_dev, nullptr, n, 2, ws->idx2, ws->dist2))) return rc;
    k_symmetric<<<cdiv(n, 256), 256, 0, ctx->stream>>>(ws->idx, ws->dist, ws->idx2, ws->dist2, n, m, better_by, match_out_dev);
    CVB_LAUNCH_CHECK(ctx);
    return 0;
}

int cvb_match_symmetric_pairs_dev(cvb_ctx *ctx, const uint8_t *a_dev, const uint32_t *n_dev, uint32_t n_max, const uint8_t *b_dev,
                                  const uint32_t *m_dev, uint32_t m_max, uint32_t better_by, uint32_t *pairs_out_dev, uint32_t cap,
                                  uint32_t *n_pairs_dev) {
    if (!ctx) return CVB_EINVAL;
    if (!a_dev || !b_dev || !n_dev || !m_dev || !pairs_out_dev || !n_pairs_dev) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    if (n_max < 2 || m_max < 2) {   // cv-sfm/src/lib.rs:3099-3101: no matches at all
        CVB_CUDA(ctx, cudaMemsetAsync(n_pairs_dev, 0, sizeof(uint32_t), ctx->stream));
        return 0;
    }
    if (!ctx->match) ctx->match = new MatchWorkspace();
    MatchWorkspace *ws = ctx->match;
    int rc;
    if ((rc = grow(ctx, &ws->idx, &ws->idx_elems, (size_t)n_max * 2))) return rc;
    if ((rc = grow(ctx, &ws->dist, &ws->dist_elems, (size_t)n_max * 2))) return rc;
    if ((rc = grow(ctx, &ws->idx2, &ws->idx2_elems, (size_t)m_max * 2))) return rc;
    if ((rc = grow(ctx, &ws->dist2, &ws->dist2_elems, (size_t)m_max * 2))) return rc;
    if ((rc = knn_dev(ctx, a_dev, n_dev, n_max, b_dev, m_dev, m_max, 2, ws->idx, ws->dist))) return rc;
    if ((rc = knn_dev(ctx, b_dev, m_dev, m_max, a_dev, n_dev, n_max, 2, ws->idx2, ws->dist2))) return rc;
    CVB_PROF(ctx, "k_symmetric_pairs", 0);
    k_symmetric_pairs<<<1, 1024, 0, ctx->stream>>>(ws->idx, ws->dist, ws->idx2, ws->dist2, n_dev, n_max, m_dev, m_max, better_by,
                                                   pairs_out_dev, cap, n_pairs_dev, nullptr);
    CVB_LAUNCH_CHECK(ctx);
    return 0;
}

int cvb_hash_bag_dev(cvb_ctx *ctx, const uint8_t *desc_dev, const uint32_t *n_dev, uint32_t n_max, const uint8_t *codewords_dev,
                     uint32_t ncode, uint8_t *hash_out_dev) {
    if (!ctx) return CVB_EINVAL;
    if (!desc_dev || !codewords_dev || !hash_out_dev || !n_dev) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (ncode == 0 || (ncode & 31)) return cvb_set_error(ctx, CVB_EINVAL, "the number of codewords must be a positive multiple of 32");
    if (((uintptr_t)hash_out_dev & 3)) return cvb_set_error(ctx, CVB_EINVAL, "hash output must be 4-byte aligned");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    CVB_CUDA(ctx, cudaMemsetAsync(hash_out_dev, 0, ncode / 8, ctx->stream));
    if (n_max == 0) return 0;
    if (!ctx->match) ctx->match = new MatchWorkspace();
    MatchWorkspace *ws = ctx->match;
    int rc;
    if ((rc = grow(ctx, &ws->idx, &ws->idx_elems, (size_t)n_max * 2))) return rc;
    if ((rc = grow(ctx, &ws->dist, &ws->dist_elems, (size_t)n_max * 2))) return rc;
    if ((rc = knn_dev(ctx, desc_dev, n_dev, n_max, codewords_dev, nullptr, ncode, 1, ws->idx, ws->dist))) return rc;
    CVB_PROF(ctx, "k_hash_set_bits", 0);
    k_hash_set_bits<<<cdiv(n_max, 256), 256, 0, ctx->stream>>>(ws->idx, n_dev, n_max, ncode, (uint32_t *)hash_out_dev);
    CVB_LAUNCH_CHECK(ctx);
    return 0;
}

int cvb_hash_bag(cvb_ctx *ctx, const uint8_t *desc, uint32_t n, const uint8_t *codewords, uint32_t ncode, uint8_t *hash_out) {
    if (!ctx) return CVB_EINVAL;
    if ((n && !desc) || !codewords || !hash_out) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (ncode == 0 || (ncode & 31)) return cvb_set_error(ctx, CVB_EINVAL, "the number of codewords must be a positive multiple of 32");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    if (!ctx->match) ctx->match = new MatchWorkspace();
    MatchWorkspace *ws = ctx->match;
    int rc;
    // layout of the staging buffers: q = features, db = [codewords | n (u32, 16-byte slot) | hash]
    const size_t cw_bytes = (size_t)ncode * 64, extra = 16 + ncode / 8;
    if ((rc = grow(ctx, &ws->q, &ws->q_bytes, (size_t)std::max<uint32_t>(n, 1) * 64))) return rc;
    if ((rc = grow(ctx, &ws->db, &ws->db_bytes, cw_bytes + extra))) return rc;
    cudaStream_t st = ctx->stream;
    uint32_t *n_slot = (uint32_t *)(ws->db + cw_bytes);
    uint8_t *hash_dev = ws->db + cw_bytes + 16;
    uint32_t *hn = (uint32_t *)cvb_pinned(ctx, 16 + ncode / 8);
    if (!hn) return cvb_set_error(ctx, CVB_ENOMEM, "page-locked scratch");
    hn[0] = n;
    if (n) CVB_CUDA(ctx, cudaMemcpyAsync(ws->q, desc, (size_t)n * 64, cudaMemcpyHostToDevice, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(ws->db, codewords, cw_bytes, cudaMemcpyHostToDevice, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(n_slot, hn, 4, cudaMemcpyHostToDevice, st));
    if ((rc = cvb_hash_bag_dev(ctx, ws->q, n_slot, n, ws->db, ncode, hash_dev))) return rc;
    CVB_CUDA(ctx, cudaMemcpyAsync(hn + 4, hash_dev, ncode / 8, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    memcpy(hash_out, hn + 4, ncode / 8);
    return 0;
}

int cvb_match_symmetric(cvb_ctx *ctx, const uint8_t *a, uint32_t n, const uint8_t *b, uint32_t m, uint32_t better_by,
                        uint32_t *pairs_out, uint32_t cap, uint32_t *n_out) {
    if (!ctx) return CVB_EINVAL;
    if (!n_out || (n && !a) || (m && !b)) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    *n_out = 0;
    if (n < 2 || m < 2) return 0;   // cv-sfm/src/lib.rs:3099-3101
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    if (!ctx->match) ctx->match = new MatchWorkspace();
    MatchWorkspace *ws = ctx->match;
    int rc;
    if ((rc = grow(ctx, &ws->q, &ws->q_bytes, (size_t)n * 64))) return rc;
    if ((rc = grow(ctx, &ws->db, &ws->db_bytes, (size_t)m * 64))) return rc;
    if ((rc = grow(ctx, &ws->idx, &ws->idx_elems, (size_t)n * 2))) return rc;
    if ((rc = grow(ctx, &ws->dist, &ws->dist_elems, (size_t)n * 2))) return rc;
    if ((rc = grow(ctx, &ws->idx2, &ws->idx2_elems, (size_t)m * 2))) return rc;
    if ((rc = grow(ctx, &ws->dist2, &ws->dist2_elems, (size_t)m * 2))) return rc;
    if ((rc = grow(ctx, &ws->flag, &ws->flag_elems, (size_t)n))) return rc;
    cudaStream_t st = ctx->stream;
    CVB_CUDA(ctx, cudaMemcpyAsync(ws->q, a, (size_t)n * 64, cudaMemcpyHostToDevice, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(ws->db, b, (size_t)m * 64, cudaMemcpyHostToDevice, st));
    if ((rc = knn_dev(ctx, ws->q, nullptr, n, ws->db, nullptr, m, 2, ws->idx, ws->dist))) return rc;
    if ((rc = knn_dev(ctx, ws->db, nullptr, m, ws->q, nullptr, n, 2, ws->idx2, ws->dist2))) return rc;
    k_symmetric<<<cdiv(n, 256), 256, 0, st>>>(ws->idx, ws->dist, ws->idx2, ws->dist2, n, m, better_by, ws->flag);
    CVB_LAUNCH_CHECK(ctx);
    const uint32_t *flag = (const uint32_t *)cvb_pinned(ctx, sizeof(uint32_t) * (size_t)n);
    if (!flag) return cvb_set_error(ctx, CVB_ENOMEM, "page-locked scratch");
    CVB_CUDA(ctx, cudaMemcpyAsync((void *)flag, ws->flag, sizeof(uint32_t) * n, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    uint32_t cnt = 0;
    for (uint32_t i = 0; i < n; i++)
        if (flag[i] != 0xffffffffu) {
            if (cnt < cap && pairs_out) { pairs_out[2 * cnt] = i; pairs_out[2 * cnt + 1] = flag[i]; }
            cnt++;
        }
    *n_out = cnt;
    if (cnt > cap) return cvb_set_error(ctx, CVB_ECAP, "pair capacity %u too small (%u needed)", cap, cnt);
    return 0;
}

}  // extern "C"
