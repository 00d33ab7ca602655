// cv_b200/csrc/lsh.cu -- exact Hamming k-NN over wide binary codes (include/cvb200_lsh.h): cv-sfm's similar-frame search
// (`lsh_to_frame.knn_values(&lsh, num)`, cv-sfm/src/lib.rs:597-668) over its 4096-bit frame hashes, k up to 1024.
//
// Semantics: distance = popcount(q ^ d) over 32 * words bits; the k smallest (distance, database index) pairs in ascending order, so
// equal distances list the lower index first (the rule of cvb_hamming_knn).  Every pair is one unique 64-bit key
// (distance << 32) | index, so the result is a plain k-smallest over unique keys: exact, and the same bytes whatever the launch
// order, split count or tie pattern.
//
// k_lsh_scan: a CTA takes Q queries and one contiguous split of the database.  Tiles of R rows are staged in shared memory with
// cp.async (double buffered); thread t computes the distance of query t / R against tile row t % R (a warp shares its query: that
// read is a broadcast).  Rows are padded to WP words, WP / 4 odd, so the 16-byte row reads of a warp are free of bank conflicts; the
// padding is zero in queries and rows alike.  Selection is a buffered top-k per query: keys below the running k-th key are appended
// to a buffer of CAP >= k + R entries; when fewer than R free slots remain, the filled part is sorted (bitonic, whole CTA), cut to k, and
// the threshold tightens to the new k-th key.  With one split the CTA writes the final lists; otherwise it writes its sorted k keys
// and k_lsh_merge runs the same selection over the per-split lists of a query (each list sorted, so a round that appends nothing
// ends that list).  No n x m matrix is materialised; the workspace is the per-split lists, bounded by the grid, not by m.
// The C names are given by lsh_abi.cu (libcvb200_lsh.so), so libcvb200.so's exports stay as they are.
#include <string.h>
#include "common.cuh"
#include "../../include/cvb200_lsh.h"

struct LshWorkspace {
    uint64_t *partial = nullptr; size_t partial_elems = 0;   // per-split sorted key lists
    uint8_t *q = nullptr; size_t q_bytes = 0;                 // host form: staged queries
    uint8_t *db = nullptr; size_t db_bytes = 0;               // host form: staged database
    uint32_t *idx = nullptr, *dist = nullptr; size_t idx_elems = 0, dist_elems = 0;   // host form: results
};

void lsh_workspace_free(LshWorkspace *w) {
    if (!w) return;
    cudaFree(w->partial); cudaFree(w->q); cudaFree(w->db); cudaFree(w->idx); cudaFree(w->dist);
    delete w;
}

namespace {

constexpr int Q = 4;                  // queries per CTA
constexpr int R = 64;                 // database rows per tile = threads per query
constexpr int NT = Q * R;             // 256 threads
constexpr int SPLIT_TILES = 16;       // fewest tiles per database split
constexpr uint64_t NONE = ~0ull;

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void cp_async4(void *dst, const void *src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async16(void *dst, const void *src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait1() { asm volatile("cp.async.wait_group 1;" ::: "memory"); }

// Shared-memory layout of both kernels: [Q][cap] keys, [Q] counts, then (scan only) [Q][WP] query words and [2][R][WP] tile words.
struct TopK {
    uint64_t *buf;
    uint32_t *cnt;
    uint32_t k, cap;
};

__device__ __forceinline__ TopK topk_layout(uint8_t *sm, uint32_t k, uint32_t cap) {
    TopK t;
    t.buf = (uint64_t *)sm;
    t.cnt = (uint32_t *)(sm + (size_t)Q * cap * sizeof(uint64_t));
    t.k = k;
    t.cap = cap;
    return t;
}

// Sorts b[0, c) ascending: bitonic over the next power of two P >= c, after padding [c, P) with NONE (P <= cap).  Whole CTA; ends
// synchronised.
__device__ void block_sort(uint64_t *b, uint32_t c) {
    uint32_t p = 1;
    while (p < c) p <<= 1;
    for (uint32_t i = c + threadIdx.x; i < p; i += NT) b[i] = NONE;
    __syncthreads();
    for (uint32_t size = 2; size <= p; size <<= 1) {
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            for (uint32_t i = threadIdx.x; i < p / 2; i += NT) {
                const uint32_t lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
                const uint64_t a = b[lo], d = b[hi];
                if ((a > d) == ((lo & size) == 0)) { b[lo] = d; b[hi] = a; }
            }
            __syncthreads();
        }
    }
}

// Called by the whole CTA after a round of appends and a barrier.  Sorts and cuts the buffer of every one of the CTA's nq queries
// that has fewer than `room` free slots (all of them when room > cap) and refreshes the caller's threshold for its own query `my_q`.
__device__ void topk_compact(const TopK &t, int nq, uint32_t room, int my_q, uint64_t &my_thr) {
#pragma unroll 1
    for (int q = 0; q < nq; q++) {
        const uint32_t c = t.cnt[q];
        if (c + room <= t.cap) continue;
        uint64_t *b = t.buf + (size_t)q * t.cap;
        block_sort(b, c);
        const uint32_t kept = min(c, t.k);
        if (q == my_q && kept == t.k) my_thr = b[t.k - 1];
        if (threadIdx.x == 0) t.cnt[q] = kept;
        __syncthreads();
    }
}

__device__ __forceinline__ void topk_append(const TopK &t, int q, uint64_t key) {
    const uint32_t pos = atomicAdd(&t.cnt[q], 1u);
    t.buf[(size_t)q * t.cap + pos] = key;
}

// Writes query q's first k keys: as (idx, dist) rows when final, else as the split's sorted key list.
__device__ void topk_store(const TopK &t, uint32_t q0, uint32_t n, uint64_t *partial, uint32_t splits, uint32_t split,
                           uint32_t *idx_out, uint32_t *dist_out) {
    for (int q = 0; q < Q; q++) {
        const uint32_t gq = q0 + q;
        if (gq >= n) break;
        const uint64_t *b = t.buf + (size_t)q * t.cap;
        const uint32_t c = t.cnt[q];
        for (uint32_t j = threadIdx.x; j < t.k; j += NT) {
            const uint64_t key = j < c ? b[j] : NONE;
            if (partial) {
                partial[((size_t)gq * splits + split) * t.k + j] = key;
            } else {
                idx_out[(size_t)gq * t.k + j] = key == NONE ? 0xffffffffu : (uint32_t)key;
                dist_out[(size_t)gq * t.k + j] = key == NONE ? 0xffffffffu : (uint32_t)(key >> 32);
            }
        }
    }
}

__device__ __forceinline__ uint32_t count_of(const uint32_t *dev, uint32_t host_max) { return dev ? min(*dev, host_max) : host_max; }

// grid = (ceil(n_max / Q), splits); split s covers database rows [s * chunk, min((s + 1) * chunk, m)).
__global__ void __launch_bounds__(NT) k_lsh_scan(const uint32_t *__restrict__ queries, const uint32_t *__restrict__ n_dev, uint32_t n_max,
                                                 const uint32_t *__restrict__ db, const uint32_t *__restrict__ m_dev, uint32_t m_max,
                                                 uint32_t words, uint32_t wp, uint32_t k, uint32_t cap, uint32_t chunk,
                                                 uint64_t *__restrict__ partial, uint32_t *__restrict__ idx_out,
                                                 uint32_t *__restrict__ dist_out) {
    extern __shared__ __align__(16) uint8_t sm[];
    const uint32_t n = count_of(n_dev, n_max), m = count_of(m_dev, m_max);
    const uint32_t q0 = blockIdx.x * Q;
    if (q0 >= n) return;
    const TopK t = topk_layout(sm, k, cap);
    uint32_t *s_q = (uint32_t *)(sm + (size_t)Q * cap * sizeof(uint64_t) + 16);
    uint32_t *s_tile = s_q + (size_t)Q * wp;                   // [2][R][wp]
    const int my_q = threadIdx.x / R, my_r = threadIdx.x % R, nq = (int)min((uint32_t)Q, n - q0);
    const bool active = my_q < nq;
    const uint32_t lo = min(blockIdx.y * chunk, m), hi = min(lo + chunk, m), rows = hi - lo;
    const uint32_t ntiles = (rows + R - 1) / R;

    if (threadIdx.x < Q) t.cnt[threadIdx.x] = 0;
    for (uint32_t i = threadIdx.x; i < Q * wp; i += NT) {
        const uint32_t q = i / wp, c = i - q * wp;
        s_q[i] = (c < words && q0 + q < n) ? queries[(size_t)(q0 + q) * words + c] : 0u;
    }
    for (uint32_t i = threadIdx.x; i < 2 * R * (wp - words); i += NT) {   // padding columns of both tile buffers
        const uint32_t r = i / (wp - words), c = words + (i - r * (wp - words));
        s_tile[(size_t)r * wp + c] = 0u;
    }
    const bool vec = (words & 3) == 0;                          // rows start on 16-byte boundaries: 16-byte copies
    const uint32_t unit = vec ? 4 : 1, upr = words / unit;
    auto stage = [&](uint32_t tile) {
        if (tile < ntiles) {
            const uint32_t first = tile * R, nrows = min((uint32_t)R, rows - first);
            const uint32_t *src = db + (size_t)(lo + first) * words;
            uint32_t *dst = s_tile + (size_t)(tile & 1) * R * wp;
            for (uint32_t i = threadIdx.x; i < nrows * upr; i += NT) {
                const uint32_t r = i / upr, c = (i - r * upr) * unit;
                if (vec) cp_async16(dst + (size_t)r * wp + c, src + (size_t)r * words + c);
                else cp_async4(dst + (size_t)r * wp + c, src + (size_t)r * words + c);
            }
        }
        cp_async_commit();
    };
    stage(0);
    stage(1);
    __syncthreads();                                           // counts and padding visible, also when there is no tile
    uint64_t thr = NONE;
    const uint4 *qv = (const uint4 *)(s_q + (size_t)my_q * wp);
    const uint32_t nv = wp / 4;
    for (uint32_t tile = 0; tile < ntiles; tile++) {
        cp_async_wait1();
        __syncthreads();
        const uint32_t row = tile * R + my_r;
        if (active && row < rows) {
            const uint4 *dv = (const uint4 *)(s_tile + ((size_t)(tile & 1) * R + my_r) * wp);
            uint32_t d = 0;
#pragma unroll 4
            for (uint32_t v = 0; v < nv; v++) {
                const uint4 a = qv[v], b = dv[v];
                d += __popc(a.x ^ b.x) + __popc(a.y ^ b.y) + __popc(a.z ^ b.z) + __popc(a.w ^ b.w);
            }
            const uint64_t key = ((uint64_t)d << 32) | (lo + row);
            if (key < thr) topk_append(t, my_q, key);
        }
        __syncthreads();                                       // appends done; tile buffer (tile & 1) is free
        stage(tile + 2);
        topk_compact(t, nq, R, my_q, thr);
    }
    topk_compact(t, nq, cap + 1, my_q, thr);                       // final sort of every buffer
    topk_store(t, q0, n, gridDim.y > 1 ? partial : nullptr, gridDim.y, blockIdx.y, idx_out, dist_out);
}

// grid = ceil(n_max / Q): the k smallest keys of the `splits` sorted lists of each query.
__global__ void __launch_bounds__(NT) k_lsh_merge(const uint64_t *__restrict__ partial, const uint32_t *__restrict__ n_dev,
                                                  uint32_t n_max, const uint32_t *__restrict__ m_dev, uint32_t m_max, uint32_t k,
                                                  uint32_t cap, uint32_t splits, uint32_t chunk, uint32_t *__restrict__ idx_out,
                                                  uint32_t *__restrict__ dist_out) {
    extern __shared__ __align__(16) uint8_t sm[];
    const uint32_t n = count_of(n_dev, n_max), m = count_of(m_dev, m_max);
    const uint32_t q0 = blockIdx.x * Q;
    if (q0 >= n) return;
    const TopK t = topk_layout(sm, k, cap);
    const int my_q = threadIdx.x / R, my_r = threadIdx.x % R, nq = (int)min((uint32_t)Q, n - q0);
    const bool active = my_q < nq;
    if (threadIdx.x < Q) t.cnt[threadIdx.x] = 0;
    __syncthreads();
    uint64_t thr = NONE;
    for (uint32_t s = 0; s < splits; s++) {
        const uint32_t lo = min(s * chunk, m), len = min(min(lo + chunk, m) - lo, k);   // valid keys of list s
        const uint64_t *list = partial + ((size_t)(q0 + my_q) * splits + s) * k;
        for (uint32_t j0 = 0; j0 < len; j0 += R) {
            bool appended = false;
            if (active && j0 + my_r < len) {
                const uint64_t key = list[j0 + my_r];
                if (key < thr) { topk_append(t, my_q, key); appended = true; }
            }
            if (!__syncthreads_or(appended)) break;              // the lists ascend: nothing later in list s can enter
            topk_compact(t, nq, R, my_q, thr);
        }
    }
    topk_compact(t, nq, cap + 1, my_q, thr);
    topk_store(t, q0, n, nullptr, 1, 0, idx_out, dist_out);
}

uint32_t padded_words(uint32_t words) {
    uint32_t wp = (words + 3) & ~3u;
    if (((wp / 4) & 1) == 0) wp += 4;
    return wp;
}

uint32_t buffer_cap(uint32_t k) {
    uint32_t need = std::max(2 * k, k + (uint32_t)R), cap = 1;
    while (cap < need) cap <<= 1;
    return cap;
}

size_t topk_smem(uint32_t cap) { return (size_t)Q * cap * sizeof(uint64_t) + 16; }

LshWorkspace *workspace(cvb_ctx *ctx) {
    if (!ctx->lsh) ctx->lsh = new LshWorkspace();
    return ctx->lsh;
}

int check_args(cvb_ctx *ctx, uint32_t words, uint32_t k, uint32_t m_max, const void *q, const void *db, const void *idx,
               const void *dist) {
    if (words < 1 || words > CVB_LSH_MAX_WORDS) return cvb_set_error(ctx, CVB_EINVAL, "words must be 1..%d (got %u)", CVB_LSH_MAX_WORDS, words);
    if (k < 1 || k > CVB_LSH_MAX_K) return cvb_set_error(ctx, CVB_EINVAL, "k must be 1..%d (got %u)", CVB_LSH_MAX_K, k);
    if (m_max >= 0xffffffffu) return cvb_set_error(ctx, CVB_EINVAL, "the database must hold fewer than 2^32 - 1 codes");
    if (!q || !db || !idx || !dist) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    return 0;
}

int knn_launch(cvb_ctx *ctx, uint32_t words, const uint8_t *q, const uint32_t *n_dev, uint32_t n_max, const uint8_t *db,
               const uint32_t *m_dev, uint32_t m_max, uint32_t k, uint32_t *idx, uint32_t *dist) {
    if (n_max == 0) return 0;
    const uint32_t wp = padded_words(words), cap = buffer_cap(k);
    const size_t scan_smem = topk_smem(cap) + sizeof(uint32_t) * (size_t)(Q + 2 * R) * wp;
    const size_t merge_smem = topk_smem(cap);
    static bool attr_set = false;   // once per process: the largest layout (k = 1024, words = 128) is 132 KB
    if (!attr_set) {
        const int most = (int)(topk_smem(buffer_cap(CVB_LSH_MAX_K)) + sizeof(uint32_t) * (size_t)(Q + 2 * R) * padded_words(CVB_LSH_MAX_WORDS));
        CVB_CUDA(ctx, cudaFuncSetAttribute(k_lsh_scan, cudaFuncAttributeMaxDynamicSharedMemorySize, most));
        CVB_CUDA(ctx, cudaFuncSetAttribute(k_lsh_merge, cudaFuncAttributeMaxDynamicSharedMemorySize, most));
        attr_set = true;
    }
    // Split the database until the grid has about two CTAs per SM, keeping at least SPLIT_TILES tiles per split: k_lsh_merge walks the
    // lists one after another, so a single query pays for every split it adds.
    const uint32_t qblocks = cdiv(n_max, Q);
    uint32_t splits = std::min(cdiv(2u * (uint32_t)ctx->num_sms, qblocks), std::max(1u, cdiv(m_max, SPLIT_TILES * R)));
    splits = std::max(splits, 1u);
    const uint32_t chunk = splits > 1 ? cdiv(m_max, splits) : std::max(m_max, 1u);
    if (splits > 1) splits = cdiv(m_max, chunk);
    LshWorkspace *ws = workspace(ctx);
    int rc;
    if (splits > 1 && (rc = ws_grow(ctx, &ws->partial, &ws->partial_elems, (size_t)n_max * splits * k))) return rc;
    cudaStream_t st = ctx->stream;
    {
        CVB_PROF(ctx, "k_lsh_scan", 4.0 * words * ((double)m_max * qblocks + n_max));
        k_lsh_scan<<<dim3(qblocks, splits), NT, scan_smem, st>>>((const uint32_t *)q, n_dev, n_max, (const uint32_t *)db, m_dev, m_max,
                                                                 words, wp, k, cap, chunk, ws->partial, idx, dist);
        CVB_LAUNCH_CHECK(ctx);
    }
    if (splits > 1) {
        CVB_PROF(ctx, "k_lsh_merge", 8.0 * n_max * splits * k);
        k_lsh_merge<<<qblocks, NT, merge_smem, st>>>(ws->partial, n_dev, n_max, m_dev, m_max, k, cap, splits, chunk, idx, dist);
        CVB_LAUNCH_CHECK(ctx);
    }
    return 0;
}

}  // namespace

int lsh_hash_knn_dev(cvb_ctx *ctx, uint32_t words, const uint8_t *queries_dev, const uint32_t *n_dev, uint32_t n_max,
                     const uint8_t *database_dev, const uint32_t *m_dev, uint32_t m_max, uint32_t k, uint32_t *idx_out_dev,
                     uint32_t *dist_out_dev) {
    if (!ctx) return CVB_EINVAL;
    int rc = check_args(ctx, words, k, m_max, queries_dev, database_dev, idx_out_dev, dist_out_dev);
    if (rc) return rc;
    if ((((uintptr_t)queries_dev | (uintptr_t)database_dev | (uintptr_t)idx_out_dev | (uintptr_t)dist_out_dev) & 15))
        return cvb_set_error(ctx, CVB_EINVAL, "device arrays must be 16-byte aligned");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    return knn_launch(ctx, words, queries_dev, n_dev, n_max, database_dev, m_dev, m_max, k, idx_out_dev, dist_out_dev);
}

int lsh_hash_knn(cvb_ctx *ctx, uint32_t words, const uint8_t *queries, uint32_t n, const uint8_t *database, uint32_t m, uint32_t k,
                 uint32_t *idx_out, uint32_t *dist_out) {
    if (!ctx) return CVB_EINVAL;
    int rc = check_args(ctx, words, k, m, queries, database, idx_out, dist_out);
    if (rc) return rc;
    if (n == 0) return 0;
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    LshWorkspace *ws = workspace(ctx);
    const size_t row = 4 * (size_t)words, nout = (size_t)n * k;
    if ((rc = ws_grow(ctx, &ws->q, &ws->q_bytes, n * row)) || (rc = ws_grow(ctx, &ws->db, &ws->db_bytes, std::max<size_t>(m, 1) * row)))
        return rc;
    if ((rc = ws_grow(ctx, &ws->idx, &ws->idx_elems, nout)) || (rc = ws_grow(ctx, &ws->dist, &ws->dist_elems, nout))) return rc;
    cudaStream_t st = ctx->stream;
    CVB_CUDA(ctx, cudaMemcpyAsync(ws->q, queries, n * row, cudaMemcpyHostToDevice, st));
    if (m) CVB_CUDA(ctx, cudaMemcpyAsync(ws->db, database, m * row, cudaMemcpyHostToDevice, st));
    if ((rc = knn_launch(ctx, words, ws->q, nullptr, n, ws->db, nullptr, m, k, ws->idx, ws->dist))) return rc;
    CVB_CUDA(ctx, cudaMemcpyAsync(idx_out, ws->idx, sizeof(uint32_t) * nout, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(dist_out, ws->dist, sizeof(uint32_t) * nout, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    return 0;
}
