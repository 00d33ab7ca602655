// cv_b200/csrc/arrsac_dev.cuh -- arrsac::Arrsac::model_inliers entirely on the device (included by geom.cu).
//
// The reference loop (external crate arrsac 0.10.0, restated for the CPU checker under the test tree; call sites
// cv-sfm/src/lib.rs:1394-1406, vslam-sandbox/src/main.rs:105-117, akaze/tests/estimate_pose.rs:63-75) is sequential in
// three places: the random draws, the adaptive likelihood-ratio test over the initial hypotheses, and the block loop
// (score, stable sort, halve, re-estimate from the best inlier set).  Round 1 ran that bookkeeping on the host with
// ~3 stream synchronisations per 64-datum block.  Here nothing returns to the host between enqueue and result:
//
//   k_ars_begin     minimal samples of all initial hypotheses from a pre-generated stream of raw u32 draws (the modulo and
//                   the rejection of repeats need n, which may only exist on the device); one CTA, 256 samples per turn, a turn
//                   commits the samples in front of its first repeat (ars_sample_block_par)
//   k_ars_estimate  eight-point / P3P / five-point per hypothesis (k_estimate's device functions); k_ars_estimate8<L>: eight-point
//                   with L lanes per hypothesis on the round-robin Jacobi (geom.cu: sym_eigen9_rr)
//   k_ars_score     one warp per (model, 32 data): inlier bits by ballot.  CameraToCamera bits come from the exact-predicate
//                   filter (c2c_filter.cuh); the predicates it leaves undecided are queued for the Jacobi evaluation
//   k_ars_resolve   the queued predicates, one per thread (k_ars_resolve_block: those of a block iteration's scoring)
//   k_ars_sprt      one CTA: the adaptive SPRT over all initial models in order.  Up to 1024 models are walked concurrently under
//                   the state in front of the chunk; a walk carries the exact likelihood ratio and both corners of nested BOXES of
//                   delta values -- f32 multiplication is monotone, so a model whose corners stop where the exact walk stops has
//                   that outcome for every delta inside the box.  Block-wide prefix sums then give the exact state in front of
//                   every model; models whose state leaves their box are walked again (all at once), everything up to the first
//                   model that raises epsilon is committed, and the next chunk starts behind it.  Then: stable top-max_candidate
//                   selection (histogram + ordered compaction + bitonic).
//   k_ars_book      one CTA per block of data: accept the new hypotheses that beat the bar, stable sort, truncate, termination
//                   test, add the next block's inliers, stable sort, halve, inlier pool of the best, next minimal samples.
//   k_ars_final     inlier list of the winner.
// The candidate table is double buffered (rows = pose + inlier count + inlier bit mask); every k_ars_book writes the
// surviving rows in sorted order into the other buffer, so there is no free list and no indirection.
//
// Batches: one launch per stage serves B independent problems.  The one-CTA kernels (begin, sprt, book, final) run B CTAs and take
// the problem from blockIdx.x; the estimate, score and resolve grids take it from blockIdx.y.  Problem pb owns ctl[pb] and the pb-th
// slice of every workspace buffer (ars_ws: strides from the launch parameters), its own staged raw-draw stream, data rows
// [pb * sdata, pb * sdata + n) and the pb-th share of the undecided-predicate queue.  A single problem is the batch of one: pb = 0
// everywhere, so its addresses, launches and results are those of the unbatched driver.
#pragma once

#define ARS_SORT_CAP 4096u     // max_candidate_hypotheses + estimations_per_block * models_per_sample must fit
#define ARS_BOOK_NT 1024
#define ARS_BOOK_SMEM (14u * ARS_SORT_CAP)
#define ARS_QCAP (1u << 20)    // queue of undecided predicates of a scoring stage (entries beyond it are evaluated in place); a batch of B
                               // problems splits it, ARS_QCAP / B entries per problem and stage

struct ArrsacCtl {
    uint32_t n, init_n, Mv, npass;
    uint32_t Hn, cur, blk_lo, blk_hi;
    uint32_t acc_hi, n_new, worst, done;
    uint32_t found, iters, nraw, q_count;     // q_count / q_count2: undecided (model, datum) predicates queued by the two initial scoring stages
    uint32_t q_count2, stat_lazy;             // stat_lazy: mask words the SPRT had to compute itself
    uint32_t stat_units0, stat_units2;        // 32-datum units scored by the two initial stages
    uint32_t stat_repairs, stat_pad;          // SPRT: models walked again with their exact state
    uint64_t rng_pos, gen_pos;
    cvb_rng gen;                 // generator positioned at raw index gen_pos (continues the stream when it is exhausted)
    cvb_pose winner;
    uint32_t n_inliers, overflow;
    uint32_t stat_chunks, stat_pass;
    uint32_t stat_walk_us, stat_commit_us;   // SPRT: time in the chunk walks / in the commit turns (globaltimer)
    uint32_t stat_perm_us, stat_turns;       // SPRT: time in the ordering step in front of the walks; commit turns in total
    uint32_t q_blk, stat_qblk;               // undecided predicates queued by the current block's scoring (queue region 0); over all blocks
    uint32_t stat_units_kept, stat_units_new; // block loop: 32-datum units of kept rows / of new models (valid poses)
    uint32_t stat_skip;                      // new-model units written 0 by early rejection instead of scored
    uint32_t stat_blk_w0, stat_blk_lt32;     // blocks with new models scored under worst == 0 / under acc_hi - worst < 32
    uint32_t stat_blk_bar0;                  // blocks whose new samples were drawn but not estimated (worst >= acc_hi)
    uint32_t retired;                        // k_ars_book has taken this problem off the batch's live count
};

struct ArrsacParams {            // launch-constant configuration (by value)
    uint32_t K, MM, kind;        // MIN_SAMPLES, models per sample, estimator kind
    uint32_t H0, ib, bs, max_cand, G;
    uint32_t W0;                 // mask words per model of the initialisation (ceil(bs * ib / 32))
    uint32_t NW;                 // mask words per candidate row (ceil(NMAX / 32))
    uint32_t NMAX;               // data capacity
    uint32_t rows;               // candidate rows per table (max_cand + G * MM)
    uint32_t prefix, cmin;       // initial scoring in two stages: all words for the first `prefix` samples; for the rest, words >= 1 only
                                 // when the first 32 data hold >= cmin inliers (the SPRT computes a missing word itself if it ever needs one)
    uint32_t early;              // block scoring stops scoring new models that can no longer beat the bar (k_ars_score phase 1)
    uint32_t nraw;               // staged raw draws per problem
    uint32_t qcap;               // queue entries per problem and scoring stage (ARS_QCAP / B)
    uint32_t sdata;              // data rows per problem (problem pb's rows start at pb * sdata)
    float lr_thr, eps0, delta0;
    double thr;
    int row0;
};

// per-problem slice sizes of the workspace buffers, in elements (the host allocates B of each, the kernels offset by pb)
struct ArsStrides {
    size_t samples0, models0, nposes0, vm, rows2, tmasks, nnew, nposes_new, newmask, samples_new, queue, a, b;
};
__host__ __device__ __forceinline__ ArsStrides ars_strides(const ArrsacParams &P) {
    ArsStrides s;
    const size_t h0 = P.H0 ? P.H0 : 1, g = P.G ? P.G : 1, m0 = P.H0 ? (size_t)P.H0 * P.MM : 1;
    s.samples0 = h0 * P.K; s.models0 = m0; s.nposes0 = h0; s.vm = m0 > ARS_SORT_CAP ? m0 : ARS_SORT_CAP;
    s.rows2 = 2 * (size_t)P.rows; s.tmasks = s.rows2 * P.NW;
    s.nnew = g * P.MM; s.nposes_new = g; s.newmask = s.nnew * P.NW; s.samples_new = g * P.K;
    s.queue = 2 * (size_t)P.qcap;
    s.a = 3 * (size_t)P.sdata; s.b = (P.kind == 1 ? 4 : 3) * (size_t)P.sdata;
    return s;
}


__device__ __forceinline__ unsigned long long ars_globaltimer() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
__device__ __forceinline__ uint64_t ars_rotl64(uint64_t x, int k) { return (x << k) | (x >> (64 - k)); }
__device__ uint32_t ars_rng_next_u32(cvb_rng *r) {
    if (r->kind == 0) {
        uint64_t *s = r->s;
        const uint64_t result = ars_rotl64(s[0] + s[3], 23) + s[0];
        const uint64_t t = s[1] << 17;
        s[2] ^= s[0]; s[3] ^= s[1]; s[1] ^= s[2]; s[0] ^= s[3]; s[2] ^= t; s[3] = ars_rotl64(s[3], 45);
        return (uint32_t)(result >> 32);
    }
    unsigned __int128 state = (unsigned __int128)r->s[0] | ((unsigned __int128)r->s[1] << 64);
    const unsigned __int128 incr = (unsigned __int128)r->s[2] | ((unsigned __int128)r->s[3] << 64);
    const unsigned __int128 MUL = ((unsigned __int128)0x2360ED051FC65DA4ull << 64) | 0x4385DF649FCCF645ull;
    state = state * MUL + incr;
    r->s[0] = (uint64_t)state; r->s[1] = (uint64_t)(state >> 64);
    const uint32_t rot = (uint32_t)(state >> 122);
    const uint64_t xsl = (uint64_t)(state >> 64) ^ (uint64_t)state;
    return (uint32_t)((xsl >> rot) | (xsl << ((64 - rot) & 63)));
}

// raw draw number pos of the caller's generator (sequential consumers only: pos never decreases)
__device__ uint32_t ars_raw_at(ArrsacCtl *ctl, const uint32_t *raw, uint64_t pos) {
    if (pos < ctl->nraw) return raw[pos];
    uint32_t v = 0;
    while (ctl->gen_pos <= pos) { v = ars_rng_next_u32(&ctl->gen); ctl->gen_pos++; }
    return v;
}

// `count` minimal samples of K distinct indices below len: next_u32() % len with rejection of repeats, exactly in the
// reference's draw order.  Called by EVERY thread of the CTA: the raw draws are staged through a shared-memory window (cooperative,
// coalesced loads; the consumer's position depends on the data, so reading them from global memory one warp-step at a time costs
// an L2 round trip per step), and warp 0 consumes them: 32/K samples per step are taken from 32 consecutive draws when none of
// them repeats inside its sample (the common case); a sample with a repeat is redone draw by draw by lane 0.
#define ARS_WIN 4096u
__device__ void ars_sample_block(ArrsacCtl *ctl, const uint32_t *raw, uint32_t len, uint32_t K, uint32_t count, uint32_t *out,
                                 const uint32_t *map, uint32_t *win /* ARS_WIN words of shared memory */, uint32_t *sh /* 4 shared words */) {
    const unsigned full = 0xffffffffu;
    const uint32_t lane = threadIdx.x & 31, hps = 32 / K;
    const uint32_t g = lane / K, k = lane % K;
    const uint32_t nraw = ctl->nraw;
    if (threadIdx.x == 0) { sh[0] = 0; *(uint64_t *)(sh + 2) = ctl->rng_pos; }
    __syncthreads();
    while (true) {
        const uint32_t h0 = sh[0];
        const uint64_t wbase = *(const uint64_t *)(sh + 2);
        if (h0 >= count) break;
        for (uint32_t i = threadIdx.x; i < ARS_WIN; i += blockDim.x) win[i] = wbase + i < nraw ? raw[wbase + i] : 0u;
        __syncthreads();
        if (threadIdx.x < 32) {
            uint64_t pos = wbase;
            uint32_t h = h0;
            while (h < count) {
                const bool in_win = pos + 32 <= wbase + ARS_WIN && pos + 32 <= nraw;
                if (!in_win && pos + 32 <= nraw) break;             // refill the window at pos
                if (in_win) {
                    const uint32_t ng = min(hps, count - h);
                    const bool act = g < ng;
                    const uint32_t s = win[(uint32_t)(pos - wbase) + lane] % len;
                    bool dup = false;
                    for (uint32_t j = 1; j < K; j++) {
                        const uint32_t o = __shfl_sync(full, s, (lane - j) & 31);
                        if (k >= j && o == s) dup = true;
                    }
                    const unsigned dm = __ballot_sync(full, act && dup);
                    const uint32_t good = dm ? (uint32_t)(__ffs(dm) - 1) / K : ng;
                    if (act && g < good) out[(size_t)(h + g) * K + k] = map ? map[s] : s;
                    h += good; pos += (uint64_t)good * K;
                    if (good == ng) continue;
                }
                if (lane == 0) {      // one sample draw by draw (a repeat inside it, or the tail of the staged stream)
                    uint32_t loc[8];
                    for (uint32_t c = 0; c < K;) {
                        const uint32_t r = (pos >= wbase && pos < wbase + ARS_WIN && pos < nraw) ? win[(uint32_t)(pos - wbase)] : ars_raw_at(ctl, raw, pos);
                        const uint32_t s = r % len;
                        pos++;
                        bool dup = false;
                        for (uint32_t j = 0; j < c; j++) dup |= loc[j] == s;
                        if (!dup) { loc[c] = s; out[(size_t)h * K + c] = map ? map[s] : s; c++; }
                    }
                }
                pos = __shfl_sync(full, pos, 0);
                h++;
            }
            if (lane == 0) { sh[0] = h; *(uint64_t *)(sh + 2) = pos; }
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) ctl->rng_pos = *(const uint64_t *)(sh + 2);
    __syncthreads();
}

// The same samples, CTA-parallel, for the big initial batch (no index map).  A sample without a repeat consumes exactly K draws, so
// thread t takes sample h0 + t from draws [p0 + t*K, p0 + (t+1)*K) -- right as long as no earlier sample of the turn met a repeat
// (probability K(K-1)/2n per sample).  Samples in front of the first repeat are committed, the thread that owns it redoes its sample
// draw by draw (the reference's loop) and the next turn starts behind it.  The tail of the staged stream goes to ars_sample_block.
__device__ void ars_sample_block_par(ArrsacCtl *ctl, const uint32_t *raw, uint32_t len, uint32_t K, uint32_t count, uint32_t *out,
                                     uint32_t *win, uint32_t *sh /* 4 shared words */) {
    const uint32_t nraw = ctl->nraw, tid = threadIdx.x;
    if (tid == 0) { sh[0] = 0; *(uint64_t *)(sh + 2) = ctl->rng_pos; }
    __syncthreads();
    while (true) {
        const uint32_t h0 = sh[0];
        const uint64_t p0 = *(const uint64_t *)(sh + 2);
        if (h0 >= count) break;
        // a turn commits the samples in front of its first repeat (one in ~2n / K(K-1) samples): wider turns mostly compute discards
        const uint32_t m = min(min((uint32_t)blockDim.x, 256u), count - h0);
        if (p0 + (uint64_t)(m + 8) * K > nraw) break;               // not enough staged draws for a whole turn (+ slack for the redo)
        __syncthreads();                                            // everyone has read sh[0] / the position
        if (tid == 0) sh[1] = m;
        __syncthreads();
        uint32_t loc[8];
        if (tid < m) {
            bool dup = false;
            for (uint32_t k = 0; k < K; k++) {
                loc[k] = raw[p0 + (uint64_t)tid * K + k] % len;
                for (uint32_t j = 0; j < k; j++) dup |= loc[j] == loc[k];
            }
            if (dup) atomicMin(&sh[1], tid);
        }
        __syncthreads();
        const uint32_t f = sh[1];
        if (tid < f)
            for (uint32_t k = 0; k < K; k++) out[(size_t)(h0 + tid) * K + k] = loc[k];
        if (f < m && tid == f) {
            // the reference's loop over this sample: its first K draws are the ones already reduced in loc[] (consumed in order, repeats
            // dropped), further draws come from the stream one at a time
            uint32_t t[8];
            for (uint32_t k = 0; k < K; k++) t[k] = loc[k];
            uint64_t pos = p0 + (uint64_t)f * K + K;
            uint32_t c = 0;
            for (uint32_t k = 0; k < K; k++) {
                bool dup = false;
                for (uint32_t j = 0; j < c; j++) dup |= loc[j] == t[k];
                if (!dup) loc[c++] = t[k];
            }
            while (c < K) {
                const uint32_t s = ars_raw_at(ctl, raw, pos) % len;
                pos++;
                bool dup = false;
                for (uint32_t j = 0; j < c; j++) dup |= loc[j] == s;
                if (!dup) loc[c++] = s;
            }
            for (uint32_t k = 0; k < K; k++) out[(size_t)(h0 + f) * K + k] = loc[k];
            sh[0] = h0 + f + 1; *(uint64_t *)(sh + 2) = pos;
        } else if (f >= m && tid == 0) {
            sh[0] = h0 + m; *(uint64_t *)(sh + 2) = p0 + (uint64_t)m * K;
        }
        __syncthreads();
    }
    const uint32_t hdone = sh[0];
    __syncthreads();
    if (tid == 0) ctl->rng_pos = *(const uint64_t *)(sh + 2);
    __syncthreads();
    if (hdone < count) ars_sample_block(ctl, raw, len, K, count - hdone, out + (size_t)hdone * K, nullptr, win, sh);
}

// ---- k_ars_begin ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(ARS_BOOK_NT) k_ars_begin(ArrsacCtl *ctl, ArrsacParams P, const uint32_t *n_dev, uint32_t n_host,
                                                            const uint32_t *raw, uint32_t *samples0) {
    __shared__ uint32_t win[ARS_WIN];
    __shared__ __align__(8) uint32_t sh[4];
    const uint32_t pb = blockIdx.x;
    ctl += pb; raw += (size_t)pb * P.nraw; samples0 += pb * ars_strides(P).samples0;
    const uint32_t n = min(n_dev ? n_dev[pb] : n_host, P.NMAX);
    if (threadIdx.x == 0) {
        ctl->n = n;
        ctl->init_n = min(P.bs * P.ib, n);
        ctl->Mv = 0; ctl->npass = 0; ctl->Hn = 0; ctl->cur = 0; ctl->blk_lo = ctl->blk_hi = ctl->acc_hi = 0;
        ctl->n_new = 0; ctl->worst = 0; ctl->found = 0; ctl->iters = 0; ctl->n_inliers = 0; ctl->overflow = 0;
        ctl->stat_chunks = 0; ctl->stat_pass = 0; ctl->q_count = 0; ctl->q_count2 = 0; ctl->stat_lazy = 0; ctl->stat_units0 = 0; ctl->stat_units2 = 0; ctl->stat_repairs = 0; ctl->stat_pad = 0; ctl->stat_walk_us = 0; ctl->stat_commit_us = 0; ctl->stat_perm_us = 0; ctl->stat_turns = 0;
        ctl->q_blk = 0; ctl->stat_qblk = 0;
        ctl->done = (n < P.K || P.H0 == 0) ? 1u : 0u;
    }
    __syncthreads();
    if (n < P.K || P.H0 == 0) return;
    ars_sample_block_par(ctl, raw, n, P.K, P.H0, samples0, win, sh);
}

// ---- k_ars_estimate ------------------------------------------------------------------------------------------------------
template <int KIND>
__global__ void __launch_bounds__(128) k_ars_estimate(const ArrsacCtl *ctl, int phase, uint32_t H_init, const double *__restrict__ a,
                                                      const double *__restrict__ b, const uint32_t *__restrict__ samples,
                                                      cvb_pose *poses, uint8_t *nposes, int row0, ArrsacParams P) {
    const uint32_t pb = blockIdx.y;
    ctl += pb;
    if (ctl->done) return;
    {
        const ArsStrides S = ars_strides(P);
        a += pb * S.a; b += pb * S.b;
        samples += pb * (phase == 0 ? S.samples0 : S.samples_new); poses += pb * (phase == 0 ? S.models0 : S.nnew);
        nposes += pb * (phase == 0 ? S.nposes0 : S.nposes_new);
    }
    const uint32_t H = phase == 0 ? H_init : ctl->n_new;
    const uint32_t h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= H) return;
    if (KIND == 2) { nposes[h] = (uint8_t)five_point(a, b, samples + (size_t)h * 5, row0, poses + (size_t)h * 40); return; }
    cvb_pose out[4];
    const int n = KIND == 0 ? eight_point(a, b, samples + (size_t)h * 8, out) : p3p(a, b, samples + (size_t)h * 3, out);
    for (int k = 0; k < n; k++) poses[(size_t)h * 4 + k] = out[k];
    nposes[h] = (uint8_t)n;
}

// Eight-point with EIGHT_LANES lanes per hypothesis, the 9x9 matrix and its eigenvectors in shared memory (128 / EIGHT_LANES hypotheses per CTA).
// The chain of 36 rotations x ~8 sweeps is what a block of the hypothesis loop waits for: a rotation is the FP64 divide / square-root
// sequence (every lane) followed by the column and row updates (split over the lanes).  (A nine-lane version with the matrix in
// REGISTERS and shuffles was measured slower than one thread; shared memory keeps the element exchange off the critical path.)
template <int EIGHT_LANES, int MINB>
__global__ void __launch_bounds__(128, MINB) k_ars_estimate8(const ArrsacCtl *ctl, int phase, uint32_t H_init, const double *__restrict__ a,
                                                       const double *__restrict__ b, const uint32_t *__restrict__ samples,
                                                       cvb_pose *poses, uint8_t *nposes, ArrsacParams P) {
    const uint32_t pb = blockIdx.y;
    ctl += pb;
    if (ctl->done) return;
    {
        const ArsStrides S = ars_strides(P);
        a += pb * S.a; b += pb * S.b;
        samples += pb * (phase == 0 ? S.samples0 : S.samples_new); poses += pb * (phase == 0 ? S.models0 : S.nnew);
        nposes += pb * (phase == 0 ? S.nposes0 : S.nposes_new);
    }
    __shared__ double sh[(128 / EIGHT_LANES) * EIGHT_SH];
    const uint32_t H = phase == 0 ? H_init : ctl->n_new;
    const uint32_t g = threadIdx.x / EIGHT_LANES, lane = threadIdx.x % EIGHT_LANES;
    const uint32_t h = blockIdx.x * (128 / EIGHT_LANES) + g;
    if (h >= H) return;                                          // whole lane groups leave together
    const unsigned mask = ((1u << EIGHT_LANES) - 1u) << ((threadIdx.x & 31) / EIGHT_LANES * EIGHT_LANES);
    cvb_pose out[4];
    const int n = eight_point_lanes<EIGHT_LANES>(a, b, samples + (size_t)h * 8, out, sh + g * EIGHT_SH, lane, mask);
    if (lane == 0) {
        for (int k = 0; k < n; k++) poses[(size_t)h * 4 + k] = out[k];
        nposes[h] = (uint8_t)n;
    }
}

// ---- k_ars_score ---------------------------------------------------------------------------------------------------------
// the exact evaluation behind a call: inlining the 4x4 Jacobi into the scoring kernels cost 148 registers (one 256-thread CTA per SM,
// FP64 pipe 30 % busy in ncu); out of line the filter path fits two CTAs per SM
__device__ __noinline__ bool ars_exact_c2c(const cvb_pose *Pz, const double *pa, const double *pb, double thr) {
    return residual_c2c(*Pz, pa, pb) < thr;
}

template <int RES>
__device__ __forceinline__ bool ars_inlier(const cvb_pose &Pz, const double *__restrict__ a, const double *__restrict__ b, uint32_t i,
                                           double thr) {
    if (RES == 1) return residual_w2c(Pz, a + 3 * (size_t)i, b + 4 * (size_t)i) < thr;
    const double *pa = a + 3 * (size_t)i, *pb = b + 3 * (size_t)i;
    int f = c2c_inlier_filter(Pz.r, Pz.t, pa, pb, thr);
    if (f < 0) f = ars_exact_c2c(&Pz, pa, pb, thr) ? 1 : 0;
    return f != 0;
}

// the scoring kernels' predicate: the exact evaluation costs ~8x the filter, so an undecided pair goes to a queue that a resolve
// kernel works off without divergence (one undecided lane would otherwise stall its warp for the whole Jacobi iteration) and
// counts as an outlier until then; `src` tells the resolve kernel which pose and mask row the entry belongs to.
// Returns 1 (inlier), 0 (certain outlier) or -1 (queued: its mask bit is 0 until k_ars_resolve* decides it).
template <int RES>
__device__ __forceinline__ int ars_inlier_queued(const cvb_pose &Pz, const double *__restrict__ a, const double *__restrict__ b, uint32_t i,
                                                 double thr, uint32_t *qc, uint2 *q, uint32_t qcap, uint32_t src) {
    if (RES == 1) return ars_inlier<RES>(Pz, a, b, i, thr) ? 1 : 0;
    const double *pa = a + 3 * (size_t)i, *pb = b + 3 * (size_t)i;
    const int f = c2c_inlier_filter(Pz.r, Pz.t, pa, pb, thr);
    if (f >= 0) return f != 0 ? 1 : 0;
    const uint32_t slot = atomicAdd(qc, 1u);
    if (slot < qcap) { q[slot] = make_uint2(src, i); return -1; }
    return ars_exact_c2c(&Pz, pa, pb, thr) ? 1 : 0;
}

// are the mask words >= 1 of an initial model computed by the scoring kernels?  (word0 = its final first mask word)
__device__ __forceinline__ bool ars_ready(uint32_t word0, uint32_t init_n, uint32_t sample, const ArrsacParams &P) {
    if (sample < P.prefix) return true;
    const uint32_t c = min(32u, init_n);
    return (uint32_t)__popc(c < 32 ? (word0 & ((1u << c) - 1)) : word0) >= P.cmin;
}

// phase 0 / 2: the initial models on data [0, init_n) -> masks0[model * W0 + w] (two stages, see ArrsacParams::prefix)
// phase 1: kept candidate rows on [blk_lo, blk_hi) merged into their mask rows; new models on [0, blk_hi) -> newmask rows
//          (nout[j]: certain outliers of new model j in [0, acc_hi) so far; zero on entry, k_ars_book clears it for the next block)
template <int RES>
__global__ void __launch_bounds__(256, 2) k_ars_score(ArrsacCtl *ctl, uint2 *__restrict__ queue, ArrsacParams P, int phase, const double *__restrict__ a,
                                                   const double *__restrict__ b, const cvb_pose *__restrict__ poses0,
                                                   const uint8_t *__restrict__ nposes0, uint32_t *__restrict__ masks0,
                                                   const cvb_pose *__restrict__ tposes, uint32_t *__restrict__ tmasks,
                                                   const cvb_pose *__restrict__ newposes, const uint8_t *__restrict__ nposes_new,
                                                   uint32_t *__restrict__ newmask, uint32_t *nout) {
    const uint32_t pb = blockIdx.y;
    ctl += pb;
    if (ctl->done) return;
    {
        const ArsStrides S = ars_strides(P);
        queue += pb * S.queue; a += pb * S.a; b += pb * S.b; poses0 += pb * S.models0; nposes0 += pb * S.nposes0;
        masks0 += pb * S.models0 * P.W0; tposes += pb * S.rows2; tmasks += pb * S.tmasks; newposes += pb * S.nnew;
        nposes_new += pb * S.nposes_new; newmask += pb * S.newmask; nout += pb * S.nnew;
    }
    const unsigned full = 0xffffffffu;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
    if (phase == 0 || phase == 2) {
        // phase 0: word 0 of every initial model, every word of the first P.prefix samples' models
        // phase 2: words >= 1 of the remaining models whose first 32 data hold >= P.cmin inliers (after k_ars_resolve fixed word 0)
        const uint32_t init_n = ctl->init_n, W = (init_n + 31) >> 5;
        // compact unit spaces (no warp iterates over units of the other stage):
        //   phase 0: [word 0 of every model | words 1.. of the prefix models]      phase 2: words 1.. of the other models
        const uint32_t nmod = P.H0 * P.MM, npre = min(P.prefix, P.H0) * P.MM, W1 = W > 0 ? W - 1 : 0;
        const uint32_t units = phase == 0 ? nmod + npre * W1 : (nmod - npre) * W1;
        uint32_t *qc = phase == 0 ? &ctl->q_count : &ctl->q_count2;
        uint2 *q = phase == 0 ? queue : queue + P.qcap;
        for (uint32_t u = warp; u < units; u += nwarps) {
            uint32_t m, w;
            if (phase == 0) { if (u < nmod) { m = u; w = 0; } else { m = (u - nmod) / W1; w = 1 + (u - nmod) % W1; } }
            else { m = npre + u / W1; w = 1 + u % W1; }
            if ((m % P.MM) >= nposes0[m / P.MM]) continue;
            if (phase == 2 && !ars_ready(masks0[(size_t)m * P.W0], init_n, m / P.MM, P)) continue;
            const uint32_t i = w * 32 + lane;
            bool bit = false;
            if (i < init_n) bit = ars_inlier_queued<RES>(poses0[m], a, b, i, P.thr, qc, q, P.qcap, m) > 0;      // queue: k_ars_resolve
            const unsigned bits = __ballot_sync(full, bit);
            if (lane == 0) { masks0[(size_t)m * P.W0 + w] = bits; atomicAdd(phase == 0 ? &ctl->stat_units0 : &ctl->stat_units2, 1u); }
        }
        return;
    }
    const uint32_t lo = ctl->blk_lo, hi = ctl->blk_hi, Hn = ctl->Hn, cur = ctl->cur;
    const uint32_t worst = ctl->worst;
    const uint32_t wlo = lo >> 5, nwb = hi > lo ? ((hi - 1) >> 5) - wlo + 1 : 0;
    const uint32_t kept_units = Hn * nwb;
    const uint32_t nnew = ctl->n_new * P.MM, nwn = (hi + 31) >> 5;
    const uint32_t units = kept_units + nnew * nwn;
    const cvb_pose *tp = tposes + (size_t)cur * P.rows;
    uint32_t *tm = tmasks + (size_t)cur * P.rows * P.NW;
    // Early rejection of new models.  k_ars_book accepts new model j only when its mask holds more than `worst` inliers in
    // [0, acc_hi); both values were written by the previous k_ars_book, which sets acc_hi = blk_lo (so does k_ars_sprt).  Once
    // bar = acc_hi - worst data of that range are CERTAIN outliers of j (filter result 0, counted in nout[j]; queued predicates are
    // not counted), j has at most `worst` inliers there and will be rejected, so its remaining mask words are written 0 instead of
    // scored.  The result stays exact:
    // k_ars_resolve_block only ORs real inliers into a word, so the popcount k_ars_book takes of j stays <= its true count <= worst
    // and j is rejected by the same test as with every word scored; the mask of a rejected model is never read again.  (bar = 0,
    // worst >= acc_hi: no new model can beat the bar, and k_ars_book leaves such a block without new models.)  New-model units run word-major -- word w of every model, then word w + 1 --
    // so that a model's early words are decided before its later ones start.  Kept rows are scored in full.
    const uint32_t bar = lo > worst ? lo - worst : 0;
    if (blockIdx.x == 0 && threadIdx.x == 0) {           // CVB_ARS_DEBUG counters
        uint32_t valid = 0;
        for (uint32_t s = 0; s < ctl->n_new; s++) valid += min((uint32_t)nposes_new[s], P.MM);
        ctl->stat_units_kept += kept_units; ctl->stat_units_new += valid * nwn;
        if (nnew) { ctl->stat_blk_w0 += worst == 0; ctl->stat_blk_lt32 += bar < 32; }
    }
    uint32_t skipped = 0;                                // units this warp wrote 0 instead of scoring
    // undecided predicates go to queue region 0 (free once the initial stages are resolved) for k_ars_resolve_block:
    // entry source r < P.rows is kept row r, P.rows + j is new model j
    for (uint32_t u = warp; u < units; u += nwarps) {
        // one predicate site for both kinds of unit (two inlined copies of the filter cost registers)
        const bool kept = u < kept_units;
        uint32_t src, w;                                 // src: queue source (kept row r, or P.rows + new model j)
        if (kept) { src = u / nwb; w = wlo + u % nwb; }
        else {
            const uint32_t v = u - kept_units, j = v % nnew;
            if ((j % P.MM) >= nposes_new[j / P.MM]) continue;
            src = P.rows + j; w = v / nnew;
            if (P.early && __ldcg(nout + j) >= bar) {          // the same address in every lane: the branch is warp-uniform
                if (lane == 0) newmask[(size_t)j * P.NW + w] = 0u;
                skipped++;
                continue;
            }
        }
        const uint32_t i = w * 32 + lane;
        const bool act = i < hi && (!kept || i >= lo);
        int f = -1;
        if (act) f = ars_inlier_queued<RES>(kept ? tp[src] : newposes[src - P.rows], a, b, i, P.thr, &ctl->q_blk, queue, P.qcap, src);
        const unsigned bits = __ballot_sync(full, f > 0);
        if (kept) {
            const unsigned range = __ballot_sync(full, act);
            if (lane == 0) { uint32_t *p = tm + (size_t)src * P.NW + w; *p = (*p & ~range) | bits; }
        } else {
            const uint32_t j = src - P.rows;
            const unsigned out = __ballot_sync(full, f == 0 && i < lo);
            if (lane == 0) {
                newmask[(size_t)j * P.NW + w] = bits;
                if (P.early && out) atomicAdd(nout + j, (uint32_t)__popc(out));
            }
        }
    }
    if (lane == 0 && skipped) atomicAdd(&ctl->stat_skip, skipped);
}

// exact evaluation of the queued predicates of the initial scoring; inliers are OR-ed into their mask word
__global__ void __launch_bounds__(256) k_ars_resolve(const ArrsacCtl *ctl, const uint2 *__restrict__ queue, int stage, ArrsacParams P,
                                                     const double *__restrict__ a, const double *__restrict__ b,
                                                     const cvb_pose *__restrict__ poses0, uint32_t *__restrict__ masks0) {
    const uint32_t pb = blockIdx.y;
    ctl += pb;
    if (ctl->done) return;
    {
        const ArsStrides S = ars_strides(P);
        queue += pb * S.queue; a += pb * S.a; b += pb * S.b; poses0 += pb * S.models0; masks0 += pb * S.models0 * P.W0;
    }
    const uint32_t cnt = min(stage == 0 ? ctl->q_count : ctl->q_count2, P.qcap);
    queue += stage == 0 ? 0 : P.qcap;
    for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e < cnt; e += gridDim.x * blockDim.x) {
        const uint2 q = queue[e];
        if (residual_c2c(poses0[q.x], a + 3 * (size_t)q.y, b + 3 * (size_t)q.y) < P.thr)
            atomicOr(&masks0[(size_t)q.x * P.W0 + (q.y >> 5)], 1u << (q.y & 31));
    }
}

// the same for the block loop's scoring (k_ars_score phase 1, in front of k_ars_book): inliers are OR-ed into the mask rows of the
// current candidate table and into newmask
__global__ void __launch_bounds__(64) k_ars_resolve_block(const ArrsacCtl *ctl, const uint2 *__restrict__ queue, ArrsacParams P,
                                                          const double *__restrict__ a, const double *__restrict__ b,
                                                          const cvb_pose *__restrict__ tposes, uint32_t *__restrict__ tmasks,
                                                          const cvb_pose *__restrict__ newposes, uint32_t *__restrict__ newmask) {
    const uint32_t pb = blockIdx.y;
    ctl += pb;
    if (ctl->done) return;
    {
        const ArsStrides S = ars_strides(P);
        queue += pb * S.queue; a += pb * S.a; b += pb * S.b; tposes += pb * S.rows2; tmasks += pb * S.tmasks;
        newposes += pb * S.nnew; newmask += pb * S.newmask;
    }
    const uint32_t cnt = min(ctl->q_blk, P.qcap), cur = ctl->cur;
    for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e < cnt; e += gridDim.x * blockDim.x) {
        const uint2 q = queue[e];
        const bool kept = q.x < P.rows;
        const size_t row = kept ? (size_t)cur * P.rows + q.x : (size_t)(q.x - P.rows);
        if (residual_c2c(kept ? tposes[row] : newposes[row], a + 3 * (size_t)q.y, b + 3 * (size_t)q.y) < P.thr)
            atomicOr(&(kept ? tmasks : newmask)[row * P.NW + (q.y >> 5)], 1u << (q.y & 31));
    }
}

// ---- block-wide helpers (ARS_BOOK_NT threads) ----------------------------------------------------------------------------
// inclusive scan of three u32 values per thread; total of component k in tot[k]
__device__ void ars_scan3(uint32_t &a, uint32_t &b, uint32_t &c, uint32_t *sm /* 3 * 32 */, uint32_t *tot /* 3 */) {
    const unsigned full = 0xffffffffu;
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t x = __shfl_up_sync(full, a, o), y = __shfl_up_sync(full, b, o), z = __shfl_up_sync(full, c, o);
        if ((int)lane >= o) { a += x; b += y; c += z; }
    }
    __syncthreads();     // protects sm / tot against the previous call's readers
    if (lane == 31) { sm[wid] = a; sm[32 + wid] = b; sm[64 + wid] = c; }
    __syncthreads();
    if (wid == 0) {
        uint32_t x = sm[lane], y = sm[32 + lane], z = sm[64 + lane];
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t p = __shfl_up_sync(full, x, o), q = __shfl_up_sync(full, y, o), r = __shfl_up_sync(full, z, o);
            if ((int)lane >= o) { x += p; y += q; z += r; }
        }
        sm[lane] = x; sm[32 + lane] = y; sm[64 + lane] = z;
        if (lane == 31) { tot[0] = x; tot[1] = y; tot[2] = z; }
    }
    __syncthreads();
    if (wid > 0) { a += sm[wid - 1]; b += sm[32 + wid - 1]; c += sm[64 + wid - 1]; }
}

__device__ uint32_t ars_block_min(uint32_t v, uint32_t *sm /* 32 */) {
    const unsigned full = 0xffffffffu;
    for (int o = 16; o; o >>= 1) v = min(v, __shfl_xor_sync(full, v, o));
    __syncthreads();
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
    __syncthreads();
    uint32_t r = sm[threadIdx.x & 31];
    for (int o = 16; o; o >>= 1) r = min(r, __shfl_xor_sync(full, r, o));
    return r;
}
__device__ uint32_t ars_block_max(uint32_t v, uint32_t *sm) { return ~ars_block_min(~v, sm); }

// ascending bitonic sort of the first P2 (power of two) u64 keys in shared memory.  Element i belongs to thread i mod blockDim.x, so
// the partners of a stage with distance j < 32 live in the same warp: such a stage needs a block barrier only when the stage in
// front of it crossed warps (of the 66 stages of 2 048 keys, 21 cross warps).
__device__ void ars_bitonic(uint64_t *keys, uint32_t P2) {
    bool prev_wide = true;
    for (uint32_t k = 2; k <= P2; k <<= 1)
        for (uint32_t j = k >> 1; j > 0; j >>= 1) {
            const bool wide = j >= 32;
            if (wide || prev_wide) __syncthreads(); else __syncwarp();
            prev_wide = wide;
            for (uint32_t i = threadIdx.x; i < P2; i += blockDim.x) {
                const uint32_t l = i ^ j;
                if (l > i) {
                    const uint64_t x = keys[i], y = keys[l];
                    const bool up = (i & k) == 0;
                    if ((x > y) == up) { keys[i] = y; keys[l] = x; }
                }
            }
        }
    __syncthreads();
}
// stable "descending by inliers" order as ascending u64 keys: (inliers desc, previous position asc); payload = source id
__device__ __forceinline__ uint64_t ars_key(uint32_t inl, uint32_t pos, uint32_t src) {
    return ((uint64_t)(0xfffffu - inl) << 32) | ((uint64_t)pos << 16) | (uint64_t)src;
}
__device__ __forceinline__ uint32_t ars_pow2(uint32_t n) { uint32_t p = 2; while (p < n) p <<= 1; return p; }

// number of set bits of a mask row in data [lo, hi)
__device__ uint32_t ars_popc_range(const uint32_t *row, uint32_t lo, uint32_t hi) {
    if (hi <= lo) return 0;
    uint32_t c = 0;
    for (uint32_t w = lo >> 5; w <= (hi - 1) >> 5; w++) {
        uint32_t x = row[w];
        const uint32_t b0 = w * 32;
        if (b0 < lo) x &= ~0u << (lo - b0);
        if (b0 + 32 > hi) x &= ~0u >> (b0 + 32 - hi);
        c += __popc(x);
    }
    return c;
}

// SPRT walk of one model over its initialisation mask (the reference's inner loop, f32 in data order): ONE pass that carries the exact
// likelihood ratio for delta = dl and, beside it, both corners of ARS_NBOX nested boxes of delta values dl (1 -+ width) (two boxes,
// widths 1/4 and 1/128: the 1024-thread CTA has 64 registers per thread, and four boxes = 9 chains + 18 multipliers spilled).
//   * f32 multiplication and division are monotone, so for every delta inside a box the ratio lies between the box's lower and upper
//     corner at every datum (upper corner: delta_hi / eps on inliers, (1 - delta_lo) / (1 - eps) on outliers; lower corner the other way).
//   * the exact walk stops at datum T (ratio > thr) or passes.  A box is VALID for this model when its upper corner does not stop in
//     front of T and its lower corner stops at T as well (or, for a passing model, when the upper corner never stops): the outcome
//     (T, inliers up to T) then holds for every delta in the box.  The widest valid box is returned ([dl, dl] when none is).
// words[w * stride] = mask word w; words at and beyond `avail` have not been computed by the scoring kernels (two-stage initial scoring):
// the walk evaluates such a word itself, stores it (walk copy and global row) and moves `avail` on.  *tested_out = the 1-based datum at
// which the ratio exceeded the threshold, 0 when the model passes; *inl_out = inliers up to there.
struct ArsLazy { const cvb_pose *pose; const double *a, *b; double thr; uint32_t *grow; uint32_t *counter; uint32_t *steps; };
#ifndef ARS_NBOX
#define ARS_NBOX 2
#endif
__device__ __forceinline__ float ars_box_width(int i) {
    constexpr float W0 = 0.25f, WS = ARS_NBOX == 2 ? 0.03125f : (ARS_NBOX == 3 ? 0.125f : 0.25f);   // 1/4, 1/128 | 1/4, 1/32, 1/256 | 1/4 .. 1/256
    float w = W0;
    for (int k = 0; k < i; k++) w *= WS;
    return w;
}
// Out of line on purpose: inlined into the 1024-thread kernel (64 registers per thread, a dozen live pointers) the multipliers and
// ratios were spilled and every step reloaded them from local memory; as a function the walk has the register file to itself.
// Returns (tested << 16 | inliers, index of the widest valid box or ARS_NBOX).
template <int RES>
__device__ __noinline__ uint2 ars_sprt_walk_multi(uint32_t *words, uint32_t stride, uint32_t init_n, float dl, float eps, float one_m_eps, float thr,
                                                  uint32_t avail, const ArsLazy *L) {
    constexpr int NB = ARS_NBOX;
    const float pe = dl / eps, ne = (1.0f - dl) / one_m_eps;
    float ph[NB], nh[NB], pl[NB], nl[NB];
    bool dead[NB];
#pragma unroll
    for (int i = 0; i < NB; i++) {
        const float wdt = ars_box_width(i);
        const float lo = dl * (1.0f - wdt), hi = dl * (1.0f + wdt);
        dead[i] = !(hi < 1.0f);                     // keeps every multiplier positive (the monotonicity argument needs it)
        ph[i] = dead[i] ? pe : hi / eps; nh[i] = dead[i] ? ne : (1.0f - lo) / one_m_eps;
        pl[i] = dead[i] ? pe : lo / eps; nl[i] = dead[i] ? ne : (1.0f - hi) / one_m_eps;
    }
    float re = 1.0f, rh[NB], rl[NB];
#pragma unroll
    for (int i = 0; i < NB; i++) rh[i] = rl[i] = 1.0f;
    uint32_t inl = 0, tested = 0;
    bool stopped = false;
    for (uint32_t w = 0; w * 32 < init_n && !stopped; w++) {
        const uint32_t cnt = min(32u, init_n - w * 32);
        if (w >= avail) {
            uint32_t bits = 0;
            for (uint32_t k = 0; k < cnt; k++)
                if (ars_inlier<RES>(*L->pose, L->a, L->b, w * 32 + k, L->thr)) bits |= 1u << k;
            words[w * stride] = bits;
            L->grow[w] = bits;
            avail = w + 1;
            atomicAdd(L->counter, 1u);
        }
        const uint32_t x = words[w * stride];
        // 0 * finite stays 0: once every chain has underflowed nothing can stop any more
        bool all0 = re == 0.0f;
#pragma unroll
        for (int i = 0; i < NB; i++) all0 = all0 && rh[i] == 0.0f;
        if (all0) {
            inl += __popc(cnt < 32 ? (x & ((1u << cnt) - 1)) : x);
            continue;
        }
        uint32_t k = 0;
        // four data per turn: the products are the sequential ones (same order), only the threshold tests are gathered
        for (; k + 4 <= cnt && !stopped; k += 4) {
            const uint32_t q = (x >> k) & 15u;
            const bool b0 = q & 1u, b1 = q & 2u, b2 = q & 4u, b3 = q & 8u;
            const float e1 = re * (b0 ? pe : ne), e2 = e1 * (b1 ? pe : ne), e3 = e2 * (b2 ? pe : ne), e4 = e3 * (b3 ? pe : ne);
            float h1[NB], h2[NB], h3[NB], h4[NB], l1[NB], l2[NB], l3[NB], l4[NB];
#pragma unroll
            for (int i = 0; i < NB; i++) {
                h1[i] = rh[i] * (b0 ? ph[i] : nh[i]); h2[i] = h1[i] * (b1 ? ph[i] : nh[i]);
                h3[i] = h2[i] * (b2 ? ph[i] : nh[i]); h4[i] = h3[i] * (b3 ? ph[i] : nh[i]);
                l1[i] = rl[i] * (b0 ? pl[i] : nl[i]); l2[i] = l1[i] * (b1 ? pl[i] : nl[i]);
                l3[i] = l2[i] * (b2 ? pl[i] : nl[i]); l4[i] = l3[i] * (b3 ? pl[i] : nl[i]);
            }
            if (!(fmaxf(fmaxf(e1, e2), fmaxf(e3, e4)) > thr)) {          // the exact walk goes on (no NaN: every factor is finite and positive)
#pragma unroll
                for (int i = 0; i < NB; i++) {
                    dead[i] |= fmaxf(fmaxf(h1[i], h2[i]), fmaxf(h3[i], h4[i])) > thr;      // upper corner stops in front of the exact walk
                    rh[i] = h4[i]; rl[i] = l4[i];
                }
                re = e4;
                inl += __popc(q);
                continue;
            }
            const int jstop = e1 > thr ? 1 : (e2 > thr ? 2 : (e3 > thr ? 3 : 4));      // first datum of the turn at which the exact ratio stops
            tested = w * 32 + k + jstop;
            inl += __popc(q & ((1u << jstop) - 1u));
#pragma unroll
            for (int i = 0; i < NB; i++) {
                const bool early = (jstop > 1 && h1[i] > thr) || (jstop > 2 && h2[i] > thr) || (jstop > 3 && h3[i] > thr);
                const float lj = jstop == 1 ? l1[i] : (jstop == 2 ? l2[i] : (jstop == 3 ? l3[i] : l4[i]));
                dead[i] |= early || !(lj > thr);                           // ... or the lower corner does not stop here
            }
            stopped = true;
        }
        for (; k < cnt && !stopped; k++) {                                 // tail of a partial word
            const bool in = (x >> k) & 1u;
            inl += in ? 1u : 0u;
            re *= in ? pe : ne;
#pragma unroll
            for (int i = 0; i < NB; i++) { rh[i] *= in ? ph[i] : nh[i]; rl[i] *= in ? pl[i] : nl[i]; }
            if (re > thr) {
                tested = w * 32 + k + 1; stopped = true;
#pragma unroll
                for (int i = 0; i < NB; i++) dead[i] |= !(rl[i] > thr);
            } else {
#pragma unroll
                for (int i = 0; i < NB; i++) dead[i] |= rh[i] > thr;
            }
        }
    }
    atomicAdd(L->steps, stopped ? tested : init_n);
    uint32_t box = NB;
#pragma unroll
    for (int i = NB - 1; i >= 0; i--)
        if (!dead[i]) box = (uint32_t)i;
    return make_uint2((tested << 16) | inl, box);
}

// both minima of a pair of block-wide values in one pass (ARS_BOOK_NT threads)
__device__ void ars_block_min2(uint32_t &a, uint32_t &b, uint32_t *sm /* 64 */) {
    const unsigned full = 0xffffffffu;
    for (int o = 16; o; o >>= 1) { a = min(a, __shfl_xor_sync(full, a, o)); b = min(b, __shfl_xor_sync(full, b, o)); }
    __syncthreads();
    if ((threadIdx.x & 31) == 0) { sm[threadIdx.x >> 5] = a; sm[32 + (threadIdx.x >> 5)] = b; }
    __syncthreads();
    a = sm[threadIdx.x & 31]; b = sm[32 + (threadIdx.x & 31)];
    for (int o = 16; o; o >>= 1) { a = min(a, __shfl_xor_sync(full, a, o)); b = min(b, __shfl_xor_sync(full, b, o)); }
}

// inclusive block-wide max scan (ARS_BOOK_NT threads)
__device__ uint32_t ars_scan_max(uint32_t v, uint32_t *sm /* 32 */) {
    const unsigned full = 0xffffffffu;
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (int o = 1; o < 32; o <<= 1) { const uint32_t x = __shfl_up_sync(full, v, o); if ((int)lane >= o) v = max(v, x); }
    __syncthreads();
    if (lane == 31) sm[wid] = v;
    __syncthreads();
    if (wid == 0) {
        uint32_t x = sm[lane];
        for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(full, x, o); if ((int)lane >= o) x = max(x, y); }
        sm[lane] = x;
    }
    __syncthreads();
    if (wid > 0) v = max(v, sm[wid - 1]);
    return v;
}

// ---- k_ars_sprt ----------------------------------------------------------------------------------------------------------
template <int RES>
__global__ void __launch_bounds__(ARS_BOOK_NT) k_ars_sprt(ArrsacCtl *ctl, ArrsacParams P, const double *__restrict__ a, const double *__restrict__ b,
                                                           const cvb_pose *__restrict__ poses0,
                                                           const uint8_t *__restrict__ nposes0, uint32_t *__restrict__ masks0,
                                                           uint32_t *__restrict__ vm, uint32_t *__restrict__ pass_id,
                                                           uint32_t *__restrict__ pass_inl, cvb_pose *tposes, uint32_t *tinl,
                                                           uint32_t *tmasks) {
    const uint32_t pb = blockIdx.x;
    ctl += pb;
    if (ctl->done) return;
    {
        const ArsStrides S = ars_strides(P);
        a += pb * S.a; b += pb * S.b; poses0 += pb * S.models0; nposes0 += pb * S.nposes0; masks0 += pb * S.models0 * P.W0;
        vm += pb * S.vm; pass_id += pb * S.models0; pass_inl += pb * S.models0; tposes += pb * S.rows2; tinl += pb * S.rows2;
        tmasks += pb * S.tmasks;
    }
    __shared__ uint32_t sm[96], tot[3];
    extern __shared__ __align__(16) unsigned char ars_dyn[];     // 8 * ARS_SORT_CAP bytes
    uint64_t *keys = (uint64_t *)ars_dyn;                        // [ARS_SORT_CAP]
    __shared__ float s_eps, s_delta;
    __shared__ uint32_t s_best, s_cursor, s_npass, s_stop, s_chunks;
    __shared__ unsigned long long s_rej_inl, s_rej_tested;
    const uint32_t tid = threadIdx.x, NT = blockDim.x;
    const uint32_t init_n = ctl->init_n;
    // A. models in reference order (sample-major, solution-minor), skipping the slots an estimator left empty
    uint32_t base = 0;
    for (uint32_t h0 = 0; h0 < P.H0; h0 += NT) {
        const uint32_t h = h0 + tid;
        const uint32_t cnt = h < P.H0 ? nposes0[h] : 0;
        uint32_t x = cnt, y = 0, z = 0;
        ars_scan3(x, y, z, sm, tot);
        const uint32_t off = base + x - cnt;
        for (uint32_t k = 0; k < cnt; k++) vm[off + k] = h * P.MM + k;
        base += tot[0];
        __syncthreads();
    }
    const uint32_t Mv = base;
    if (tid == 0) {
        ctl->Mv = Mv;
        s_eps = P.eps0; s_delta = P.delta0; s_best = 0; s_cursor = 0; s_npass = 0; s_rej_inl = 0; s_rej_tested = 0; s_chunks = 0;
    }
    __syncthreads();
    // B. adaptive SPRT.  A chunk of up to NT models is walked concurrently under the state (epsilon, delta) in front of the chunk; the
    // one-pass walk returns every model's outcome together with the widest BOX of delta values for which that outcome is certain
    // (ars_sprt_walk_multi; epsilon is fixed inside a chunk).  Block-wide prefix sums over the outcomes give the delta in front of every
    // position.  Positions whose delta lies outside their box are walked again -- all of them at once, each with the delta its current
    // predecessors give it -- and the sums are redone: the first such position is final after one turn (everything in front of it is),
    // a later one unless a repaired predecessor changed its outcome, in which case its delta leaves its new box and it comes back.
    // When no position in front of the first epsilon-raising model violates its box, everything up to and including that model is
    // committed by the positions' own threads, and the next chunk starts behind it.
    //  * for the walk, models are assigned to threads with the long walks (models the scoring kernels gave all their mask words)
    //    first, so that a warp of quickly rejected models costs a few instructions instead of waiting for one long walk among its lanes.
    uint32_t *smw = (uint32_t *)keys;                    // [8][NT] mask words by chunk position (keys[] is free until phase C)
    __shared__ float o_lo[ARS_BOOK_NT], o_hi[ARS_BOOK_NT], o_d[ARS_BOOK_NT];
    __shared__ uint32_t o_ti[ARS_BOOK_NT];               // outcome by position: tested << 16 | inliers at the stop (init_n < 8192)
    __shared__ uint16_t perm[ARS_BOOK_NT];
    //  * the chunk doubles (64 .. NT) while it is committed whole and restarts small behind an epsilon change: models walked under a
    //    stale (smaller) epsilon survive longer than they will, and those the two-stage scoring gave one mask word would evaluate the
    //    missing words themselves, one predicate after the other.
    __shared__ uint32_t s_chunk;
    __shared__ unsigned long long s_t_walk, s_t_commit, s_t_perm;
    __shared__ uint32_t s_turns;
    const bool words_in_smem = P.W0 <= 8;
    if (tid == 0) { s_chunk = 64; s_t_walk = 0; s_t_commit = 0; s_t_perm = 0; s_turns = 0; }
    __syncthreads();
    while (true) {
        const uint32_t c0 = s_cursor;
        if (c0 >= Mv) break;
        const float eps = s_eps, delta = s_delta;
        const uint32_t best0 = s_best, np0 = s_npass;
        const unsigned long long ri0 = s_rej_inl, rt0 = s_rej_tested;
        const uint32_t j = tid, cnt = min(s_chunk, Mv - c0);
        unsigned long long t_a = 0;
        if (tid == 0) t_a = ars_globaltimer();
        const float one_m_eps = 1.0f - eps;
        // 1. positions with all mask words first
        {
            bool rdy = false;
            if (j < cnt) { const uint32_t idj = vm[c0 + j]; rdy = ars_ready(masks0[(size_t)idj * P.W0], init_n, idj / P.MM, P); }
            uint32_t x = (j < cnt && rdy) ? 1 : 0, y = (j < cnt && !rdy) ? 1 : 0, z = 0;
            ars_scan3(x, y, z, sm, tot);
            if (j < cnt) perm[rdy ? x - 1 : tot[0] + y - 1] = (uint16_t)j;
            __syncthreads();
        }
        if (tid == 0) { const unsigned long long t_b = ars_globaltimer(); s_t_perm += t_b - t_a; t_a = t_b; }
        // 2. thread t walks position perm[t]
        auto walk_position = [&](uint32_t pos, float dl) {
            const uint32_t id = vm[c0 + pos];
            uint32_t *grow = masks0 + (size_t)id * P.W0, *row = grow;
            uint32_t stride = 1;
            uint32_t avail = ars_ready(grow[0], init_n, id / P.MM, P) ? P.W0 : 1u;     // words the scoring kernels computed
            if (words_in_smem) {
                const uint32_t wn = min(avail, (init_n + 31) >> 5);       // words behind the data count were never written (nor are they walked)
                for (uint32_t w = 0; w < wn; w++) smw[w * NT + pos] = grow[w];
                row = smw + pos; stride = NT;
            }
            const ArsLazy LZ = {poses0 + id, a, b, P.thr, grow, &ctl->stat_lazy, &ctl->stat_pad};
            const uint2 res = ars_sprt_walk_multi<RES>(row, stride, init_n, dl, eps, one_m_eps, P.lr_thr, avail, &LZ);
            float blo = dl, bhi = dl;
            if (res.y < ARS_NBOX) { const float wdt = ars_box_width((int)res.y); blo = dl * (1.0f - wdt); bhi = dl * (1.0f + wdt); }
            o_ti[pos] = res.x;
            o_lo[pos] = blo; o_hi[pos] = bhi;
        };
        if (tid < cnt) walk_position(perm[tid], delta);
        __syncthreads();
        if (tid == 0) { const unsigned long long t_b = ars_globaltimer(); s_t_walk += t_b - t_a; t_a = t_b; }
        // 3. commit: thread j owns position j
        const bool hv = j < cnt;
        while (true) {
            const uint32_t oti = hv ? o_ti[j] : 0u;
            const uint32_t tested = oti >> 16, inl = oti & 0xffffu;
            const bool pass = hv && tested == 0, rej = hv && tested != 0;
            uint32_t a_ri = rej ? inl : 0, a_rt = rej ? tested : 0, a_pc = pass ? 1 : 0;
            if (tid == 0) s_turns++;
            ars_scan3(a_ri, a_rt, a_pc, sm, tot);                             // inclusive: rejected inliers / tested data / passes
            float dj = 0.0f;                                                   // delta estimate right behind this position (valid ones only)
            if (rej) {
                const float d = (float)(ri0 + a_ri) / (float)(rt0 + a_rt);
                if (d > 0.0f && d < eps) dj = d;
            }
            o_d[j] = dj;
            __syncthreads();
            // 1-based position of the last valid estimate in front of position j
            const uint32_t lv_exc = ars_scan_max((j > 0 && j <= cnt && o_d[j - 1] != 0.0f) ? j : 0u, sm);
            const float db = lv_exc ? o_d[lv_exc - 1] : delta;                 // delta in front of this position
            const bool viol = hv && !(db >= o_lo[j] && db <= o_hi[j]);
            const bool e2 = pass && inl > best0;
            uint32_t fv = viol ? j : (uint32_t)NT, fe = e2 ? j : (uint32_t)NT;
            ars_block_min2(fv, fe, sm);
            if (fv < NT && fv <= fe) {                                         // walked under a state that is not their own
                if (viol && j <= fe) { walk_position(j, db); atomicAdd(&ctl->stat_repairs, 1u); }
                __syncthreads();
                continue;
            }
            const uint32_t last = min(fe, cnt - 1);
            if (pass && j <= last) { const uint32_t p = np0 + a_pc - 1; pass_id[p] = vm[c0 + j]; pass_inl[p] = inl; }
            if (j == last) {                                                   // publish the state behind position `last`
                s_rej_inl = ri0 + a_ri; s_rej_tested = rt0 + a_rt;
                s_npass = np0 + a_pc;
                s_cursor = c0 + last + 1;
                s_chunks++;
                s_delta = dj != 0.0f ? dj : db;
                s_chunk = fe < NT ? 64u : min((uint32_t)NT, 2u * cnt);
                if (fe < NT) {
                    s_best = inl;
                    const float e = (float)inl / (float)init_n;
                    if (e > eps && e < 1.0f) s_eps = e; else if (e >= 1.0f) s_eps = 0.999f;
                }
            }
            break;
        }
        __syncthreads();
        if (tid == 0) s_t_commit += ars_globaltimer() - t_a;
    }
    __syncthreads();
    if (tid == 0) { ctl->stat_walk_us = (uint32_t)(s_t_walk / 1000); ctl->stat_commit_us = (uint32_t)(s_t_commit / 1000);
                    ctl->stat_perm_us = (uint32_t)(s_t_perm / 1000); ctl->stat_turns = s_turns; }
    // C. stable top-max_cand by inliers: threshold from a histogram, ordered compaction, bitonic on (inliers desc, order asc)
    const uint32_t npass = s_npass;
    uint32_t *hist = (uint32_t *)keys;      // init_n + 1 <= 32 * W0 + 1 bins (host guarantees <= 2 * ARS_SORT_CAP)
    for (uint32_t i = tid; i <= init_n; i += NT) hist[i] = 0;
    __syncthreads();
    for (uint32_t i = tid; i < npass; i += NT) atomicAdd(&hist[pass_inl[i]], 1u);
    __syncthreads();
    if (tid == 0) {
        uint32_t T = 0, need = 0;
        if (npass > P.max_cand) {
            uint32_t cum = 0;
            for (int v = (int)init_n; v >= 0; v--) {
                if (cum + hist[v] >= P.max_cand) { T = (uint32_t)v; need = P.max_cand - cum; break; }
                cum += hist[v];
            }
        }
        s_stop = T; s_best = need;        // reuse: threshold value, how many of the entries equal to it are taken
        ctl->npass = npass; ctl->stat_chunks = s_chunks;
    }
    __syncthreads();
    const uint32_t T = s_stop, need = s_best;
    const bool all = npass <= P.max_cand;
    __syncthreads();
    uint32_t ngt = 0, neq = 0;
    for (uint32_t i0 = 0; i0 < npass; i0 += NT) {
        const uint32_t i = i0 + tid;
        const uint32_t v = i < npass ? pass_inl[i] : 0;
        const bool gt = i < npass && (all || v > T), eq = i < npass && !all && v == T;
        uint32_t x = gt ? 1 : 0, y = eq ? 1 : 0, z = 0;
        ars_scan3(x, y, z, sm, tot);
        // position among the selected = (greater-than entries before) + min(equal entries before, need)
        const uint32_t eq_before = neq + y - (eq ? 1 : 0);
        const bool take = gt || (eq && eq_before < need);
        if (take) {
            const uint32_t p = ngt + (x - (gt ? 1 : 0)) + min(eq_before, need);
            keys[p] = ars_key(v, p, 0);
            vm[p] = pass_id[i];                    // vm is free again: model id by selection position
        }
        ngt += tot[0];
        neq += tot[1];
        __syncthreads();
    }
    const uint32_t nsel = ngt + min(neq, need);
    // NOTE: selection positions are already in pass order, i.e. keys carry (inliers, position); sort them
    const uint32_t Hn = nsel;
    const uint32_t P2 = ars_pow2(max(Hn, 2u));
    for (uint32_t i = Hn + tid; i < P2; i += NT) keys[i] = ~0ull;
    ars_bitonic(keys, P2);
    // D. candidate table 0 in sorted order: pose, inliers, mask (initialisation words, rest zero)
    for (uint32_t r = tid / 32; r < Hn; r += NT / 32) {
        const uint32_t lane = tid & 31;
        const uint64_t kx = keys[r];
        const uint32_t p = (uint32_t)(kx >> 16) & 0xffffu;
        const uint32_t id = vm[p];
        const double *src = (const double *)(poses0 + id);
        double *dst = (double *)(tposes + r);
        if (lane < 12) dst[lane] = src[lane];
        if (lane == 0) tinl[r] = 0xfffffu - (uint32_t)(kx >> 32);
        for (uint32_t w = lane; w < P.NW; w += 32) tmasks[(size_t)r * P.NW + w] = w < P.W0 ? masks0[(size_t)id * P.W0 + w] : 0u;
    }
    __syncthreads();
    if (tid == 0) {
        const uint32_t n = ctl->n;
        ctl->Hn = Hn; ctl->cur = 0; ctl->stat_pass = npass;
        ctl->acc_hi = init_n; ctl->blk_lo = init_n; ctl->blk_hi = min(init_n + P.bs, n);
        ctl->n_new = 0; ctl->worst = 0;
        if (!(init_n < n && Hn > 1)) {
            ctl->done = 1; ctl->found = Hn >= 1 ? 1 : 0;
            if (Hn >= 1) ctl->winner = tposes[0];
        }
    }
}

// ---- k_ars_book ----------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(ARS_BOOK_NT) k_ars_book(ArrsacCtl *ctl, ArrsacParams P, const uint32_t *__restrict__ raw,
                                                           cvb_pose *tposes, uint32_t *tinl, uint32_t *tmasks,
                                                           const cvb_pose *__restrict__ newposes, const uint8_t *__restrict__ nposes_new,
                                                           const uint32_t *__restrict__ newmask, uint32_t *__restrict__ pool,
                                                           uint32_t *__restrict__ samples_new, uint32_t *__restrict__ nout,
                                                           uint32_t *live, unsigned long long loop_cond) {
    // loop_cond: the handle of the graph's WHILE node when the block loop is a device-side loop (0 = unrolled launches);
    // the node re-runs its body while the value is non-zero.  *live counts the problems of the batch still in the loop: the CTA
    // that retires a finished problem decrements it, and the one that takes it to zero -- only that one -- ends the loop.
    const uint32_t pb = blockIdx.x;
    ctl += pb;
    auto retire = [&]() {                                        // thread 0, once per problem
        if (ctl->retired) return;
        ctl->retired = 1;
        if (atomicSub(live, 1u) == 1u && loop_cond) cudaGraphSetConditional(loop_cond, 0);
    };
    if (ctl->done) { if (threadIdx.x == 0) retire(); return; }
    {
        const ArsStrides S = ars_strides(P);
        raw += (size_t)pb * P.nraw; tposes += pb * S.rows2; tinl += pb * S.rows2; tmasks += pb * S.tmasks; newposes += pb * S.nnew;
        nposes_new += pb * S.nposes_new; newmask += pb * S.newmask; pool += (size_t)pb * P.NMAX; samples_new += pb * S.samples_new;
        nout += pb * S.nnew;
    }
    __shared__ __align__(8) uint32_t sm[96];
    __shared__ uint32_t tot[3];
    extern __shared__ __align__(16) unsigned char ars_dyn[];     // ARS_BOOK_SMEM bytes
    uint64_t *keys = (uint64_t *)ars_dyn;                                        // [ARS_SORT_CAP]
    uint32_t *e_inl = (uint32_t *)(ars_dyn + 8 * ARS_SORT_CAP);                  // inliers by entry position (part 1 order)
    uint16_t *e_src = (uint16_t *)(ars_dyn + 12 * ARS_SORT_CAP);                 // source: < rows -> kept row of the current table, else rows + new model
    const uint32_t tid = threadIdx.x, NT = blockDim.x;
    if (tid == 0) { ctl->stat_qblk += ctl->q_blk; ctl->q_blk = 0; }      // this block's queue has been resolved
    const uint32_t cur = ctl->cur, Hk = ctl->Hn, n = ctl->n;
    const uint32_t acc_hi = ctl->acc_hi, lo = ctl->blk_lo, hi = ctl->blk_hi, worst = ctl->worst;
    const uint32_t nnew = ctl->n_new * P.MM;
    const cvb_pose *tp = tposes + (size_t)cur * P.rows;
    const uint32_t *ti = tinl + (size_t)cur * P.rows;
    const uint32_t *tm = tmasks + (size_t)cur * P.rows * P.NW;
    // ---- part 1: new hypotheses that beat the bar join the candidates (in generation order), stable sort, truncate
    for (uint32_t r = tid; r < Hk; r += NT) { e_inl[r] = ti[r]; e_src[r] = (uint16_t)r; keys[r] = ars_key(ti[r], r, r); }
    uint32_t total = Hk;
    for (uint32_t j0 = 0; j0 < nnew; j0 += NT) {
        const uint32_t j = j0 + tid;
        uint32_t inl = 0;
        bool acc = false;
        if (j < nnew && (j % P.MM) < nposes_new[j / P.MM]) {
            inl = ars_popc_range(newmask + (size_t)j * P.NW, 0, acc_hi);
            acc = inl > worst;
        }
        uint32_t x = acc ? 1 : 0, y = 0, z = 0;
        ars_scan3(x, y, z, sm, tot);
        if (acc) {
            const uint32_t p = total + x - 1;
            if (p < ARS_SORT_CAP) { e_inl[p] = inl; e_src[p] = (uint16_t)(P.rows + j); keys[p] = ars_key(inl, p, p); }
        }
        total += tot[0];
        __syncthreads();
    }
    uint32_t P2 = ars_pow2(max(total, 2u));
    for (uint32_t i = total + tid; i < P2; i += NT) keys[i] = ~0ull;
    ars_bitonic(keys, P2);
    const uint32_t Hn1 = min(total, P.max_cand);
    // termination test of the reference's loop head (start < n && H.n > 1)
    if (!(lo < n && Hn1 > 1)) {
        if (tid == 0) {
            ctl->done = 1; ctl->found = Hn1 >= 1 ? 1 : 0;
            if (Hn1 >= 1) {
                const uint32_t src = e_src[(uint32_t)keys[0] & 0xffffu];
                ctl->winner = src < P.rows ? tp[src] : newposes[src - P.rows];
            }
            retire();
        }
        return;
    }
    // ---- part 2: add this block's inliers, stable sort, halve
    // entry positions of the survivors of part 1 in their sorted order -> new keys (inliers + block count, rank, entry)
    __syncthreads();
    uint64_t mykeys[ARS_SORT_CAP / ARS_BOOK_NT];
    uint32_t nk = 0;
    for (uint32_t r = tid; r < Hn1; r += NT) {
        const uint32_t e = (uint32_t)keys[r] & 0xffffu;
        const uint32_t src = e_src[e];
        const uint32_t *row = src < P.rows ? tm + (size_t)src * P.NW : newmask + (size_t)(src - P.rows) * P.NW;
        const uint32_t inl = e_inl[e] + ars_popc_range(row, lo, hi);
        e_inl[e] = inl;
        mykeys[nk++] = ars_key(inl, r, e);
    }
    __syncthreads();
    nk = 0;
    for (uint32_t r = tid; r < Hn1; r += NT) keys[r] = mykeys[nk++];
    P2 = ars_pow2(max(Hn1, 2u));
    for (uint32_t i = Hn1 + tid; i < P2; i += NT) keys[i] = ~0ull;
    ars_bitonic(keys, P2);
    const uint32_t keep = max(Hn1 / 2, 1u);
    const uint32_t worst_next = e_inl[(uint32_t)keys[keep - 1] & 0xffffu];      // the bar of this block's new hypotheses (read before keys[] is reused)
    // surviving rows, in order, into the other table
    cvb_pose *np_ = tposes + (size_t)(cur ^ 1) * P.rows;
    uint32_t *ni = tinl + (size_t)(cur ^ 1) * P.rows;
    uint32_t *nm = tmasks + (size_t)(cur ^ 1) * P.rows * P.NW;
    const uint32_t nwords = (hi + 31) >> 5;
    for (uint32_t r = tid / 32; r < keep; r += NT / 32) {
        const uint32_t lane = tid & 31;
        const uint32_t e = (uint32_t)keys[r] & 0xffffu;
        const uint32_t src = e_src[e];
        const double *ps = (const double *)(src < P.rows ? tp + src : newposes + (src - P.rows));
        const uint32_t *row = src < P.rows ? tm + (size_t)src * P.NW : newmask + (size_t)(src - P.rows) * P.NW;
        double *pd = (double *)(np_ + r);
        if (lane < 12) pd[lane] = ps[lane];
        if (lane == 0) ni[r] = e_inl[e];
        for (uint32_t w = lane; w < P.NW; w += 32) nm[(size_t)r * P.NW + w] = w < nwords ? row[w] : 0u;
    }
    __syncthreads();
    // inlier pool of the best candidate over [0, hi)
    uint32_t npool = 0;
    for (uint32_t w0 = 0; w0 < nwords; w0 += NT) {
        const uint32_t w = w0 + tid;
        uint32_t x = 0;
        if (w < nwords) {
            x = nm[w];
            if (w * 32 + 32 > hi) x &= ~0u >> (w * 32 + 32 - hi);
        }
        uint32_t c = __popc(x), y = 0, z = 0;
        const uint32_t mine = c;
        ars_scan3(c, y, z, sm, tot);
        uint32_t p = npool + c - mine;
        while (x) { const int b = __ffs(x) - 1; x &= x - 1; pool[p++] = w * 32 + b; }
        npool += tot[0];
        __syncthreads();
    }
    const bool gen = npool >= P.K && P.G > 0;
    if (gen) ars_sample_block(ctl, raw, npool, P.K, P.G, samples_new, pool, (uint32_t *)keys /* free: the keys were consumed above */, sm + 64);
    for (uint32_t j = tid; j < P.G * P.MM; j += NT) nout[j] = 0;     // the next block's scoring counts its new models' outliers from 0
    __syncthreads();
    if (tid == 0) {
        // A new hypothesis joins the candidates only with more than worst_next inliers in [0, hi).  When worst_next >= hi none can,
        // whatever its pose: its sample is still drawn above (the generator advances exactly as in the reference), but it is neither
        // estimated nor scored.
        const bool bar0 = worst_next >= hi;
        ctl->worst = worst_next;
        ctl->n_new = gen && !bar0 ? P.G : 0;
        ctl->stat_blk_bar0 += gen && bar0;
        ctl->cur = cur ^ 1; ctl->Hn = keep;
        ctl->acc_hi = hi; ctl->blk_lo = hi; ctl->blk_hi = min(hi + P.bs, n);
        ctl->iters++;
    }
}

// ---- k_ars_final ---------------------------------------------------------------------------------------------------------
template <int RES>
__global__ void __launch_bounds__(ARS_BOOK_NT) k_ars_final(ArrsacCtl *ctl, ArrsacParams P, const double *__restrict__ a,
                                                            const double *__restrict__ b, cvb_pose *model_out, uint32_t *inliers_out,
                                                            uint32_t cap, uint32_t *n_inliers_out, int32_t *found_out) {
    __shared__ uint32_t sm[96], tot[3];
    const uint32_t pb = blockIdx.x;
    {
        const ArsStrides S = ars_strides(P);
        ctl += pb; a += pb * S.a; b += pb * S.b;
        if (model_out) model_out += pb;
        if (inliers_out) inliers_out += (size_t)pb * cap;
        if (n_inliers_out) n_inliers_out += pb;
        if (found_out) found_out += pb;
    }
    const uint32_t tid = threadIdx.x, NT = blockDim.x;
    const uint32_t n = ctl->n;
    const bool found = ctl->found != 0;
    uint32_t cnt = 0;
    if (found) {
        const cvb_pose W = ctl->winner;
        if (tid == 0 && model_out) *model_out = W;
        for (uint32_t i0 = 0; i0 < n; i0 += NT) {
            const uint32_t i = i0 + tid;
            const bool in = i < n && ars_inlier<RES>(W, a, b, i, P.thr);
            uint32_t x = in ? 1 : 0, y = 0, z = 0;
            ars_scan3(x, y, z, sm, tot);
            if (in) { const uint32_t p = cnt + x - 1; if (inliers_out && p < cap) inliers_out[p] = i; }
            cnt += tot[0];
            __syncthreads();
        }
    }
    if (tid == 0) {
        ctl->n_inliers = cnt;
        ctl->overflow = (inliers_out && cnt > cap) ? 1u : 0u;
        if (n_inliers_out) *n_inliers_out = cnt;
        if (found_out) *found_out = found ? 1 : 0;
    }
}
