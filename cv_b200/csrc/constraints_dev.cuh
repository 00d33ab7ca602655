// cv_b200/csrc/constraints_dev.cuh -- cv-sfm's three-view constraints on the device (include/cvb200_constraints.h):
// VSlam::generate_view_constraints (cv-sfm/src/lib.rs:2438-2516) for many query views of one reconstruction snapshot, and the acceptance
// of record_view_constraints (lib.rs:2092-2109).  Included by geom.cu after the triangulators, init_dev.cuh (init_block_rank) and the
// three-view optimisers (no -rdc).
//
// Stages, each one launch: per observation its pose and bearings (k_con_gather_obs); per landmark the robust flag (k_con_robust); then per
// chunk of queries, one CTA per query unless said otherwise: the ordered robust list and the kept coviews (k_con_lists), one bitset over
// the robust list per kept coview (k_con_bits), every coview pair's count as a popcount of an AND, one warp per pair (k_con_pairs), the
// stable descending sort and the unique-first order (k_con_order), the two pre-checks of optimize_three_view in that order until the take
// limit (k_con_select), the packed optimisation rows (k_con_offsets, k_con_pack), one optimiser launch over every selected problem
// (k_three_view_opt when the batch fits one CTA per SM, else k_three_view_opt_warp; the two give the same bits), and the rescale and
// outputs (k_con_finish).  Nothing in a query's result depends on the other queries or on the chunking.
#pragma once

constexpr uint32_t CON_NONE = 0xffffffffu;
constexpr unsigned long long CON_NO_KEY = ~0ull;

struct ConParams {
    double inc, bp_min_cos;
    uint32_t V, min_obs, covis_min, opt_min, opt_max, bp_min, max_c, min_new;
};
// one query of a chunk: the host fills q and the bases, k_con_lists R and K, k_con_order T and U, k_con_select the rest
struct ConQuery {
    uint32_t q, out;                     // query view, its position in the call's queries
    uint32_t rbase;                      // robust list (u32) and selection sort buffer (u64, sbase) bases
    uint32_t R, K;                       // robust landmarks, kept coviews
    uint32_t words, bbase;               // bitset words per coview, bitset base
    uint32_t P, n2, kbase, obase, sbase, s2;   // pairs, their sort length and bases, the selection sort length
    uint32_t T, U;                       // triples kept, unique triples
    uint32_t ns, cand, few_lm, few_bp;   // constraints selected, candidates looked at, the two None counts
};

__device__ __forceinline__ void con_pair_views(uint32_t p, uint32_t K, uint32_t &a, uint32_t &b) {   // tuple_combinations order
    uint32_t i = 0, rem = p;
    while (rem >= K - 1 - i) { rem -= K - 1 - i; i++; }
    a = i;
    b = i + 1 + rem;
}
// the feature of landmark l in view v (CSR consistency makes it exist for the views the caller asks about)
__device__ __forceinline__ uint32_t con_feature(const uint32_t *lm_off, const uint32_t *obs, uint32_t l, uint32_t v) {
    for (uint32_t o = lm_off[l]; o < lm_off[l + 1]; o++)
        if (obs[2 * (size_t)o] == v) return obs[2 * (size_t)o + 1];
    return CON_NONE;
}
// A * B of isometries (nalgebra: rotation A.R B.R, translation A.t + A.R B.t)
__device__ __forceinline__ void con_pose_mul(const cvb_pose &A, const cvb_pose &B, cvb_pose *o) {
    for (int i = 0; i < 3; i++)
        for (int c = 0; c < 3; c++) o->r[3 * i + c] = A.r[3 * i] * B.r[c] + A.r[3 * i + 1] * B.r[3 + c] + A.r[3 * i + 2] * B.r[6 + c];
    double sh[3];
    rotv(A.r, B.t, sh);
    for (int i = 0; i < 3; i++) o->t[i] = A.t[i] + sh[i];
}

// the world-frame bearing of an observation: pose^-1's rotation applied to the bearing (lib.rs:2985-2988)
__device__ __forceinline__ void world_bearing(const cvb_pose &P, const double *b, double *o) {
    for (int r = 0; r < 3; r++) o[r] = P.r[r] * b[0] + P.r[3 + r] * b[1] + P.r[6 + r] * b[2];
}
// are_observations_robust (lib.rs:2907-2934) over the n world-frame bearings world[o0 ..): at least min_obs of them, and some pair
// i < j, in tuple_combinations order, with 1 - a.b > inc
__device__ __forceinline__ bool observations_robust(const double *world, uint32_t o0, uint32_t n, uint32_t min_obs, double inc) {
    bool ok = n >= min_obs, incident = false;
    for (uint32_t i = 0; ok && !incident && i < n; i++)
        for (uint32_t j = i + 1; !incident && j < n; j++)
            incident = 1.0 - dot3(world + 3 * (size_t)(o0 + i), world + 3 * (size_t)(o0 + j)) > inc;
    return ok && incident;
}
// per observation: the view's pose, the bearing, and the world-frame bearing
__global__ void __launch_bounds__(256) k_con_gather_obs(const cvb_pose *__restrict__ poses, const uint32_t *__restrict__ view_off,
                                                        const double *__restrict__ bear, const uint32_t *__restrict__ obs, uint32_t n_obs,
                                                        cvb_pose *__restrict__ obs_pose, double *__restrict__ obs_bear,
                                                        double *__restrict__ obs_world) {
    const uint32_t o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= n_obs) return;
    const uint32_t v = obs[2 * (size_t)o], f = obs[2 * (size_t)o + 1];
    const cvb_pose P = poses[v];
    const double *b = bear + 3 * ((size_t)view_off[v] + f);
    obs_pose[o] = P;
    for (int r = 0; r < 3; r++) obs_bear[3 * (size_t)o + r] = b[r];
    world_bearing(P, b, obs_world + 3 * (size_t)o);
}
// triangulate_landmark_robust (lib.rs:2907-2934, 2975-3000) of the landmark whose n gathered observations start at o0: 0 when its
// observations are not robust, 1 when the triangulator returns None, 2 when it returns the point p
__device__ __forceinline__ int robust_landmark_point(const cvb_triangulator &T, uint32_t o0, uint32_t n, const cvb_pose *obs_pose,
                                                     const double *obs_bear, const double *obs_world, double *W, uint32_t min_obs,
                                                     double inc, double *p) {
    if (!observations_robust(obs_world, o0, n, min_obs, inc)) return 0;
    return triangulate_observations(T, obs_pose + o0, obs_bear + 3 * (size_t)o0, n, W ? W + 6 * (size_t)o0 : nullptr, p) ? 2 : 1;
}
// triangulate_landmark_robust is Some; one thread per landmark
__global__ void __launch_bounds__(128) k_con_robust(cvb_triangulator T, const uint32_t *__restrict__ lm_off, uint32_t L,
                                                    const cvb_pose *__restrict__ obs_pose, const double *__restrict__ obs_bear,
                                                    const double *__restrict__ obs_world, double *__restrict__ W, ConParams prm,
                                                    uint8_t *__restrict__ robust) {
    const uint32_t l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= L) return;
    const uint32_t o0 = lm_off[l], n = lm_off[l + 1] - o0;
    double p[4];
    robust[l] = robust_landmark_point(T, o0, n, obs_pose, obs_bear, obs_world, W, prm.min_obs, prm.inc, p) == 2 ? 1 : 0;
}
// view_covisibilities (lib.rs:2535-2556): the query's robust landmarks in feature order, the landmarks per other view, and the coviews
// kept (lib.rs:2443-2450), ascending; cnt (Qc x V, zeroed) counts, kidx (Qc x V) is the kept position or CON_NONE, kview the kept views
__global__ void __launch_bounds__(256) k_con_lists(const uint32_t *__restrict__ view_off, const uint32_t *__restrict__ view_lm,
                                                   const uint32_t *__restrict__ lm_off, const uint32_t *__restrict__ obs,
                                                   const uint8_t *__restrict__ robust, ConParams prm, ConQuery *__restrict__ qs,
                                                   uint32_t *__restrict__ rlist, uint32_t *__restrict__ cnt, uint32_t *__restrict__ kidx,
                                                   uint32_t *__restrict__ kview) {
    __shared__ uint32_t s_warp[32];
    ConQuery &Q = qs[blockIdx.x];
    const uint32_t q = Q.q, f0 = view_off[q], nf = view_off[q + 1] - f0, V = prm.V;
    uint32_t *rl = rlist + Q.rbase, *c = cnt + (size_t)blockIdx.x * V, *ki = kidx + (size_t)blockIdx.x * V,
             *kv = kview + (size_t)blockIdx.x * V;
    uint32_t base = 0;
    for (uint32_t i0 = 0; i0 < nf; i0 += blockDim.x) {
        const uint32_t i = i0 + threadIdx.x;
        const uint32_t l = i < nf ? view_lm[f0 + i] : 0;
        const bool keep = i < nf && robust[l];
        uint32_t tot;
        const uint32_t r = init_block_rank(keep, s_warp, tot);
        if (keep) rl[base + r] = l;
        base += tot;
    }
    const uint32_t R = base;
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < R; i += blockDim.x) {
        const uint32_t l = rl[i];
        for (uint32_t o = lm_off[l]; o < lm_off[l + 1]; o++) {
            const uint32_t v = obs[2 * (size_t)o];
            if (v != q) atomicAdd(&c[v], 1u);
        }
    }
    __syncthreads();
    base = 0;
    for (uint32_t v0 = 0; v0 < V; v0 += blockDim.x) {
        const uint32_t v = v0 + threadIdx.x;
        const bool keep = v < V && c[v] > 0 && c[v] >= prm.covis_min;
        uint32_t tot;
        const uint32_t r = init_block_rank(keep, s_warp, tot);
        if (v < V) ki[v] = keep ? base + r : CON_NONE;
        if (keep) kv[base + r] = v;
        base += tot;
    }
    if (threadIdx.x == 0) { Q.R = R; Q.K = base; }
}
// per kept coview a bitset over the query's robust list: bit i when the coview observes landmark rlist[i] (bits zeroed)
__global__ void __launch_bounds__(256) k_con_bits(const uint32_t *__restrict__ lm_off, const uint32_t *__restrict__ obs, ConParams prm,
                                                  const ConQuery *__restrict__ qs, const uint32_t *__restrict__ rlist,
                                                  const uint32_t *__restrict__ kidx, uint32_t *__restrict__ bits) {
    const ConQuery &Q = qs[blockIdx.x];
    const uint32_t *ki = kidx + (size_t)blockIdx.x * prm.V;
    uint32_t *bt = bits + Q.bbase;
    for (uint32_t i = threadIdx.x; i < Q.R; i += blockDim.x) {
        const uint32_t l = rlist[Q.rbase + i];
        for (uint32_t o = lm_off[l]; o < lm_off[l + 1]; o++) {
            const uint32_t v = obs[2 * (size_t)o];
            if (v == Q.q || ki[v] == CON_NONE) continue;
            atomicOr(&bt[(size_t)ki[v] * Q.words + i / 32], 1u << (i % 32));
        }
    }
}
// lib.rs:2463-2481, one warp per pair of kept coviews: the filtered list's length, and the sort key (descending count, then combination
// order) of a pair that keeps the minimum; the sort buffer's tail and the other pairs get CON_NO_KEY
__global__ void __launch_bounds__(256) k_con_pairs(ConParams prm, const ConQuery *__restrict__ qs, const uint32_t *__restrict__ bits,
                                                   unsigned long long *__restrict__ keys, uint32_t *__restrict__ pcount) {
    const ConQuery &Q = qs[blockIdx.y];
    const uint32_t lane = threadIdx.x & 31, p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (p >= Q.n2) return;
    unsigned long long key = CON_NO_KEY;
    if (p < Q.P) {
        uint32_t a, b;
        con_pair_views(p, Q.K, a, b);
        const uint32_t *ba = bits + Q.bbase + (size_t)a * Q.words, *bb = bits + Q.bbase + (size_t)b * Q.words;
        uint32_t c = 0;
        for (uint32_t w = lane; w < Q.words; w += 32) c += __popc(ba[w] & bb[w]);
        for (int d = 16; d; d >>= 1) c += __shfl_down_sync(0xffffffffu, c, d);
        if (lane == 0) pcount[Q.obase + p] = c;
        if (c >= prm.covis_min) key = ((unsigned long long)(0xffffffffu - c) << 32) | p;
    }
    if (lane == 0) keys[Q.kbase + p] = key;
}
// bitonic sort of n (a power of two) keys, ascending, by one CTA
__device__ void con_bitonic(unsigned long long *buf, uint32_t n) {
    __syncthreads();
    for (uint32_t k = 2; k <= n; k <<= 1)
        for (uint32_t j = k >> 1; j > 0; j >>= 1) {
            for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
                const uint32_t ixj = i ^ j;
                if (ixj > i) {
                    const unsigned long long x = buf[i], y = buf[ixj];
                    if ((x > y) == ((i & k) == 0)) { buf[i] = y; buf[ixj] = x; }
                }
            }
            __syncthreads();
        }
}
// lib.rs:2483-2508: the kept triples sorted (stable: the key holds the combination index), the unique pass -- `any` stops at the first
// view it inserts, and the pass stops at the take limit -- and the evaluation order: unique first, then the rest in sorted order
__global__ void __launch_bounds__(1024) k_con_order(ConParams prm, ConQuery *__restrict__ qs, const uint32_t *__restrict__ kept_views,
                                                    unsigned long long *__restrict__ keys, uint32_t *__restrict__ visited,
                                                    uint32_t *__restrict__ order) {
    ConQuery &Q = qs[blockIdx.x];
    unsigned long long *k = keys + Q.kbase;
    con_bitonic(k, Q.n2);
    if (threadIdx.x != 0) return;
    const uint32_t *kv = kept_views + (size_t)blockIdx.x * prm.V;
    uint32_t *vis = visited + (size_t)blockIdx.x * ((prm.V + 31) / 32), *ord = order + Q.obase;
    uint32_t T = 0;
    while (T < Q.P && k[T] != CON_NO_KEY) T++;
    uint32_t U = 0;
    for (uint32_t t = 0; t < T && U < prm.max_c; t++) {
        uint32_t a, b;
        con_pair_views((uint32_t)k[t], Q.K, a, b);
        uint32_t v[3] = {Q.q, kv[a], kv[b]};
        for (int x = 0; x < 2; x++)
            for (int y = 0; y < 2 - x; y++)
                if (v[y] > v[y + 1]) { const uint32_t s = v[y]; v[y] = v[y + 1]; v[y + 1] = s; }
        for (int x = 0; x < 3; x++) {
            const uint32_t bit = 1u << (v[x] % 32);
            if (!(vis[v[x] / 32] & bit)) {
                vis[v[x] / 32] |= bit;
                ord[U++] = t;
                k[t] |= 1ull << 31;          // marks a unique triple (combination indices stay below 2^31)
                break;
            }
        }
    }
    uint32_t n = U;
    for (uint32_t t = 0; t < T; t++)
        if (!(k[t] & (1ull << 31))) ord[n++] = t;
    Q.T = T;
    Q.U = U;
}
// lib.rs:2509-2515 with optimize_three_view's checks in front of the optimiser (lib.rs:1939-2018), candidate after candidate in the
// evaluation order until max_c succeed: the rows [v0, v1, v2 bearings] of the first opt_max landmarks by descending observation count
// (stable: the key holds the position in the query's robust list), their robust bearing pairs, and the problem's poses and scale
__global__ void __launch_bounds__(256) k_con_select(const cvb_pose *__restrict__ poses, const uint32_t *__restrict__ view_off,
                                                    const double *__restrict__ bear, const uint32_t *__restrict__ lm_off,
                                                    const uint32_t *__restrict__ obs, ConParams prm, ConQuery *__restrict__ qs,
                                                    const uint32_t *__restrict__ rlist, const uint32_t *__restrict__ kept_views,
                                                    const uint32_t *__restrict__ bits, const unsigned long long *__restrict__ keys,
                                                    const uint32_t *__restrict__ pcount, const uint32_t *__restrict__ order,
                                                    unsigned long long *__restrict__ sortbuf, double *__restrict__ rows,
                                                    cvb_pose *__restrict__ prob_poses, uint32_t *__restrict__ prob_n,
                                                    uint32_t *__restrict__ prob_views, double *__restrict__ prob_scale) {
    __shared__ uint32_t s_warp[32];
    __shared__ unsigned long long s_pairs[8];
    ConQuery &Q = qs[blockIdx.x];
    const uint32_t *rl = rlist + Q.rbase, *kv = kept_views + (size_t)blockIdx.x * prm.V;
    unsigned long long *sb = sortbuf + Q.sbase;
    const size_t pb = (size_t)blockIdx.x * prm.max_c;
    uint32_t ns = 0, cand = 0, few_lm = 0, few_bp = 0;
    for (uint32_t t = 0; t < Q.T && ns < prm.max_c; t++) {
        const uint32_t p = (uint32_t)(keys[Q.kbase + order[Q.obase + t]] & 0x7fffffffu), n = pcount[Q.obase + p];
        cand++;
        if (n < prm.opt_min) { few_lm++; continue; }
        uint32_t a, b;
        con_pair_views(p, Q.K, a, b);
        const uint32_t *ba = bits + Q.bbase + (size_t)a * Q.words, *bb = bits + Q.bbase + (size_t)b * Q.words;
        uint32_t n2 = 1;
        while (n2 < n) n2 <<= 1;
        uint32_t base = 0;
        for (uint32_t i0 = 0; i0 < Q.R; i0 += blockDim.x) {
            const uint32_t i = i0 + threadIdx.x;
            const bool keep = i < Q.R && ((ba[i / 32] & bb[i / 32]) >> (i % 32) & 1u);
            uint32_t tot;
            const uint32_t r = init_block_rank(keep, s_warp, tot);
            if (keep) {
                const uint32_t l = rl[i];
                sb[base + r] = ((unsigned long long)(0xffffffffu - (lm_off[l + 1] - lm_off[l])) << 32) | i;
            }
            base += tot;
        }
        for (uint32_t i = n + threadIdx.x; i < n2; i += blockDim.x) sb[i] = CON_NO_KEY;
        con_bitonic(sb, n2);
        uint32_t v[3] = {Q.q, kv[a], kv[b]};
        for (int x = 0; x < 2; x++)
            for (int y = 0; y < 2 - x; y++)
                if (v[y] > v[y + 1]) { const uint32_t s = v[y]; v[y] = v[y + 1]; v[y + 1] = s; }
        const uint32_t m = min(n, prm.opt_max);
        double *rw = rows + (pb + ns) * prm.opt_max * 9;
        for (uint32_t i = threadIdx.x; i < m; i += blockDim.x) {
            const uint32_t l = rl[(uint32_t)sb[i]];
            for (int x = 0; x < 3; x++) {
                const double *src = bear + 3 * ((size_t)view_off[v[x]] + con_feature(lm_off, obs, l, v[x]));
                for (int k = 0; k < 3; k++) rw[9 * (size_t)i + 3 * x + k] = src[k];
            }
        }
        __syncthreads();
        unsigned long long cnt = 0;
        for (uint32_t i = threadIdx.x; i < m; i += blockDim.x) {
            const double *x = rw + 9 * (size_t)i;
            for (uint32_t j = i + 1; j < m; j++) {
                const double *y = rw + 9 * (size_t)j;
                cnt += 1.0 - dot3(x, y) > prm.bp_min_cos && 1.0 - dot3(x + 3, y + 3) > prm.bp_min_cos &&
                       1.0 - dot3(x + 6, y + 6) > prm.bp_min_cos;
            }
        }
        for (int d = 16; d; d >>= 1) cnt += __shfl_down_sync(0xffffffffu, cnt, d);
        if ((threadIdx.x & 31) == 0) s_pairs[threadIdx.x >> 5] = cnt;
        __syncthreads();
        unsigned long long bp = 0;
        for (uint32_t w = 0; w < (blockDim.x >> 5); w++) bp += s_pairs[w];
        __syncthreads();
        if (bp < prm.bp_min) { few_bp++; continue; }
        if (threadIdx.x == 0) {
            cvb_pose inv0, first, second;
            pose_inverse(poses[v[0]], &inv0);
            con_pose_mul(poses[v[1]], inv0, &first);
            con_pose_mul(poses[v[2]], inv0, &second);
            prob_poses[2 * (pb + ns)] = first;
            prob_poses[2 * (pb + ns) + 1] = second;
            prob_scale[pb + ns] = norm3(first.t) + norm3(second.t);
            prob_n[pb + ns] = m;
            for (int x = 0; x < 3; x++) prob_views[3 * (pb + ns) + x] = v[x];
        }
        ns++;
    }
    for (uint32_t k = ns + threadIdx.x; k < prm.max_c; k += blockDim.x) prob_n[pb + k] = 0;
    if (threadIdx.x == 0) { Q.ns = ns; Q.cand = cand; Q.few_lm = few_lm; Q.few_bp = few_bp; }
}
// the packed offsets of the chunk's B = Qc x max_c problems (unused ones are empty); one thread
__global__ void k_con_offsets(uint32_t B, const uint32_t *__restrict__ prob_n, uint32_t *__restrict__ offsets) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    uint32_t off = 0;
    for (uint32_t b = 0; b < B; b++) { offsets[b] = off; off += prob_n[b]; }
    offsets[B] = off;
}
// problem blockIdx.x's rows to its packed place
__global__ void __launch_bounds__(256) k_con_pack(uint32_t opt_max, const uint32_t *__restrict__ prob_n, const uint32_t *__restrict__ offsets,
                                                  const double *__restrict__ rows, double *__restrict__ packed) {
    const uint32_t b = blockIdx.x, n = prob_n[b] * 9;
    const double *src = rows + (size_t)b * opt_max * 9;
    double *dst = packed + 9 * (size_t)offsets[b];
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) dst[i] = src[i];
}
// lib.rs:2039-2061 and 2097-2102: the optimised poses scaled back to the original scale, the constraints, counts and acceptance
__global__ void __launch_bounds__(64) k_con_finish(ConParams prm, const ConQuery *__restrict__ qs, const cvb_pose *__restrict__ opt_out,
                                                   const uint32_t *__restrict__ upd, const uint32_t *__restrict__ prob_n,
                                                   const uint32_t *__restrict__ prob_views, const double *__restrict__ prob_scale,
                                                   cvb_view_constraint *__restrict__ out, cvb_view_constraints_result *__restrict__ res,
                                                   cvb_view_constraints_stats *__restrict__ stats) {
    const ConQuery &Q = qs[blockIdx.x];
    const size_t pb = (size_t)blockIdx.x * prm.max_c;
    for (uint32_t k = threadIdx.x; k < Q.ns; k += blockDim.x) {
        cvb_pose first = opt_out[2 * (pb + k)], second = opt_out[2 * (pb + k) + 1];
        const double rel = prob_scale[pb + k] / (norm3(first.t) + norm3(second.t));
        for (int i = 0; i < 3; i++) { first.t[i] = first.t[i] * rel; second.t[i] = second.t[i] * rel; }
        cvb_view_constraint c;
        for (int x = 0; x < 3; x++) c.views[x] = prob_views[3 * (pb + k) + x];
        c.landmarks = prob_n[pb + k];
        c.poses[0] = first;
        c.poses[1] = second;
        out[(size_t)Q.out * prm.max_c + k] = c;
    }
    if (threadIdx.x != 0) return;
    cvb_view_constraints_result r;
    r.n_constraints = Q.ns;
    r.accepted = !(Q.ns < prm.min_new && Q.ns + 1 < prm.V);
    res[Q.out] = r;
    if (stats) {
        cvb_view_constraints_stats s;
        s.robust_landmarks = Q.R; s.coviews = Q.K; s.triples = Q.T; s.unique_triples = Q.U; s.candidates = Q.cand;
        s.few_landmarks = Q.few_lm; s.few_bearing_pairs = Q.few_bp;
        uint32_t u = 0;
        for (uint32_t k = 0; k < Q.ns; k++) u += upd[pb + k];
        s.updates = u;
        stats[Q.out] = s;
    }
}
