// cv_b200/csrc/init_dev.cuh -- cv-sfm's three-view initialisation on the device (include/cvb200_init.h): the part of
// VSlam::init_reconstruction that chooses the initial triple from the two-view options (cv-sfm/src/lib.rs:986-1303).
// Included by geom.cu after the triangulators, the robustness test and k_three_view_opt, which these kernels call (no -rdc).
//
// The pairs of taking-part options are evaluated speculatively, a wave of W pairs at a time (W = the device's SM count), slot w of a
// wave holding pair base + w.  Every stage is one launch over the wave; a slot that is no longer running returns at once.  After a wave
// k_init_decide records the first decisive slot (accepted, or the bearing-pair None) and the host reads that one word.
#pragma once

constexpr int INIT_RUNNING = -1;                         // a slot still being evaluated (the final outcomes are CVB_INIT_PAIR_*)
constexpr uint32_t INIT_NONE_FEATURE = 0xffffffffu;      // no match of this center feature in the option's map

struct InitFrames { uint32_t center; uint32_t f[CVB_ARRSAC_BATCH_MAX]; };
struct InitCtl {
    uint32_t K, P;                                       // options taking part, pairs of them
    int32_t decided, slot;                               // the decisive pair (-1: none yet) and its slot in the last wave
    uint32_t list[CVB_ARRSAC_BATCH_MAX];                 // option positions that take part, in option order
};
struct InitSlot {
    int32_t outcome;
    uint32_t pair, a, b;                                 // pair index, first / second option position
    uint32_t n_common, cnt_scale, cnt_flag, n_opti, n_use, n_opti0, robust_min, updates, n_robust, n_comb, n_first, n_second;
    double median;
    unsigned long long bpairs;
};
struct InitParams {
    double inc, bp_min_cos, max_cos, max_sine;
    uint32_t min_scales, limit, bp_min, min_robust;
};

// Exclusive rank of `flag` among the CTA's threads in thread order, and the CTA's total (blockDim.x a multiple of 32).
__device__ __forceinline__ uint32_t init_block_rank(bool flag, uint32_t *s_warp, uint32_t &total) {
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const unsigned m = __ballot_sync(0xffffffffu, flag);
    if (lane == 0) s_warp[warp] = __popc(m);
    __syncthreads();
    uint32_t before = 0, tot = 0;
    for (uint32_t k = 0; k < nw; k++) { const uint32_t v = s_warp[k]; if (k < warp) before += v; tot += v; }
    __syncthreads();
    total = tot;
    return before + __popc(m & ((1u << lane) - 1u));
}

__device__ __forceinline__ const double *init_bearing(const double *bear, uint32_t cap, uint32_t frame, uint32_t feature) {
    return bear + ((size_t)frame * cap + feature) * 3;
}
// the (c, f, s) bearings of common triple i of slot w, contiguous as the robustness test takes them
__device__ __forceinline__ void init_triple(const double *bear, uint32_t cap, const InitFrames &fr, const InitSlot &S, const uint32_t *tri3,
                                            double *B) {
    const double *c = init_bearing(bear, cap, fr.center, tri3[0]), *f = init_bearing(bear, cap, fr.f[S.a], tri3[1]),
                 *s = init_bearing(bear, cap, fr.f[S.b], tri3[2]);
    for (int k = 0; k < 3; k++) { B[k] = c[k]; B[3 + k] = f[k]; B[6 + k] = s[k]; }
}

// the options that take part (lib.rs:977-985, 1421) and the number of their pairs; once per call
__global__ void k_init_setup(const uint32_t *__restrict__ n_inl, const int32_t *__restrict__ found, uint32_t F, uint32_t min_matches,
                             InitCtl *__restrict__ ctl) {
    if (threadIdx.x != 0) return;
    uint32_t K = 0;
    for (uint32_t f = 0; f < F; f++)
        if (found[f] != 0 && n_inl[f] >= min_matches) ctl->list[K++] = f;
    ctl->K = K;
    ctl->P = K * (K - (K > 0)) / 2;
    ctl->decided = -1;
    ctl->slot = -1;
}
// per option a center feature -> option feature map of its inlier matches (map preset to INIT_NONE_FEATURE)
__global__ void __launch_bounds__(256) k_init_maps(const uint32_t *__restrict__ pairs, const uint32_t *__restrict__ inliers,
                                                   const uint32_t *__restrict__ n_inl, const int32_t *__restrict__ found, uint32_t cap,
                                                   uint32_t *__restrict__ map) {
    const uint32_t f = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
    if (!found[f] || i >= min(n_inl[f], cap)) return;
    const uint32_t *m = pairs + ((size_t)f * cap + inliers[(size_t)f * cap + i]) * 2;
    map[(size_t)f * cap + m[0]] = m[1];
}
// slot w <- pair base + w in tuple_combinations order, with the options' two-view poses
__global__ void k_init_begin(const InitCtl *__restrict__ ctl, uint32_t base, uint32_t W, const cvb_pose *__restrict__ model,
                             InitSlot *__restrict__ slots, cvb_pose *__restrict__ poses) {
    const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= W) return;
    InitSlot S;
    memset(&S, 0, sizeof(S));
    const uint32_t p = base + w;
    S.pair = p;
    if (p >= ctl->P) { S.outcome = CVB_INIT_PAIR_NOT_EVALUATED; slots[w] = S; return; }
    uint32_t i = 0, rem = p;
    while (rem >= ctl->K - 1 - i) { rem -= ctl->K - 1 - i; i++; }
    S.a = ctl->list[i];
    S.b = ctl->list[i + 1 + rem];
    S.outcome = INIT_RUNNING;
    slots[w] = S;
    poses[2 * w] = model[S.a];
    poses[2 * w + 1] = model[S.b];
}
// common (lib.rs:991-998): the first option's matches, in order, whose center feature the second option also matched
__global__ void __launch_bounds__(256) k_init_common(const uint32_t *__restrict__ pairs, const uint32_t *__restrict__ inliers,
                                                     const uint32_t *__restrict__ n_inl, const uint32_t *__restrict__ map, uint32_t cap,
                                                     InitSlot *__restrict__ slots, uint32_t *__restrict__ common) {
    __shared__ uint32_t s_warp[32];
    InitSlot &S = slots[blockIdx.x];
    if (S.outcome != INIT_RUNNING) return;
    const uint32_t a = S.a, b = S.b, n = min(n_inl[a], cap);
    uint32_t *out = common + (size_t)blockIdx.x * cap * 3, base = 0;
    for (uint32_t i0 = 0; i0 < n; i0 += blockDim.x) {
        const uint32_t i = i0 + threadIdx.x;
        uint32_t c = 0, f = 0, s = INIT_NONE_FEATURE;
        if (i < n) {
            const uint32_t *m = pairs + ((size_t)a * cap + inliers[(size_t)a * cap + i]) * 2;
            c = m[0]; f = m[1]; s = map[(size_t)b * cap + c];
        }
        uint32_t tot;
        const bool keep = s != INIT_NONE_FEATURE;
        const uint32_t r = init_block_rank(keep, s_warp, tot);
        if (keep) { out[3 * (base + r)] = c; out[3 * (base + r) + 1] = f; out[3 * (base + r) + 2] = s; }
        base += tot;
    }
    if (threadIdx.x == 0) S.n_common = base;
}

// per common triple, one thread each:
//   MODE 0 (lib.rs:1002-1038): robust with (1.0, incidence), both relative triangulations give points, |fp|^2 / |sp|^2 is normal
//   MODE 1 (lib.rs:1064-1083, 1140-1159): robust with (max_cos, incidence) -> bit 0
//   MODE 2 (lib.rs:1193-1210, 1248-1268): bit 0 robust with (max_cos, 0.0) (combined), bit 1 robust with (max_cos, incidence)
template <int MODE>
__global__ void __launch_bounds__(128) k_init_flags(cvb_triangulator T, const double *__restrict__ bear, uint32_t cap, InitFrames fr,
                                                    const uint32_t *__restrict__ common, const cvb_pose *__restrict__ poses, InitParams prm,
                                                    double max_cos, InitSlot *__restrict__ slots, uint8_t *__restrict__ flags,
                                                    double *__restrict__ ratio) {
    const uint32_t w = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
    InitSlot &S = slots[w];
    if (S.outcome != INIT_RUNNING || i >= S.n_common) return;
    double B[9];
    init_triple(bear, cap, fr, S, common + ((size_t)w * cap + i) * 3, B);
    const cvb_pose first = poses[2 * w], second = poses[2 * w + 1];
    uint8_t fl = 0;
    if (MODE == 0) {
        double fp[4], sp[4];
        if (tri_landmark_robust(T, first, second, B, 1.0, prm.inc) && triangulate_relative(T, first, B, B + 3, fp) && fp[3] != 0.0 &&
            triangulate_relative(T, second, B, B + 6, sp) && sp[3] != 0.0) {
            const double f3[3] = {fp[0] / fp[3], fp[1] / fp[3], fp[2] / fp[3]}, s3[3] = {sp[0] / sp[3], sp[1] / sp[3], sp[2] / sp[3]};
            const double r = dot3(f3, f3) / dot3(s3, s3);
            if (isfinite(r) && fabs(r) >= DBL_MIN) { fl = 1; ratio[(size_t)w * cap + i] = r; atomicAdd(&S.cnt_scale, 1u); }
        }
    } else if (MODE == 1) {
        fl = tri_landmark_robust(T, first, second, B, max_cos, prm.inc);
        if (fl) atomicAdd(&S.cnt_flag, 1u);
    } else {
        const bool comb = tri_landmark_robust(T, first, second, B, prm.max_cos, 0.0);
        const bool rob = tri_landmark_robust(T, first, second, B, prm.max_cos, prm.inc);
        fl = (comb ? 1 : 0) | (rob ? 2 : 0);
        if (comb) atomicAdd(&S.n_comb, 1u);
        if (rob) atomicAdd(&S.n_robust, 1u);
    }
    flags[(size_t)w * cap + i] = fl;
}
// lib.rs:1212-1246: the first (blockIdx.z = 0) or second (1) option's matches whose center feature the other option did not match and
// that pass is_bi_landmark_robust(pose, c, x, maximum_sine_distance) = epipolar::loss(t, R c, x) < maximum_sine_distance (lib.rs:1306-1317)
__global__ void __launch_bounds__(128) k_init_bi_flags(const double *__restrict__ bear, uint32_t cap, InitFrames fr,
                                                       const uint32_t *__restrict__ pairs, const uint32_t *__restrict__ inliers,
                                                       const uint32_t *__restrict__ n_inl, const uint32_t *__restrict__ map,
                                                       const cvb_pose *__restrict__ poses, InitParams prm, InitSlot *__restrict__ slots,
                                                       uint8_t *__restrict__ flags_first, uint8_t *__restrict__ flags_second) {
    const uint32_t w = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x, z = blockIdx.z;
    InitSlot &S = slots[w];
    if (S.outcome != INIT_RUNNING) return;
    const uint32_t me = z ? S.b : S.a, other = z ? S.a : S.b;
    if (i >= min(n_inl[me], cap)) return;
    const uint32_t *m = pairs + ((size_t)me * cap + inliers[(size_t)me * cap + i]) * 2;
    bool keep = map[(size_t)other * cap + m[0]] == INIT_NONE_FEATURE;
    if (keep) {
        const cvb_pose P = poses[2 * w + z];
        double rc[3];
        rotv(P.r, init_bearing(bear, cap, fr.center, m[0]), rc);
        keep = epipolar_loss(P.t, rc, init_bearing(bear, cap, fr.f[me], m[1])) < prm.max_sine;
    }
    (z ? flags_second : flags_first)[(size_t)w * cap + i] = keep;
    if (keep) atomicAdd(z ? &S.n_second : &S.n_first, 1u);
}
// lib.rs:1039-1059: too few scales rejects the pair; otherwise the median of the kept ratios (a bitonic sort of the slot's sort buffer,
// n2 a power of two >= cap; the value at len / 2 does not depend on the order the ratios were kept in) scales the second translation
__global__ void __launch_bounds__(256) k_init_median(uint32_t cap, uint32_t n2, InitParams prm, const uint8_t *__restrict__ flags,
                                                     const double *__restrict__ ratio, InitSlot *__restrict__ slots, double *__restrict__ sortbuf,
                                                     cvb_pose *__restrict__ poses) {
    __shared__ uint32_t s_warp[32];
    InitSlot &S = slots[blockIdx.x];
    if (S.outcome != INIT_RUNNING) return;
    const uint32_t n = S.cnt_scale;
    if (n < prm.min_scales) {
        if (threadIdx.x == 0) S.outcome = CVB_INIT_PAIR_FEW_SCALES;
        return;
    }
    double *buf = sortbuf + (size_t)blockIdx.x * n2;
    const uint8_t *fl = flags + (size_t)blockIdx.x * cap;
    const double *rt = ratio + (size_t)blockIdx.x * cap;
    uint32_t base = 0;
    for (uint32_t i0 = 0; i0 < S.n_common; i0 += blockDim.x) {
        const uint32_t i = i0 + threadIdx.x;
        const bool keep = i < S.n_common && fl[i];
        uint32_t tot;
        const uint32_t r = init_block_rank(keep, s_warp, tot);
        if (keep) buf[base + r] = rt[i];
        base += tot;
    }
    uint32_t len = 1;
    while (len < n) len <<= 1;
    for (uint32_t i = n + threadIdx.x; i < len; i += blockDim.x) buf[i] = INFINITY;
    __syncthreads();
    for (uint32_t k = 2; k <= len; k <<= 1)
        for (uint32_t j = k >> 1; j > 0; j >>= 1) {
            for (uint32_t i = threadIdx.x; i < len; i += blockDim.x) {
                const uint32_t ixj = i ^ j;
                if (ixj > i) {
                    const double x = buf[i], y = buf[ixj];
                    if ((x > y) == ((i & k) == 0)) { buf[i] = y; buf[ixj] = x; }
                }
            }
            __syncthreads();
        }
    if (threadIdx.x == 0) {
        const double med = sqrt(buf[n / 2]);
        S.median = med;
        cvb_pose &P = poses[2 * blockIdx.x + 1];
        for (int k = 0; k < 3; k++) P.t[k] = P.t[k] * med;    // CameraToCamera::scale: the translation only (cv-core/src/pose.rs:37-41)
    }
}
constexpr uint32_t INIT_SZ_RECOUNT = 1, INIT_SZ_FIRST = 2, INIT_SZ_BEARING = 4, INIT_SZ_CHECK = 8;
// The optimisation set's size and the checks in front of each optimisation; then the packed offsets of the wave's sets (a slot that is
// not running gets an empty set, so k_three_view_opt returns at once for it).  One thread.
//   RECOUNT: n_opti = min(flagged, three_view_optimization_landmarks) (the take-limit of lib.rs:1082, 1158)
//   FIRST:   robust_minimum_matches = n_opti / 2 (lib.rs:1110)
//   BEARING: fewer robust bearing pairs than robust_view_num_robust_bearing_pair: the call's None (lib.rs:1100-1106)
//   CHECK:   fewer than 32 (lib.rs:1118, 1167), or at most robust_minimum_matches (lib.rs:1126, 1175), rejects the pair
__global__ void k_init_sizes(uint32_t W, uint32_t mode, InitParams prm, InitSlot *__restrict__ slots, uint32_t *__restrict__ offsets) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    uint32_t off = 0;
    for (uint32_t w = 0; w < W; w++) {
        InitSlot &S = slots[w];
        offsets[w] = off;
        S.n_use = 0;
        if (S.outcome != INIT_RUNNING) continue;
        if (mode & INIT_SZ_RECOUNT) { S.n_opti = min(S.cnt_flag, prm.limit); S.cnt_flag = 0; }
        if (mode & INIT_SZ_FIRST) { S.n_opti0 = S.n_opti; S.robust_min = S.n_opti / 2; }
        if ((mode & INIT_SZ_BEARING) && S.bpairs < prm.bp_min) { S.outcome = CVB_INIT_PAIR_BEARING_PAIRS; continue; }
        if (mode & INIT_SZ_CHECK) {
            if (S.n_opti < 32) { S.outcome = CVB_INIT_PAIR_FEW_MATCHES; continue; }
            if (S.n_opti <= S.robust_min) { S.outcome = CVB_INIT_PAIR_HALF_MATCHES; continue; }
        }
        S.n_use = S.n_opti;
        off += S.n_opti;
    }
    offsets[W] = off;
}
// the first n_use flagged common triples, in order, as [c, f, s] bearing rows at the slot's packed offset
__global__ void __launch_bounds__(256) k_init_gather(const double *__restrict__ bear, uint32_t cap, InitFrames fr,
                                                     const uint32_t *__restrict__ common, const uint8_t *__restrict__ flags,
                                                     const InitSlot *__restrict__ slots, const uint32_t *__restrict__ offsets,
                                                     double *__restrict__ obs) {
    __shared__ uint32_t s_warp[32];
    const InitSlot &S = slots[blockIdx.x];
    const uint32_t lim = S.n_use, n = S.n_common;
    if (lim == 0) return;
    double *out = obs + 9 * (size_t)offsets[blockIdx.x];
    const uint8_t *fl = flags + (size_t)blockIdx.x * cap;
    const uint32_t *cm = common + (size_t)blockIdx.x * cap * 3;
    uint32_t base = 0;
    for (uint32_t i0 = 0; i0 < n && base < lim; i0 += blockDim.x) {
        const uint32_t i = i0 + threadIdx.x;
        const bool keep = i < n && (fl[i] & 1);
        uint32_t tot;
        const uint32_t r = init_block_rank(keep, s_warp, tot);
        if (keep && base + r < lim) init_triple(bear, cap, fr, S, cm + 3 * (size_t)i, out + 9 * (size_t)(base + r));
        base += tot;
    }
}
// lib.rs:1085-1096: pairs (i < j) of the first optimisation set whose c, f and s bearings all have 1 - a.b above the minimum; thread i
// counts its partners j > i
__global__ void __launch_bounds__(128) k_init_bearing_pairs(const double *__restrict__ obs, const uint32_t *__restrict__ offsets,
                                                            double min_cos, InitSlot *__restrict__ slots) {
    const uint32_t w = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
    InitSlot &S = slots[w];
    const uint32_t L = S.n_use;
    unsigned long long cnt = 0;
    if (i < L) {
        const double *o = obs + 9 * (size_t)offsets[w], *a = o + 9 * (size_t)i;
        for (uint32_t j = i + 1; j < L; j++) {
            const double *b = o + 9 * (size_t)j;
            cnt += 1.0 - dot3(a, b) > min_cos && 1.0 - dot3(a + 3, b + 3) > min_cos && 1.0 - dot3(a + 6, b + 6) > min_cos;
        }
    }
    for (int d = 16; d; d >>= 1) cnt += __shfl_down_sync(0xffffffffu, cnt, d);
    if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(&S.bpairs, cnt);
}
// after k_three_view_opt: the optimised poses become the slot's poses
__global__ void k_init_post_opt(uint32_t W, const cvb_pose *__restrict__ opt_out, const uint32_t *__restrict__ upd, InitSlot *__restrict__ slots,
                                cvb_pose *__restrict__ poses) {
    const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= W || slots[w].n_use == 0) return;
    poses[2 * w] = opt_out[2 * w];
    poses[2 * w + 1] = opt_out[2 * w + 1];
    slots[w].updates += upd[w];
}
// lib.rs:1281-1300: the final robust count decides a pair that is still running
__global__ void k_init_accept(uint32_t W, InitParams prm, InitSlot *__restrict__ slots) {
    const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= W) return;
    InitSlot &S = slots[w];
    if (S.outcome != INIT_RUNNING) return;
    if (S.n_robust <= S.robust_min) S.outcome = CVB_INIT_PAIR_HALF_ROBUST;
    else if (S.n_robust < prm.min_robust) S.outcome = CVB_INIT_PAIR_FEW_ROBUST;
    else S.outcome = CVB_INIT_PAIR_ACCEPTED;
}
// the first decisive slot of the wave, and the statistics of the wave's pairs up to it (the reference never evaluates later pairs)
__global__ void k_init_decide(uint32_t W, const InitSlot *__restrict__ slots, InitCtl *__restrict__ ctl, cvb_init_pair_stats *__restrict__ stats) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    for (uint32_t w = 0; w < W; w++) {
        const InitSlot &S = slots[w];
        if (S.outcome == CVB_INIT_PAIR_NOT_EVALUATED) break;
        if (stats) {
            cvb_init_pair_stats st;
            st.outcome = S.outcome; st.first = S.a; st.second = S.b; st.scales = S.cnt_scale; st.median_scale = S.median;
            st.bearing_pairs = S.bpairs; st.common = S.n_common; st.opti = S.n_opti0; st.updates = S.updates; st.robust = S.n_robust;
            stats[S.pair] = st;
        }
        if (S.outcome == CVB_INIT_PAIR_ACCEPTED || S.outcome == CVB_INIT_PAIR_BEARING_PAIRS) {
            ctl->decided = (int32_t)S.pair;
            ctl->slot = (int32_t)w;
            break;
        }
    }
}
// the result header and, for an accepted pair, its lists in the reference's order (lib.rs:1193-1246)
__global__ void __launch_bounds__(256) k_init_finish(const InitCtl *__restrict__ ctl, const InitSlot *__restrict__ slots, uint32_t cap,
                                                     const uint32_t *__restrict__ pairs, const uint32_t *__restrict__ inliers,
                                                     const uint32_t *__restrict__ n_inl, const uint32_t *__restrict__ common,
                                                     const uint8_t *__restrict__ flags, const uint8_t *__restrict__ flags_first,
                                                     const uint8_t *__restrict__ flags_second, const cvb_pose *__restrict__ poses,
                                                     cvb_init_result *__restrict__ res, uint32_t *__restrict__ combined,
                                                     uint32_t *__restrict__ first_matches, uint32_t *__restrict__ second_matches) {
    __shared__ uint32_t s_warp[32];
    const int32_t w = ctl->slot;
    const InitSlot *S = w >= 0 ? slots + w : nullptr;
    const bool acc = S && S->outcome == CVB_INIT_PAIR_ACCEPTED;
    if (threadIdx.x == 0) {
        cvb_init_result R;
        memset(&R, 0, sizeof(R));
        R.n_pairs = ctl->P;
        if (S) {
            R.status = acc ? CVB_INIT_ACCEPTED : CVB_INIT_NONE_BEARING_PAIRS;
            R.pair = S->pair; R.first = S->a; R.second = S->b;
        }
        if (acc) {
            R.n_combined = S->n_comb; R.n_first_matches = S->n_first; R.n_second_matches = S->n_second;
            R.first_pose = poses[2 * w]; R.second_pose = poses[2 * w + 1];
        }
        *res = R;
    }
    if (!acc) return;
    uint32_t base = 0;
    const uint8_t *fl = flags + (size_t)w * cap;
    const uint32_t *cm = common + (size_t)w * cap * 3;
    for (uint32_t i0 = 0; i0 < S->n_common; i0 += blockDim.x) {
        const uint32_t i = i0 + threadIdx.x;
        const bool keep = i < S->n_common && (fl[i] & 1);
        uint32_t tot;
        const uint32_t r = init_block_rank(keep, s_warp, tot);
        if (keep) for (int k = 0; k < 3; k++) combined[3 * (size_t)(base + r) + k] = cm[3 * (size_t)i + k];
        base += tot;
    }
    for (int z = 0; z < 2; z++) {
        const uint32_t me = z ? S->b : S->a, n = min(n_inl[me], cap);
        const uint8_t *fz = (z ? flags_second : flags_first) + (size_t)w * cap;
        uint32_t *out = z ? second_matches : first_matches;
        base = 0;
        for (uint32_t i0 = 0; i0 < n; i0 += blockDim.x) {
            const uint32_t i = i0 + threadIdx.x;
            const bool keep = i < n && fz[i];
            uint32_t tot;
            const uint32_t r = init_block_rank(keep, s_warp, tot);
            if (keep) {
                const uint32_t *m = pairs + ((size_t)me * cap + inliers[(size_t)me * cap + i]) * 2;
                out[2 * (size_t)(base + r)] = m[0]; out[2 * (size_t)(base + r) + 1] = m[1];
            }
            base += tot;
        }
    }
}
