// cv_b200/csrc/register_dev.cuh -- cv-sfm's frame registration on the device (include/cvb200_register.h): VSlam::register_frame /
// register_frame_subset (cv-sfm/src/lib.rs:1452-1812) for one new frame against one reconstruction snapshot.  Included by geom.cu after
// constraints_dev.cuh (world_bearing, robust_landmark_point, con_bitonic), the triangulators, epipolar_loss and k_single_view_opt (no -rdc).
//
// One subset is a fixed chain of launches with no host round trip: the exact 3-NN of the new range in every matched view
// (cvb_hamming_knn_dev, one launch per view), the candidate merge and decision per feature (k_reg_candidates), the in-order append to the
// accumulated match list (k_reg_append), the claim count and the sort keys (k_reg_claims, k_reg_keys), the stable sort and the scratch
// layout (k_reg_order), the observation gather and the robust point of each match tuple, computed once per call (k_reg_gather), the
// compaction of matches_3d (k_reg_compact), P3P ARRSAC on the device count (cvb_arrsac_p3p_dev), the inlier take (k_reg_take), then
// filter_loop_iterations + 1 rounds of k_single_view_opt, the consistency of every match under the new pose (k_reg_consistent) and a
// compaction, and the final counts and matches (k_reg_final).  Every kernel after a failed decision sees RegCtl.status and does nothing;
// the optimiser's offsets are set to an empty problem.  The host waits once per subset, for the status and the generator commit.
#pragma once

constexpr uint32_t REG_NONE = 0xffffffffu;

struct RegParams {
    double max_sin, max_cos, inc;
    uint32_t better_by, min_obs, min_landmarks, num_matches, iters, min_robust_landmarks;
};
// one entry of original_matches: landmark a, landmark b (REG_NONE for a single landmark), feature
struct RegMatch { uint32_t a, b, f; };

// the device state of one call; the fields after n_orig are per subset (k_reg_begin clears them)
struct RegCtl {
    cvb_pose model;                  // the consensus' model
    cvb_pose pose[2];                // the optimiser's input and output, alternating
    uint32_t n_orig;                 // original_matches accumulated over the call
    int32_t status, found;
    uint32_t iteration, n_kept, n_3d, cons_n, n_inl, n_cur, robust_min, final_robust, final_matches, iters_entered, final_stage;
    uint32_t filter[CVB_REGISTER_STATS_ITERATIONS];
    uint32_t opt_off[2];             // k_single_view_opt's offsets: {0, n} or the empty problem {0, 0}
    uint32_t opt_upd;
};

__global__ void k_reg_begin(RegCtl *ctl) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const uint32_t n = ctl->n_orig;
    memset((char *)&ctl->status, 0, sizeof(RegCtl) - offsetof(RegCtl, status));
    ctl->n_orig = n;
}

// are_landmarks_sharing_view (lib.rs:1435-1449)
__device__ __forceinline__ bool reg_sharing_view(const uint32_t *lm_off, const uint32_t *obs, uint32_t a, uint32_t b) {
    for (uint32_t i = lm_off[a]; i < lm_off[a + 1]; i++)
        for (uint32_t j = lm_off[b]; j < lm_off[b + 1]; j++)
            if (obs[2 * (size_t)i] == obs[2 * (size_t)j]) return true;
    return false;
}
// lib.rs:1468-1541, one thread per feature of the range [r0, r0 + n): the best three landmarks by (best distance, landmark) kept as a
// sorted list while the candidates stream in (a landmark already in the list only lowers its distance; one not in it replaces the last
// entry when its key is smaller -- a landmark that left the list can never re-enter with a smaller key, so the list is exact), then the
// decision; dec[i] = (a, b) with a = REG_NONE for no match.  Fewer than three distinct landmarks: the reference's unwrap panics.
__global__ void __launch_bounds__(128) k_reg_candidates(const uint32_t *__restrict__ knn_idx, const uint32_t *__restrict__ knn_dist, uint32_t n,
                                                        uint32_t H, const uint32_t *__restrict__ vbase, const uint32_t *__restrict__ view_lm,
                                                        const uint32_t *__restrict__ lm_off, const uint32_t *__restrict__ obs,
                                                        uint32_t better_by, uint2 *__restrict__ dec, RegCtl *__restrict__ ctl) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t bl[3], bd[3], cnt = 0;
    for (uint32_t h = 0; h < H; h++)
        for (int k = 0; k < 3; k++) {
            const size_t e = ((size_t)h * n + i) * 3 + k;
            const uint32_t j = knn_idx[e];
            if (j == REG_NONE) continue;
            const uint32_t l = view_lm[vbase[h] + j], d = knn_dist[e];
            int p = -1;
            for (uint32_t s = 0; s < cnt; s++) if (bl[s] == l) p = (int)s;
            if (p >= 0) {
                if (d >= bd[p]) continue;
                bd[p] = d;
            } else if (cnt < 3) {
                p = (int)cnt++;
                bl[p] = l; bd[p] = d;
            } else {
                if (d > bd[2] || (d == bd[2] && l > bl[2])) continue;
                p = 2;
                bl[2] = l; bd[2] = d;
            }
            for (; p > 0 && (bd[p] < bd[p - 1] || (bd[p] == bd[p - 1] && bl[p] < bl[p - 1])); p--) {
                const uint32_t tl = bl[p], td = bd[p];
                bl[p] = bl[p - 1]; bd[p] = bd[p - 1]; bl[p - 1] = tl; bd[p - 1] = td;
            }
        }
    uint2 r = make_uint2(REG_NONE, REG_NONE);
    if (cnt < 3) {
        ctl->status = CVB_REGISTER_PANIC;
    } else if (bd[0] + better_by <= bd[1]) {
        r.x = bl[0];
    } else if (bd[1] + better_by <= bd[2] && !reg_sharing_view(lm_off, obs, bl[0], bl[1])) {
        r.x = bl[0]; r.y = bl[1];
    }
    dec[i] = r;
}
// the range's decisions appended to original_matches in feature order (lib.rs:1533-1540); one CTA
__global__ void __launch_bounds__(1024) k_reg_append(const uint2 *__restrict__ dec, uint32_t n, uint32_t r0, RegMatch *__restrict__ orig,
                                                     RegCtl *__restrict__ ctl) {
    __shared__ uint32_t s_warp[32];
    uint32_t base = ctl->n_orig;
    for (uint32_t i0 = 0; i0 < n; i0 += blockDim.x) {
        const uint32_t i = i0 + threadIdx.x;
        const uint2 d = i < n ? dec[i] : make_uint2(REG_NONE, REG_NONE);
        uint32_t tot;
        const uint32_t r = init_block_rank(d.x != REG_NONE, s_warp, tot);
        if (d.x != REG_NONE) orig[base + r] = RegMatch{d.x, d.y, r0 + i};
        base += tot;
    }
    if (threadIdx.x == 0) ctl->n_orig = base;
}
// landmark_counts (lib.rs:1552-1555): counts (L, zeroed) of every landmark of the whole list
__global__ void __launch_bounds__(256) k_reg_claims(const RegMatch *__restrict__ orig, const RegCtl *__restrict__ ctl, uint32_t *__restrict__ counts) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (ctl->status || i >= ctl->n_orig) return;
    const RegMatch m = orig[i];
    atomicAdd(&counts[m.a], 1u);
    if (m.b != REG_NONE) atomicAdd(&counts[m.b], 1u);
}
// lib.rs:1558-1576: the sort key of every match the claim filter keeps (descending summed observation count, then list position), and
// CON_NO_KEY for the others and the tail up to n2
__global__ void __launch_bounds__(256) k_reg_keys(const RegMatch *__restrict__ orig, const uint32_t *__restrict__ counts,
                                                  const uint32_t *__restrict__ lm_off, const RegCtl *__restrict__ ctl, uint32_t n2,
                                                  unsigned long long *__restrict__ keys) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n2) return;
    unsigned long long key = CON_NO_KEY;
    if (!ctl->status && i < ctl->n_orig) {
        const RegMatch m = orig[i];
        if (counts[m.a] == 1 && (m.b == REG_NONE || counts[m.b] == 1)) {
            uint32_t sum = lm_off[m.a + 1] - lm_off[m.a];
            if (m.b != REG_NONE) sum += lm_off[m.b + 1] - lm_off[m.b];
            key = ((unsigned long long)(0xffffffffu - sum) << 32) | i;
        }
    }
    keys[i] = key;
}
// an exclusive scan of one value per thread over the CTA (total: the sum)
__device__ __forceinline__ uint32_t reg_block_scan(uint32_t v, uint32_t *s_warp, uint32_t &total) {
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    uint32_t x = v;
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= (uint32_t)d) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    uint32_t before = 0, tot = 0;
    for (uint32_t k = 0; k < nw; k++) { const uint32_t w = s_warp[k]; if (k < warp) before += w; tot += w; }
    __syncthreads();
    total = tot;
    return before + x - v;
}
// the stable sort (the key holds the list position), the kept count, and per kept match its list index and the base of its
// observations in the scratch: a's observations, b's, and one slot for the new (pose, bearing); one CTA
__global__ void __launch_bounds__(1024) k_reg_order(unsigned long long *__restrict__ keys, uint32_t n2, const RegMatch *__restrict__ orig,
                                                    const uint32_t *__restrict__ lm_off, RegCtl *__restrict__ ctl, uint32_t *__restrict__ list,
                                                    uint32_t *__restrict__ soff) {
    __shared__ uint32_t s_warp[32], s_kept;
    __shared__ int s_status;
    if (threadIdx.x == 0) { s_status = ctl->status; s_kept = 0; }
    __syncthreads();
    if (s_status) return;
    con_bitonic(keys, n2);
    for (uint32_t i = threadIdx.x; i < n2; i += blockDim.x)
        if (keys[i] != CON_NO_KEY && (i + 1 == n2 || keys[i + 1] == CON_NO_KEY)) s_kept = i + 1;
    __syncthreads();
    const uint32_t K = s_kept;
    uint32_t base = 0;
    for (uint32_t i0 = 0; i0 < K; i0 += blockDim.x) {
        const uint32_t i = i0 + threadIdx.x;
        uint32_t c = 0, li = 0;
        if (i < K) {
            li = (uint32_t)keys[i];
            const RegMatch m = orig[li];
            c = lm_off[m.a + 1] - lm_off[m.a] + 1;
            if (m.b != REG_NONE) c += lm_off[m.b + 1] - lm_off[m.b];
        }
        uint32_t tot;
        const uint32_t r = reg_block_scan(c, s_warp, tot);
        if (i < K) { list[i] = li; soff[i] = base + r; }
        base += tot;
    }
    if (threadIdx.x == 0) ctl->n_kept = K;
}
// per kept match: its observations (pose, bearing, world-frame bearing) gathered at its scratch base, a's first (lib.rs:2958-2970); and,
// the first time the call meets the tuple, its robust point (triangulate_landmark_robust / triangulate_merged_landmark_robust):
// rob = 1 when there is none, 2 when pt holds it
__global__ void __launch_bounds__(128) k_reg_gather(cvb_triangulator T, RegParams prm, const RegCtl *__restrict__ ctl,
                                                    const RegMatch *__restrict__ orig, const uint32_t *__restrict__ list,
                                                    const uint32_t *__restrict__ soff, const cvb_pose *__restrict__ poses,
                                                    const uint32_t *__restrict__ view_off, const double *__restrict__ bear,
                                                    const uint32_t *__restrict__ lm_off, const uint32_t *__restrict__ obs,
                                                    cvb_pose *__restrict__ sp, double *__restrict__ sb, double *__restrict__ sw,
                                                    double *__restrict__ W, double *__restrict__ pt, uint8_t *__restrict__ rob) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (ctl->status || i >= ctl->n_kept) return;
    const uint32_t li = list[i], s = soff[i];
    const RegMatch m = orig[li];
    uint32_t k = 0;
    for (int x = 0; x < 2; x++) {
        const uint32_t l = x ? m.b : m.a;
        if (l == REG_NONE) break;
        for (uint32_t o = lm_off[l]; o < lm_off[l + 1]; o++, k++) {
            const uint32_t v = obs[2 * (size_t)o], f = obs[2 * (size_t)o + 1];
            const cvb_pose P = poses[v];
            const double *b = bear + 3 * ((size_t)view_off[v] + f);
            sp[s + k] = P;
            for (int r = 0; r < 3; r++) sb[3 * (size_t)(s + k) + r] = b[r];
            world_bearing(P, b, sw + 3 * (size_t)(s + k));
        }
    }
    if (rob[li]) return;
    double p[4];
    const int r = robust_landmark_point(T, s, k, sp, sb, sw, W, prm.min_obs, prm.inc, p);
    if (r == 2)
        for (int c = 0; c < 4; c++) pt[4 * (size_t)li + c] = p[c];
    rob[li] = r == 2 ? 2 : 1;
}
// the gate in front of every optimisation (lib.rs:1650, 1701), by thread 0 of a one-CTA kernel once n_cur is known: it == iters is the
// final stage
__device__ __forceinline__ void reg_gate(const RegParams &prm, RegCtl *ctl, uint32_t it) {
    if (ctl->status == 0) {
        const uint32_t n = ctl->n_cur;
        if (it < prm.iters) {
            if (it < CVB_REGISTER_STATS_ITERATIONS) ctl->filter[it] = n;
            ctl->iters_entered = it + 1;
            if (n <= ctl->robust_min) { ctl->status = CVB_REGISTER_FILTER_HALF; ctl->iteration = it; }
        } else {
            ctl->final_stage = n;
            if (n <= ctl->robust_min) ctl->status = CVB_REGISTER_FINAL_HALF;
        }
    }
    ctl->opt_off[0] = 0;
    ctl->opt_off[1] = ctl->status == 0 ? ctl->n_cur : 0;
}
// matches_3d in list order (lib.rs:1583-1611), or after an optimisation the consistent matches with a robust point, capped at
// single_view_optimization_num_matches (lib.rs:1663-1692); rows: the new bearing and the homogeneous world point.  One CTA.
__global__ void __launch_bounds__(1024) k_reg_compact(int loop, uint32_t gate_it, RegParams prm, RegCtl *__restrict__ ctl,
                                                      const RegMatch *__restrict__ orig, const uint32_t *__restrict__ list,
                                                      const uint8_t *__restrict__ rob, const double *__restrict__ pt,
                                                      const uint8_t *__restrict__ cons, const double *__restrict__ new_bear,
                                                      double *__restrict__ rows_b, double *__restrict__ rows_w) {
    __shared__ uint32_t s_warp[32];
    __shared__ int s_status;
    if (threadIdx.x == 0) s_status = ctl->status;
    __syncthreads();
    const uint32_t K = ctl->n_kept, cap = loop ? prm.num_matches : 0xffffffffu;
    uint32_t base = 0;
    if (!s_status)
        for (uint32_t i0 = 0; i0 < K && base < cap; i0 += blockDim.x) {
            const uint32_t i = i0 + threadIdx.x;
            const uint32_t li = i < K ? list[i] : 0;
            const bool keep = i < K && rob[li] == 2 && (!loop || cons[i]);
            uint32_t tot;
            const uint32_t r = init_block_rank(keep, s_warp, tot);
            if (keep && base + r < cap) {
                const uint32_t o = base + r, f = orig[li].f;
                for (int c = 0; c < 3; c++) rows_b[3 * (size_t)o + c] = new_bear[3 * (size_t)f + c];
                for (int c = 0; c < 4; c++) rows_w[4 * (size_t)o + c] = pt[4 * (size_t)li + c];
            }
            base += tot;
        }
    if (threadIdx.x != 0) return;
    const uint32_t n = min(base, cap);
    if (!loop) {
        ctl->n_3d = n;
        if (ctl->status == 0 && n < prm.min_landmarks) ctl->status = CVB_REGISTER_FEW_ROBUST_LANDMARKS;
        ctl->cons_n = ctl->status == 0 ? n : 0;
        return;
    }
    if (ctl->status == 0) ctl->n_cur = n;
    reg_gate(prm, ctl, gate_it);
}
// lib.rs:1619-1641: None, or the inliers' rows in the consensus' order up to the cap, robust_minimum_matches and the starting pose
__global__ void __launch_bounds__(1024) k_reg_take(RegParams prm, RegCtl *__restrict__ ctl, const uint32_t *__restrict__ inl,
                                                   const double *__restrict__ m3d_b, const double *__restrict__ m3d_w,
                                                   double *__restrict__ rows_b, double *__restrict__ rows_w) {
    __shared__ int s_status;
    if (threadIdx.x == 0) {
        if (ctl->status == 0 && !ctl->found) ctl->status = CVB_REGISTER_NO_CONSENSUS;
        s_status = ctl->status;
    }
    __syncthreads();
    const uint32_t n = s_status ? 0 : min(ctl->n_inl, prm.num_matches);
    for (uint32_t k = threadIdx.x; k < n; k += blockDim.x) {
        const uint32_t d = inl[k];
        for (int c = 0; c < 3; c++) rows_b[3 * (size_t)k + c] = m3d_b[3 * (size_t)d + c];
        for (int c = 0; c < 4; c++) rows_w[4 * (size_t)k + c] = m3d_w[4 * (size_t)d + c];
    }
    if (threadIdx.x != 0) return;
    if (!s_status) {
        ctl->n_cur = n;
        ctl->robust_min = n / 2;
        ctl->pose[0] = ctl->model;
    }
    reg_gate(prm, ctl, 0);
}
// is_observation_consistent (lib.rs:2622-2655) of every kept match under pose[slot]: one other observation is is_bi_landmark_robust
// (lib.rs:1306-1318); more are triangulated with the new (pose, bearing) appended in the match's scratch slot
__global__ void __launch_bounds__(128) k_reg_consistent(cvb_triangulator T, RegParams prm, const RegCtl *__restrict__ ctl, uint32_t slot,
                                                        const RegMatch *__restrict__ orig, const uint32_t *__restrict__ list,
                                                        const uint32_t *__restrict__ soff, const uint32_t *__restrict__ lm_off,
                                                        const double *__restrict__ new_bear, cvb_pose *__restrict__ sp,
                                                        double *__restrict__ sb, double *__restrict__ W, uint8_t *__restrict__ cons) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (ctl->status || i >= ctl->n_kept) return;
    const cvb_pose pose = ctl->pose[slot];
    const RegMatch m = orig[list[i]];
    const uint32_t s = soff[i];
    uint32_t k = lm_off[m.a + 1] - lm_off[m.a];
    if (m.b != REG_NONE) k += lm_off[m.b + 1] - lm_off[m.b];
    const double *bearing = new_bear + 3 * (size_t)m.f;
    bool ok;
    if (k == 1) {
        cvb_pose inv, tot;
        double a[3];
        pose_inverse(pose, &inv);
        pose_mul(sp[s], inv, &tot);
        rotv(tot.r, bearing, a);
        ok = epipolar_loss(tot.t, a, sb + 3 * (size_t)s) < prm.max_sin;
    } else {
        sp[s + k] = pose;
        for (int c = 0; c < 3; c++) sb[3 * (size_t)(s + k) + c] = bearing[c];
        double p[4];
        ok = triangulate_observations(T, sp + s, sb + 3 * (size_t)s, k + 1, W ? W + 6 * (size_t)s : nullptr, p);
        for (uint32_t j = 0; ok && j <= k; j++) ok = transformed_cosine_distance(sp[s + j], p, sb + 3 * (size_t)(s + j)) < prm.max_cos;
    }
    cons[i] = ok;
}
// lib.rs:1713-1775 under the final pose: final_num_robust_matches, the consistent matches in list order of original_matches (ascending
// feature), the last two decisions, and the result and statistics of the subset.  One CTA.
__global__ void __launch_bounds__(1024) k_reg_final(RegParams prm, RegCtl *__restrict__ ctl, uint32_t slot, uint32_t subset,
                                                    const RegMatch *__restrict__ orig, const uint32_t *__restrict__ list,
                                                    const uint8_t *__restrict__ rob, const uint8_t *__restrict__ cons, uint8_t *__restrict__ fin,
                                                    cvb_register_match *__restrict__ out, cvb_register_result *__restrict__ res,
                                                    cvb_register_stats *__restrict__ stats) {
    __shared__ uint32_t s_warp[32], s_robust;
    __shared__ int s_status;
    if (threadIdx.x == 0) { s_status = ctl->status; s_robust = 0; }
    __syncthreads();
    uint32_t nm = 0;
    if (!s_status) {
        const uint32_t n = ctl->n_orig, K = ctl->n_kept;
        for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) fin[i] = 0;
        __syncthreads();
        uint32_t robust = 0;
        for (uint32_t i = threadIdx.x; i < K; i += blockDim.x) {
            const uint32_t li = list[i];
            fin[li] = cons[i];
            robust += cons[i] && rob[li] == 2;
        }
        atomicAdd(&s_robust, robust);
        __syncthreads();
        for (uint32_t i0 = 0; i0 < n; i0 += blockDim.x) {
            const uint32_t i = i0 + threadIdx.x;
            const bool keep = i < n && fin[i];
            uint32_t tot;
            const uint32_t r = init_block_rank(keep, s_warp, tot);
            if (keep) {
                const RegMatch m = orig[i];
                out[nm + r] = cvb_register_match{m.f, m.a, m.b};
            }
            nm += tot;
        }
    }
    if (threadIdx.x != 0) return;
    if (ctl->status == 0) {
        ctl->final_robust = s_robust;
        if (s_robust <= ctl->robust_min) {
            ctl->status = CVB_REGISTER_FINAL_ROBUST_HALF;
        } else {
            ctl->final_matches = nm;
            if (nm < prm.min_robust_landmarks) ctl->status = CVB_REGISTER_FEW_MATCHES;
        }
    }
    cvb_register_result r;
    memset(&r, 0, sizeof(r));
    r.status = ctl->status;
    r.iteration = ctl->iteration;
    r.n_inliers = ctl->found ? ctl->n_inl : 0;
    if (r.status == CVB_REGISTER_OK) { r.n_matches = nm; r.pose = ctl->pose[slot]; }
    *res = r;
    if (stats) {   // a panic ends the subset before anything is counted
        cvb_register_stats s;
        memset(&s, 0, sizeof(s));
        s.subsets = subset;
        if (r.status != CVB_REGISTER_PANIC) {
            s.matches = ctl->n_orig; s.claimed = ctl->n_kept; s.matches_3d = ctl->n_3d;
            s.inliers = ctl->found ? ctl->n_inl : 0; s.final_robust = ctl->final_robust; s.final_matches = ctl->final_matches;
            s.iterations = ctl->iters_entered; s.final_stage_matches = ctl->final_stage;
            for (int k = 0; k < CVB_REGISTER_STATS_ITERATIONS; k++) s.filter_matches[k] = ctl->filter[k];
        }
        *stats = s;
    }
}
