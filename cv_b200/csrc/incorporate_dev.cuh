// cv_b200/csrc/incorporate_dev.cuh -- the two CSR edits of cv-sfm's frame incorporation on the device (include/cvb200_incorporate.h):
// add_view with merge_landmarks, and the replay of optimize_reconstruction's remove_view / split_landmark / split_observation edits.
// Included by geom.cu after register_dev.cuh (no -rdc).
//
// Both edits are stable compactions.  Each element (landmark, new feature, view, observation, constraint) writes a pair of counts; one
// exclusive scan of those pairs gives every element its output index and its output offset at once.  The scan is the CTA-count pattern
// of k_exp_scan / k_exp_compact on wider data: per-tile sums (k_inc_tile_sums), one CTA scanning the tile sums (k_inc_scan_tiles), then
// every tile scanned in place from its tile offset (k_inc_scan_apply).  Placement kernels then copy each element to its place.
//
// Every read of an offset array is clamped to the array it indexes (inc_range), and every write is checked against the capacity of its
// output, so that a caller's broken precondition (inconsistent CSRs, out-of-range matches or states) gives wrong output, never an
// out-of-bounds access.
#pragma once

constexpr int INC_NT = 256;
constexpr int INC_ITEMS = 4;
constexpr uint32_t INC_TILE = INC_NT * INC_ITEMS;
#define INC_NONE 0xffffffffu

__device__ __forceinline__ uint2 inc_add(uint2 a, uint2 b) { return make_uint2(a.x + b.x, a.y + b.y); }

// the clamped range [o0, o1) of row i of an offset array over n entries
__device__ __forceinline__ void inc_range(const uint32_t *__restrict__ off, uint32_t i, uint32_t n, uint32_t &o0, uint32_t &o1) {
    o0 = min(off[i], n);
    o1 = min(max(off[i + 1], o0), n);
}

// exclusive scan of one pair per thread over a CTA of INC_NT threads; total gets the CTA's sum
__device__ uint2 inc_block_scan(uint2 v, uint2 &total) {
    __shared__ uint2 s_w[INC_NT / 32];
    const uint32_t lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    uint2 x = v;
    for (int o = 1; o < 32; o <<= 1) {
        const uint2 y = make_uint2(__shfl_up_sync(0xffffffffu, x.x, o), __shfl_up_sync(0xffffffffu, x.y, o));
        if ((int)lane >= o) x = inc_add(x, y);
    }
    if (lane == 31) s_w[w] = x;
    __syncthreads();
    if (w == 0) {
        uint2 s = lane < INC_NT / 32 ? s_w[lane] : make_uint2(0, 0);
        for (int o = 1; o < INC_NT / 32; o <<= 1) {
            const uint2 y = make_uint2(__shfl_up_sync(0xffffffffu, s.x, o), __shfl_up_sync(0xffffffffu, s.y, o));
            if ((int)lane >= o) s = inc_add(s, y);
        }
        if (lane < INC_NT / 32) s_w[lane] = s;
    }
    __syncthreads();
    const uint2 pre = w ? s_w[w - 1] : make_uint2(0, 0);
    total = s_w[INC_NT / 32 - 1];
    __syncthreads();   // s_w may be reused by the caller's next scan
    return make_uint2(x.x - v.x + pre.x, x.y - v.y + pre.y);
}

// the sum of every tile of INC_TILE pairs
__global__ void __launch_bounds__(INC_NT) k_inc_tile_sums(uint32_t n, const uint2 *__restrict__ a, uint2 *__restrict__ tile_sum) {
    const size_t i0 = (size_t)blockIdx.x * INC_TILE + (size_t)threadIdx.x * INC_ITEMS;
    uint2 s = make_uint2(0, 0);
    for (int k = 0; k < INC_ITEMS; k++)
        if (i0 + k < n) s = inc_add(s, a[i0 + k]);
    uint2 tot;
    inc_block_scan(s, tot);
    if (threadIdx.x == 0) tile_sum[blockIdx.x] = tot;
}
// exclusive scan of the nt tile sums in place, the grand total into *total; one CTA
__global__ void __launch_bounds__(INC_NT) k_inc_scan_tiles(uint32_t nt, uint2 *__restrict__ tile_sum, uint2 *__restrict__ total) {
    uint2 carry = make_uint2(0, 0);
    for (uint32_t b = 0; b < nt; b += INC_NT) {
        const uint32_t i = b + threadIdx.x;
        const uint2 v = i < nt ? tile_sum[i] : make_uint2(0, 0);
        uint2 tot;
        const uint2 e = inc_block_scan(v, tot);
        if (i < nt) tile_sum[i] = inc_add(carry, e);
        carry = inc_add(carry, tot);
    }
    if (threadIdx.x == 0) *total = carry;
}
// every tile's pairs replaced by their exclusive prefix sums
__global__ void __launch_bounds__(INC_NT) k_inc_scan_apply(uint32_t n, uint2 *__restrict__ a, const uint2 *__restrict__ tile_off) {
    const size_t i0 = (size_t)blockIdx.x * INC_TILE + (size_t)threadIdx.x * INC_ITEMS;
    uint2 v[INC_ITEMS], s = make_uint2(0, 0);
    for (int k = 0; k < INC_ITEMS; k++) {
        v[k] = i0 + k < n ? a[i0 + k] : make_uint2(0, 0);
        s = inc_add(s, v[k]);
    }
    uint2 tot;
    uint2 p = inc_add(tile_off[blockIdx.x], inc_block_scan(s, tot));
    for (int k = 0; k < INC_ITEMS; k++) {
        if (i0 + k < n) a[i0 + k] = p;
        p = inc_add(p, v[k]);
    }
}

// ---- add_view ---------------------------------------------------------------------------------------------------------------------------
// role[l]: INC_NONE, or (m << 1) | is_b for the match m naming landmark l; featm[f]: the match of new feature f, or INC_NONE.  Both arrays
// are set to INC_NONE before.  *merges counts the matches with two landmarks.
__global__ void k_av_roles(uint32_t M, const cvb_register_match *__restrict__ matches, uint32_t L, uint32_t N, uint32_t *__restrict__ role,
                           uint32_t *__restrict__ featm, uint32_t *__restrict__ merges) {
    const uint32_t m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= M) return;
    const cvb_register_match t = matches[m];
    if (t.feature < N) featm[t.feature] = m;
    if (t.landmark_a < L) role[t.landmark_a] = m << 1;
    if (t.landmark_b != CVB_REGISTER_NONE) {
        if (t.landmark_b < L) role[t.landmark_b] = (m << 1) | 1u;
        atomicAdd(merges, 1u);
    }
}
// per element i < L + N: (present, observation count).  Landmark l: b of a merge (0, 0); a of a match (1, |a| + |b| + 1) or (1, |a| + 1);
// otherwise (1, |l|).  New feature f = i - L: (1, 1) when unmatched, else (0, 0).
__global__ void k_av_counts(uint32_t L, uint32_t N, uint32_t n_obs, const uint32_t *__restrict__ lm_off, const uint32_t *__restrict__ role,
                            const uint32_t *__restrict__ featm, const cvb_register_match *__restrict__ matches, uint2 *__restrict__ cnt) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= L + N) return;
    uint2 c = make_uint2(0, 0);
    if (i < L) {
        const uint32_t r = role[i];
        uint32_t o0, o1;
        inc_range(lm_off, i, n_obs, o0, o1);
        if (r == INC_NONE) {
            c = make_uint2(1, o1 - o0);
        } else if (!(r & 1u)) {
            uint32_t n = o1 - o0 + 1;
            const uint32_t b = matches[r >> 1].landmark_b;
            if (b < L) {
                uint32_t b0, b1;
                inc_range(lm_off, b, n_obs, b0, b1);
                n += b1 - b0;
            }
            c = make_uint2(1, n);
        }
    } else if (featm[i - L] == INC_NONE) {
        c = make_uint2(1, 1);
    }
    cnt[i] = c;
}
// per element i < L + N, after the scan of cnt: its landmark offset and observations (a's, then b's, then (V, feature)), and the landmark
// map of the old landmarks.  cap_l / cap_o: the capacities of lm_off_out (rows before the last) and obs_out (pairs).
__global__ void k_av_place(uint32_t V, uint32_t L, uint32_t N, uint32_t n_obs, const uint32_t *__restrict__ lm_off, const uint32_t *__restrict__ obs,
                           const uint32_t *__restrict__ role, const uint32_t *__restrict__ featm, const cvb_register_match *__restrict__ matches,
                           const uint2 *__restrict__ cnt, uint32_t cap_l, uint32_t cap_o, uint32_t *__restrict__ lm_off_out,
                           uint32_t *__restrict__ obs_out, uint32_t *__restrict__ lmap) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= L + N) return;
    const uint2 c = cnt[i];
    if (i >= L) {
        const uint32_t f = i - L;
        if (featm[f] != INC_NONE) return;
        if (c.x < cap_l) lm_off_out[c.x] = c.y;
        if (c.y < cap_o) { obs_out[2 * (size_t)c.y] = V; obs_out[2 * (size_t)c.y + 1] = f; }
        return;
    }
    const uint32_t r = role[i];
    if (r != INC_NONE && (r & 1u)) {    // b: merged into a
        const uint32_t a = matches[r >> 1].landmark_a;
        lmap[i] = a < L ? cnt[a].x : INC_NONE;
        return;
    }
    lmap[i] = c.x;
    if (c.x < cap_l) lm_off_out[c.x] = c.y;
    uint32_t k = c.y, o0, o1;
    inc_range(lm_off, i, n_obs, o0, o1);
    for (uint32_t o = o0; o < o1; o++, k++)
        if (k < cap_o) { obs_out[2 * (size_t)k] = obs[2 * (size_t)o]; obs_out[2 * (size_t)k + 1] = obs[2 * (size_t)o + 1]; }
    if (r == INC_NONE) return;
    const cvb_register_match t = matches[r >> 1];
    if (t.landmark_b < L) {
        inc_range(lm_off, t.landmark_b, n_obs, o0, o1);
        for (uint32_t o = o0; o < o1; o++, k++)
            if (k < cap_o) { obs_out[2 * (size_t)k] = obs[2 * (size_t)o]; obs_out[2 * (size_t)k + 1] = obs[2 * (size_t)o + 1]; }
    }
    if (k < cap_o) { obs_out[2 * (size_t)k] = V; obs_out[2 * (size_t)k + 1] = t.feature; }
}
// the view CSR's landmarks: every old entry through the landmark map, then the new view's (its match's a, or its own singleton)
__global__ void k_av_features(uint32_t nf, uint32_t L, uint32_t N, const uint32_t *__restrict__ view_lm, const uint32_t *__restrict__ lmap,
                              const uint32_t *__restrict__ featm, const cvb_register_match *__restrict__ matches, const uint2 *__restrict__ cnt,
                              uint32_t *__restrict__ view_lm_out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nf + N) return;
    uint32_t l;
    if (i < nf) {
        l = view_lm[i];
        l = l < L ? lmap[l] : INC_NONE;
    } else {
        const uint32_t f = i - nf, m = featm[f];
        if (m == INC_NONE) {
            l = cnt[L + f].x;
        } else {
            const uint32_t a = matches[m].landmark_a;
            l = a < L ? lmap[a] : INC_NONE;
        }
    }
    view_lm_out[i] = l;
}
// the closing rows and the counts
__global__ void k_av_finish(uint32_t V, uint32_t nf, uint32_t N, const uint2 *__restrict__ total, const uint32_t *__restrict__ merges,
                            uint32_t cap_l, uint32_t *__restrict__ view_off_out, uint32_t *__restrict__ lm_off_out,
                            cvb_incorporate_counts *__restrict__ counts) {
    const uint2 t = *total;
    if (t.x <= cap_l) lm_off_out[t.x] = t.y;
    view_off_out[V + 1] = nf + N;
    cvb_incorporate_counts c;
    c.V = V + 1;
    c.n_features = nf + N;
    c.L = t.x;
    c.n_observations = t.y;
    c.C = 0;
    c.merges = *merges;
    *counts = c;
}

// ---- apply_optimization -----------------------------------------------------------------------------------------------------------------
// per view: (kept, its feature count when kept)
__global__ void k_ap_view_counts(uint32_t V, uint32_t nf, const uint32_t *__restrict__ view_off, const uint8_t *__restrict__ vstate,
                                 uint2 *__restrict__ vcnt) {
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    uint32_t f0, f1;
    inc_range(view_off, v, nf, f0, f1);
    vcnt[v] = vstate[v] == CVB_RECON_VIEW_KEPT ? make_uint2(1, f1 - f0) : make_uint2(0, 0);
}
// per landmark: (has a KEPT observation, KEPT observations)
__global__ void k_ap_landmark_counts(uint32_t L, uint32_t n_obs, const uint32_t *__restrict__ lm_off, const uint8_t *__restrict__ ostate,
                                     uint2 *__restrict__ lcnt) {
    const uint32_t l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= L) return;
    uint32_t o0, o1, k = 0;
    inc_range(lm_off, l, n_obs, o0, o1);
    for (uint32_t o = o0; o < o1; o++) k += ostate[o] == CVB_RECON_OBS_KEPT;
    lcnt[l] = make_uint2(k ? 1u : 0u, k);
}
// per observation: (SPLIT, 0); per constraint: (all three views kept, 0)
__global__ void k_ap_split_counts(uint32_t n_obs, const uint8_t *__restrict__ ostate, uint2 *__restrict__ scnt) {
    const uint32_t o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o < n_obs) scnt[o] = make_uint2(ostate[o] == CVB_RECON_OBS_SPLIT ? 1u : 0u, 0);
}
__global__ void k_ap_constraint_counts(uint32_t C, uint32_t V, const cvb_view_constraint *__restrict__ cons, const uint8_t *__restrict__ vstate,
                                       uint2 *__restrict__ ccnt) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    bool keep = true;
    for (int k = 0; k < 3; k++) {
        const uint32_t v = cons[c].views[k];
        keep = keep && v < V && vstate[v] == CVB_RECON_VIEW_KEPT;
    }
    ccnt[c] = make_uint2(keep ? 1u : 0u, 0);
}
// the new feature index of (v, f) after the scan of vcnt, or INC_NONE for a removed view or a feature out of range
__device__ __forceinline__ uint32_t ap_feature(uint32_t v, uint32_t f, uint32_t V, uint32_t nf, const uint32_t *__restrict__ view_off,
                                               const uint8_t *__restrict__ vstate, const uint2 *__restrict__ vcnt) {
    if (v >= V || vstate[v] != CVB_RECON_VIEW_KEPT) return INC_NONE;
    uint32_t f0, f1;
    inc_range(view_off, v, nf, f0, f1);
    return f < f1 - f0 ? vcnt[v].y + f : INC_NONE;
}
// per view, after the scan: its pose, view offset and map entry
__global__ void k_ap_views(uint32_t V, const cvb_pose *__restrict__ poses, const uint8_t *__restrict__ vstate, const uint2 *__restrict__ vcnt,
                           cvb_pose *__restrict__ poses_out, uint32_t *__restrict__ view_off_out, uint32_t *__restrict__ vmap) {
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    if (vstate[v] != CVB_RECON_VIEW_KEPT) { vmap[v] = INC_NONE; return; }
    const uint2 c = vcnt[v];
    poses_out[c.x] = poses[v];
    view_off_out[c.x] = c.y;
    vmap[v] = c.x;
}
// one warp per kept view: its features' bearings, descriptors (16-byte rows of four uint4) and colours, in order
__global__ void __launch_bounds__(256) k_ap_feature_rows(uint32_t V, uint32_t nf, const uint32_t *__restrict__ view_off,
                                                         const uint8_t *__restrict__ vstate, const uint2 *__restrict__ vcnt,
                                                         const double *__restrict__ bear, const uint4 *__restrict__ desc,
                                                         const uint8_t *__restrict__ colors, double *__restrict__ bear_out,
                                                         uint4 *__restrict__ desc_out, uint8_t *__restrict__ colors_out) {
    const uint32_t v = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (v >= V || vstate[v] != CVB_RECON_VIEW_KEPT) return;
    uint32_t f0, f1;
    inc_range(view_off, v, nf, f0, f1);
    const size_t d0 = vcnt[v].y;
    for (uint32_t j = lane; j < f1 - f0; j += 32) {
        const size_t s = f0 + j, d = d0 + j;
        if (d >= nf) break;
        for (int k = 0; k < 3; k++) bear_out[3 * d + k] = bear[3 * s + k];
        if (desc)
            for (int k = 0; k < 4; k++) desc_out[4 * d + k] = desc[4 * s + k];
        if (colors)
            for (int k = 0; k < 3; k++) colors_out[3 * d + k] = colors[3 * s + k];
    }
}
// per landmark, after the scans: its KEPT observations in order (views renumbered), its features' new landmark, its map entry
__global__ void k_ap_landmarks(uint32_t V, uint32_t nf, uint32_t L, uint32_t n_obs, const uint32_t *__restrict__ view_off,
                               const uint8_t *__restrict__ vstate, const uint2 *__restrict__ vcnt, const uint32_t *__restrict__ lm_off,
                               const uint32_t *__restrict__ obs, const uint8_t *__restrict__ ostate, const uint2 *__restrict__ lcnt,
                               const uint2 *__restrict__ ltotal, uint32_t *__restrict__ lm_off_out, uint32_t *__restrict__ obs_out,
                               uint32_t *__restrict__ view_lm_out, uint32_t *__restrict__ lmap) {
    const uint32_t l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= L) return;
    const uint2 c = lcnt[l];
    const uint32_t next = l + 1 < L ? lcnt[l + 1].x : ltotal->x;
    if (next == c.x) { lmap[l] = INC_NONE; return; }   // no KEPT observation
    lmap[l] = c.x;
    lm_off_out[c.x] = c.y;
    uint32_t o0, o1, k = c.y;
    inc_range(lm_off, l, n_obs, o0, o1);
    for (uint32_t o = o0; o < o1; o++) {
        if (ostate[o] != CVB_RECON_OBS_KEPT) continue;
        const uint32_t v = obs[2 * (size_t)o], f = obs[2 * (size_t)o + 1];
        const uint32_t nv = v < V && vstate[v] == CVB_RECON_VIEW_KEPT ? vcnt[v].x : INC_NONE;
        if (k < n_obs) { obs_out[2 * (size_t)k] = nv; obs_out[2 * (size_t)k + 1] = f; }
        k++;
        const uint32_t j = ap_feature(v, f, V, nf, view_off, vstate, vcnt);
        if (j < nf) view_lm_out[j] = c.x;
    }
}
// per SPLIT observation, after the scans: a landmark of its own after the kept ones, in observation order
__global__ void k_ap_splits(uint32_t V, uint32_t nf, uint32_t L, uint32_t n_obs, const uint32_t *__restrict__ view_off,
                            const uint8_t *__restrict__ vstate, const uint2 *__restrict__ vcnt, const uint32_t *__restrict__ obs,
                            const uint8_t *__restrict__ ostate, const uint2 *__restrict__ scnt, const uint2 *__restrict__ ltotal,
                            uint32_t *__restrict__ lm_off_out, uint32_t *__restrict__ obs_out, uint32_t *__restrict__ view_lm_out) {
    const uint32_t o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= n_obs || ostate[o] != CVB_RECON_OBS_SPLIT) return;
    const uint2 t = *ltotal;
    const uint32_t r = scnt[o].x, l = t.x + r, k = t.y + r;
    if (l < L + n_obs) lm_off_out[l] = k;
    const uint32_t v = obs[2 * (size_t)o], f = obs[2 * (size_t)o + 1];
    if (k < n_obs) {
        obs_out[2 * (size_t)k] = v < V && vstate[v] == CVB_RECON_VIEW_KEPT ? vcnt[v].x : INC_NONE;
        obs_out[2 * (size_t)k + 1] = f;
    }
    const uint32_t j = ap_feature(v, f, V, nf, view_off, vstate, vcnt);
    if (j < nf) view_lm_out[j] = l;
}
// per constraint, after the scan: the kept ones in order, their views renumbered
__global__ void k_ap_constraints(uint32_t C, const cvb_view_constraint *__restrict__ cons, const uint2 *__restrict__ ccnt,
                                 const uint2 *__restrict__ ctotal, const uint2 *__restrict__ vcnt, cvb_view_constraint *__restrict__ cons_out) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    const uint32_t r = ccnt[c].x, next = c + 1 < C ? ccnt[c + 1].x : ctotal->x;
    if (next == r) return;   // dropped (its views were checked in k_ap_constraint_counts)
    cvb_view_constraint x = cons[c];
    for (int k = 0; k < 3; k++) x.views[k] = vcnt[x.views[k]].x;
    cons_out[r] = x;
}
// the closing rows and the counts
__global__ void k_ap_finish(const uint2 *__restrict__ vtotal, const uint2 *__restrict__ ltotal, const uint2 *__restrict__ stotal,
                            const uint2 *__restrict__ ctotal, uint32_t cap_l, uint32_t *__restrict__ view_off_out, uint32_t *__restrict__ lm_off_out,
                            cvb_incorporate_counts *__restrict__ counts) {
    const uint2 vt = *vtotal, lt = *ltotal, st = *stotal;
    view_off_out[vt.x] = vt.y;
    const uint32_t l = lt.x + st.x, n = lt.y + st.x;
    if (l <= cap_l) lm_off_out[l] = n;
    cvb_incorporate_counts c;
    c.V = vt.x;
    c.n_features = vt.y;
    c.L = l;
    c.n_observations = n;
    c.C = ctotal->x;
    c.merges = 0;
    *counts = c;
}

// ---- incorporate_frame's glue -----------------------------------------------------------------------------------------------------------
// remove_view of the new view V as apply_optimization's states: its observations DROPPED, every other KEPT
__global__ void k_inc_reject_states(uint32_t n_obs, uint32_t V, const uint32_t *__restrict__ obs, uint8_t *__restrict__ ostate) {
    const uint32_t o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o < n_obs) ostate[o] = obs[2 * (size_t)o] == V ? CVB_RECON_OBS_DROPPED : CVB_RECON_OBS_KEPT;
}
// a map from the input to the output: first[i] (INC_NONE, or an index < n_mid) through second[]; a nullptr map is the identity
__global__ void k_inc_compose(uint32_t n, const uint32_t *__restrict__ first, uint32_t n_mid, const uint32_t *__restrict__ second,
                              uint32_t *__restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t m = first ? first[i] : i;
    out[i] = !second ? m : (m < n_mid ? second[m] : INC_NONE);
}
