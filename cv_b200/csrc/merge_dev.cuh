// cv_b200/csrc/merge_dev.cuh -- the move edit of cv-sfm's incorporate_reconstruction on the device (include/cvb200_merge.h): a source
// reconstruction's views appended to a destination snapshot under a WorldToWorld, their landmarks mapped or created.  Included by
// geom.cu after incorporate_dev.cuh (its scan, inc_range and INC_NONE; no -rdc).
//
// The moved views are S's views without skip_view, in order, so the moved rows of S's view CSR keep their order and only shift past
// skip_view's rows: the pose transform, the view offsets and the feature rows need no scan.  The landmarks do: one scan over the pairs
// (present, observations) of D's landmarks followed by S's feature rows, where a row is present when it is the first moved (view, feature)
// of an unmapped S landmark, gives D's landmark offsets and every created landmark its index (creation order: moved-view order, then
// feature order) and offset at once.  Each S landmark then places its moved observations at its target's tail, ranked by view, so that
// they come in moved-view order whatever the order of S's landmark CSR.
//
// As in incorporate_dev.cuh, reads of offset arrays are clamped and writes are checked against the output capacities, so that a broken
// precondition (inconsistent CSRs, a non-injective or out-of-range landmark map) gives wrong output, never an out-of-bounds access.
#pragma once

// the moved index of S view v, or INC_NONE for skip_view
__device__ __forceinline__ uint32_t mg_moved(uint32_t v, uint32_t skip) { return v == skip ? INC_NONE : v - (skip < v ? 1u : 0u); }

// world_transform = dest^-1 * src (WorldToWorld::from_camera_poses, cv-core/src/pose.rs:322); one thread
__global__ void k_mg_world(const cvb_pose *__restrict__ dest, const cvb_pose *__restrict__ src, cvb_pose *__restrict__ wt) {
    cvb_pose inv;
    pose_inverse(*dest, &inv);
    con_pose_mul(inv, *src, wt);
}

// per S view v != skip: its pose P_v * world_transform^-1 and its view offset, at view V + its moved index
__global__ void k_mg_views(uint32_t VS, uint32_t skip, uint32_t V, uint32_t nf, uint32_t nf_s, const cvb_pose *__restrict__ poses_s,
                           const uint32_t *__restrict__ vo_s, const cvb_pose *__restrict__ wt, cvb_pose *__restrict__ poses_out,
                           uint32_t *__restrict__ vo_out) {
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= VS) return;
    const uint32_t q = mg_moved(v, skip);
    if (q == INC_NONE) return;
    uint32_t s0 = 0, s1 = 0, f0, f1;
    if (skip < VS) inc_range(vo_s, skip, nf_s, s0, s1);
    inc_range(vo_s, v, nf_s, f0, f1);
    cvb_pose inv;
    pose_inverse(*wt, &inv);
    con_pose_mul(poses_s[v], inv, &poses_out[V + q]);
    vo_out[V + q] = nf + f0 - (skip < v ? s1 - s0 : 0u);
}

// per S landmark: its moved observations n and the S row of the first of them (smallest view; feature order within a view is the row
// order); D's tail count app[landmark_map[l]] = n when mapped, otherwise the pair (1, n) at the first row's element L + row.  cnt's row
// elements and app are zeroed before.
__global__ void k_mg_landmark_counts(uint32_t LS, uint32_t n_obs_s, uint32_t VS, uint32_t nf_s, uint32_t skip, uint32_t L,
                                     const uint32_t *__restrict__ lo_s, const uint32_t *__restrict__ obs_s, const uint32_t *__restrict__ vo_s,
                                     const uint32_t *__restrict__ lmap_in, uint32_t *__restrict__ app, uint2 *__restrict__ cnt,
                                     uint32_t *__restrict__ first) {
    const uint32_t l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= LS) return;
    uint32_t o0, o1, n = 0, bv = INC_NONE, row = INC_NONE;
    inc_range(lo_s, l, n_obs_s, o0, o1);
    for (uint32_t o = o0; o < o1; o++) {
        const uint32_t v = obs_s[2 * (size_t)o], f = obs_s[2 * (size_t)o + 1];
        if (v >= VS || v == skip) continue;
        uint32_t f0, f1;
        inc_range(vo_s, v, nf_s, f0, f1);
        if (f >= f1 - f0) continue;
        n++;
        if (v < bv) { bv = v; row = f0 + f; }
    }
    first[l] = row;
    const uint32_t d = lmap_in[l];
    if (d < L) app[d] = n;
    else if (row != INC_NONE) cnt[L + row] = make_uint2(1, n);
}

// per D landmark: (1, its observations + the appended ones)
__global__ void k_mg_dest_counts(uint32_t L, uint32_t n_obs, const uint32_t *__restrict__ lo, const uint32_t *__restrict__ app,
                                 uint2 *__restrict__ cnt) {
    const uint32_t d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= L) return;
    uint32_t o0, o1;
    inc_range(lo, d, n_obs, o0, o1);
    cnt[d] = make_uint2(1, o1 - o0 + app[d]);
}

// per D landmark, after the scan: its offset and its own observations
__global__ void k_mg_dest_place(uint32_t L, uint32_t n_obs, const uint32_t *__restrict__ lo, const uint32_t *__restrict__ obs,
                                const uint2 *__restrict__ cnt, uint32_t cap_o, uint32_t *__restrict__ lo_out, uint32_t *__restrict__ obs_out) {
    const uint32_t d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= L) return;
    uint32_t o0, o1, k = cnt[d].y;
    lo_out[d] = min(k, cap_o);
    inc_range(lo, d, n_obs, o0, o1);
    for (uint32_t o = o0; o < o1; o++, k++)
        if (k < cap_o) { obs_out[2 * (size_t)k] = obs[2 * (size_t)o]; obs_out[2 * (size_t)k + 1] = obs[2 * (size_t)o + 1]; }
}

// per S landmark, after the scan: its target (the map's entry or its created landmark), written to the source landmark map; a created
// landmark's offset; its moved observations at the target's tail, each ranked by the moved observations of smaller views
__global__ void k_mg_landmark_place(uint32_t LS, uint32_t n_obs_s, uint32_t VS, uint32_t nf_s, uint32_t skip, uint32_t V, uint32_t L,
                                    uint32_t n_obs, const uint32_t *__restrict__ lo_s, const uint32_t *__restrict__ obs_s,
                                    const uint32_t *__restrict__ vo_s, const uint32_t *__restrict__ lmap_in, const uint32_t *__restrict__ lo,
                                    const uint2 *__restrict__ cnt, const uint32_t *__restrict__ first, uint32_t cap_l, uint32_t cap_o,
                                    uint32_t *__restrict__ lo_out, uint32_t *__restrict__ obs_out, uint32_t *__restrict__ tgt) {
    const uint32_t l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= LS) return;
    const uint32_t d0 = lmap_in[l], row = first[l];
    uint32_t d = INC_NONE, base = 0;
    if (d0 < L) {
        uint32_t a0, a1;
        inc_range(lo, d0, n_obs, a0, a1);
        d = d0;
        base = cnt[d0].y + (a1 - a0);
    } else if (row < nf_s) {
        const uint2 c = cnt[L + row];
        d = c.x;
        base = c.y;
        if (d < cap_l) lo_out[d] = min(base, cap_o);
    }
    tgt[l] = d;
    if (d == INC_NONE) return;
    uint32_t o0, o1;
    inc_range(lo_s, l, n_obs_s, o0, o1);
    for (uint32_t o = o0; o < o1; o++) {
        const uint32_t v = obs_s[2 * (size_t)o], f = obs_s[2 * (size_t)o + 1];
        if (v >= VS || v == skip) continue;
        uint32_t f0, f1;
        inc_range(vo_s, v, nf_s, f0, f1);
        if (f >= f1 - f0) continue;
        uint32_t rank = 0;
        for (uint32_t p = o0; p < o1; p++) {
            const uint32_t w = obs_s[2 * (size_t)p];
            rank += w < v && w != skip;
        }
        const uint32_t k = base + rank;
        if (k < cap_o) { obs_out[2 * (size_t)k] = V + mg_moved(v, skip); obs_out[2 * (size_t)k + 1] = f; }
    }
}

// one warp per moved view: its feature rows (landmark through tgt, bearing, descriptor as four uint4, colour) after D's rows
__global__ void __launch_bounds__(256) k_mg_feature_rows(uint32_t VS, uint32_t skip, uint32_t nf, uint32_t nf_s, uint32_t LS,
                                                         const uint32_t *__restrict__ vo_s, const uint32_t *__restrict__ vl_s,
                                                         const double *__restrict__ bear_s, const uint4 *__restrict__ desc_s,
                                                         const uint8_t *__restrict__ col_s, const uint32_t *__restrict__ tgt, uint32_t cap_f,
                                                         uint32_t *__restrict__ vl_out, double *__restrict__ bear_out, uint4 *__restrict__ desc_out,
                                                         uint8_t *__restrict__ col_out) {
    const uint32_t v = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (v >= VS || v == skip) return;
    uint32_t s0 = 0, s1 = 0, f0, f1;
    if (skip < VS) inc_range(vo_s, skip, nf_s, s0, s1);
    inc_range(vo_s, v, nf_s, f0, f1);
    const size_t d0 = (size_t)nf + f0 - (skip < v ? s1 - s0 : 0u);
    for (uint32_t j = lane; j < f1 - f0; j += 32) {
        const size_t s = f0 + j, d = d0 + j;
        if (d >= cap_f) break;
        const uint32_t l = vl_s[s];
        vl_out[d] = l < LS ? tgt[l] : INC_NONE;
        for (int k = 0; k < 3; k++) bear_out[3 * d + k] = bear_s[3 * s + k];
        if (desc_s)
            for (int k = 0; k < 4; k++) desc_out[4 * d + k] = desc_s[4 * s + k];
        if (col_s)
            for (int k = 0; k < 3; k++) col_out[3 * d + k] = col_s[3 * s + k];
    }
}

// the closing rows and the counts.  With consistent CSRs the totals fit the capacities (cap_l landmarks, cap_o observations); with S's
// landmark CSR out of step with its view CSR the observation total can exceed cap_o, and it is clamped, as every landmark offset is, so
// that the calls that read the snapshot next stay inside its buffers
__global__ void k_mg_finish(uint32_t V, uint32_t Q, uint32_t nf_out, const uint2 *__restrict__ total, uint32_t cap_l, uint32_t cap_o,
                            uint32_t *__restrict__ vo_out, uint32_t *__restrict__ lo_out, cvb_incorporate_counts *__restrict__ counts) {
    const uint2 t = *total;
    const uint32_t nl = min(t.x, cap_l), no = min(t.y, cap_o);
    vo_out[V + Q] = nf_out;
    lo_out[nl] = no;
    cvb_incorporate_counts c;
    c.V = V + Q;
    c.n_features = nf_out;
    c.L = nl;
    c.n_observations = no;
    c.C = 0;
    c.merges = 0;
    *counts = c;
}

// try_merge_reconstructions' landmark_to_landmark: S landmark of s_view's feature -> add_view's landmark_a of its match
__global__ void k_mg_ltl(uint32_t M, const cvb_register_match *__restrict__ matches, uint32_t N, const uint32_t *__restrict__ vl_view,
                         uint32_t LS, uint32_t L, const uint32_t *__restrict__ amap, uint32_t *__restrict__ ltl) {
    const uint32_t m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= M) return;
    const cvb_register_match t = matches[m];
    if (t.feature >= N) return;
    const uint32_t ls = vl_view[t.feature];
    if (ls < LS) ltl[ls] = t.landmark_a < L ? amap[t.landmark_a] : INC_NONE;
}
