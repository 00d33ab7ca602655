// cv_b200/csrc/try_init_dev.cuh -- add_reconstruction on the device (include/cvb200_try_init.h): three frames of the frame store and the
// three match lists of init_reconstruction to the first snapshot of a reconstruction.  Included by geom.cu after incorporate_dev.cuh (its
// scan, inc_range and INC_NONE; no -rdc).
//
// The feature counts and list lengths are read on the device, so every kernel is a grid-stride loop over the capacity.  A mapping pass
// scatters the list entries into per-view feature -> center landmark arrays and their inverses (center landmark -> feature); the entries
// are unique by precondition, so it needs no atomics.  One scan over the 3 cap elements (center features, then the first view's, then the
// second's) of the pairs (is a landmark, its observations) gives every landmark its index and its observation offset at once: a center
// feature is landmark c with 1 + [mapped into view 1] + [mapped into view 2] observations, a feature of view 1 or 2 is a new landmark
// with one observation when it is not mapped.  A placement pass then writes the view CSR with its row gathers, the landmark offsets and
// the observations in view order.
//
// As in incorporate_dev.cuh, list entries are clamped to the feature counts and every write is checked against the output capacity, so a
// broken precondition (repeated entries) gives wrong output, never an out-of-bounds access.
#pragma once

struct TiFrames { uint32_t f[3]; };   // the frames of views 0, 1, 2

// the clamped feature counts of the three frames
__device__ __forceinline__ uint32_t ti_count(const uint32_t *__restrict__ n, uint32_t frame, uint32_t cap) { return min(n[frame], cap); }

// every map entry to INC_NONE: fmap[v][f] (feature f of view v = 1, 2 -> center feature) and cmap[v][c] (center feature c -> feature of
// view v = 1, 2), four arrays of cap entries
__global__ void __launch_bounds__(256) k_ti_clear(uint32_t n, uint32_t *__restrict__ maps) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) maps[i] = INC_NONE;
}

// the list entries scattered into the maps; an entry outside the counts is skipped
__global__ void __launch_bounds__(256) k_ti_map(uint32_t cap, TiFrames fr, const uint32_t *__restrict__ n, const cvb_init_result *__restrict__ ir,
                                                const uint32_t *__restrict__ comb, const uint32_t *__restrict__ fm, const uint32_t *__restrict__ sm,
                                                uint32_t *__restrict__ fmap1, uint32_t *__restrict__ fmap2, uint32_t *__restrict__ cmap1,
                                                uint32_t *__restrict__ cmap2) {
    const uint32_t nc = ti_count(n, fr.f[0], cap), n1 = ti_count(n, fr.f[1], cap), n2 = ti_count(n, fr.f[2], cap);
    const uint32_t kc = min(ir->n_combined, cap), k1 = min(ir->n_first_matches, cap), k2 = min(ir->n_second_matches, cap);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += gridDim.x * blockDim.x) {
        if (i < k1) {
            const uint32_t c = fm[2 * (size_t)i], f = fm[2 * (size_t)i + 1];
            if (c < nc && f < n1) { fmap1[f] = c; cmap1[c] = f; }
        }
        if (i < k2) {
            const uint32_t c = sm[2 * (size_t)i], s = sm[2 * (size_t)i + 1];
            if (c < nc && s < n2) { fmap2[s] = c; cmap2[c] = s; }
        }
        if (i < kc) {
            const uint32_t c = comb[3 * (size_t)i], f = comb[3 * (size_t)i + 1], s = comb[3 * (size_t)i + 2];
            if (c < nc && f < n1) { fmap1[f] = c; cmap1[c] = f; }
            if (c < nc && s < n2) { fmap2[s] = c; cmap2[c] = s; }
        }
    }
}

// element e of the 3 cap: (is a landmark, its observations), in the order center, first, second
__global__ void __launch_bounds__(256) k_ti_counts(uint32_t cap, TiFrames fr, const uint32_t *__restrict__ n, const uint32_t *__restrict__ fmap1,
                                                   const uint32_t *__restrict__ fmap2, const uint32_t *__restrict__ cmap1,
                                                   const uint32_t *__restrict__ cmap2, uint2 *__restrict__ cnt) {
    const uint32_t nc = ti_count(n, fr.f[0], cap), n1 = ti_count(n, fr.f[1], cap), n2 = ti_count(n, fr.f[2], cap);
    for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e < 3 * cap; e += gridDim.x * blockDim.x) {
        const uint32_t v = e / cap, j = e - v * cap;
        uint2 c = make_uint2(0, 0);
        if (v == 0 && j < nc) c = make_uint2(1, 1 + (cmap1[j] != INC_NONE) + (cmap2[j] != INC_NONE));
        else if (v == 1 && j < n1 && fmap1[j] == INC_NONE) c = make_uint2(1, 1);
        else if (v == 2 && j < n2 && fmap2[j] == INC_NONE) c = make_uint2(1, 1);
        cnt[e] = c;
    }
}

// after the scan, per element: its feature row (landmark, bearing, descriptor as four uint4, colour) and, when it is a landmark, its
// offset and observations
__global__ void __launch_bounds__(256) k_ti_place(uint32_t cap, TiFrames fr, const uint32_t *__restrict__ n, const double *__restrict__ bear,
                                                  const uint4 *__restrict__ desc, const uint8_t *__restrict__ col,
                                                  const uint32_t *__restrict__ fmap1, const uint32_t *__restrict__ fmap2,
                                                  const uint32_t *__restrict__ cmap1, const uint32_t *__restrict__ cmap2,
                                                  const uint2 *__restrict__ cnt, uint32_t *__restrict__ vl_out, double *__restrict__ bear_out,
                                                  uint4 *__restrict__ desc_out, uint8_t *__restrict__ col_out, uint32_t *__restrict__ lo_out,
                                                  uint32_t *__restrict__ obs_out) {
    const uint32_t nc = ti_count(n, fr.f[0], cap), n1 = ti_count(n, fr.f[1], cap), n2 = ti_count(n, fr.f[2], cap);
    const uint32_t cap3 = 3 * cap;
    for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e < cap3; e += gridDim.x * blockDim.x) {
        const uint32_t v = e / cap, j = e - v * cap;
        const uint32_t nv = v == 0 ? nc : (v == 1 ? n1 : n2);
        if (j >= nv) continue;
        const uint2 p = cnt[e];
        const uint32_t fv = v == 0 ? INC_NONE : (v == 1 ? fmap1[j] : fmap2[j]);
        const uint32_t lm = v == 0 ? j : (fv != INC_NONE ? fv : p.x);
        const size_t d = (size_t)(v == 0 ? 0 : (v == 1 ? nc : nc + n1)) + j;
        const size_t s = (size_t)(v == 0 ? fr.f[0] : (v == 1 ? fr.f[1] : fr.f[2])) * cap + j;
        vl_out[d] = lm;
        for (int k = 0; k < 3; k++) bear_out[3 * d + k] = bear[3 * s + k];
        for (int k = 0; k < 4; k++) desc_out[4 * d + k] = desc[4 * s + k];
        if (col)
            for (int k = 0; k < 3; k++) col_out[3 * d + k] = col[3 * s + k];
        if (v != 0 && fv != INC_NONE) continue;   // an observation of a center landmark, placed by the center element
        if (p.x < cap3) lo_out[p.x] = min(p.y, cap3);
        uint32_t k = p.y;
        auto put = [&](uint32_t view, uint32_t f) {
            if (k < cap3) { obs_out[2 * (size_t)k] = view; obs_out[2 * (size_t)k + 1] = f; }
            k++;
        };
        put(v, j);
        if (v == 0) {
            if (cmap1[j] != INC_NONE) put(1, cmap1[j]);
            if (cmap2[j] != INC_NONE) put(2, cmap2[j]);
        }
    }
}

// the poses, the view offsets, the closing landmark offset, the constraint and the counts; one thread
__global__ void k_ti_finish(uint32_t cap, TiFrames fr, const uint32_t *__restrict__ n, const cvb_init_result *__restrict__ ir,
                            const uint2 *__restrict__ total, cvb_pose *__restrict__ poses_out, uint32_t *__restrict__ vo_out,
                            uint32_t *__restrict__ lo_out, cvb_view_constraint *__restrict__ cons_out,
                            cvb_incorporate_counts *__restrict__ counts) {
    const uint32_t nc = ti_count(n, fr.f[0], cap), n1 = ti_count(n, fr.f[1], cap), n2 = ti_count(n, fr.f[2], cap);
    cvb_pose id;
    for (int k = 0; k < 9; k++) id.r[k] = k % 4 == 0 ? 1.0 : 0.0;
    for (int k = 0; k < 3; k++) id.t[k] = 0.0;
    poses_out[0] = id;
    poses_out[1] = ir->first_pose;
    poses_out[2] = ir->second_pose;
    vo_out[0] = 0;
    vo_out[1] = nc;
    vo_out[2] = nc + n1;
    vo_out[3] = nc + n1 + n2;
    const uint2 t = *total;
    const uint32_t nl = min(t.x, 3 * cap), no = min(t.y, 3 * cap);
    lo_out[nl] = no;
    cvb_view_constraint c;
    c.views[0] = 0;
    c.views[1] = 1;
    c.views[2] = 2;
    c.landmarks = 0;
    c.poses[0] = ir->first_pose;
    c.poses[1] = ir->second_pose;
    cons_out[0] = c;
    cvb_incorporate_counts k;
    k.V = 3;
    k.n_features = nc + n1 + n2;
    k.L = nl;
    k.n_observations = no;
    k.C = 1;
    k.merges = 0;
    *counts = k;
}
