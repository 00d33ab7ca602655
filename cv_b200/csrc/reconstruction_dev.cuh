// cv_b200/csrc/reconstruction_dev.cuh -- cv-sfm's reconstruction optimisation on the device (include/cvb200_reconstruction.h):
// VSlam::optimize_reconstruction (cv-sfm/src/lib.rs:2343-2355), its pose graph (apply_constraints) and its observation filter
// (filter_non_robust_observations), as a pure function of a reconstruction snapshot.  Included by geom.cu after constraints_dev.cuh
// (world_bearing, observations_robust), the triangulators and the optimiser helpers (no -rdc).
//
// Per round: the live constraints' edges in a per-view CSR (k_rec_count, k_rec_scan, k_rec_place: a stable counting sort, the edge
// transforms with it); every Jacobi step in one cooperative launch (k_rec_steps: one thread per edge writes its se3 term, a grid barrier,
// one warp per view adds its terms in list order and updates the pose into the other half of a ping-pong buffer, a grid barrier, the stop
// rules); the views left (k_rec_present); the filter, one thread per landmark (k_rec_filter); its verdict (k_rec_judge).  k_rec_finish
// writes the outputs.  RecCtl carries the status and the current half of the ping-pong buffers between launches, so the host never
// waits inside the call.
#pragma once

constexpr int32_t REC_RUNNING = -1;
constexpr int REC_NT = 256;

struct RecParams {
    double rate, max_sin, max_cos, inc;
    uint32_t V, C, iters, min_obs_cfg, min_robust;
};
struct RecCtl {
    int32_t status;
    uint32_t round, step;
    uint32_t cur;                        // the half of the pose / state buffers that holds the current ones
    uint32_t panic;                      // a present view reached a removed one in this step's edges
    uint32_t updated[2], small[2];       // per step parity: views updated, and of them through rotation_small
    uint32_t small_total, split;
    uint32_t min_obs;                    // min(robust_minimum_observations, views present) of this round's filter
    uint32_t robust_before, robust_after;
};

// Skew3::from(Rotation3) (so3.rs:263-275): nalgebra's scaled_axis, NaN mapped to zero
__device__ void rot_log(const double *m, double *w) {
    const double angle = acos((m[0] + m[4] + m[8] - 1.0) / 2.0);
    const double a[3] = {m[7] - m[5], m[2] - m[6], m[3] - m[1]};
    const double sq = dot3(a, a);
    if (sq > DBL_EPSILON * DBL_EPSILON) {
        const double n = sqrt(sq);
        for (int i = 0; i < 3; i++) w[i] = a[i] / n * angle;
    } else {
        w[0] = w[1] = w[2] = 0.0;
    }
    if (any_nan3(w)) w[0] = w[1] = w[2] = 0.0;
}
// Rotation3::from_matrix (from_matrix_eps with f64::EPSILON, an identity guess; the loop bound is the header's)
__device__ void rot_from_matrix(const double *m, double *rot) {
    for (int i = 0; i < 9; i++) rot[i] = (i % 4 == 0) ? 1.0 : 0.0;
    for (int it = 0; it < CVB_RECON_FROM_MATRIX_MAX_ITERATIONS; it++) {
        double axis[3] = {0.0, 0.0, 0.0}, denom = 0.0;
        for (int c = 0; c < 3; c++) {
            const double rc[3] = {rot[c], rot[3 + c], rot[6 + c]}, mc[3] = {m[c], m[3 + c], m[6 + c]};
            double x[3];
            cross3(rc, mc, x);
            for (int i = 0; i < 3; i++) axis[i] = c == 0 ? x[i] : axis[i] + x[i];
            denom = c == 0 ? dot3(rc, mc) : denom + dot3(rc, mc);
        }
        const double d = fabs(denom) + DBL_EPSILON;
        const double aa[3] = {axis[0] / d, axis[1] / d, axis[2] / d};
        if (!(dot3(aa, aa) > DBL_EPSILON * DBL_EPSILON)) break;
        double Rd[9], Rn[9];
        rot_from_scaled_axis(aa, Rd);   // from_axis_angle(aa / |aa|, |aa|)
        for (int r = 0; r < 3; r++)
            for (int c = 0; c < 3; c++) Rn[3 * r + c] = Rd[3 * r] * rot[c] + Rd[3 * r + 1] * rot[3 + c] + Rd[3 * r + 2] * rot[6 + c];
        for (int i = 0; i < 9; i++) rot[i] = Rn[i];
    }
}
// Rotation3::from(Skew3) (so3.rs:248-261); returns whether rotation_small was taken
__device__ bool rot_exp(const double *w, double *R) {
    if (dot3(w, w) <= DBL_EPSILON) {
        const double m[9] = {1.0, -w[2], w[1], w[2], 1.0, -w[0], -w[1], w[0], 1.0};
        rot_from_matrix(m, R);
        return true;
    }
    rot_from_scaled_axis(w, R);
    return false;
}
// a constraint that contains no removed view (and, as a precondition, only distinct views below V)
__device__ __forceinline__ bool rec_live(const cvb_view_constraint &c, uint32_t V, const uint8_t *S) {
    const uint32_t a = c.views[0], b = c.views[1], d = c.views[2];
    return a < V && b < V && d < V && a != b && a != d && b != d && S[a] == CVB_RECON_VIEW_KEPT && S[b] == CVB_RECON_VIEW_KEPT &&
           S[d] == CVB_RECON_VIEW_KEPT;
}

__global__ void k_rec_init(RecCtl *ctl) {
    RecCtl c;
    memset(&c, 0, sizeof(c));
    c.status = REC_RUNNING;
    *ctl = c;
}
// two edges per view of every live constraint (deg zeroed)
__global__ void __launch_bounds__(256) k_rec_count(RecParams prm, const RecCtl *ctl, const cvb_view_constraint *__restrict__ cons,
                                                   const uint8_t *sbuf, uint32_t *deg) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= prm.C || ctl->status != REC_RUNNING) return;
    const uint8_t *S = sbuf + (size_t)ctl->cur * prm.V;
    const cvb_view_constraint &k = cons[c];
    if (!rec_live(k, prm.V, S)) return;
    for (int x = 0; x < 3; x++) atomicAdd(&deg[k.views[x]], 2u);
}
// exclusive scan of deg into edge_off [V + 1]; one thread
__global__ void k_rec_scan(RecParams prm, const RecCtl *ctl, const uint32_t *deg, uint32_t *edge_off) {
    if (threadIdx.x != 0 || blockIdx.x != 0 || ctl->status != REC_RUNNING) return;
    uint32_t off = 0;
    for (uint32_t v = 0; v < prm.V; v++) { edge_off[v] = off; off += deg[v]; }
    edge_off[prm.V] = off;
}
// flatten_constraints (lib.rs:2519-2532) with edge_constraints (lib.rs:167-180), one warp per view: the live constraints in order, a
// ballot over 32 of them at a time, each containing the view writes its two edges at the view's running position
__global__ void __launch_bounds__(256) k_rec_place(RecParams prm, const RecCtl *ctl, const cvb_view_constraint *__restrict__ cons,
                                                   const uint8_t *sbuf, const uint32_t *edge_off, uint32_t *edge_view, uint32_t *edge_other,
                                                   cvb_pose *edge_T) {
    const uint32_t lane = threadIdx.x & 31, v = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (v >= prm.V || ctl->status != REC_RUNNING) return;
    const uint8_t *S = sbuf + (size_t)ctl->cur * prm.V;
    uint32_t pos = edge_off[v];
    if (pos == edge_off[v + 1]) return;
    for (uint32_t c0 = 0; c0 < prm.C; c0 += 32) {
        const uint32_t c = c0 + lane;
        int slot = -1;
        if (c < prm.C && rec_live(cons[c], prm.V, S))
            for (int x = 0; x < 3; x++) if (cons[c].views[x] == v) slot = x;
        const uint32_t ball = __ballot_sync(0xffffffffu, slot >= 0);
        if (slot >= 0) {
            const cvb_view_constraint &k = cons[c];
            const uint32_t p = pos + 2 * __popc(ball & ((1u << lane) - 1));
            cvb_pose T[2], inv, f2s;
            uint32_t other[2];
            if (slot == 0) {
                pose_inverse(k.poses[1], &T[0]); other[0] = k.views[2];
                pose_inverse(k.poses[0], &T[1]); other[1] = k.views[1];
            } else {
                pose_inverse(k.poses[0], &inv);
                pose_mul(k.poses[1], inv, &f2s);   // first_to_second = second * first^-1
                if (slot == 1) {
                    T[0] = k.poses[0]; other[0] = k.views[0];
                    pose_inverse(f2s, &T[1]); other[1] = k.views[2];
                } else {
                    T[0] = f2s; other[0] = k.views[1];
                    T[1] = k.poses[1]; other[1] = k.views[0];
                }
            }
            for (int x = 0; x < 2; x++) { edge_view[p + x] = v; edge_other[p + x] = other[x]; edge_T[p + x] = T[x]; }
        }
        pos += 2 * __popc(ball);
    }
}
// se3 of T * P_other * P_view^-1 (constrain_view, lib.rs:1913-1924): the translation, then Skew3::from(rotation)
__device__ void rec_edge_se3(const cvb_pose &T, const cvb_pose &Po, const cvb_pose &Pv, double *out) {
    cvb_pose inv, a, d;
    pose_inverse(Pv, &inv);
    pose_mul(T, Po, &a);
    pose_mul(a, inv, &d);
    double w[3];
    rot_log(d.r, w);
    for (int i = 0; i < 3; i++) { out[i] = d.t[i]; out[3 + i] = w[i]; }
}
// apply_constraints' steps (lib.rs:2358-2414), persistent over a grid that is all resident (cooperative launch).  Pose and state buffers
// are ping-pong halves, read at ctl->cur and written at the other; a step that stops the call is not committed.  The buffers written in
// the kernel are read without __restrict__ / const so that no load goes through the non-coherent path.
__global__ void __launch_bounds__(REC_NT) k_rec_steps(RecParams prm, RecCtl *ctl, const uint32_t *__restrict__ edge_off,
                                                      const uint32_t *__restrict__ edge_view, const uint32_t *__restrict__ edge_other,
                                                      const cvb_pose *__restrict__ edge_T, double *se3, cvb_pose *pbuf, uint8_t *sbuf,
                                                      uint32_t round) {
    namespace cg = cooperative_groups;
    cg::grid_group grid = cg::this_grid();
    if (ctl->status != REC_RUNNING) return;
    const uint32_t V = prm.V, E = edge_off[V];
    const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x, nth = gridDim.x * blockDim.x, lane = threadIdx.x & 31;
    uint32_t cur = ctl->cur;
    volatile RecCtl *vc = ctl;
    if (tid == 0) { ctl->updated[0] = 0; ctl->small[0] = 0; }
    for (uint32_t s = 0; s < prm.iters; s++) {
        const cvb_pose *P = pbuf + (size_t)cur * V;
        cvb_pose *Pn = pbuf + (size_t)(cur ^ 1) * V;
        const uint8_t *S = sbuf + (size_t)cur * V;
        uint8_t *Sn = sbuf + (size_t)(cur ^ 1) * V;
        for (uint32_t e = tid; e < E; e += nth) {
            const uint32_t v = edge_view[e], u = edge_other[e];
            if (S[v] != CVB_RECON_VIEW_KEPT) continue;
            if (S[u] != CVB_RECON_VIEW_KEPT) { vc->panic = 1; continue; }
            rec_edge_se3(edge_T[e], P[u], P[v], se3 + 6 * (size_t)e);
        }
        grid.sync();
        if (vc->panic) {
            if (tid == 0) { ctl->status = CVB_RECON_PANIC; ctl->round = round; ctl->step = s; }
            break;
        }
        // every thread has read the previous step's counters by now: the next step's may be reset
        if (tid == 0) { vc->updated[(s + 1) & 1] = 0; vc->small[(s + 1) & 1] = 0; }
        for (uint32_t v = tid >> 5; v < V; v += nth >> 5) {
            const uint32_t e0 = edge_off[v], e1 = edge_off[v + 1];
            if (S[v] != CVB_RECON_VIEW_KEPT || e0 == e1) {
                if (lane == 0) { Pn[v] = P[v]; Sn[v] = S[v] != CVB_RECON_VIEW_KEPT ? S[v] : (uint8_t)CVB_RECON_VIEW_NO_EDGES; }
                continue;
            }
            // Iterator::sum from zero in list order; lane j holds edge b + j, and every lane adds them all in order
            double acc[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
            for (uint32_t b = e0; b < e1; b += 32) {
                double x[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
                if (b + lane < e1)
                    for (int c = 0; c < 6; c++) x[c] = se3[6 * (size_t)(b + lane) + c];
                const uint32_t n = min(32u, e1 - b);
                for (uint32_t i = 0; i < n; i++)
                    for (int c = 0; c < 6; c++) acc[c] = acc[c] + __shfl_sync(0xffffffffu, x[c], i);
            }
            if (lane != 0) continue;
            double d[6];
            bool finite = true;
            for (int c = 0; c < 6; c++) { d[c] = acc[c] * prm.rate; finite = finite && isfinite(d[c]); }
            if (!finite) { Pn[v] = P[v]; Sn[v] = CVB_RECON_VIEW_NON_FINITE; continue; }
            cvb_pose D, out;
            const bool small = rot_exp(d + 3, D.r);
            for (int i = 0; i < 3; i++) D.t[i] = d[i];
            pose_mul(D, P[v], &out);
            Pn[v] = out;
            Sn[v] = CVB_RECON_VIEW_KEPT;
            atomicAdd((uint32_t *)&vc->updated[s & 1], 1u);
            if (small) atomicAdd((uint32_t *)&vc->small[s & 1], 1u);
        }
        grid.sync();
        if (vc->updated[s & 1] < 3) {
            if (tid == 0) { ctl->status = CVB_RECON_REMOVED_CONSTRAINTS; ctl->round = round; ctl->step = s; }
            break;
        }
        if (tid == 0) vc->small_total += vc->small[s & 1];
        cur ^= 1;
    }
    if (tid == 0) ctl->cur = cur;
}
// the views left, hence robust_minimum_observations' cap; one CTA
__global__ void __launch_bounds__(256) k_rec_present(RecParams prm, RecCtl *ctl, const uint8_t *sbuf) {
    __shared__ uint32_t s_n;
    if (ctl->status != REC_RUNNING) return;
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    const uint8_t *S = sbuf + (size_t)ctl->cur * prm.V;
    uint32_t n = 0;
    for (uint32_t v = threadIdx.x; v < prm.V; v += blockDim.x) n += S[v] == CVB_RECON_VIEW_KEPT;
    atomicAdd(&s_n, n);
    __syncthreads();
    if (threadIdx.x == 0) { ctl->min_obs = min(prm.min_obs_cfg, s_n); ctl->robust_before = 0; ctl->robust_after = 0; }
}
// filter_non_robust_observations (lib.rs:2657-2757), one thread per landmark: its observations of present views that are still in it,
// gathered in order at the front of its own CSR range (gi: their input positions), the robust test before, the split decisions, the
// robust test after over the observations that stay
__global__ void __launch_bounds__(128) k_rec_filter(cvb_triangulator T, RecParams prm, RecCtl *ctl, const cvb_pose *pbuf, const uint8_t *sbuf,
                                                    const uint32_t *__restrict__ view_off, const double *__restrict__ bear,
                                                    const uint32_t *__restrict__ lm_off, const uint32_t *__restrict__ obs, uint32_t L,
                                                    uint8_t *obs_state, cvb_pose *gp, double *gb, double *gw, uint32_t *gi, double *W) {
    const uint32_t l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= L || ctl->status != REC_RUNNING) return;
    const cvb_pose *P = pbuf + (size_t)ctl->cur * prm.V;
    const uint8_t *S = sbuf + (size_t)ctl->cur * prm.V;
    const uint32_t o0 = lm_off[l], n_in = lm_off[l + 1] - o0, min_obs = ctl->min_obs;
    uint32_t m = 0;
    for (uint32_t i = 0; i < n_in; i++) {
        const uint32_t o = o0 + i, v = obs[2 * (size_t)o], f = obs[2 * (size_t)o + 1];
        if (S[v] != CVB_RECON_VIEW_KEPT) { obs_state[o] = CVB_RECON_OBS_DROPPED; continue; }
        if (obs_state[o] != CVB_RECON_OBS_KEPT) continue;
        const uint32_t q = o0 + m++;
        const double *b = bear + 3 * ((size_t)view_off[v] + f);
        gi[q] = o;
        gp[q] = P[v];
        for (int r = 0; r < 3; r++) gb[3 * (size_t)q + r] = b[r];
        world_bearing(P[v], b, gw + 3 * (size_t)q);
    }
    const cvb_pose *Pl = gp + o0;
    const double *Bl = gb + 3 * (size_t)o0;
    double *Wl = gw + 3 * (size_t)o0;
    const bool before = observations_robust(gw, o0, m, min_obs, prm.inc);
    uint32_t split = 0;
    if (m == 2) {   // is_bi_landmark_robust (lib.rs:1306-1318), else split_landmark
        cvb_pose inv, tot;
        double fb[3];
        pose_inverse(Pl[0], &inv);
        pose_mul(Pl[1], inv, &tot);
        rotv(tot.r, Bl, fb);
        if (!(epipolar_loss(tot.t, fb, Bl + 3) < prm.max_sin)) { obs_state[gi[o0 + 1]] = CVB_RECON_OBS_SPLIT; split = 1; }
    } else if (m >= 3) {
        double p[4];
        if (!triangulate_observations(T, Pl, Bl, m, W ? W + 6 * (size_t)o0 : nullptr, p)) {   // split_landmark keeps the first
            for (uint32_t k = 1; k < m; k++) obs_state[gi[o0 + k]] = CVB_RECON_OBS_SPLIT;
            split = m - 1;
        } else {   // split_observation refuses the last remaining observation
            for (uint32_t k = 0; k < m; k++)
                if (transformed_cosine_distance(Pl[k], p, Bl + 3 * (size_t)k) > prm.max_cos && m - split >= 2) {
                    obs_state[gi[o0 + k]] = CVB_RECON_OBS_SPLIT;
                    split++;
                }
        }
    }
    uint32_t kept = 0;
    for (uint32_t k = 0; k < m; k++)
        if (obs_state[gi[o0 + k]] == CVB_RECON_OBS_KEPT) {
            for (int r = 0; r < 3; r++) Wl[3 * (size_t)kept + r] = Wl[3 * (size_t)k + r];
            kept++;
        }
    const bool after = observations_robust(gw, o0, kept, min_obs, prm.inc);
    if (before) atomicAdd(&ctl->robust_before, 1u);
    if (after) atomicAdd(&ctl->robust_after, 1u);
    if (split) atomicAdd(&ctl->split, split);
}
// lib.rs:2744-2755: too few robust landmarks removes the reconstruction
__global__ void k_rec_judge(RecParams prm, RecCtl *ctl, uint32_t round) {
    if (threadIdx.x != 0 || blockIdx.x != 0 || ctl->status != REC_RUNNING) return;
    if (ctl->robust_after < prm.min_robust) { ctl->status = CVB_RECON_REMOVED_FILTER; ctl->round = round; ctl->step = prm.iters; }
}
// the outputs; one CTA
__global__ void __launch_bounds__(256) k_rec_finish(RecParams prm, const RecCtl *ctl, const cvb_pose *pbuf, const uint8_t *sbuf,
                                                    uint32_t rounds, cvb_recon_result *res, cvb_pose *poses_out, uint8_t *view_state) {
    __shared__ uint32_t s_removed;
    if (threadIdx.x == 0) s_removed = 0;
    __syncthreads();
    const cvb_pose *P = pbuf + (size_t)ctl->cur * prm.V;
    const uint8_t *S = sbuf + (size_t)ctl->cur * prm.V;
    uint32_t removed = 0;
    for (uint32_t v = threadIdx.x; v < prm.V; v += blockDim.x) {
        poses_out[v] = P[v];
        view_state[v] = S[v];
        removed += S[v] != CVB_RECON_VIEW_KEPT;
    }
    atomicAdd(&s_removed, removed);
    __syncthreads();
    if (threadIdx.x != 0) return;
    cvb_recon_result r;
    const bool kept = ctl->status == REC_RUNNING;
    r.status = kept ? CVB_RECON_KEPT : ctl->status;
    r.round = kept ? rounds : ctl->round;
    r.step = kept ? 0 : ctl->step;
    r.views_removed = s_removed;
    r.robust_before = ctl->robust_before;
    r.robust_after = ctl->robust_after;
    r.observations_split = ctl->split;
    r.small_angle_updates = ctl->small_total;
    *res = r;
}
