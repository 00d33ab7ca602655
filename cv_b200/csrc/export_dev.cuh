// cv_b200/csrc/export_dev.cuh -- cv-sfm's reconstruction export on the device (include/cvb200_export.h): triangulate_landmark_robust for
// every landmark, export_reconstruction's point cloud and cameras, and normalize_reconstruction, on a reconstruction snapshot.  Included
// by geom.cu after constraints_dev.cuh (k_con_gather_obs, robust_landmark_point, con_pose_mul), init_dev.cuh (init_block_rank) and the
// triangulators (no -rdc).
//
// Stages, each one launch: per observation its pose and bearings (k_con_gather_obs); per landmark (or per landmark of one view) the robust
// point and its state, and per CTA the POINT count (k_exp_robust); the exclusive scan of those counts (k_exp_scan, one thread); the stable
// compaction of the points and their colours (k_exp_compact); one warp per view for the mean distances and the cameras (k_exp_cameras);
// for the normalisation the first view's mean (k_exp_first_mean, one warp) and the transform of every pose and constraint
// (k_exp_normalize).
#pragma once

constexpr int EXP_NT = 128;
// the mean of no values, written as these bits (f64::NAN) rather than computed, so that it does not depend on how a NaN propagates
#define EXP_EMPTY_MEAN __longlong_as_double(0x7ff8000000000000ll)

// one warp: the mean distance of view v (the Mean of lib.rs:2252-2257, 2315-2324).  The lanes transform one feature's point each; every
// lane then folds the 32 values in feature order, since the running mean is a non-associative recurrence.  n: the values folded.
__device__ double exp_view_mean(uint32_t v, const cvb_pose &P, const uint32_t *__restrict__ view_off, const uint32_t *__restrict__ view_lm,
                                const double *__restrict__ points, const uint8_t *__restrict__ state, uint32_t &n) {
    const uint32_t lane = threadIdx.x & 31, f0 = view_off[v], nf = view_off[v + 1] - f0;
    double avg = 0.0;
    n = 0;
    for (uint32_t b = 0; b < nf; b += 32) {
        double d = 0.0;
        bool ok = false;
        if (b + lane < nf) {
            const uint32_t l = view_lm[f0 + b + lane];
            const uint8_t s = state[l];
            if (s == CVB_EXPORT_POINT || s == CVB_EXPORT_AT_INFINITY) {
                const double *h = points + 4 * (size_t)l;
                double q[4];
                for (int r = 0; r < 3; r++) q[r] = ((P.r[3 * r] * h[0] + P.r[3 * r + 1] * h[1]) + P.r[3 * r + 2] * h[2]) + P.t[r] * h[3];
                q[3] = ((0.0 * h[0] + 0.0 * h[1]) + 0.0 * h[2]) + 1.0 * h[3];
                from_homogeneous(q);   // pose.transform returns a CameraPoint (Projective::from_homogeneous)
                const double w = q[3];
                if (w != 0.0) {
                    const double x[3] = {q[0] / w, q[1] / w, q[2] / w};
                    d = norm3(x);
                    ok = true;
                }
            }
        }
        const uint32_t ball = __ballot_sync(0xffffffffu, ok);
        for (uint32_t i = 0; i < 32; i++) {
            const double x = __shfl_sync(0xffffffffu, d, i);
            if (ball >> i & 1u) {
                n++;
                avg = avg + (x - avg) / (double)n;
            }
        }
    }
    return n ? avg : EXP_EMPTY_MEAN;
}

// triangulate_landmark_robust for landmark list[i] (list == nullptr: landmark i); the POINT landmarks of the CTA counted into block_cnt
__global__ void __launch_bounds__(EXP_NT) k_exp_robust(cvb_triangulator T, const uint32_t *__restrict__ lm_off, const uint32_t *__restrict__ list,
                                                       uint32_t n, const cvb_pose *__restrict__ obs_pose, const double *__restrict__ obs_bear,
                                                       const double *__restrict__ obs_world, double *__restrict__ W, uint32_t min_obs, double inc,
                                                       double *__restrict__ points, uint8_t *__restrict__ state, uint32_t *__restrict__ block_cnt) {
    __shared__ uint32_t s_warp[EXP_NT / 32];
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    bool point = false;
    if (i < n) {
        const uint32_t l = list ? list[i] : i, o0 = lm_off[l], m = lm_off[l + 1] - o0;
        double p[4] = {0.0, 0.0, 0.0, 0.0};
        const int r = robust_landmark_point(T, o0, m, obs_pose, obs_bear, obs_world, W, min_obs, inc, p);
        uint8_t s = CVB_EXPORT_NOT_ROBUST;
        if (r == 1) s = CVB_EXPORT_TRI_FAILED;
        if (r == 2) s = p[3] == 0.0 ? CVB_EXPORT_AT_INFINITY : CVB_EXPORT_POINT;
        if (r != 2) p[0] = p[1] = p[2] = p[3] = 0.0;
        for (int k = 0; k < 4; k++) points[4 * (size_t)l + k] = p[k];
        state[l] = s;
        point = s == CVB_EXPORT_POINT;
    }
    if (!block_cnt) return;
    uint32_t tot;
    init_block_rank(point, s_warp, tot);
    if (threadIdx.x == 0) block_cnt[blockIdx.x] = tot;
}
// exclusive scan of the nb CTA counts in place, the total into *n_points; one thread
__global__ void k_exp_scan(uint32_t nb, uint32_t *block_cnt, uint32_t *n_points) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    uint32_t off = 0;
    for (uint32_t b = 0; b < nb; b++) { const uint32_t c = block_cnt[b]; block_cnt[b] = off; off += c; }
    *n_points = off;
}
// the POINT landmarks in landmark order: Point3::from_homogeneous, and the colour of the first observation (lib.rs:2293-2307)
__global__ void __launch_bounds__(EXP_NT) k_exp_compact(uint32_t L, const double *__restrict__ points4, const uint8_t *__restrict__ state,
                                                        const uint32_t *__restrict__ block_off, const uint32_t *__restrict__ view_off,
                                                        const uint32_t *__restrict__ lm_off, const uint32_t *__restrict__ obs,
                                                        const uint8_t *__restrict__ colors, double *__restrict__ out_points,
                                                        uint8_t *__restrict__ out_colors) {
    __shared__ uint32_t s_warp[EXP_NT / 32];
    const uint32_t l = blockIdx.x * blockDim.x + threadIdx.x;
    const bool point = l < L && state[l] == CVB_EXPORT_POINT;
    uint32_t tot;
    const uint32_t r = init_block_rank(point, s_warp, tot);
    if (!point) return;
    const size_t k = (size_t)block_off[blockIdx.x] + r;
    const double *h = points4 + 4 * (size_t)l;
    for (int c = 0; c < 3; c++) out_points[3 * k + c] = h[c] / h[3];
    const uint32_t o = lm_off[l], v = obs[2 * (size_t)o], f = obs[2 * (size_t)o + 1];
    const uint8_t *src = colors + 3 * ((size_t)view_off[v] + f);
    for (int c = 0; c < 3; c++) out_colors[3 * k + c] = src[c];
}
// one warp per view: the mean distance and the ExportCamera (lib.rs:2309-2333)
__global__ void __launch_bounds__(256) k_exp_cameras(uint32_t V, const cvb_pose *__restrict__ poses, const uint32_t *__restrict__ view_off,
                                                     const uint32_t *__restrict__ view_lm, const double *__restrict__ points,
                                                     const uint8_t *__restrict__ state, cvb_export_camera *__restrict__ cameras,
                                                     double *__restrict__ mean_distance) {
    const uint32_t v = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (v >= V) return;
    const cvb_pose P = poses[v];
    uint32_t n;
    const double mean = exp_view_mean(v, P, view_off, view_lm, points, state, n);
    if ((threadIdx.x & 31) != 0) return;
    cvb_pose c2w;
    pose_inverse(P, &c2w);
    const double origin[3] = {0.0, 0.0, 0.0}, down[3] = {-0.0, -1.0, -0.0}, z[3] = {0.0, 0.0, 1.0};
    cvb_export_camera c;
    double o[3];
    rotv(c2w.r, origin, o);
    for (int i = 0; i < 3; i++) c.optical_center[i] = o[i] + c2w.t[i];
    rotv(c2w.r, down, c.up_direction);
    rotv(c2w.r, z, c.forward_direction);
    c.focal_length = n ? mean * 0.01 : EXP_EMPTY_MEAN;
    cameras[v] = c;
    if (mean_distance) mean_distance[v] = mean;
}
// one warp: the first view's mean distance and whether it is normal (lib.rs:2248-2261)
__global__ void k_exp_first_mean(uint32_t first, const cvb_pose *__restrict__ poses, const uint32_t *__restrict__ view_off,
                                 const uint32_t *__restrict__ view_lm, const double *__restrict__ points, const uint8_t *__restrict__ state,
                                 cvb_normalize_result *__restrict__ res) {
    uint32_t n;
    const double mean = exp_view_mean(first, poses[first], view_off, view_lm, points, state, n);
    if (threadIdx.x != 0) return;
    cvb_normalize_result r;
    r.normalized = isfinite(mean) && fabs(mean) >= DBL_MIN;
    r.robust_points = n;
    r.mean_distance = mean;
    *res = r;
}
// lib.rs:2263-2282: every pose P_v * P_first^-1 with its translation scaled by 1 / mean, every constraint's translations scaled; the
// inputs copied when the mean is not normal.  Thread i handles view i and constraint i.
__global__ void __launch_bounds__(256) k_exp_normalize(uint32_t V, uint32_t C, uint32_t first, const cvb_pose *__restrict__ poses,
                                                       const cvb_view_constraint *__restrict__ cons, const cvb_normalize_result *__restrict__ res,
                                                       cvb_pose *__restrict__ poses_out, cvb_view_constraint *__restrict__ cons_out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool go = res->normalized != 0;
    const double s = 1.0 / res->mean_distance;
    if (i < V) {
        cvb_pose P = poses[i];
        if (go) {
            cvb_pose T;
            pose_inverse(poses[first], &T);
            con_pose_mul(poses[i], T, &P);
            for (int k = 0; k < 3; k++) P.t[k] = P.t[k] * s;
        }
        poses_out[i] = P;
    }
    if (i < C) {
        cvb_view_constraint c = cons[i];
        if (go)
            for (int x = 0; x < 2; x++)
                for (int k = 0; k < 3; k++) c.poses[x].t[k] = c.poses[x].t[k] * s;
        cons_out[i] = c;
    }
}
