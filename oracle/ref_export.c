/* oracle/ref_export.c -- TEST INFRASTRUCTURE (CPU oracle), not product code.  The oracle of include/cvb200_export.h: cv-sfm's
 * triangulate_landmark_robust (cv-sfm/src/lib.rs:2907-2934, 2975-3000), export_reconstruction without the file (lib.rs:2285-2340) and
 * normalize_reconstruction (lib.rs:2241-2283), restated loop for loop in the reference's order on the host inputs of the entry points and
 * with their outputs.  As the reference does, every view's mean distance triangulates each of its landmarks again.  Built on
 * ref_triangulate_observations (ref_triangulation.c).  Landmarks, and views, are independent, so OpenMP spreads them over threads; every
 * running mean keeps its order.  average's Mean and nalgebra's operations are restated as the header states them. */
#include <math.h>
#include <omp.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "ref_triangulation.h"

enum { POINT = 0, NOT_ROBUST = 1, TRI_FAILED = 2, AT_INFINITY = 3 };

typedef struct {   /* == cvb_export_cfg */
    double robust_observation_incidence_minimum_cosine_distance;
    uint32_t robust_minimum_observations;
} ref_export_cfg;
typedef struct { double optical_center[3], up_direction[3], forward_direction[3], focal_length; } ref_export_camera;   /* == cvb_export_camera */
typedef struct { int32_t normalized; uint32_t robust_points; double mean_distance; } ref_normalize_result;   /* == cvb_normalize_result */
typedef struct { uint32_t views[3], landmarks; ref_pose poses[2]; } ref_view_constraint;                      /* == cvb_view_constraint */

/* the snapshot every function reads */
typedef struct {
    const ref_export_cfg *cfg;
    const ref_triangulator *tri;
    uint32_t V;
    const ref_pose *poses;
    const uint32_t *vo, *vl;
    const double *bear;
    const uint32_t *lo, *obs;
} snap;

static double dot3(const double *a, const double *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
static double norm3(const double *a) { return sqrt(dot3(a, a)); }
static void rotv(const double *R, const double *v, double *o) { for (int r = 0; r < 3; r++) o[r] = dot3(R + 3 * r, v); }
static void pose_inverse(const ref_pose *P, ref_pose *o) {
    double nt[3] = {-P->t[0], -P->t[1], -P->t[2]}, R[9];
    for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) R[3 * r + c] = P->R[3 * c + r];
    rotv(R, nt, o->t);
    memcpy(o->R, R, 72);
}
static void pose_mul(const ref_pose *A, const ref_pose *B, ref_pose *o) {   /* A * B */
    ref_pose r;
    for (int i = 0; i < 3; i++)
        for (int c = 0; c < 3; c++) r.R[3 * i + c] = A->R[3 * i] * B->R[c] + A->R[3 * i + 1] * B->R[3 + c] + A->R[3 * i + 2] * B->R[6 + c];
    for (int i = 0; i < 3; i++) r.t[i] = A->t[i] + dot3(A->R + 3 * i, B->t);
    *o = r;
}

/* triangulate_landmark_robust: the state, and the WorldPoint in p when it is Some */
static int robust_landmark(const snap *s, uint32_t l, double *p) {
    const uint32_t o0 = s->lo[l], n = s->lo[l + 1] - o0;
    const uint32_t min_obs = s->cfg->robust_minimum_observations < s->V ? s->cfg->robust_minimum_observations : s->V;
    ref_pose *P = malloc(sizeof(ref_pose) * (n ? n : 1));
    double *B = malloc(sizeof(double) * 3 * (n ? n : 1)), *W = malloc(sizeof(double) * 3 * (n ? n : 1));
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t v = s->obs[2 * (size_t)(o0 + i)], f = s->obs[2 * (size_t)(o0 + i) + 1];
        P[i] = s->poses[v];
        memcpy(B + 3 * (size_t)i, s->bear + 3 * ((size_t)s->vo[v] + f), 24);
        ref_pose inv;   /* pose.inverse().isometry() * bearing: the rotation only */
        pose_inverse(&P[i], &inv);
        rotv(inv.R, B + 3 * (size_t)i, W + 3 * (size_t)i);
    }
    int robust = 0;   /* are_observations_robust: the count, then any pair in tuple_combinations order */
    if (n >= min_obs)
        for (uint32_t i = 0; i < n && !robust; i++)
            for (uint32_t j = i + 1; j < n && !robust; j++)
                robust = 1.0 - dot3(W + 3 * (size_t)i, W + 3 * (size_t)j) > s->cfg->robust_observation_incidence_minimum_cosine_distance;
    int state = NOT_ROBUST;
    if (robust) state = !ref_triangulate_observations(s->tri, P, B, (int)n, p, NULL) ? TRI_FAILED : (p[3] == 0.0 ? AT_INFINITY : POINT);
    free(P); free(B); free(W);
    return state;
}

/* the Mean of v.landmarks' robust points' distances (lib.rs:2250-2257, 2315-2324), each landmark triangulated again */
static double view_mean(const snap *s, uint32_t v, uint32_t *count) {
    const ref_pose *P = &s->poses[v];
    double avg = 0.0;
    uint32_t n = 0;
    for (uint32_t j = s->vo[v]; j < s->vo[v + 1]; j++) {
        double h[4];
        const int st = robust_landmark(s, s->vl[j], h);
        if (st != POINT && st != AT_INFINITY) continue;
        /* pose.transform(wp): to_homogeneous() * h, then Projective::from_homogeneous */
        double q[4];
        for (int r = 0; r < 3; r++) q[r] = ((P->R[3 * r] * h[0] + P->R[3 * r + 1] * h[1]) + P->R[3 * r + 2] * h[2]) + P->t[r] * h[3];
        q[3] = ((0.0 * h[0] + 0.0 * h[1]) + 0.0 * h[2]) + 1.0 * h[3];
        if (signbit(q[3])) for (int i = 0; i < 4; i++) q[i] = -q[i];
        const double nq = norm3(q);
        for (int i = 0; i < 4; i++) q[i] /= nq;
        /* .point()?: Point3::from_homogeneous, then coords.norm() */
        if (q[3] == 0.0) continue;
        const double x[3] = {q[0] / q[3], q[1] / q[3], q[2] / q[3]};
        const double d = norm3(x);
        n++;   /* Mean::add */
        avg += (d - avg) / (double)n;
    }
    *count = n;
    if (n) return avg;
    const uint64_t nan_bits = 0x7ff8000000000000ull;   /* f64::NAN */
    double nan;
    memcpy(&nan, &nan_bits, 8);
    return nan;
}

int ref_robust_landmarks(const ref_export_cfg *cfg, const ref_triangulator *tri, uint32_t V, const ref_pose *poses, const uint32_t *vo,
                         const uint32_t *vl, const double *bear, uint32_t L, const uint32_t *lo, const uint32_t *obs, double *points,
                         uint8_t *state, int threads) {
    if (threads > 0) omp_set_num_threads(threads);
    const snap s = {cfg, tri, V, poses, vo, vl, bear, lo, obs};
#pragma omp parallel for schedule(dynamic, 64)
    for (uint32_t l = 0; l < L; l++) {
        double p[4] = {0.0, 0.0, 0.0, 0.0};
        const int st = robust_landmark(&s, l, p);
        if (st == NOT_ROBUST || st == TRI_FAILED) p[0] = p[1] = p[2] = p[3] = 0.0;
        memcpy(points + 4 * (size_t)l, p, 32);
        state[l] = (uint8_t)st;
    }
    return 0;
}

int ref_export_reconstruction(const ref_export_cfg *cfg, const ref_triangulator *tri, uint32_t V, const ref_pose *poses, const uint32_t *vo,
                              const uint32_t *vl, const double *bear, const uint8_t *colors, uint32_t L, const uint32_t *lo,
                              const uint32_t *obs, double *points, uint8_t *point_colors, uint32_t *n_points, ref_export_camera *cameras,
                              double *mean_distance, int threads) {
    if (threads > 0) omp_set_num_threads(threads);
    const snap s = {cfg, tri, V, poses, vo, vl, bear, lo, obs};
    /* the point cloud: triangulate_landmark_robust(..).and_then(Projective::point), with the first observation's colour */
    double *h = malloc(sizeof(double) * 4 * (L ? L : 1));
    uint8_t *st = malloc(L ? L : 1);
#pragma omp parallel for schedule(dynamic, 64)
    for (uint32_t l = 0; l < L; l++) st[l] = (uint8_t)robust_landmark(&s, l, h + 4 * (size_t)l);
    uint32_t k = 0;
    for (uint32_t l = 0; l < L; l++) {
        if (st[l] != POINT) continue;
        const double *p = h + 4 * (size_t)l;
        for (int c = 0; c < 3; c++) points[3 * (size_t)k + c] = p[c] / p[3];
        const uint32_t v = obs[2 * (size_t)lo[l]], f = obs[2 * (size_t)lo[l] + 1];
        memcpy(point_colors + 3 * (size_t)k, colors + 3 * ((size_t)vo[v] + f), 3);
        k++;
    }
    *n_points = k;
    free(h); free(st);
    /* the cameras */
#pragma omp parallel for schedule(dynamic, 1)
    for (uint32_t v = 0; v < V; v++) {
        uint32_t n;
        const double mean = view_mean(&s, v, &n);
        ref_pose c2w;
        pose_inverse(&poses[v], &c2w);
        const double origin[3] = {0.0, 0.0, 0.0}, down[3] = {-0.0, -1.0, -0.0}, z[3] = {0.0, 0.0, 1.0};
        ref_export_camera c;
        double o[3];
        rotv(c2w.R, origin, o);
        for (int i = 0; i < 3; i++) c.optical_center[i] = o[i] + c2w.t[i];
        rotv(c2w.R, down, c.up_direction);
        rotv(c2w.R, z, c.forward_direction);
        c.focal_length = mean * 0.01;
        cameras[v] = c;
        if (mean_distance) mean_distance[v] = mean;
    }
    return 0;
}

int ref_normalize_reconstruction(const ref_export_cfg *cfg, const ref_triangulator *tri, uint32_t V, const ref_pose *poses, const uint32_t *vo,
                                 const uint32_t *vl, const double *bear, uint32_t L, const uint32_t *lo, const uint32_t *obs,
                                 const ref_view_constraint *cons, uint32_t C, uint32_t first, ref_pose *poses_out,
                                 ref_view_constraint *cons_out, ref_normalize_result *res) {
    (void)L;
    const snap s = {cfg, tri, V, poses, vo, vl, bear, lo, obs};
    uint32_t n;
    const double mean = view_mean(&s, first, &n);
    res->normalized = isnormal(mean) ? 1 : 0;
    res->robust_points = n;
    res->mean_distance = mean;
    memcpy(poses_out, poses, sizeof(ref_pose) * V);
    if (C) memcpy(cons_out, cons, sizeof(ref_view_constraint) * C);
    if (!res->normalized) return 0;
    const double rescale = 1.0 / mean;
    ref_pose T;
    pose_inverse(&poses[first], &T);
    for (uint32_t v = 0; v < V; v++) {
        pose_mul(&poses[v], &T, &poses_out[v]);
        for (int i = 0; i < 3; i++) poses_out[v].t[i] *= rescale;
    }
    for (uint32_t c = 0; c < C; c++)
        for (int k = 0; k < 2; k++)
            for (int i = 0; i < 3; i++) cons_out[c].poses[k].t[i] *= rescale;
    return 0;
}
