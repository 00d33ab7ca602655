/* oracle/ref_register.c -- TEST INFRASTRUCTURE (CPU oracle), not product code.  The oracle of include/cvb200_register.h: cv-sfm's
 * register_frame / register_frame_subset (cv-sfm/src/lib.rs:1452-1812), restated loop for loop in the reference's order on the host
 * inputs of cvb_register_frame and with its outputs.  As the reference does, it runs one exact 3-NN per feature and view
 * (ref_hamming_knn), triangulates every match's robust point again wherever the reference asks for it, and re-triangulates every match in
 * every consistency pass.  Built on ref_arrsac (kind 1, P3P), ref_single_view_optimize_l2, ref_triangulate_observations and
 * ref_epipolar_loss.  The unpinned choices are the header's: exact k-NN with ties to the lower index, the best three landmarks by
 * (distance, landmark), observations in the caller's order.  Single-threaded. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "ref_triangulation.h"

void ref_hamming_knn(const uint8_t *q, uint32_t n, const uint8_t *db, uint32_t m, uint32_t k, uint32_t *idx_out, uint32_t *dist_out);

enum { OK = 0, FEW_ROBUST_LANDMARKS, NO_CONSENSUS, FILTER_HALF, FINAL_HALF, FINAL_ROBUST_HALF, FEW_MATCHES, PANIC };
#define NONE 0xffffffffu
#define STATS_ITERATIONS 16

typedef struct {   /* == cvb_register_cfg */
    double single_view_optimization_rate, maximum_sine_distance, maximum_cosine_distance,
        robust_observation_incidence_minimum_cosine_distance;
    uint32_t single_view_match_better_by, single_view_initial_features, single_view_minimum_landmarks,
        single_view_optimization_num_matches, single_view_filter_loop_iterations, single_view_patience,
        single_view_minimum_robust_landmarks, robust_minimum_observations;
} ref_register_cfg;
typedef struct { uint32_t feature, landmark_a, landmark_b; } ref_register_match;                                   /* == cvb_register_match */
typedef struct { int32_t status; uint32_t iteration, n_matches, n_inliers; ref_pose pose; } ref_register_result;   /* == cvb_register_result */
typedef struct {   /* == cvb_register_stats */
    uint32_t subsets, matches, claimed, matches_3d, inliers, final_robust, final_matches, iterations;
    uint32_t filter_matches[STATS_ITERATIONS];
    uint32_t final_stage_matches, reserved[3];
} ref_register_stats;

typedef struct { uint32_t a, b, f; } match;   /* ArrayVec<LandmarkKey, 2> (b = NONE: one landmark) and the feature */

typedef struct {
    const ref_register_cfg *cfg;
    const ref_triangulator *tri;
    uint32_t V, L;
    const ref_pose *poses;
    const uint32_t *vo, *vl;
    const double *bear;
    const uint8_t *desc;
    const uint32_t *lo, *obs;
    const uint8_t *new_desc;
    const double *new_bear;
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
    double sh[3];
    rotv(A->R, B->t, sh);
    for (int i = 0; i < 3; i++) r.t[i] = A->t[i] + sh[i];
    *o = r;
}
static void from_homogeneous(double *p) {   /* Projective::from_homogeneous (cv-core/src/point.rs:20-25) */
    if (signbit(p[3])) for (int i = 0; i < 4; i++) p[i] = -p[i];
    const double n = norm3(p);
    for (int i = 0; i < 4; i++) p[i] /= n;
}
/* 1 - pose.transform(point).bearing().dot(bearing) */
static double transformed_cosine_distance(const ref_pose *P, const double *point_h, const double *bearing) {
    double q[4];
    for (int r = 0; r < 3; r++) q[r] = dot3(P->R + 3 * r, point_h) + P->t[r] * point_h[3];
    q[3] = point_h[3];
    from_homogeneous(q);
    return 1.0 - dot3(q, bearing);
}

/* landmark_pose_bearings of the match's landmarks, a's first (lib.rs:340-354); returns the count; P, B hold one slot more */
static uint32_t pose_bearings(const snap *s, const match *m, ref_pose **P, double **B) {
    uint32_t n = s->lo[m->a + 1] - s->lo[m->a];
    if (m->b != NONE) n += s->lo[m->b + 1] - s->lo[m->b];
    *P = malloc(sizeof(ref_pose) * (n + 1));
    *B = malloc(sizeof(double) * 3 * (n + 1));
    uint32_t k = 0;
    for (int x = 0; x < 2; x++) {
        const uint32_t l = x ? m->b : m->a;
        if (l == NONE) break;
        for (uint32_t o = s->lo[l]; o < s->lo[l + 1]; o++, k++) {
            const uint32_t v = s->obs[2 * (size_t)o], f = s->obs[2 * (size_t)o + 1];
            (*P)[k] = s->poses[v];
            memcpy(*B + 3 * (size_t)k, s->bear + 3 * ((size_t)s->vo[v] + f), 24);
        }
    }
    return n;
}

/* triangulate_landmark_robust / triangulate_merged_landmark_robust (lib.rs:2907-3000): 1 and the WorldPoint in p when Some */
static int robust_point(const snap *s, const match *m, double *p) {
    ref_pose *P;
    double *B;
    const uint32_t n = pose_bearings(s, m, &P, &B);
    const uint32_t min_obs = s->cfg->robust_minimum_observations < s->V ? s->cfg->robust_minimum_observations : s->V;
    double *W = malloc(sizeof(double) * 3 * (n + 1));
    for (uint32_t i = 0; i < n; i++) {   /* pose.inverse().isometry() * bearing: the rotation only */
        ref_pose inv;
        pose_inverse(&P[i], &inv);
        rotv(inv.R, B + 3 * (size_t)i, W + 3 * (size_t)i);
    }
    int robust = 0;
    if (n >= min_obs)
        for (uint32_t i = 0; i < n && !robust; i++)
            for (uint32_t j = i + 1; j < n && !robust; j++)
                robust = 1.0 - dot3(W + 3 * (size_t)i, W + 3 * (size_t)j) > s->cfg->robust_observation_incidence_minimum_cosine_distance;
    const int ok = robust && ref_triangulate_observations(s->tri, P, B, (int)n, p, NULL);
    free(P); free(B); free(W);
    return ok;
}

/* is_observation_consistent (lib.rs:2622-2655) of the new (pose, bearing) against the match's landmarks' observations */
static int consistent(const snap *s, const ref_pose *pose, const match *m) {
    ref_pose *P;
    double *B;
    const uint32_t n = pose_bearings(s, m, &P, &B);
    const double *bearing = s->new_bear + 3 * (size_t)m->f;
    int ok;
    if (n == 1) {   /* is_bi_landmark_robust (lib.rs:1306-1318) of other_pose * pose^-1 */
        ref_pose inv, tot;
        double a[3];
        pose_inverse(pose, &inv);
        pose_mul(&P[0], &inv, &tot);
        rotv(tot.R, bearing, a);
        ok = ref_epipolar_loss(tot.t, a, B) < s->cfg->maximum_sine_distance;
    } else {
        P[n] = *pose;
        memcpy(B + 3 * (size_t)n, bearing, 24);
        double p[4];
        ok = ref_triangulate_observations(s->tri, P, B, (int)n + 1, p, NULL);
        for (uint32_t j = 0; ok && j <= n; j++) ok = transformed_cosine_distance(&P[j], p, B + 3 * (size_t)j) < s->cfg->maximum_cosine_distance;
    }
    free(P); free(B);
    return ok;
}

/* are_landmarks_sharing_view (lib.rs:1435-1449) */
static int sharing_view(const snap *s, uint32_t a, uint32_t b) {
    for (uint32_t i = s->lo[a]; i < s->lo[a + 1]; i++)
        for (uint32_t j = s->lo[b]; j < s->lo[b + 1]; j++)
            if (s->obs[2 * (size_t)i] == s->obs[2 * (size_t)j]) return 1;
    return 0;
}

static uint32_t obs_count(const snap *s, const match *m) {
    uint32_t c = s->lo[m->a + 1] - s->lo[m->a];
    if (m->b != NONE) c += s->lo[m->b + 1] - s->lo[m->b];
    return c;
}

/* matches_3d: (bearing, world point) of the matches (in order) that pass `keep` and have a robust point, up to cap */
static uint32_t build_3d(const snap *s, const match *list, uint32_t n, const ref_pose *pose, uint32_t cap, double *rb, double *rw) {
    uint32_t k = 0;
    for (uint32_t i = 0; i < n && k < cap; i++) {
        if (pose && !consistent(s, pose, &list[i])) continue;
        double p[4];
        if (!robust_point(s, &list[i], p)) continue;
        memcpy(rb + 3 * (size_t)k, s->new_bear + 3 * (size_t)list[i].f, 24);
        memcpy(rw + 4 * (size_t)k, p, 32);
        k++;
    }
    return k;
}

/* register_frame_subset (lib.rs:1452-1776); orig / n_orig: the accumulated original_matches */
static int subset(const snap *s, const uint32_t *view_matches, uint32_t H, uint32_t r0, uint32_t r1, match *orig, uint32_t *n_orig,
                  const ref_arrsac_cfg *ars, ref_rng *rng, ref_register_result *res, ref_register_match *out, uint32_t *inl_out,
                  ref_register_stats *st) {
    const ref_register_cfg *cfg = s->cfg;
    uint32_t idx[3], dist[3];
    uint32_t *cl = malloc(sizeof(uint32_t) * (3 * (size_t)H + 1)), *cd = malloc(sizeof(uint32_t) * (3 * (size_t)H + 1));
    for (uint32_t f = r0; f < r1; f++) {
        uint32_t nc = 0;   /* raw_landmark_matches, then the best distance per landmark */
        for (uint32_t h = 0; h < H; h++) {
            const uint32_t v = view_matches[h], m = s->vo[v + 1] - s->vo[v];
            ref_hamming_knn(s->new_desc + 64 * (size_t)f, 1, s->desc + 64 * (size_t)s->vo[v], m, 3, idx, dist);
            for (int k = 0; k < 3; k++) {
                if (idx[k] == NONE) continue;
                const uint32_t l = s->vl[s->vo[v] + idx[k]];
                uint32_t e = 0;
                while (e < nc && cl[e] != l) e++;
                if (e == nc) { cl[nc] = l; cd[nc] = dist[k]; nc++; }
                else if (cd[e] > dist[k]) cd[e] = dist[k];
            }
        }
        if (nc < 3) {   /* landmark_matches.next().unwrap() */
            free(cl); free(cd);
            res->status = PANIC;
            return PANIC;
        }
        uint32_t bl[3], bd[3];   /* the best three by (distance, landmark) */
        for (int t = 0; t < 3; t++) {
            uint32_t best = NONE;
            for (uint32_t e = 0; e < nc; e++) {
                int taken = 0;
                for (int u = 0; u < t; u++) taken |= bl[u] == cl[e];
                if (taken) continue;
                if (best == NONE || cd[e] < cd[best] || (cd[e] == cd[best] && cl[e] < cl[best])) best = e;
            }
            bl[t] = cl[best]; bd[t] = cd[best];
        }
        if (bd[0] + cfg->single_view_match_better_by <= bd[1]) {
            orig[(*n_orig)++] = (match){bl[0], NONE, f};
        } else if (bd[1] + cfg->single_view_match_better_by <= bd[2]) {
            if (!sharing_view(s, bl[0], bl[1])) orig[(*n_orig)++] = (match){bl[0], bl[1], f};
        }
    }
    free(cl); free(cd);
    st->matches = *n_orig;
    /* the claim filter and the stable sort by descending summed observation count (lib.rs:1551-1576) */
    uint32_t *counts = calloc(s->L ? s->L : 1, sizeof(uint32_t));
    for (uint32_t i = 0; i < *n_orig; i++) {
        counts[orig[i].a]++;
        if (orig[i].b != NONE) counts[orig[i].b]++;
    }
    match *list = malloc(sizeof(match) * (*n_orig ? *n_orig : 1));
    uint32_t n = 0;
    for (uint32_t i = 0; i < *n_orig; i++)
        if (counts[orig[i].a] == 1 && (orig[i].b == NONE || counts[orig[i].b] == 1)) list[n++] = orig[i];
    free(counts);
    for (uint32_t i = 1; i < n; i++) {   /* insertion sort: stable */
        const match x = list[i];
        const uint32_t c = obs_count(s, &x);
        uint32_t j = i;
        while (j > 0 && obs_count(s, &list[j - 1]) < c) { list[j] = list[j - 1]; j--; }
        list[j] = x;
    }
    st->claimed = n;
    double *mb = malloc(sizeof(double) * 3 * (n ? n : 1)), *mw = malloc(sizeof(double) * 4 * (n ? n : 1));
    double *rb = malloc(sizeof(double) * 3 * (n ? n : 1)), *rw = malloc(sizeof(double) * 4 * (n ? n : 1));
    uint32_t *inl = malloc(sizeof(uint32_t) * (n ? n : 1));
    int status = OK;
    ref_pose pose;
    const uint32_t n3d = build_3d(s, list, n, NULL, NONE, mb, mw);
    st->matches_3d = n3d;
    uint32_t ninl = 0, len = 0, robust_min = 0;
    if (n3d < cfg->single_view_minimum_landmarks) { status = FEW_ROBUST_LANDMARKS; goto done; }
    if (!ref_arrsac(ars, 1, mb, mw, n3d, rng, &pose, inl, &ninl)) { status = NO_CONSENSUS; goto done; }
    st->inliers = ninl;
    res->n_inliers = ninl;
    if (inl_out) memcpy(inl_out, inl, sizeof(uint32_t) * ninl);
    len = ninl < cfg->single_view_optimization_num_matches ? ninl : cfg->single_view_optimization_num_matches;
    for (uint32_t k = 0; k < len; k++) {
        memcpy(rb + 3 * (size_t)k, mb + 3 * (size_t)inl[k], 24);
        memcpy(rw + 4 * (size_t)k, mw + 4 * (size_t)inl[k], 32);
    }
    robust_min = len / 2;
    for (uint32_t it = 0; it < cfg->single_view_filter_loop_iterations; it++) {
        if (it < STATS_ITERATIONS) st->filter_matches[it] = len;
        st->iterations = it + 1;
        if (len <= robust_min) { status = FILTER_HALF; res->iteration = it; goto done; }
        ref_single_view_optimize_l2(&pose, cfg->single_view_optimization_rate, cfg->single_view_patience, rb, rw, len);
        len = build_3d(s, list, n, &pose, cfg->single_view_optimization_num_matches, rb, rw);
    }
    st->final_stage_matches = len;
    if (len <= robust_min) { status = FINAL_HALF; goto done; }
    ref_single_view_optimize_l2(&pose, cfg->single_view_optimization_rate, cfg->single_view_patience, rb, rw, len);
    uint32_t final_robust = 0;
    for (uint32_t i = 0; i < n; i++) {
        double p[4];
        if (consistent(s, &pose, &list[i]) && robust_point(s, &list[i], p)) final_robust++;
    }
    st->final_robust = final_robust;
    if (final_robust <= robust_min) { status = FINAL_ROBUST_HALF; goto done; }
    uint32_t nm = 0;
    for (uint32_t i = 0; i < n; i++)
        if (consistent(s, &pose, &list[i])) out[nm++] = (ref_register_match){list[i].f, list[i].a, list[i].b};
    for (uint32_t i = 1; i < nm; i++) {   /* the HashMap, listed ascending by feature */
        const ref_register_match x = out[i];
        uint32_t j = i;
        while (j > 0 && out[j - 1].feature > x.feature) { out[j] = out[j - 1]; j--; }
        out[j] = x;
    }
    st->final_matches = nm;
    if (nm < cfg->single_view_minimum_robust_landmarks) { status = FEW_MATCHES; goto done; }
    res->n_matches = nm;
    res->pose = pose;
done:
    free(list); free(mb); free(mw); free(rb); free(rw); free(inl);
    res->status = status;
    return status;
}

/* register_frame (lib.rs:1781-1812) */
int ref_register_frame(const ref_register_cfg *cfg, const ref_triangulator *tri, const ref_arrsac_cfg *ars, ref_rng *rng, uint32_t V,
                       const ref_pose *poses, const uint32_t *vo, const uint32_t *vl, const double *bear, const uint8_t *desc, uint32_t L,
                       const uint32_t *lo, const uint32_t *obs, const uint8_t *new_desc, const double *new_bear, uint32_t N,
                       const uint32_t *view_matches, uint32_t H, ref_register_result *res, ref_register_match *out, uint32_t *inliers,
                       ref_register_stats *stats) {
    if (N && cfg->single_view_initial_features == 0) return 1;   /* the subset range would stay empty forever */
    const snap s = {cfg, tri, V, L, poses, vo, vl, bear, desc, lo, obs, new_desc, new_bear};
    match *orig = malloc(sizeof(match) * (N ? N : 1));
    uint32_t n_orig = 0, r0 = 0, r1 = cfg->single_view_initial_features < N ? cfg->single_view_initial_features : N, subsets = 0;
    ref_register_stats st;
    for (;;) {
        memset(res, 0, sizeof(*res));
        memset(&st, 0, sizeof(st));
        st.subsets = ++subsets;
        const int status = subset(&s, view_matches, H, r0, r1, orig, &n_orig, ars, rng, res, out, inliers, &st);
        if (status == OK || status == PANIC || r1 == N) break;
        r0 = r1;
        r1 = 2 * (uint64_t)r1 < N ? 2 * r1 : N;
    }
    if (stats) *stats = st;
    free(orig);
    return 0;
}
