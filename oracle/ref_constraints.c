/* oracle/ref_constraints.c -- TEST INFRASTRUCTURE (CPU oracle), not product code.  The oracle of include/cvb200_constraints.h: cv-sfm's
 * generate_view_constraints (cv-sfm/src/lib.rs:2438-2516) and record_view_constraints' acceptance (lib.rs:2092-2109), restated one query
 * at a time, sequentially, on the host inputs of cvb_view_constraints and with its outputs.  Built on ref_triangulate_observations
 * (ref_triangulation.c) and ref_three_view_optimize_l2 (ref_optimize.c, adaptive, sums in landmark order).  The orders the reference
 * leaves undefined are fixed as the header says: coviews ascending, stable sorts, no shuffle, observations in the caller's order. */
#include <math.h>
#include <omp.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "ref_triangulation.h"

uint32_t ref_three_view_optimize_l2(ref_pose poses[2], int adaptive, double rate, uint32_t iterations, const double *obs, uint32_t n);

typedef struct {   /* == cvb_constraints_cfg */
    double robust_observation_incidence_minimum_cosine_distance, robust_view_bearing_pair_minimum_cosine_distance;
    uint32_t robust_minimum_observations, robust_view_num_robust_bearing_pair, optimization_robust_covisibility_minimum_landmarks,
        optimization_minimum_landmarks, optimization_maximum_landmarks, optimization_maximum_three_view_constraints,
        optimization_minimum_new_constraints, constraint_patience;
} ref_constraints_cfg;
typedef struct { uint32_t views[3], landmarks; ref_pose poses[2]; } ref_view_constraint;        /* == cvb_view_constraint */
typedef struct { uint32_t n_constraints; int32_t accepted; } ref_view_constraints_result;      /* == cvb_view_constraints_result */
typedef struct {                                                                               /* == cvb_view_constraints_stats */
    uint32_t robust_landmarks, coviews, triples, unique_triples, candidates, few_landmarks, few_bearing_pairs, updates;
} ref_view_constraints_stats;

static double dot3(const double *a, const double *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
static double norm3(const double *a) { return sqrt(dot3(a, a)); }
static void pose_inverse(const ref_pose *P, ref_pose *o) {
    double nt[3] = {-P->t[0], -P->t[1], -P->t[2]}, R[9];
    for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) R[3 * r + c] = P->R[3 * c + r];
    for (int r = 0; r < 3; r++) o->t[r] = dot3(R + 3 * r, nt);
    memcpy(o->R, R, 72);
}
static void pose_mul(const ref_pose *A, const ref_pose *B, ref_pose *o) {   /* A * B */
    for (int i = 0; i < 3; i++)
        for (int c = 0; c < 3; c++) o->R[3 * i + c] = A->R[3 * i] * B->R[c] + A->R[3 * i + 1] * B->R[3 + c] + A->R[3 * i + 2] * B->R[6 + c];
    for (int i = 0; i < 3; i++) o->t[i] = A->t[i] + dot3(A->R + 3 * i, B->t);
}
static int cmp_u64(const void *x, const void *y) { const uint64_t a = *(const uint64_t *)x, b = *(const uint64_t *)y; return (a > b) - (a < b); }

typedef struct {
    uint32_t V, L;
    const ref_pose *poses;
    const uint32_t *vo, *vl, *lo, *obs;
    const double *bear;
} snap;
static const double *bearing(const snap *S, uint32_t v, uint32_t f) { return S->bear + 3 * ((size_t)S->vo[v] + f); }
static uint32_t feature_of(const snap *S, uint32_t l, uint32_t v) {
    for (uint32_t o = S->lo[l]; o < S->lo[l + 1]; o++) if (S->obs[2 * o] == v) return S->obs[2 * o + 1];
    return 0xffffffffu;
}
static int observes(const snap *S, uint32_t l, uint32_t v) { return feature_of(S, l, v) != 0xffffffffu; }

/* lib.rs:2907-2934, 2975-3000 */
static int landmark_robust(const snap *S, const ref_constraints_cfg *cfg, const ref_triangulator *tri, uint32_t l) {
    const uint32_t o0 = S->lo[l], n = S->lo[l + 1] - o0, mn = cfg->robust_minimum_observations < S->V ? cfg->robust_minimum_observations : S->V;
    if (n < mn) return 0;
    double *w = malloc(sizeof(double) * 3 * (n ? n : 1)), *B = malloc(sizeof(double) * 3 * (n ? n : 1));
    ref_pose *P = malloc(sizeof(ref_pose) * (n ? n : 1));
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t v = S->obs[2 * (o0 + i)], f = S->obs[2 * (o0 + i) + 1];
        const ref_pose *Q = &S->poses[v];
        const double *b = bearing(S, v, f);
        P[i] = *Q;
        memcpy(B + 3 * i, b, 24);
        for (int r = 0; r < 3; r++) w[3 * i + r] = Q->R[r] * b[0] + Q->R[3 + r] * b[1] + Q->R[6 + r] * b[2];
    }
    int inc = 0;
    for (uint32_t i = 0; i < n && !inc; i++)
        for (uint32_t j = i + 1; j < n && !inc; j++) inc = 1.0 - dot3(w + 3 * i, w + 3 * j) > cfg->robust_observation_incidence_minimum_cosine_distance;
    int ok = 0;
    if (inc) { double p[4]; ok = ref_triangulate_observations(tri, P, B, (int)n, p, NULL); }
    free(w); free(B); free(P);
    return ok;
}

static void sort3(uint32_t *v) {
    for (int x = 0; x < 2; x++)
        for (int y = 0; y < 2 - x; y++)
            if (v[y] > v[y + 1]) { const uint32_t s = v[y]; v[y] = v[y + 1]; v[y + 1] = s; }
}

static void one_query(const snap *S, const ref_constraints_cfg *cfg, const uint8_t *robust, uint32_t q, ref_view_constraint *out,
                      ref_view_constraints_result *res, ref_view_constraints_stats *st) {
    const uint32_t V = S->V, maxc = cfg->optimization_maximum_three_view_constraints, cmin = cfg->optimization_robust_covisibility_minimum_landmarks;
    memset(st, 0, sizeof(*st));
    /* view_covisibilities: per coview, q's robust landmarks it observes, in q's feature order (as positions in q's robust list) */
    const uint32_t nf = S->vo[q + 1] - S->vo[q];
    uint32_t *rl = malloc(sizeof(uint32_t) * (nf ? nf : 1)), R = 0;
    for (uint32_t j = 0; j < nf; j++) { const uint32_t l = S->vl[S->vo[q] + j]; if (robust[l]) rl[R++] = l; }
    uint32_t *cnt = calloc(V, sizeof(uint32_t)), *kept = malloc(sizeof(uint32_t) * V), K = 0;
    for (uint32_t i = 0; i < R; i++)
        for (uint32_t o = S->lo[rl[i]]; o < S->lo[rl[i] + 1]; o++) if (S->obs[2 * o] != q) cnt[S->obs[2 * o]]++;
    for (uint32_t v = 0; v < V; v++) if (cnt[v] > 0 && cnt[v] >= cmin) kept[K++] = v;
    /* triples in combination order, then sorted by descending count (ties: combination order) */
    const uint64_t P = (uint64_t)K * (K - (K > 0)) / 2;
    uint64_t *keys = malloc(sizeof(uint64_t) * (P ? P : 1));
    uint32_t *pa = malloc(sizeof(uint32_t) * (P ? P : 1)), *pb = malloc(sizeof(uint32_t) * (P ? P : 1)), *pc = malloc(sizeof(uint32_t) * (P ? P : 1));
    uint32_t T = 0, p = 0;
    for (uint32_t a = 0; a < K; a++)
        for (uint32_t b = a + 1; b < K; b++, p++) {
            uint32_t c = 0;
            for (uint32_t i = 0; i < R; i++) c += observes(S, rl[i], kept[a]) && observes(S, rl[i], kept[b]);
            pa[p] = a; pb[p] = b; pc[p] = c;
            if (c >= cmin) keys[T++] = ((uint64_t)(0xffffffffu - c) << 32) | p;
        }
    qsort(keys, T, sizeof(uint64_t), cmp_u64);
    /* the unique pass (any() short-circuits; the pass stops at the take limit), then the rest in sorted order */
    uint8_t *vis = calloc(V, 1), *uniq = calloc(T ? T : 1, 1);
    uint32_t *ord = malloc(sizeof(uint32_t) * (T ? T : 1)), U = 0;
    for (uint32_t t = 0; t < T && U < maxc; t++) {
        const uint32_t pp = (uint32_t)keys[t];
        uint32_t v[3] = {q, kept[pa[pp]], kept[pb[pp]]};
        sort3(v);
        for (int x = 0; x < 3; x++)
            if (!vis[v[x]]) { vis[v[x]] = 1; uniq[t] = 1; ord[U++] = t; break; }
    }
    uint32_t n = U;
    for (uint32_t t = 0; t < T; t++) if (!uniq[t]) ord[n++] = t;
    st->robust_landmarks = R; st->coviews = K; st->triples = T; st->unique_triples = U;
    /* optimize_three_view over that order until maxc succeed */
    const uint32_t omax = cfg->optimization_maximum_landmarks;
    uint64_t *lk = malloc(sizeof(uint64_t) * (R ? R : 1));
    double *rows = malloc(sizeof(double) * 9 * (omax ? omax : 1));
    uint32_t ns = 0;
    for (uint32_t t = 0; t < T && ns < maxc; t++) {
        const uint32_t pp = (uint32_t)keys[ord[t]], c = pc[pp];
        st->candidates++;
        if (c < cfg->optimization_minimum_landmarks) { st->few_landmarks++; continue; }
        const uint32_t a = kept[pa[pp]], b = kept[pb[pp]];
        uint32_t m = 0;
        for (uint32_t i = 0; i < R; i++)
            if (observes(S, rl[i], a) && observes(S, rl[i], b))
                lk[m++] = ((uint64_t)(0xffffffffu - (S->lo[rl[i] + 1] - S->lo[rl[i]])) << 32) | i;
        qsort(lk, m, sizeof(uint64_t), cmp_u64);
        if (m > omax) m = omax;
        uint32_t v[3] = {q, a, b};
        sort3(v);
        for (uint32_t i = 0; i < m; i++) {
            const uint32_t l = rl[(uint32_t)lk[i]];
            for (int x = 0; x < 3; x++) memcpy(rows + 9 * i + 3 * x, bearing(S, v[x], feature_of(S, l, v[x])), 24);
        }
        uint64_t bp = 0;
        const double mc = cfg->robust_view_bearing_pair_minimum_cosine_distance;
        for (uint32_t i = 0; i < m; i++)
            for (uint32_t j = i + 1; j < m; j++) {
                const double *x = rows + 9 * i, *y = rows + 9 * j;
                bp += 1.0 - dot3(x, y) > mc && 1.0 - dot3(x + 3, y + 3) > mc && 1.0 - dot3(x + 6, y + 6) > mc;
            }
        if (bp < cfg->robust_view_num_robust_bearing_pair) { st->few_bearing_pairs++; continue; }
        ref_pose inv0, pz[2];
        pose_inverse(&S->poses[v[0]], &inv0);
        pose_mul(&S->poses[v[1]], &inv0, &pz[0]);
        pose_mul(&S->poses[v[2]], &inv0, &pz[1]);
        const double scale = norm3(pz[0].t) + norm3(pz[1].t);
        st->updates += ref_three_view_optimize_l2(pz, 1, 0.0, cfg->constraint_patience, rows, m);
        const double rel = scale / (norm3(pz[0].t) + norm3(pz[1].t));
        for (int k = 0; k < 3; k++) { pz[0].t[k] = pz[0].t[k] * rel; pz[1].t[k] = pz[1].t[k] * rel; }
        ref_view_constraint *C = &out[ns++];
        memcpy(C->views, v, sizeof(v));
        C->landmarks = m;
        C->poses[0] = pz[0];
        C->poses[1] = pz[1];
    }
    res->n_constraints = ns;
    res->accepted = !(ns < cfg->optimization_minimum_new_constraints && ns + 1 < V);
    free(rl); free(cnt); free(kept); free(keys); free(pa); free(pb); free(pc); free(vis); free(uniq); free(ord); free(lk); free(rows);
}

/* the layout of cvb_view_constraints (host arrays, already validated); out: Q x optimization_maximum_three_view_constraints.  Queries run
 * on `threads` OpenMP threads (0: OpenMP's default); each is sequential. */
int ref_view_constraints(const ref_constraints_cfg *cfg, const ref_triangulator *tri, uint32_t V, const ref_pose *poses, const uint32_t *vo,
                         const uint32_t *vl, const double *bear, uint32_t L, const uint32_t *lo, const uint32_t *obs, const uint32_t *queries,
                         uint32_t Q, ref_view_constraint *out, ref_view_constraints_result *res, ref_view_constraints_stats *stats,
                         int threads) {
    if (tri->method < REF_TRI_LINEAR_EIGEN || tri->method > REF_TRI_MEAN_MEAN) return -1;
    const snap S = {V, L, poses, vo, vl, lo, obs, bear};
    uint8_t *robust = malloc(L ? L : 1);
    const int nt = threads > 0 ? threads : omp_get_max_threads();
#pragma omp parallel for schedule(dynamic) num_threads(nt)
    for (uint32_t l = 0; l < L; l++) robust[l] = (uint8_t)landmark_robust(&S, cfg, tri, l);
#pragma omp parallel for schedule(dynamic) num_threads(nt)
    for (uint32_t i = 0; i < Q; i++) {
        ref_view_constraints_stats st;
        one_query(&S, cfg, robust, queries[i], out + (size_t)i * cfg->optimization_maximum_three_view_constraints, &res[i], &st);
        if (stats) stats[i] = st;
    }
    free(robust);
    return 0;
}
