/* oracle/ref_reconstruction.c -- TEST INFRASTRUCTURE (CPU oracle), not product code.  The oracle of include/cvb200_reconstruction.h:
 * cv-sfm's optimize_reconstruction (cv-sfm/src/lib.rs:2343-2355) -- apply_constraints (lib.rs:2358-2414) with constrain_view
 * (:1892-1936), flatten_constraints (:2519-2532) and edge_constraints (:167-180), then filter_non_robust_observations (:2657-2757) --
 * restated step by step in the reference's order on the host inputs of cvb_optimize_reconstruction and with its outputs.  Built on
 * ref_triangulate_observations (ref_triangulation.c) and ref_epipolar_loss (ref_optimize.c).  Views of one step are independent (each
 * reads the previous step's poses), so OpenMP spreads them, and the landmarks of one filter, over threads; every sum keeps its order.
 * nalgebra 0.30.1's scaled_axis, from_axis_angle and from_matrix are restated as the header states them. */
#include <float.h>
#include <math.h>
#include <omp.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "ref_triangulation.h"

double ref_epipolar_loss(const double *t, const double *a, const double *b);

#define FROM_MATRIX_MAX_ITERATIONS 64   /* == CVB_RECON_FROM_MATRIX_MAX_ITERATIONS */
enum { RUNNING = -1, KEPT = 0, REMOVED_CONSTRAINTS = 1, REMOVED_FILTER = 2, PANIC = 3 };
enum { VIEW_KEPT = 0, VIEW_NO_EDGES = 1, VIEW_NON_FINITE = 2 };
enum { OBS_KEPT = 0, OBS_SPLIT = 1, OBS_DROPPED = 2 };

typedef struct {   /* == cvb_recon_cfg */
    double graph_optimization_rate, maximum_sine_distance, maximum_cosine_distance, robust_observation_incidence_minimum_cosine_distance;
    uint32_t optimization_iterations, reconstruction_optimization_iterations, robust_minimum_observations, minimum_robust_landmarks;
} ref_recon_cfg;
typedef struct { uint32_t views[3], landmarks; ref_pose poses[2]; } ref_view_constraint;   /* == cvb_view_constraint */
typedef struct {                                                                           /* == cvb_recon_result */
    int32_t status;
    uint32_t round, step, views_removed, robust_before, robust_after, observations_split, small_angle_updates;
} ref_recon_result;

static double dot3(const double *a, const double *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
static double norm3(const double *a) { return sqrt(dot3(a, a)); }
static void cross3(const double *a, const double *b, double *o) {
    const double r0 = a[1] * b[2] - a[2] * b[1], r1 = a[2] * b[0] - a[0] * b[2], r2 = a[0] * b[1] - a[1] * b[0];
    o[0] = r0; o[1] = r1; o[2] = r2;
}
static void pose_inverse(const ref_pose *P, ref_pose *o) {
    double nt[3] = {-P->t[0], -P->t[1], -P->t[2]}, R[9];
    for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) R[3 * r + c] = P->R[3 * c + r];
    for (int r = 0; r < 3; r++) o->t[r] = dot3(R + 3 * r, nt);
    memcpy(o->R, R, 72);
}
static void pose_mul(const ref_pose *A, const ref_pose *B, ref_pose *o) {   /* A * B */
    ref_pose r;
    for (int i = 0; i < 3; i++)
        for (int c = 0; c < 3; c++) r.R[3 * i + c] = A->R[3 * i] * B->R[c] + A->R[3 * i + 1] * B->R[3 + c] + A->R[3 * i + 2] * B->R[6 + c];
    for (int i = 0; i < 3; i++) r.t[i] = A->t[i] + dot3(A->R + 3 * i, B->t);
    *o = r;
}
/* Projective::from_homogeneous (cv-core/src/point.rs:20-25) */
static void from_homogeneous(double *p) {
    if (signbit(p[3])) for (int i = 0; i < 4; i++) p[i] = -p[i];
    double n = norm3(p);
    for (int i = 0; i < 4; i++) p[i] /= n;
}
/* 1 - pose.transform(point).bearing() . bearing */
static double transformed_cosine_distance(const ref_pose *P, const double *point_h, const double *bearing) {
    double q[4];
    for (int r = 0; r < 3; r++) q[r] = dot3(P->R + 3 * r, point_h) + P->t[r] * point_h[3];
    q[3] = point_h[3];
    from_homogeneous(q);
    return 1.0 - dot3(q, bearing);
}
/* nalgebra from_axis_angle(v / |v|, |v|) (Rotation3::from_scaled_axis) */
static void rot_from_scaled_axis(const double *v, double *R) {
    const double angle = norm3(v);
    if (angle == 0.0) { memset(R, 0, 72); R[0] = R[4] = R[8] = 1.0; return; }
    const double ux = v[0] / angle, uy = v[1] / angle, uz = v[2] / angle;
    const double sqx = ux * ux, sqy = uy * uy, sqz = uz * uz, s = sin(angle), c = cos(angle), omc = 1.0 - c;
    R[0] = sqx + (1.0 - sqx) * c; R[1] = ux * uy * omc - uz * s; R[2] = ux * uz * omc + uy * s;
    R[3] = ux * uy * omc + uz * s; R[4] = sqy + (1.0 - sqy) * c; R[5] = uy * uz * omc - ux * s;
    R[6] = ux * uz * omc - uy * s; R[7] = uy * uz * omc + ux * s; R[8] = sqz + (1.0 - sqz) * c;
}
/* Skew3::from(Rotation3) (so3.rs:263-275): scaled_axis = axis * angle, NaN mapped to zero */
static void rot_log(const double *m, double *w) {
    const double angle = acos((m[0] + m[4] + m[8] - 1.0) / 2.0);
    const double a[3] = {m[7] - m[5], m[2] - m[6], m[3] - m[1]};
    const double sq = dot3(a, a);
    if (sq > DBL_EPSILON * DBL_EPSILON) { const double n = sqrt(sq); for (int i = 0; i < 3; i++) w[i] = a[i] / n * angle; }
    else w[0] = w[1] = w[2] = 0.0;
    if (isnan(w[0]) || isnan(w[1]) || isnan(w[2])) w[0] = w[1] = w[2] = 0.0;
}
/* Rotation3::from_matrix: from_matrix_eps(m, f64::EPSILON, unbounded (bounded here), identity) */
static void rot_from_matrix(const double *m, double *rot) {
    memset(rot, 0, 72); rot[0] = rot[4] = rot[8] = 1.0;
    for (int it = 0; it < FROM_MATRIX_MAX_ITERATIONS; it++) {
        double axis[3], denom = 0.0;
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
        rot_from_scaled_axis(aa, Rd);
        for (int r = 0; r < 3; r++)
            for (int c = 0; c < 3; c++) Rn[3 * r + c] = Rd[3 * r] * rot[c] + Rd[3 * r + 1] * rot[3 + c] + Rd[3 * r + 2] * rot[6 + c];
        memcpy(rot, Rn, 72);
    }
}
/* Rotation3::from(Skew3) (so3.rs:248-261); 1 when rotation_small was taken */
static int rot_exp(const double *w, double *R) {
    if (dot3(w, w) <= DBL_EPSILON) {
        const double m[9] = {1.0, -w[2], w[1], w[2], 1.0, -w[0], -w[1], w[0], 1.0};
        rot_from_matrix(m, R);
        return 1;
    }
    rot_from_scaled_axis(w, R);
    return 0;
}
static void world_bearing(const ref_pose *P, const double *b, double *o) {
    for (int r = 0; r < 3; r++) o[r] = P->R[r] * b[0] + P->R[3 + r] * b[1] + P->R[6 + r] * b[2];
}
/* are_observations_robust (lib.rs:2907-2934) */
static int observations_robust(const double *w, uint32_t n, uint32_t min_obs, double inc) {
    if (n < min_obs) return 0;
    for (uint32_t i = 0; i < n; i++)
        for (uint32_t j = i + 1; j < n; j++)
            if (1.0 - dot3(w + 3 * (size_t)i, w + 3 * (size_t)j) > inc) return 1;
    return 0;
}

typedef struct { uint32_t other; ref_pose T; } edge;

int ref_optimize_reconstruction(const ref_recon_cfg *cfg, const ref_triangulator *tri, uint32_t V, const ref_pose *poses, const uint32_t *vo,
                                const double *bear, uint32_t L, const uint32_t *lo, const uint32_t *obs, const ref_view_constraint *cons,
                                uint32_t C, ref_recon_result *res, ref_pose *poses_out, uint8_t *view_state, uint8_t *obs_state, int threads) {
    if (threads > 0) omp_set_num_threads(threads);
    const uint32_t no = lo[L];
    ref_pose *P = malloc(sizeof(ref_pose) * (V ? V : 1)), *Pn = malloc(sizeof(ref_pose) * (V ? V : 1));
    uint8_t *S = calloc(V ? V : 1, 1), *Sn = calloc(V ? V : 1, 1);
    uint32_t *eoff = malloc(sizeof(uint32_t) * (V + 1)), *cur = malloc(sizeof(uint32_t) * (V ? V : 1));
    edge *E = malloc(sizeof(edge) * (C ? 6 * (size_t)C : 1));
    memcpy(P, poses, sizeof(ref_pose) * V);
    memset(obs_state, OBS_KEPT, no);
    memset(res, 0, sizeof(*res));
    int32_t status = RUNNING;
    uint32_t small_total = 0, split_total = 0;
    for (uint32_t round = 0; round < cfg->reconstruction_optimization_iterations && status == RUNNING; round++) {
        /* flatten_constraints: the constraints left after remove_view, six edges each in edge_constraints' order */
        memset(eoff, 0, sizeof(uint32_t) * (V + 1));
        for (uint32_t c = 0; c < C; c++) {
            const uint32_t *w = cons[c].views;
            if (S[w[0]] || S[w[1]] || S[w[2]]) continue;
            for (int x = 0; x < 3; x++) eoff[w[x] + 1] += 2;
        }
        for (uint32_t v = 0; v < V; v++) { eoff[v + 1] += eoff[v]; cur[v] = eoff[v]; }
        for (uint32_t c = 0; c < C; c++) {
            const uint32_t *w = cons[c].views;
            if (S[w[0]] || S[w[1]] || S[w[2]]) continue;
            const ref_pose *first = &cons[c].poses[0], *second = &cons[c].poses[1];
            ref_pose inv_first, f2s;
            pose_inverse(first, &inv_first);
            pose_mul(second, &inv_first, &f2s);
            edge *e;
            e = &E[cur[w[0]]++]; e->other = w[2]; pose_inverse(second, &e->T);
            e = &E[cur[w[0]]++]; e->other = w[1]; e->T = inv_first;
            e = &E[cur[w[1]]++]; e->other = w[0]; e->T = *first;
            e = &E[cur[w[1]]++]; e->other = w[2]; pose_inverse(&f2s, &e->T);
            e = &E[cur[w[2]]++]; e->other = w[1]; e->T = f2s;
            e = &E[cur[w[2]]++]; e->other = w[0]; e->T = *second;
        }
        /* compute_momentum_bundle_adjust, then apply_bundle_adjust */
        for (uint32_t s = 0; s < cfg->optimization_iterations; s++) {
            int panic = 0;
            uint32_t updated = 0, small = 0;
#pragma omp parallel for schedule(dynamic, 4) reduction(| : panic) reduction(+ : updated, small)
            for (uint32_t v = 0; v < V; v++) {
                Pn[v] = P[v];
                Sn[v] = S[v];
                if (S[v]) continue;
                if (eoff[v] == eoff[v + 1]) { Sn[v] = VIEW_NO_EDGES; continue; }
                ref_pose inv;
                pose_inverse(&P[v], &inv);
                double acc[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
                int bad = 0;
                for (uint32_t k = eoff[v]; k < eoff[v + 1]; k++) {
                    if (S[E[k].other]) { bad = 1; break; }   /* views[other_view] of a removed key panics */
                    ref_pose a, d;
                    pose_mul(&E[k].T, &P[E[k].other], &a);
                    pose_mul(&a, &inv, &d);
                    double w[3];
                    rot_log(d.R, w);
                    for (int i = 0; i < 3; i++) { acc[i] = acc[i] + d.t[i]; acc[3 + i] = acc[3 + i] + w[i]; }
                }
                if (bad) { panic = 1; continue; }
                double dl[6];
                int finite = 1;
                for (int i = 0; i < 6; i++) { dl[i] = acc[i] * cfg->graph_optimization_rate; finite = finite && isfinite(dl[i]); }
                if (!finite) { Sn[v] = VIEW_NON_FINITE; continue; }
                ref_pose D;
                small += rot_exp(dl + 3, D.R);
                memcpy(D.t, dl, 24);
                pose_mul(&D, &P[v], &Pn[v]);
                updated++;
            }
            if (panic) { status = PANIC; res->round = round; res->step = s; break; }
            if (updated < 3) { status = REMOVED_CONSTRAINTS; res->round = round; res->step = s; break; }
            small_total += small;
            ref_pose *tp = P; P = Pn; Pn = tp;
            uint8_t *ts = S; S = Sn; Sn = ts;
        }
        if (status != RUNNING) break;
        /* filter_non_robust_observations */
        uint32_t present = 0;
        for (uint32_t v = 0; v < V; v++) present += S[v] == VIEW_KEPT;
        const uint32_t min_obs = cfg->robust_minimum_observations < present ? cfg->robust_minimum_observations : present;
        uint32_t before = 0, after = 0, split = 0;
#pragma omp parallel for schedule(dynamic, 64) reduction(+ : before, after, split)
        for (uint32_t l = 0; l < L; l++) {
            const uint32_t o0 = lo[l], n_in = lo[l + 1] - o0;
            ref_pose *Pl = malloc(sizeof(ref_pose) * (n_in ? n_in : 1));
            double *Bl = malloc(sizeof(double) * 3 * (n_in ? n_in : 1)), *Wl = malloc(sizeof(double) * 3 * (n_in ? n_in : 1));
            uint32_t *gi = malloc(sizeof(uint32_t) * (n_in ? n_in : 1)), m = 0;
            for (uint32_t i = 0; i < n_in; i++) {
                const uint32_t o = o0 + i, v = obs[2 * (size_t)o], f = obs[2 * (size_t)o + 1];
                if (S[v]) { obs_state[o] = OBS_DROPPED; continue; }
                if (obs_state[o] != OBS_KEPT) continue;
                gi[m] = o;
                Pl[m] = P[v];
                memcpy(Bl + 3 * (size_t)m, bear + 3 * ((size_t)vo[v] + f), 24);
                world_bearing(&P[v], Bl + 3 * (size_t)m, Wl + 3 * (size_t)m);
                m++;
            }
            before += observations_robust(Wl, m, min_obs, cfg->robust_observation_incidence_minimum_cosine_distance);
            uint32_t sp = 0;
            if (m == 2) {
                ref_pose inv, tot;
                double fb[3];
                pose_inverse(&Pl[0], &inv);
                pose_mul(&Pl[1], &inv, &tot);
                for (int r = 0; r < 3; r++) fb[r] = dot3(tot.R + 3 * r, Bl);
                if (!(ref_epipolar_loss(tot.t, fb, Bl + 3) < cfg->maximum_sine_distance)) { obs_state[gi[1]] = OBS_SPLIT; sp = 1; }
            } else if (m >= 3) {
                double p[4];
                if (!ref_triangulate_observations(tri, Pl, Bl, (int)m, p, NULL)) {
                    for (uint32_t k = 1; k < m; k++) obs_state[gi[k]] = OBS_SPLIT;
                    sp = m - 1;
                } else {
                    for (uint32_t k = 0; k < m; k++)
                        if (transformed_cosine_distance(&Pl[k], p, Bl + 3 * (size_t)k) > cfg->maximum_cosine_distance && m - sp >= 2) {
                            obs_state[gi[k]] = OBS_SPLIT;
                            sp++;
                        }
                }
            }
            uint32_t kept = 0;
            for (uint32_t k = 0; k < m; k++)
                if (obs_state[gi[k]] == OBS_KEPT) { memmove(Wl + 3 * (size_t)kept, Wl + 3 * (size_t)k, 24); kept++; }
            after += observations_robust(Wl, kept, min_obs, cfg->robust_observation_incidence_minimum_cosine_distance);
            split += sp;
            free(Pl); free(Bl); free(Wl); free(gi);
        }
        res->robust_before = before;
        res->robust_after = after;
        split_total += split;
        if (after < cfg->minimum_robust_landmarks) { status = REMOVED_FILTER; res->round = round; res->step = cfg->optimization_iterations; }
    }
    if (status == RUNNING) { status = KEPT; res->round = cfg->reconstruction_optimization_iterations; res->step = 0; }
    res->status = status;
    res->observations_split = split_total;
    res->small_angle_updates = small_total;
    uint32_t removed = 0;
    for (uint32_t v = 0; v < V; v++) { poses_out[v] = P[v]; view_state[v] = S[v]; removed += S[v] != VIEW_KEPT; }
    res->views_removed = removed;
    free(P); free(Pn); free(S); free(Sn); free(eoff); free(cur); free(E);
    return 0;
}
