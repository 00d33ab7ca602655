/* oracle/ref_init.c -- TEST INFRASTRUCTURE (CPU oracle), not product code.  The oracle of include/cvb200_init.h: cv-sfm's
 * VSlam::init_reconstruction from the two-view options on (cv-sfm/src/lib.rs:986-1303), restated sequentially, pair after pair in
 * tuple_combinations order, on the same inputs as cvb_init_reconstruction_dev (host copies) and with the same outputs.  It is built on
 * the existing restatements: ref_is_tri_landmark_robust_tri and ref_triangulate_relative (ref_triangulation.c), ref_epipolar_loss and
 * ref_three_view_optimize_l2 (ref_optimize.c).  Like the device, it keeps `common` in first-match order where the reference shuffles it
 * with VSlam's generator (lib.rs:999). */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "ref_triangulation.h"

typedef struct {   /* == cvb_init_cfg */
    double robust_observation_incidence_minimum_cosine_distance, robust_view_bearing_pair_minimum_cosine_distance, maximum_cosine_distance,
        maximum_sine_distance;
    uint32_t two_view_minimum_robust_matches, three_view_minimum_relative_scales, three_view_optimization_landmarks,
        robust_view_num_robust_bearing_pair, three_view_filter_loop_iterations, three_view_patience, three_view_minimum_robust_matches, reserved;
} ref_init_cfg;
typedef struct {   /* == cvb_init_result */
    int32_t status;
    uint32_t pair, first, second, n_pairs, n_combined, n_first_matches, n_second_matches;
    ref_pose first_pose, second_pose;
} ref_init_result;
typedef struct {   /* == cvb_init_pair_stats */
    int32_t outcome;
    uint32_t first, second, scales;
    double median_scale;
    uint64_t bearing_pairs;
    uint32_t common, opti, updates, robust;
} ref_init_pair_stats;

enum { NONE = 0, ACCEPTED = 1, NONE_BEARING_PAIRS = 2 };
enum { P_NOT_EVALUATED = 0, P_ACCEPTED, P_BEARING_PAIRS, P_FEW_SCALES, P_FEW_MATCHES, P_HALF_MATCHES, P_HALF_ROBUST, P_FEW_ROBUST };
#define NO_FEATURE 0xffffffffu

static double dot3(const double *a, const double *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
static int cmp_double(const void *x, const void *y) { const double a = *(const double *)x, b = *(const double *)y; return (a > b) - (a < b); }

typedef struct {
    const ref_triangulator *tri;
    const double *bear;
    uint32_t cap, fc, ff, fs;   /* frames of center, first, second */
    const uint32_t *common;     /* n x 3 */
    uint32_t n;
} pair_ctx;

static void triple(const pair_ctx *P, uint32_t i, double *B) {
    const uint32_t *t = P->common + 3 * (size_t)i;
    memcpy(B, P->bear + ((size_t)P->fc * P->cap + t[0]) * 3, 24);
    memcpy(B + 3, P->bear + ((size_t)P->ff * P->cap + t[1]) * 3, 24);
    memcpy(B + 6, P->bear + ((size_t)P->fs * P->cap + t[2]) * 3, 24);
}
static int robust(const pair_ctx *P, const ref_pose *first, const ref_pose *second, uint32_t i, double max_cos, double inc) {
    double B[9];
    triple(P, i, B);
    return ref_is_tri_landmark_robust_tri(P->tri, first, second, B, B + 3, B + 6, max_cos, inc);
}
/* lib.rs:1064-1083, 1140-1159: the first `limit` robust triples of common, in order, as [c, f, s] rows */
static uint32_t opti_set(const pair_ctx *P, const ref_pose *first, const ref_pose *second, double max_cos, double inc, uint32_t limit,
                         double *obs) {
    uint32_t k = 0;
    for (uint32_t i = 0; i < P->n && k < limit; i++)
        if (robust(P, first, second, i, max_cos, inc)) triple(P, i, obs + 9 * (size_t)k++);
    return k;
}

int ref_init_reconstruction(const ref_init_cfg *cfg, const ref_triangulator *tri, const double *bear, uint32_t cap, uint32_t center,
                            const uint32_t *options, uint32_t F, const uint32_t *pairs, const uint32_t *n_pairs, const ref_pose *model,
                            const uint32_t *inliers, const uint32_t *n_inl, const int32_t *found, ref_init_result *res, uint32_t *combined,
                            uint32_t *first_matches, uint32_t *second_matches, ref_init_pair_stats *stats) {
    (void)n_pairs;
    memset(res, 0, sizeof(*res));
    if (stats && F > 1) memset(stats, 0, sizeof(*stats) * ((size_t)F * (F - 1) / 2));
    uint32_t list[64], K = 0;
    for (uint32_t f = 0; f < F && f < 64; f++)
        if (found[f] && n_inl[f] >= cfg->two_view_minimum_robust_matches) list[K++] = f;   /* lib.rs:977-985, 1421 */
    res->n_pairs = K * (K - (K > 0)) / 2;
    uint32_t *map = malloc(sizeof(uint32_t) * (size_t)(F ? F : 1) * cap), *common = malloc(sizeof(uint32_t) * 3 * (size_t)cap);
    double *ratios = malloc(sizeof(double) * (size_t)cap), *obs = malloc(sizeof(double) * 9 * (size_t)cap);
    memset(map, 0xff, sizeof(uint32_t) * (size_t)(F ? F : 1) * cap);
    for (uint32_t f = 0; f < F; f++) {
        if (!found[f]) continue;
        for (uint32_t i = 0; i < n_inl[f] && i < cap; i++) {
            const uint32_t *m = pairs + ((size_t)f * cap + inliers[(size_t)f * cap + i]) * 2;
            map[(size_t)f * cap + m[0]] = m[1];
        }
    }
    const double inc = cfg->robust_observation_incidence_minimum_cosine_distance, max_cos = cfg->maximum_cosine_distance;
    const uint32_t limit = cfg->three_view_optimization_landmarks;
    uint32_t pidx = 0;
    int done = 0;
    for (uint32_t x = 0; x < K && !done; x++)
        for (uint32_t y = x + 1; y < K && !done; y++, pidx++) {
            const uint32_t a = list[x], b = list[y];
            ref_init_pair_stats st;
            memset(&st, 0, sizeof(st));
            st.first = a; st.second = b;
            /* lib.rs:991-998 */
            pair_ctx P = {tri, bear, cap, center, options[a], options[b], common, 0};
            for (uint32_t i = 0; i < n_inl[a] && i < cap; i++) {
                const uint32_t *m = pairs + ((size_t)a * cap + inliers[(size_t)a * cap + i]) * 2;
                const uint32_t s = map[(size_t)b * cap + m[0]];
                if (s == NO_FEATURE) continue;
                common[3 * (size_t)P.n] = m[0]; common[3 * (size_t)P.n + 1] = m[1]; common[3 * (size_t)P.n + 2] = s;
                P.n++;
            }
            st.common = P.n;
            ref_pose first = model[a], second = model[b];
            /* lib.rs:1002-1059 */
            uint32_t ns = 0;
            for (uint32_t i = 0; i < P.n; i++) {
                double B[9], fp[4], sp[4];
                triple(&P, i, B);
                if (!ref_is_tri_landmark_robust_tri(tri, &first, &second, B, B + 3, B + 6, 1.0, inc)) continue;
                if (!ref_triangulate_relative(tri, &first, B, B + 3, fp) || fp[3] == 0.0) continue;
                if (!ref_triangulate_relative(tri, &second, B, B + 6, sp) || sp[3] == 0.0) continue;
                const double f3[3] = {fp[0] / fp[3], fp[1] / fp[3], fp[2] / fp[3]}, s3[3] = {sp[0] / sp[3], sp[1] / sp[3], sp[2] / sp[3]};
                const double r = dot3(f3, f3) / dot3(s3, s3);
                if (isnormal(r)) ratios[ns++] = r;
            }
            st.scales = ns;
            int outcome = 0;
            if (ns < cfg->three_view_minimum_relative_scales) outcome = P_FEW_SCALES;
            else {
                qsort(ratios, ns, sizeof(double), cmp_double);
                const double med = sqrt(ratios[ns / 2]);
                st.median_scale = med;
                for (int k = 0; k < 3; k++) second.t[k] = second.t[k] * med;
                /* lib.rs:1064-1110 */
                uint32_t n = opti_set(&P, &first, &second, 1.0, inc, limit, obs);
                st.opti = n;
                uint64_t bp = 0;
                for (uint32_t i = 0; i < n; i++)
                    for (uint32_t j = i + 1; j < n; j++) {
                        const double *u = obs + 9 * (size_t)i, *v = obs + 9 * (size_t)j;
                        const double m = cfg->robust_view_bearing_pair_minimum_cosine_distance;
                        bp += 1.0 - dot3(u, v) > m && 1.0 - dot3(u + 3, v + 3) > m && 1.0 - dot3(u + 6, v + 6) > m;
                    }
                st.bearing_pairs = bp;
                if (bp < cfg->robust_view_num_robust_bearing_pair) outcome = P_BEARING_PAIRS;
                else {
                    const uint32_t robust_min = n / 2;
                    /* lib.rs:1112-1187 */
                    for (uint32_t it = 0; it <= cfg->three_view_filter_loop_iterations && !outcome; it++) {
                        if (n < 32) { outcome = P_FEW_MATCHES; break; }
                        if (n <= robust_min) { outcome = P_HALF_MATCHES; break; }
                        ref_pose pp[2] = {first, second};
                        st.updates += ref_three_view_optimize_l2(pp, 0, 0.001, cfg->three_view_patience, obs, n);
                        first = pp[0]; second = pp[1];
                        if (it < cfg->three_view_filter_loop_iterations) n = opti_set(&P, &first, &second, max_cos, inc, limit, obs);
                    }
                    if (!outcome) {
                        /* lib.rs:1248-1292 */
                        uint32_t nr = 0;
                        for (uint32_t i = 0; i < P.n; i++) nr += robust(&P, &first, &second, i, max_cos, inc);
                        st.robust = nr;
                        if (nr <= robust_min) outcome = P_HALF_ROBUST;
                        else if (nr < cfg->three_view_minimum_robust_matches) outcome = P_FEW_ROBUST;
                        else outcome = P_ACCEPTED;
                    }
                }
            }
            st.outcome = outcome;
            if (stats) stats[pidx] = st;
            if (outcome == P_BEARING_PAIRS) {
                res->status = NONE_BEARING_PAIRS; res->pair = pidx; res->first = a; res->second = b;
                done = 1;
            } else if (outcome == P_ACCEPTED) {
                res->status = ACCEPTED; res->pair = pidx; res->first = a; res->second = b;
                res->first_pose = first; res->second_pose = second;
                /* lib.rs:1193-1246 */
                uint32_t nc = 0;
                for (uint32_t i = 0; i < P.n; i++)
                    if (robust(&P, &first, &second, i, max_cos, 0.0)) memcpy(combined + 3 * (size_t)nc++, common + 3 * (size_t)i, 12);
                res->n_combined = nc;
                for (int z = 0; z < 2; z++) {
                    const uint32_t me = z ? b : a, other = z ? a : b;
                    const ref_pose *pose = z ? &second : &first;
                    uint32_t *out = z ? second_matches : first_matches, k = 0;
                    for (uint32_t i = 0; i < n_inl[me] && i < cap; i++) {
                        const uint32_t *m = pairs + ((size_t)me * cap + inliers[(size_t)me * cap + i]) * 2;
                        if (map[(size_t)other * cap + m[0]] != NO_FEATURE) continue;
                        const double *c = bear + ((size_t)center * cap + m[0]) * 3, *o = bear + ((size_t)options[me] * cap + m[1]) * 3;
                        double rc[3];
                        for (int r = 0; r < 3; r++) rc[r] = dot3(pose->R + 3 * r, c);
                        if (ref_epipolar_loss(pose->t, rc, o) < cfg->maximum_sine_distance) { out[2 * (size_t)k] = m[0]; out[2 * (size_t)k + 1] = m[1]; k++; }
                    }
                    if (z) res->n_second_matches = k; else res->n_first_matches = k;
                }
                done = 1;
            }
        }
    free(map); free(common); free(ratios); free(obs);
    return 0;
}
