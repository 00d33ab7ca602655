/* oracle/ref_optimize_l1.c -- TEST INFRASTRUCTURE (CPU oracle), not product code.
 *
 * Plain-C restatement of cv-optimize's L1 (Weiszfeld) pose optimizers, the oracle of include/cvb200_opt.h:
 *   - cv-optimize/src/single_view_optimizer.rs:4-14,16-78   landmark_delta, single_view_simple_optimize_l1
 *   - cv-optimize/src/three_view_optimizer.rs:7-21,23-124   landmark_gradients, three_view_simple_optimize_l1
 *   - cv-core/src/so3.rs:23-34,57-60,123-125                Se3TangentSpace::new (NaN -> zero), isometry(), l1()
 * The gradients are ref_optimize.c's (ref_world_pose_gradient, ref_three_view_gradients); the pose algebra is restated here as
 * ref_optimize.c states it for the L2 optimizers (nalgebra's from_scaled_axis, isometry product and inverse).
 *
 * Quirks kept as the reference has them:
 *   - g.l1() normalises each half of the gradient; a zero half normalises to NaN and Se3TangentSpace::new zeroes it, so such a
 *     landmark adds 0 to l1sum but still 1/(tscale eps) to ts and 1/eps to rs.
 *   - delta = l1sum.scale(rate).scale_translation(ts.recip()).scale_rotation(rs.recip()): times rate first, then times the reciprocal.
 *   - the patience rule looks at the unnormalised |l1sum.t|, |l1sum.r|; one counter over all four norms in the three-view loop.
 *   - tscale: |t| of the current WorldToCamera pose (single view), |t0| + |t1| of the inverted poses (three view), every iteration.
 *   - no argument is rejected: eps = 0, negative rates and zero iterations give the reference's IEEE results.
 * `order` selects how the per-iteration sums are added: REF_SUM_LANDMARK as the reference's `for` loops, REF_SUM_DEVICE as the
 * kernels do, so that the device's deviation from the reference can be measured rather than guessed.
 * Only tests/ and scripts/ may use this file. */
#include "ref_optimize_l1.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>

static double dot3(const double *a, const double *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
static double norm3(const double *a) { return sqrt(dot3(a, a)); }
static void rotv(const double *R, const double *v, double *o) { for (int r = 0; r < 3; r++) o[r] = dot3(R + 3 * r, v); }
static int any_nan3(const double *v) { return isnan(v[0]) || isnan(v[1]) || isnan(v[2]); }
static void normalize3(const double *v, double *o) { double n = norm3(v); o[0] = v[0] / n; o[1] = v[1] / n; o[2] = v[2] / n; }

/* Projective::from_homogeneous (cv-core/src/point.rs:20-25) */
static void from_homogeneous(double *p) {
    if (signbit(p[3])) for (int i = 0; i < 4; i++) p[i] = -p[i];
    double n = norm3(p);
    for (int i = 0; i < 4; i++) p[i] /= n;
}
/* nalgebra Rotation3::from_scaled_axis -> from_axis_angle */
static void rot_from_scaled_axis(const double *v, double *R) {
    const double angle = norm3(v);
    if (angle == 0.0) { memset(R, 0, 72); R[0] = R[4] = R[8] = 1.0; return; }
    const double ux = v[0] / angle, uy = v[1] / angle, uz = v[2] / angle;
    const double sqx = ux * ux, sqy = uy * uy, sqz = uz * uz, s = sin(angle), c = cos(angle), omc = 1.0 - c;
    R[0] = sqx + (1.0 - sqx) * c; R[1] = ux * uy * omc - uz * s; R[2] = ux * uz * omc + uy * s;
    R[3] = ux * uy * omc + uz * s; R[4] = sqy + (1.0 - sqy) * c; R[5] = uy * uz * omc - ux * s;
    R[6] = ux * uz * omc - uy * s; R[7] = uy * uz * omc + ux * s; R[8] = sqz + (1.0 - sqz) * c;
}
/* pose <- Se3TangentSpace{trans, rot}.isometry() * pose   (so3.rs:57-60) */
static void apply_delta(const double *trans, const double *rot, ref_pose *P) {
    double Rd[9], td[3], Rn[9], tn[3];
    rot_from_scaled_axis(rot, Rd);
    rotv(Rd, trans, td);
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) Rn[3 * r + c] = Rd[3 * r] * P->R[c] + Rd[3 * r + 1] * P->R[3 + c] + Rd[3 * r + 2] * P->R[6 + c];
    rotv(Rd, P->t, tn);
    for (int r = 0; r < 3; r++) tn[r] = td[r] + tn[r];
    memcpy(P->R, Rn, 72); memcpy(P->t, tn, 24);
}
static void pose_inverse(const ref_pose *P, ref_pose *o) {
    double nt[3] = {-P->t[0], -P->t[1], -P->t[2]}, R[9];
    for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) R[3 * r + c] = P->R[3 * c + r];
    rotv(R, nt, o->t); memcpy(o->R, R, 72);
}
/* single_view_optimizer.rs:4-14: None when the transformed point has w == 0 */
static int landmark_delta(const ref_pose *P, const double *bearing, const double *world, double *tg, double *rg) {
    double q[4];
    for (int r = 0; r < 3; r++) q[r] = dot3(P->R + 3 * r, world) + P->t[r] * world[3];
    q[3] = world[3];
    from_homogeneous(q);
    if (q[3] == 0.0) return 0;
    double p[3] = {q[0] / q[3], q[1] / q[3], q[2] / q[3]};
    ref_world_pose_gradient(p, bearing, tg, rg);
    return 1;
}

/* one landmark's terms of one pose: v = [g.l1().t, g.l1().r, 1/(|g.t| + tscale eps), 1/(|g.r| + eps)]
 * (single_view_optimizer.rs:36-38, three_view_optimizer.rs:53-55) */
static void l1_terms(const double *tg, const double *rg, double tse, double eps, double *v) {
    normalize3(tg, v); normalize3(rg, v + 3);
    if (any_nan3(v)) v[0] = v[1] = v[2] = 0.0;
    if (any_nan3(v + 3)) v[3] = v[4] = v[5] = 0.0;
    v[6] = 1.0 / (norm3(tg) + tse);
    v[7] = 1.0 / (norm3(rg) + eps);
}
/* delta of one pose from its sums s = [l1sum (6), ts, rs] */
static void l1_delta(const double *s, double rate, double *d) {
    const double it = 1.0 / s[6], ir = 1.0 / s[7];
    for (int k = 0; k < 3; k++) { d[k] = (s[k] * rate) * it; d[3 + k] = (s[3 + k] * rate) * ir; }
}

/* The per-iteration sums of nv slots.  REF_SUM_LANDMARK: one running sum per slot, landmark after landmark.  REF_SUM_DEVICE:
 * landmark i goes to partial sum i mod REF_OPT_NT (a thread's strided loop), each warp of 32 partial sums is reduced by the
 * shuffle-down tree (offsets 16, 8, 4, 2, 1 into lane 0), then the warp totals are added in warp order (block_sum in geom.cu). */
typedef struct { int order, nv; double *part; } summer;
static void sum_begin(summer *s) {
    memset(s->part, 0, sizeof(double) * (size_t)s->nv * (s->order == REF_SUM_DEVICE ? REF_OPT_NT : 1));
}
static void sum_add(summer *s, uint32_t i, const double *v) {
    double *p = s->part + (s->order == REF_SUM_DEVICE ? (size_t)(i % REF_OPT_NT) * s->nv : 0);
    for (int k = 0; k < s->nv; k++) p[k] += v[k];
}
static void sum_end(summer *s, double *out) {
    const int nv = s->nv;
    if (s->order != REF_SUM_DEVICE) { memcpy(out, s->part, sizeof(double) * nv); return; }
    for (int k = 0; k < nv; k++) {
        double total = 0.0;
        for (int w = 0; w < REF_OPT_NT / 32; w++) {
            double lane[32];
            for (int l = 0; l < 32; l++) lane[l] = s->part[(size_t)(32 * w + l) * nv + k];
            for (int o = 16; o; o >>= 1)
                for (int l = 0; l < o; l++) lane[l] += lane[l + o];
            total = w == 0 ? lane[0] : total + lane[0];
        }
        out[k] = total;
    }
}

uint32_t ref_single_view_optimize_l1(ref_pose *pose, double epsilon, double rate, uint32_t iterations, const double *bearings,
                                     const double *world, uint32_t n, int order) {
    if (n == 0) return 0;
    summer S = {order, 8, malloc(sizeof(double) * 8 * REF_OPT_NT)};
    double best_t = INFINITY, best_r = INFINITY;
    uint32_t no_improve = 0, updates = 0;
    for (uint32_t it = 0; it < iterations; it++) {
        const double tse = norm3(pose->t) * epsilon;
        double tg[3], rg[3], v[8], s[8], d[6];
        sum_begin(&S);
        for (uint32_t i = 0; i < n; i++)
            if (landmark_delta(pose, bearings + 3 * (size_t)i, world + 4 * (size_t)i, tg, rg)) {
                l1_terms(tg, rg, tse, epsilon, v);
                sum_add(&S, i, v);
            }
        sum_end(&S, s);
        l1_delta(s, rate, d);
        no_improve++;
        const double t = norm3(s), r = norm3(s + 3);
        if (best_t > t) { best_t = t; no_improve = 0; }
        if (best_r > r) { best_r = r; no_improve = 0; }
        if (no_improve >= 50) break;
        apply_delta(d, d + 3, pose); updates++;
        if (it == iterations - 1) break;
    }
    free(S.part);
    return updates;
}

uint32_t ref_three_view_optimize_l1(ref_pose poses[2], double epsilon, double rate, uint32_t iterations, const double *obs, uint32_t n,
                                    int order) {
    if (n == 0) return 0;
    summer S = {order, 16, malloc(sizeof(double) * 16 * REF_OPT_NT)};
    ref_pose P[2];
    pose_inverse(&poses[0], &P[0]); pose_inverse(&poses[1], &P[1]);
    double best[2][2] = {{INFINITY, INFINITY}, {INFINITY, INFINITY}};
    uint32_t no_improve = 0, updates = 0;
    for (uint32_t it = 0; it < iterations; it++) {
        const double tse = (norm3(P[0].t) + norm3(P[1].t)) * epsilon;
        double g[12], v[16], s[16], d[12], sv[8];
        sum_begin(&S);
        for (uint32_t i = 0; i < n; i++) {
            const double *o = obs + 9 * (size_t)i;
            double f[3], sb[3];
            rotv(P[0].R, o + 3, f); rotv(P[1].R, o + 6, sb);       /* landmark_gradients (:7-21) */
            ref_three_view_gradients(o, f, P[0].t, sb, P[1].t, g);
            for (int p = 0; p < 2; p++) {                          /* v = [l1 of pose 0, l1 of pose 1, ts0, rs0, ts1, rs1] */
                l1_terms(g + 6 * p, g + 6 * p + 3, tse, epsilon, sv);
                memcpy(v + 6 * p, sv, 48);
                v[12 + 2 * p] = sv[6]; v[13 + 2 * p] = sv[7];
            }
            sum_add(&S, i, v);
        }
        sum_end(&S, s);
        for (int p = 0; p < 2; p++) {
            memcpy(sv, s + 6 * p, 48); sv[6] = s[12 + 2 * p]; sv[7] = s[13 + 2 * p];
            l1_delta(sv, rate, d + 6 * p);
        }
        no_improve++;
        for (int p = 0; p < 2; p++) {
            const double t = norm3(s + 6 * p), r = norm3(s + 6 * p + 3);
            if (best[p][0] > t) { best[p][0] = t; no_improve = 0; }
            if (best[p][1] > r) { best[p][1] = r; no_improve = 0; }
        }
        if (no_improve >= 50) break;
        apply_delta(d, d + 3, &P[0]); apply_delta(d + 6, d + 9, &P[1]); updates++;
        if (it == iterations - 1) break;
    }
    pose_inverse(&P[0], &poses[0]); pose_inverse(&P[1], &poses[1]);
    free(S.part);
    return updates;
}
