/* oracle/ref_merge.c -- CPU oracle of the move edit of include/cvb200_merge.h (test infrastructure): VSlam::incorporate_reconstruction's
 * loop over the source views (cv-sfm/src/lib.rs:1824-1878) restated on a slot map, without its constraint pass (oracle/pyoracle_merge.py
 * calls the constraints oracle one view at a time, with remove_view between the calls, as the reference does).
 *
 * The destination's landmarks are growable observation lists; a view insert appends; landmark_map is the HashMap<LandmarkKey,
 * LandmarkKey> of the reference, here an array over the source landmarks.  The result is written as a CSR snapshot in the pinned orders of
 * the header.  Poses: world_transform^-1 = (R^T, R^T (-t)) and P_v * that, each sum over k = 0, 1, 2 left to right (-ffp-contract=off). */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define NONE 0xffffffffu

typedef struct { double R[9], t[3]; } ref_pose;
typedef struct { uint32_t V, n_features, L, n_observations, C, merges; } ref_counts;
typedef struct { uint32_t *obs; uint32_t n, cap; } lm_list;

static double dot3(const double *a, const double *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
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
static void push(lm_list *l, uint32_t v, uint32_t f) {
    if (l->n == l->cap) {
        l->cap = l->cap ? 2 * l->cap : 4;
        l->obs = realloc(l->obs, sizeof(uint32_t) * 2 * l->cap);
    }
    l->obs[2 * l->n] = v;
    l->obs[2 * l->n + 1] = f;
    l->n++;
}

/* world_transform = dest^-1 * src (WorldToWorld::from_camera_poses) */
void ref_world_transform(const ref_pose *dest, const ref_pose *src, ref_pose *wt) {
    ref_pose inv;
    pose_inverse(dest, &inv);
    pose_mul(&inv, src, wt);
}

/* The move.  Outputs with capacities V + VS, nf + nf_S, L + nf_S, n_obs + nf_S; src_vmap [VS], src_lmap [LS] (before any removal). */
int ref_move(uint32_t V, const ref_pose *poses, const uint32_t *vo, const uint32_t *vl, const double *bear, const uint8_t *desc, const uint8_t *col,
             uint32_t L, const uint32_t *lo, const uint32_t *obs, uint32_t VS, const ref_pose *poses_s, const uint32_t *vo_s, const uint32_t *vl_s,
             const double *bear_s, const uint8_t *desc_s, const uint8_t *col_s, uint32_t LS, uint32_t skip, const ref_pose *wt,
             const uint32_t *landmark_map, ref_pose *poses_out, uint32_t *vo_out, uint32_t *vl_out, double *bear_out, uint8_t *desc_out,
             uint8_t *col_out, uint32_t *lo_out, uint32_t *obs_out, uint32_t *src_vmap, uint32_t *src_lmap, ref_counts *counts) {
    const uint32_t nf = vo[V], nf_s = vo_s[VS];
    uint32_t cap = L + nf_s, nl = L;
    lm_list *lms = calloc(cap ? cap : 1, sizeof(lm_list));
    for (uint32_t l = 0; l < L; l++)
        for (uint32_t o = lo[l]; o < lo[l + 1]; o++) push(&lms[l], obs[2 * o], obs[2 * o + 1]);
    uint32_t *map = malloc(sizeof(uint32_t) * (LS ? LS : 1));
    for (uint32_t l = 0; l < LS; l++) map[l] = landmark_map[l];
    memcpy(poses_out, poses, sizeof(ref_pose) * V);
    memcpy(vo_out, vo, sizeof(uint32_t) * (V + 1));
    memcpy(vl_out, vl, sizeof(uint32_t) * nf);
    memcpy(bear_out, bear, sizeof(double) * 3 * nf);
    if (desc_out) memcpy(desc_out, desc, 64 * (size_t)nf);
    if (col_out) memcpy(col_out, col, 3 * (size_t)nf);
    ref_pose dest_to_src;
    pose_inverse(wt, &dest_to_src);
    uint32_t nv = V, row = nf;
    for (uint32_t v = 0; v < VS; v++) {
        if (v == skip) { src_vmap[v] = NONE; continue; }
        const uint32_t dv = nv++;   /* views.insert appends */
        src_vmap[v] = dv;
        pose_mul(&poses_s[v], &dest_to_src, &poses_out[dv]);
        vo_out[dv] = row;
        for (uint32_t f = 0; f < vo_s[v + 1] - vo_s[v]; f++, row++) {
            const uint32_t s = vo_s[v] + f, sl = vl_s[s];
            uint32_t dl = map[sl];
            if (dl != NONE) {
                push(&lms[dl], dv, f);
            } else {
                dl = nl++;   /* add_landmark */
                push(&lms[dl], dv, f);
                map[sl] = dl;
            }
            vl_out[row] = dl;
            memcpy(bear_out + 3 * (size_t)row, bear_s + 3 * (size_t)s, 24);
            if (desc_out) memcpy(desc_out + 64 * (size_t)row, desc_s + 64 * (size_t)s, 64);
            if (col_out) memcpy(col_out + 3 * (size_t)row, col_s + 3 * (size_t)s, 3);
        }
    }
    vo_out[nv] = row;
    uint32_t k = 0;
    for (uint32_t l = 0; l < nl; l++) {
        lo_out[l] = k;
        memcpy(obs_out + 2 * (size_t)k, lms[l].obs, sizeof(uint32_t) * 2 * lms[l].n);
        k += lms[l].n;
        free(lms[l].obs);
    }
    lo_out[nl] = k;
    for (uint32_t l = 0; l < LS; l++) src_lmap[l] = map[l];
    counts->V = nv; counts->n_features = row; counts->L = nl; counts->n_observations = k; counts->C = 0; counts->merges = 0;
    free(lms);
    free(map);
    return 0;
}
