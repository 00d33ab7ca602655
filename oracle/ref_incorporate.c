/* oracle/ref_incorporate.c -- TEST INFRASTRUCTURE (CPU oracle), not product code.  The oracle of include/cvb200_incorporate.h's two CSR
 * edits: cv-sfm's add_view with merge_landmarks (cv-sfm/src/lib.rs:432-483, 699-721), and remove_view / split_observation (lib.rs:517-588)
 * replayed from cvb_optimize_reconstruction's states.  The snapshot is loaded into a slot map of its own (landmarks and views as slots that
 * are inserted at the end and removed in place), the reference's functions run on it loop for loop, and the survivors are written back as
 * CSR in slot order, which is the header's pinned order.  Single-threaded.
 *
 * The replay of an optimisation splits first, then removes views: a SPLIT observation was split while its landmark still had another
 * observation, and every DROPPED one only lowers that count, so splitting first lets every recorded split succeed, as it did in the
 * reference, whatever the interleaving of rounds was. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define NONE 0xffffffffu
enum { VIEW_KEPT = 0 };
enum { OBS_KEPT = 0, OBS_SPLIT = 1, OBS_DROPPED = 2 };

typedef struct { double r[9], t[3]; } ref_pose;
typedef struct { uint32_t views[3]; uint32_t landmarks; ref_pose poses[2]; } ref_constraint;    /* == cvb_view_constraint */
typedef struct { uint32_t feature, landmark_a, landmark_b; } ref_match;                         /* == cvb_register_match */
typedef struct { uint32_t V, n_features, L, n_observations, C, merges; } ref_counts;            /* == cvb_incorporate_counts */

typedef struct { uint32_t n, cap, *obs; int alive; uint32_t merged_into; } landmark;   /* observations: (view, feature) pairs */
typedef struct { uint32_t n, first, *lm; int alive; ref_pose pose; } view;            /* lm[feature]; first: its row in the input CSR */

typedef struct {
    view *v; uint32_t nv;
    landmark *l; uint32_t nl, capl;
} recon;

static void lm_push(landmark *l, uint32_t v, uint32_t f) {
    if (l->n == l->cap) {
        l->cap = l->cap ? 2 * l->cap : 4;
        l->obs = (uint32_t *)realloc(l->obs, sizeof(uint32_t) * 2 * l->cap);
    }
    l->obs[2 * l->n] = v;
    l->obs[2 * l->n + 1] = f;
    l->n++;
}
/* the observation of view v, or NONE */
static uint32_t lm_find(const landmark *l, uint32_t v) {
    for (uint32_t i = 0; i < l->n; i++)
        if (l->obs[2 * i] == v) return i;
    return NONE;
}
static void lm_remove_at(landmark *l, uint32_t i) {   /* HashMap::remove; the other observations keep their order */
    memmove(l->obs + 2 * i, l->obs + 2 * i + 2, sizeof(uint32_t) * 2 * (l->n - i - 1));
    l->n--;
}
static uint32_t add_landmark(recon *r, uint32_t v, uint32_t f) {   /* lib.rs:487-500 */
    if (r->nl == r->capl) {
        r->capl = r->capl ? 2 * r->capl : 16;
        r->l = (landmark *)realloc(r->l, sizeof(landmark) * r->capl);
    }
    landmark *l = &r->l[r->nl];
    memset(l, 0, sizeof(*l));
    l->alive = 1;
    l->merged_into = NONE;
    lm_push(l, v, f);
    return r->nl++;
}

static void load(recon *r, uint32_t V, uint32_t extra_views, const ref_pose *poses, const uint32_t *vo, const uint32_t *vl, uint32_t L,
                 const uint32_t *lo, const uint32_t *obs) {
    memset(r, 0, sizeof(*r));
    r->v = (view *)calloc(V + extra_views + 1, sizeof(view));
    r->nv = V;
    for (uint32_t v = 0; v < V; v++) {
        r->v[v].n = vo[v + 1] - vo[v];
        r->v[v].first = vo[v];
        r->v[v].lm = (uint32_t *)malloc(sizeof(uint32_t) * (r->v[v].n + 1));
        memcpy(r->v[v].lm, vl + vo[v], sizeof(uint32_t) * r->v[v].n);
        r->v[v].alive = 1;
        r->v[v].pose = poses[v];
    }
    r->capl = L + 16;
    r->l = (landmark *)calloc(r->capl, sizeof(landmark));
    r->nl = L;
    for (uint32_t l = 0; l < L; l++) {
        r->l[l].alive = 1;
        r->l[l].merged_into = NONE;
        for (uint32_t o = lo[l]; o < lo[l + 1]; o++) lm_push(&r->l[l], obs[2 * o], obs[2 * o + 1]);
    }
}
static void release(recon *r) {
    for (uint32_t v = 0; v < r->nv; v++) free(r->v[v].lm);
    for (uint32_t l = 0; l < r->nl; l++) free(r->l[l].obs);
    free(r->v);
    free(r->l);
}

/* merge_landmarks (lib.rs:699-721): 0, or -1 where its assert! fires (the two share a view) */
static int merge_landmarks(recon *r, uint32_t a, uint32_t b) {
    landmark *lb = &r->l[b];
    lb->alive = 0;
    lb->merged_into = a;
    for (uint32_t i = 0; i < lb->n; i++) {
        const uint32_t v = lb->obs[2 * i], f = lb->obs[2 * i + 1];
        r->v[v].lm[f] = a;
        if (lm_find(&r->l[a], v) != NONE) return -1;
        lm_push(&r->l[a], v, f);
    }
    return 0;
}

/* remove_view (lib.rs:517-546), without its constraints (the writer drops those) */
static int remove_view(recon *r, uint32_t v) {
    view *w = &r->v[v];
    for (uint32_t f = 0; f < w->n; f++) {
        landmark *l = &r->l[w->lm[f]];
        if (l->n == 0) return -1;   /* "landmark had 0 observations" */
        if (l->n == 1) {
            l->alive = 0;
            l->n = 0;
        } else {
            const uint32_t i = lm_find(l, v);
            if (i != NONE) lm_remove_at(l, i);
        }
    }
    w->alive = 0;
    return 0;
}

/* split_observation (lib.rs:552-588) */
static int split_observation(recon *r, uint32_t v, uint32_t f) {
    const uint32_t old = r->v[v].lm[f];
    if (r->l[old].n < 2) return 0;
    lm_remove_at(&r->l[old], lm_find(&r->l[old], v));
    r->v[v].lm[f] = add_landmark(r, v, f);
    return 1;
}

/* the survivors as CSR in slot order; lmap[l] for the first L0 slots (a merged slot maps to its landmark_a's index), vmap[v] for the first
 * V0 views; the per-feature rows (bearings, descriptors, colours) follow their views from the input rows (or the new frame's for view
 * new_view) */
static void write_back(const recon *r, uint32_t L0, uint32_t V0, uint32_t new_view, const double *bear, const uint8_t *desc, const uint8_t *col,
                       const double *new_bear, const uint8_t *new_desc, const uint8_t *new_col, const ref_constraint *cons, uint32_t C,
                       ref_pose *poses_out, uint32_t *vo_out, uint32_t *vl_out, double *bear_out, uint8_t *desc_out, uint8_t *col_out,
                       uint32_t *lo_out, uint32_t *obs_out, ref_constraint *cons_out, uint32_t *vmap, uint32_t *lmap, ref_counts *cnt) {
    uint32_t *lidx = (uint32_t *)malloc(sizeof(uint32_t) * (r->nl + 1)), *vidx = (uint32_t *)malloc(sizeof(uint32_t) * (r->nv + 1));
    uint32_t nl = 0, no = 0, nv = 0, nf = 0;
    for (uint32_t l = 0; l < r->nl; l++) lidx[l] = r->l[l].alive ? nl++ : NONE;
    for (uint32_t v = 0; v < r->nv; v++) vidx[v] = r->v[v].alive ? nv++ : NONE;
    for (uint32_t l = 0; l < r->nl; l++) {
        if (!r->l[l].alive) continue;
        lo_out[lidx[l]] = no;
        for (uint32_t i = 0; i < r->l[l].n; i++, no++) {
            obs_out[2 * no] = vidx[r->l[l].obs[2 * i]];
            obs_out[2 * no + 1] = r->l[l].obs[2 * i + 1];
        }
    }
    lo_out[nl] = no;
    for (uint32_t v = 0; v < r->nv; v++) {
        const view *w = &r->v[v];
        if (!w->alive) continue;
        poses_out[vidx[v]] = w->pose;
        vo_out[vidx[v]] = nf;
        for (uint32_t f = 0; f < w->n; f++, nf++) {
            vl_out[nf] = lidx[w->lm[f]];
            const int is_new = v == new_view;
            const size_t s = (size_t)(is_new ? f : w->first + f);
            memcpy(bear_out + 3 * (size_t)nf, (is_new ? new_bear : bear) + 3 * s, sizeof(double) * 3);
            const uint8_t *d = is_new ? new_desc : desc, *c = is_new ? new_col : col;   /* NULL: the rows are not kept */
            if (desc_out && d) memcpy(desc_out + 64 * (size_t)nf, d + 64 * s, 64);
            if (col_out && c) memcpy(col_out + 3 * (size_t)nf, c + 3 * s, 3);
        }
    }
    vo_out[nv] = nf;
    uint32_t nc = 0;
    for (uint32_t c = 0; c < C; c++) {   /* remove_view's retain: constraints of removed views go, the rest keep their order */
        const uint32_t *w = cons[c].views;
        if (!r->v[w[0]].alive || !r->v[w[1]].alive || !r->v[w[2]].alive) continue;
        cons_out[nc] = cons[c];
        for (int k = 0; k < 3; k++) cons_out[nc].views[k] = vidx[w[k]];
        nc++;
    }
    for (uint32_t v = 0; v < V0 && vmap; v++) vmap[v] = vidx[v];
    for (uint32_t l = 0; l < L0; l++) {
        const uint32_t m = r->l[l].merged_into;
        lmap[l] = r->l[l].alive ? lidx[l] : (m != NONE ? lidx[m] : NONE);
    }
    cnt->V = nv;
    cnt->n_features = nf;
    cnt->L = nl;
    cnt->n_observations = no;
    cnt->C = nc;
    free(lidx);
    free(vidx);
}

/* add_view (lib.rs:432-483) of one view of N features; matches ascending by feature.  0, or -1 for merge_landmarks' assert!. */
int ref_add_view(uint32_t V, const ref_pose *poses, const uint32_t *vo, const uint32_t *vl, const double *bear, const uint8_t *desc,
                 const uint8_t *col, uint32_t L, const uint32_t *lo, const uint32_t *obs, const ref_pose *new_pose, const double *new_bear,
                 const uint8_t *new_desc, const uint8_t *new_col, uint32_t N, const ref_match *matches, uint32_t M, ref_pose *poses_out,
                 uint32_t *vo_out, uint32_t *vl_out, double *bear_out, uint8_t *desc_out, uint8_t *col_out, uint32_t *lo_out, uint32_t *obs_out,
                 uint32_t *lmap, ref_counts *cnt) {
    recon r;
    load(&r, V, 1, poses, vo, vl, L, lo, obs);
    view *w = &r.v[V];
    w->alive = 1;
    w->pose = *new_pose;
    w->lm = (uint32_t *)malloc(sizeof(uint32_t) * (N + 1));
    r.nv = V + 1;
    uint32_t merged = 0, m = 0;
    int rc = 0;
    for (uint32_t f = 0; f < N; f++) {
        uint32_t l;
        if (m < M && matches[m].feature == f) {
            l = matches[m].landmark_a;
            if (matches[m].landmark_b != NONE) {
                merged++;
                if (merge_landmarks(&r, l, matches[m].landmark_b)) { rc = -1; break; }
            }
            lm_push(&r.l[l], V, f);
            m++;
        } else {
            l = add_landmark(&r, V, f);
        }
        w->lm[w->n++] = l;
    }
    if (rc == 0) {
        write_back(&r, L, 0, V, bear, desc, col, new_bear, new_desc, new_col, NULL, 0, poses_out, vo_out, vl_out, bear_out, desc_out, col_out,
                   lo_out, obs_out, NULL, NULL, lmap, cnt);
        cnt->merges = merged;
    }
    release(&r);
    return rc;
}

/* the edits optimize_reconstruction made, from its states: every SPLIT observation split (observation-CSR order), then every removed view
 * removed (view order).  0, or -1 where remove_view would panic. */
int ref_apply_optimization(uint32_t V, const ref_pose *poses, const uint32_t *vo, const uint32_t *vl, const double *bear, const uint8_t *desc,
                           const uint8_t *col, uint32_t L, const uint32_t *lo, const uint32_t *obs, const ref_constraint *cons, uint32_t C,
                           const uint8_t *vstate, const uint8_t *ostate, ref_pose *poses_out, uint32_t *vo_out, uint32_t *vl_out,
                           double *bear_out, uint8_t *desc_out, uint8_t *col_out, uint32_t *lo_out, uint32_t *obs_out, ref_constraint *cons_out,
                           uint32_t *vmap, uint32_t *lmap, ref_counts *cnt) {
    recon r;
    load(&r, V, 0, poses, vo, vl, L, lo, obs);
    int rc = 0;
    for (uint32_t o = 0; o < lo[L]; o++)
        if (ostate[o] == OBS_SPLIT) split_observation(&r, obs[2 * o], obs[2 * o + 1]);
    for (uint32_t v = 0; v < V && rc == 0; v++)
        if (vstate[v] != VIEW_KEPT) rc = remove_view(&r, v);
    if (rc == 0) {
        write_back(&r, L, V, NONE, bear, desc, col, NULL, NULL, NULL, cons, C, poses_out, vo_out, vl_out, bear_out, desc_out, col_out, lo_out,
                   obs_out, cons_out, vmap, lmap, cnt);
        cnt->merges = 0;
    }
    release(&r);
    return rc;
}
