/* oracle/ref_try_init.c -- CPU oracle of add_reconstruction in include/cvb200_try_init.h (test infrastructure): VSlamData::add_reconstruction
 * (cv-sfm/src/lib.rs:377-427) restated on slot maps as three add_views (lib.rs:432-483).
 *
 * The reconstruction's landmarks are growable observation lists keyed by view (a view insert appends, a second insert for the same view
 * replaces that view's feature, as HashMap::insert does); first_landmarks / second_landmarks are the reference's HashMap<usize,
 * LandmarkKey>, here arrays over the view's features collected in the reference's order (first_matches, then combined: a later entry for
 * the same feature replaces an earlier one).  The row gathers of bearings, descriptors and colours are plain copies and are left to
 * oracle/pyoracle_try_init.py.  The result is written as the view CSR (landmark per feature), the landmark CSR and the counts. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define NONE 0xffffffffu

typedef struct { uint32_t *obs; uint32_t n, cap; } lm_list;
typedef struct { lm_list *lm; uint32_t L, cap; } recon;

static void insert_obs(lm_list *l, uint32_t v, uint32_t f) {   /* landmark.observations.insert(view, feature) */
    for (uint32_t i = 0; i < l->n; i++)
        if (l->obs[2 * i] == v) { l->obs[2 * i + 1] = f; return; }
    if (l->n == l->cap) {
        l->cap = l->cap ? 2 * l->cap : 4;
        l->obs = realloc(l->obs, sizeof(uint32_t) * 2 * l->cap);
    }
    l->obs[2 * l->n] = v;
    l->obs[2 * l->n + 1] = f;
    l->n++;
}

static uint32_t add_landmark(recon *r, uint32_t v, uint32_t f) {
    if (r->L == r->cap) {
        r->cap = r->cap ? 2 * r->cap : 64;
        r->lm = realloc(r->lm, sizeof(lm_list) * r->cap);
    }
    lm_list *l = &r->lm[r->L];
    memset(l, 0, sizeof(*l));
    insert_obs(l, v, f);
    return r->L++;
}

/* add_view of view v with N features; existing[f]: the landmark of feature f, or NONE */
static void add_view(recon *r, uint32_t v, uint32_t N, const uint32_t *existing, uint32_t *vl) {
    for (uint32_t f = 0; f < N; f++) {
        const uint32_t l = existing ? existing[f] : NONE;
        if (l != NONE) insert_obs(&r->lm[l], v, f);
        vl[f] = l != NONE ? l : add_landmark(r, v, f);
    }
}

/* n_c, n_f, n_s: the three frames' feature counts; comb [K][3], fm [K1][2], sm [K2][2].  Outputs: vo [4], vl [n_c + n_f + n_s],
 * lo [L + 1], obs [n_obs][2] (capacity n_c + n_f + n_s each), counts [4]: n_features, L, n_observations, landmark count of view 0.
 * Returns 0, or -1 where the reference would index out of bounds. */
int ref_add_reconstruction(uint32_t n_c, uint32_t n_f, uint32_t n_s, const uint32_t *comb, uint32_t K, const uint32_t *fm, uint32_t K1,
                           const uint32_t *sm, uint32_t K2, uint32_t *vo, uint32_t *vl, uint32_t *lo, uint32_t *obs, uint32_t *counts) {
    recon r = {NULL, 0, 0};
    uint32_t *m1 = malloc(sizeof(uint32_t) * (n_f + 1)), *m2 = malloc(sizeof(uint32_t) * (n_s + 1));
    int rc = 0;
    for (uint32_t i = 0; i < n_f; i++) m1[i] = NONE;
    for (uint32_t i = 0; i < n_s; i++) m2[i] = NONE;
    vo[0] = 0;
    vo[1] = n_c;
    vo[2] = n_c + n_f;
    vo[3] = n_c + n_f + n_s;
    add_view(&r, 0, n_c, NULL, vl);   /* every center feature a new landmark */
    /* first_landmarks: first_matches then combined, (f, center view's landmark of c) */
    for (uint32_t i = 0; i < K1 + K && !rc; i++) {
        const uint32_t c = i < K1 ? fm[2 * i] : comb[3 * (i - K1)], f = i < K1 ? fm[2 * i + 1] : comb[3 * (i - K1) + 1];
        if (c >= n_c || f >= n_f) rc = -1;
        else m1[f] = vl[c];
    }
    for (uint32_t i = 0; i < K2 + K && !rc; i++) {
        const uint32_t c = i < K2 ? sm[2 * i] : comb[3 * (i - K2)], s = i < K2 ? sm[2 * i + 1] : comb[3 * (i - K2) + 2];
        if (c >= n_c || s >= n_s) rc = -1;
        else m2[s] = vl[c];
    }
    if (!rc) {
        add_view(&r, 1, n_f, m1, vl + n_c);
        add_view(&r, 2, n_s, m2, vl + n_c + n_f);
        uint32_t k = 0;
        for (uint32_t l = 0; l < r.L; l++) {
            lo[l] = k;
            for (uint32_t i = 0; i < r.lm[l].n; i++, k++) {
                obs[2 * k] = r.lm[l].obs[2 * i];
                obs[2 * k + 1] = r.lm[l].obs[2 * i + 1];
            }
        }
        lo[r.L] = k;
        counts[0] = n_c + n_f + n_s;
        counts[1] = r.L;
        counts[2] = k;
        counts[3] = n_c;
    }
    for (uint32_t l = 0; l < r.L; l++) free(r.lm[l].obs);
    free(r.lm);
    free(m1);
    free(m2);
    return rc;
}
