// cv_b200/csrc/akaze.cu -- host orchestration + C ABI of the AKAZE extractor.
// Mirrors akaze::Akaze::extract_from_gray_float_image (akaze/src/lib.rs:309-339): allocate_evolutions
// (evolution.rs:80-126) and the FED schedule (fed_tau.rs:26-93) run on the host exactly as in the
// reference (tiny f64 scalar work); every per-pixel and per-keypoint stage is a CUDA kernel.
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <atomic>
#include <vector>
#include "../../include/cvb200_stages.h"
#include "akaze_kernels.cuh"
#include "common.cuh"

using namespace akz;

namespace {

struct EvoHost {
    int w = 0, h = 0;
    uint32_t octave = 0, sublevel = 0;
    double esigma = 0, etime = 0;
    uint32_t sigma = 0;       // detector_response.rs:13  round(esigma*derivative_factor/ratio)
    float quat = 0;           // sigma^4 as f32            detector_response.rs:39
    float norm = 0, middle = 0;  // derivatives.rs:57-61
    std::vector<double> tau;  // fed_tau_steps
    size_t off = 0;           // offset of the level inside a pyramid plane (floats)
    bool new_octave = false;
};

bool is_prime_u64(uint64_t n) {
    if (n < 2) return false;
    for (uint64_t d = 2; d * d <= n; d++)
        if (n % d == 0) return false;
    return true;
}

// fed_tau.rs:26-93 (M = 1, reordering = true)
std::vector<double> fed_tau_by_process_time(double T, double tau_max) {
    double t = T / 1.0;
    long n = (long)(ceil(sqrt(3.0 * t / tau_max + 0.25) - 0.5 - 1.0e-8) + 0.5);
    std::vector<double> out;
    if (n <= 0) return out;
    double scale = 3.0 * t / (tau_max * (double)(n * (n + 1)));
    std::vector<double> tau((size_t)n);
    for (long k = 0; k < n; k++) {
        double c = 1.0 / (4.0 * (double)n + 2.0);
        double d = scale * tau_max / 2.0;
        double hh = cos(3.14159265358979323846 * (2.0 * (double)k + 1.0) * c);
        tau[(size_t)k] = d / (hh * hh);
    }
    long kappa = n / 2, prime = n + 1;
    while (!is_prime_u64((uint64_t)prime)) prime++;
    long k = 0;
    for (long i = 0; i < n; i++) {
        long index = ((k + 1) * kappa) % prime - 1;
        while (index >= n || index < 0) {   // usize wrap-around of `x % prime - 1` when the remainder is 0
            k++;
            index = ((k + 1) * kappa) % prime - 1;
        }
        k++;
        out.push_back(tau[(size_t)index]);
    }
    return out;
}

}  // namespace

// image.rs:349-374 (also cvb_gaussian_kernel of include/cvb200_filter.h)
void gaussian_kernel_host(float r, int ks, float *out) {
    int half = ks / 2;
    float sum = 0.f;
    for (int i = -half; i <= half; i++) {
        float x = (float)i;
        volatile float denom = sqrtf(2.0f * 3.14159265358979323846f) * r;
        volatile float e = expf(-(x * x) / (2.0f * (r * r)));
        float val = (1.0f / denom) * e;
        out[i + half] = val;
        sum += val;
    }
    for (int i = 0; i < ks; i++) out[i] /= sum;
}

// cvb_half_size(_dev) of include/cvb200_filter.h: the extractor's kernel on packed planes
int half_size_launch(cvb_ctx *ctx, const float *in, float *out, uint32_t batch, uint32_t w, uint32_t h) {
    const unsigned hw = w / 2, hh = h / 2;
    dim3 blk(32, 8), grd(cdiv(hw, 32), cdiv(hh, 8), batch);
    CVB_PROF(ctx, "k_half_size", 4.0 * ((double)w * h + (double)hw * hh) * batch);
    k_half_size<<<grd, blk, 0, ctx->stream>>>(in, out, (int)w, (int)h, (size_t)w * h, (size_t)hw * hh);
    CVB_LAUNCH_CHECK(ctx);
    return 0;
}

namespace {

int make_gauss_taps(float r, Taps *t) {
    int radius = (int)ceilf(2.0f * r);   // image.rs:385
    int ks = radius * 2 + 1;
    if (ks > MAXK) return -1;
    t->ks = ks;
    memset(t->k, 0, sizeof(t->k));
    gaussian_kernel_host(r, ks, t->k);
    return 0;
}

}  // namespace

struct AkazeWorkspace {
    cvb_akaze_cfg cfg{};
    uint32_t w = 0, h = 0, batch = 0;
    std::vector<EvoHost> evo;
    EvoTable table{};
    size_t plane_floats = 0;   // sum of level sizes
    size_t p0 = 0;             // w*h
    unsigned capc = 0, capk = 0;
    Taps g0{}, g1{};
    // device memory
    float *img = nullptr;
    float *Lt = nullptr, *Lsm = nullptr, *Lx = nullptr, *Ly = nullptr, *Lflow = nullptr, *Ldet = nullptr;
    float *tmpA = nullptr, *tmpB = nullptr, *tmpC = nullptr;
    bool fuse_blur_scharr = true;   // one launch per evolution for Lsmooth + Lflow (CVB_NO_FUSE_BLUR=1: the two separate kernels)
    bool fuse_det = true;           // one launch per octave for Lx, Ly, Ldet + extrema mask (CVB_NO_FUSE_DET=1: the three separate kernels)
    double *g2 = nullptr;
    unsigned long long *gmax = nullptr;
    unsigned *hist = nullptr, *npoints = nullptr;
    double *kc = nullptr;
    float *inv_k = nullptr;
    int *evo_octave = nullptr;
    unsigned *rowcount = nullptr, *rowoff = nullptr, *ncand = nullptr;
    Cand *cand = nullptr;
    cvb_keypoint *cache = nullptr, *refined = nullptr, *sorted = nullptr;
    unsigned *ncache = nullptr, *nneed = nullptr, *nsorted = nullptr, *nvalid = nullptr, *rank = nullptr;   // nneed: unclamped cache count
    unsigned char *keep = nullptr, *valid = nullptr, *ok = nullptr, *desc_tmp = nullptr;
    unsigned *overflow = nullptr;
    CUtensorMap *tmaps = nullptr;      // device: [3][MAX_EVO] per-evolution maps (deriv1 source, Lx, Ly) for the TMA-staged tiles
    bool use_tma = false;
    int tma_mask = 3;                  // CVB_TMA_MASK: 1 k_blur_v3, 2 k_blur_scharr_pm, 4 k_deriv1_v3, 8 k_deriv2_v3.  Default: the two blur kernels
                                       // (the single-stage TMA path stages wider boxes than the derivative kernels' classic path reads)
    SupScratch sup{};
    bool suppress_seq = false;   // CVB_SUPPRESS_SEQ=1: serial reference kernel (debug / A-B check)
    bool suppress_par_only = false;   // CVB_SUPPRESS_GLOBAL=1: force the global-memory parallel kernel
    unsigned *sup_fallback = nullptr;
    unsigned char *tile_evo = nullptr;   // evolution index of every 32x64 tile (all-evolution launches)
    MaskLayout mask_layout{};
    unsigned *extrema_mask = nullptr;
    bool deriv_v3 = true;                // all derivative sigmas <= 5: column-strip kernels
    OrientTables *ot = nullptr;
    DescTables *dt = nullptr;
    // outputs owned by the workspace for the host-pointer API
    cvb_keypoint *kp_out = nullptr;
    unsigned char *desc_out = nullptr;
    unsigned *n_out = nullptr;
    unsigned cap_out = 0;
    std::vector<void *> allocs;
    std::vector<void *> kp_allocs;   // the buffers sized by capc / capk, replaced when a frame needs more (grow_keypoint_capacity)
    bool has_run = false;
    // second stream for the detector response of finished octaves (overlaps the latency-bound coarse octaves)
    cudaStream_t aux = nullptr;
    cudaEvent_t ev_fork[8] = {}, ev_join = nullptr;
    // CUDA graphs of the whole extractor, keyed by the caller's buffers
    struct GraphEntry { const void *img; void *kp, *desc, *n; unsigned B, cap; cudaGraphExec_t exec; };
    std::vector<GraphEntry> graphs;
    uint64_t launches_per_graph = 0;
    bool use_graph = true;       // CVB_NO_GRAPH=1 disables
    bool use_aux = true;         // CVB_NO_AUX_STREAM=1 disables
    // staged calls (include/cvb200_stages.h): the ticket of the scale space the planes hold (0: none; an extract or a rebuild
    // replaces the planes and so clears it) and its batch
    uint64_t ticket = 0;
    unsigned ss_batch = 0;
    DescTables *dt_side = nullptr;   // descriptor tables of a describe config other than the workspace's own
    int dt_side_pattern = 0, dt_side_nch = 0;
    // grow-only buffers of the staged calls, sized by the call
    cvb_keypoint *st_kp = nullptr, *st_kp_out = nullptr;
    unsigned char *st_ok = nullptr, *st_desc = nullptr, *st_desc_out = nullptr;
    unsigned *st_off = nullptr, *st_n = nullptr, *st_need = nullptr;
    size_t st_kp_n = 0, st_kp_out_n = 0, st_ok_n = 0, st_desc_n = 0, st_desc_out_n = 0, st_off_n = 0, st_n_n = 0, st_need_n = 0;
};

void akaze_workspace_free(AkazeWorkspace *ws) {
    if (!ws) return;
    for (auto &g : ws->graphs) cudaGraphExecDestroy(g.exec);
    if (ws->aux) cudaStreamDestroy(ws->aux);
    for (cudaEvent_t e : ws->ev_fork) if (e) cudaEventDestroy(e);
    if (ws->ev_join) cudaEventDestroy(ws->ev_join);
    for (void *p : ws->allocs) cudaFree(p);
    for (void *p : ws->kp_allocs) cudaFree(p);
    for (void *p : {(void *)ws->st_kp, (void *)ws->st_kp_out, (void *)ws->st_ok, (void *)ws->st_desc, (void *)ws->st_desc_out,
                    (void *)ws->st_off, (void *)ws->st_n, (void *)ws->st_need})
        if (p) cudaFree(p);
    delete ws;
}

namespace {

// ---- TMA tensor maps (cuTensorMapEncodeTiled resolved through the runtime: libcvb200.so keeps no link dependency on libcuda)
#ifndef CVB_TMA_DEFAULT
#define CVB_TMA_DEFAULT 1          // CVB_TMA=1 / 0 overrides at run time
#endif
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);
EncodeTiledFn encode_tiled_fn() {
    static EncodeTiledFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void *p = nullptr;
        cudaDriverEntryPointQueryResult qr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) == cudaSuccess && qr == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}
// 3-D f32 map (x, y, frame) of `B` planes of w x h floats, `bstride` floats apart; box = boxw x boxh x 1.  false: TMA not usable here
bool make_tmap(CUtensorMap *out, const float *base, int w, int h, unsigned B, size_t bstride, int boxw, int boxh) {
    EncodeTiledFn fn = encode_tiled_fn();
    memset(out, 0, sizeof(*out));
    if (!fn || ((uintptr_t)base & 15) || (w & 3) || (bstride & 3) || boxw > 256 || boxh > 256 || w < 1 || h < 1) return false;
    const cuuint64_t dims[3] = {(cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)std::max(B, 1u)};
    const cuuint64_t strides[2] = {(cuuint64_t)w * 4, (cuuint64_t)(B > 1 ? bstride : (size_t)w * h) * 4};
    const cuuint32_t box[3] = {(cuuint32_t)boxw, (cuuint32_t)boxh, 1};
    const cuuint32_t es[3] = {1, 1, 1};
    return fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, (void *)base, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
              CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}


// fused FED steps per launch (halo grows with it); CVB_FED_FUSE=1..FED_SMAX overrides for experiments
int fed_fuse_steps() {
    static int v = 0;
    if (!v) { const char *env = getenv("CVB_FED_FUSE"); v = env ? std::min(std::max(atoi(env), 1), FED_SMAX) : FED_FUSE_DEFAULT; }
    return v;
}

template <typename T>
int dalloc_into(cvb_ctx *ctx, std::vector<void *> &list, T **p, size_t n) {
    void *q = nullptr;
    cudaError_t e = cudaMalloc(&q, std::max<size_t>(n, 1) * sizeof(T));
    if (e != cudaSuccess) return cvb_set_error(ctx, CVB_ENOMEM, "cudaMalloc(%zu bytes): %s", n * sizeof(T), cudaGetErrorString(e));
    list.push_back(q);
    *p = (T *)q;
    return 0;
}

template <typename T>
int dalloc(cvb_ctx *ctx, AkazeWorkspace *ws, T **p, size_t n) { return dalloc_into(ctx, ws->allocs, p, n); }

// the buffers of the keypoint stages sized by the workspace's capacities: capc candidates, capk cached keypoints (per frame)
int alloc_keypoint_buffers(cvb_ctx *ctx, AkazeWorkspace *ws) {
    const size_t B = ws->batch;
    int rc = 0;
#define DK(p, n) do { rc = dalloc_into(ctx, ws->kp_allocs, &ws->p, (n)); if (rc) return rc; } while (0)
    DK(cand, B * ws->capc);
    DK(sup.state, B * ws->capc); DK(sup.alive, B * ws->capc); DK(sup.rdy, B * ws->capc);
    DK(sup.key, B * ws->capc); DK(sup.rank, B * ws->capc); DK(sup.next, B * ws->capc);
    DK(cache, B * ws->capk); DK(refined, B * ws->capk); DK(sorted, B * ws->capk); DK(rank, B * ws->capk);
    DK(keep, B * ws->capk); DK(valid, B * ws->capk); DK(ok, B * ws->capk); DK(desc_tmp, B * ws->capk * 64);
#undef DK
    return 0;
}

// Grow the capacities to at least (need_c, need_k), keeping every plane (and so a staged scale space and its ticket).  The
// captured graphs hold the old buffers and are dropped.  The keypoint-stage buffers hold nothing between calls.  The new set is
// allocated before the old one is freed: when an allocation fails, the workspace keeps its buffers and capacities and stays usable.
int grow_keypoint_capacity(cvb_ctx *ctx, AkazeWorkspace *ws, size_t need_c, size_t need_k) {
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    for (auto &g : ws->graphs) cudaGraphExecDestroy(g.exec);
    ws->graphs.clear();
    AkazeWorkspace *nw = new AkazeWorkspace();
    nw->batch = ws->batch;
    // an eighth more than the count, so that a run of similar frames does not grow again at every frame
    nw->capc = need_c > ws->capc ? (unsigned)std::min<size_t>(need_c + need_c / 8, 0xffffffffu) : ws->capc;
    nw->capk = need_k > ws->capk ? (unsigned)std::min<size_t>(need_k + need_k / 8, 0xffffffffu) : ws->capk;
    const int rc = alloc_keypoint_buffers(ctx, nw);
    if (rc) {
        for (void *p : nw->kp_allocs) cudaFree(p);
        delete nw;
        return rc;
    }
    for (void *p : ws->kp_allocs) cudaFree(p);
    ws->kp_allocs = std::move(nw->kp_allocs);
    ws->capc = nw->capc; ws->capk = nw->capk;
    ws->cand = nw->cand;
    ws->sup.state = nw->sup.state; ws->sup.alive = nw->sup.alive; ws->sup.rdy = nw->sup.rdy;
    ws->sup.key = nw->sup.key; ws->sup.rank = nw->sup.rank; ws->sup.next = nw->sup.next;
    ws->cache = nw->cache; ws->refined = nw->refined; ws->sorted = nw->sorted; ws->rank = nw->rank;
    ws->keep = nw->keep; ws->valid = nw->valid; ws->ok = nw->ok; ws->desc_tmp = nw->desc_tmp;
    delete nw;   // its buffers now belong to ws
    return 0;
}

bool same_cfg(const cvb_akaze_cfg &a, const cvb_akaze_cfg &b) { return memcmp(&a, &b, sizeof(a)) == 0; }

// evolution.rs:46-58,80-126 + per-level sizes from the half_size chain (image.rs:155-156, lib.rs:219-221)
int plan_evolutions(cvb_ctx *ctx, AkazeWorkspace *ws) {
    const cvb_akaze_cfg &c = ws->cfg;
    ws->evo.clear();
    for (uint32_t octave = 0; octave < c.max_octave_evolution; octave++) {
        double rfactor = 1.0 / (double)(1ull << octave);   // 2.0f64.powi(-octave)
        uint32_t lh = (uint32_t)((double)ws->h * rfactor), lw = (uint32_t)((double)ws->w * rfactor);
        uint32_t smallest = std::min(lw, lh);
        if (smallest < 40) continue;
        uint32_t sub = smallest < 80 ? 1 : c.num_sublevels;
        for (uint32_t s = 0; s < sub; s++) {
            EvoHost e;
            e.octave = octave; e.sublevel = s;
            e.esigma = c.base_scale_offset * pow(2.0, (double)s / (double)c.num_sublevels + (double)octave);
            e.etime = 0.5 * (e.esigma * e.esigma);
            ws->evo.push_back(e);
        }
    }
    if (ws->evo.empty()) return 0;
    if (ws->evo.size() > (size_t)MAX_EVO) return cvb_set_error(ctx, CVB_EUNSUPPORTED, "more than %d evolutions", MAX_EVO);
    int lw = (int)ws->w, lh = (int)ws->h;
    size_t off = 0;
    int rowbase = 0, tilebase = 0;
    for (size_t i = 0; i < ws->evo.size(); i++) {
        EvoHost &e = ws->evo[i];
        e.new_octave = i > 0 && e.octave > ws->evo[i - 1].octave;
        if (e.new_octave) { lw /= 2; lh /= 2; }
        e.w = lw; e.h = lh; e.off = off;
        off += (size_t)lw * lh;
        off = (off + 63) & ~(size_t)63;   // 256-byte aligned levels
        if (i > 0) {
            e.tau = fed_tau_by_process_time(e.etime - ws->evo[i - 1].etime, 0.25);
            if (e.tau.size() > (size_t)MAX_TAU) return cvb_set_error(ctx, CVB_EUNSUPPORTED, "too many FED steps");
        }
        double ratio = (double)(1ull << e.octave);
        double ss = round(e.esigma * c.derivative_factor / ratio);
        e.sigma = (uint32_t)ss;
        e.quat = (float)(ss * ss * ss * ss);
        double wv = 10.0 / 3.0;
        e.norm = (float)(1.0 / (2.0 * (double)e.sigma * (wv + 2.0)));
        e.middle = e.norm * (float)wv;
        if (e.sigma == 1) { e.norm = 3.0f; e.middle = 10.0f; }   // derivatives.rs:24-26,43-45: sigma 1 -> simple (un-normalised) Scharr
        if (e.sigma < 1 || e.sigma > 16) return cvb_set_error(ctx, CVB_EUNSUPPORTED, "derivative sigma %u out of range", e.sigma);
        EvoDev &d = ws->table.e[i];
        d.w = e.w; d.h = e.h; d.off = e.off; d.octave = (int)e.octave;
        d.size = (float)(e.esigma * c.derivative_factor);
        d.rowbase = rowbase; d.pad = 0;
        d.tilebase = tilebase; d.sigma = (int)e.sigma; d.norm = e.norm; d.middle = e.middle; d.quat = e.quat;
        rowbase += e.h;
        tilebase += (int)(cdiv((unsigned)e.w, SW3) * cdiv((unsigned)e.h, SH3));
    }
    ws->table.n = (int)ws->evo.size();
    ws->table.total_rows = rowbase;
    ws->table.total_tiles = tilebase;
    ws->table.pad = 0;
    ws->plane_floats = off;
    return 0;
}

// descriptor tables (descriptors.rs:64-96,117-124,188-201) of one (descriptor_pattern_size, descriptor_channels)
int make_desc_tables(cvb_ctx *ctx, int pattern, int nch, DescTables *dt) {
    memset(dt, 0, sizeof(*dt));
    if (pattern < 1 || pattern > DESC_MAXLAT) return cvb_set_error(ctx, CVB_EUNSUPPORTED, "descriptor_pattern_size %d out of range", pattern);
    const float size_mult[3] = {1.0f, 2.0f / 3.0f, 1.0f / 2.0f};
    int base[3], ncell = 0;
    for (int lvl = 0; lvl < 3; lvl++) {
        int step = (int)ceilf((float)pattern * size_mult[lvl]);
        base[lvl] = ncell;
        int per_axis = 0;
        for (int i = -pattern; i < pattern; i += step) per_axis++;
        if (per_axis != lvl + 2) return cvb_set_error(ctx, CVB_EUNSUPPORTED, "descriptor_pattern_size %d: grid %d has %d cells per axis", pattern, lvl, per_axis);
        for (int i = -pattern; i < pattern; i += step)
            for (int j = -pattern; j < pattern; j += step) {
                dt->ci[ncell] = (short)i; dt->cj[ncell] = (short)j; dt->cstep[ncell] = (short)step;
                ncell++;
            }
    }
    dt->ncells = ncell;
    int kmax = -pattern;
    for (int c = 0; c < ncell; c++) kmax = std::max(kmax, dt->ci[c] + dt->cstep[c] - 1);
    dt->nlat = kmax + pattern + 1;
    if (dt->nlat > DESC_MAXLAT) return cvb_set_error(ctx, CVB_EUNSUPPORTED, "descriptor_pattern_size %d needs a %d-point lattice (max %d)", pattern, dt->nlat, DESC_MAXLAT);
    int bit = 0;
    for (int lvl = 0; lvl < 3; lvl++) {
        int count = (lvl + 2) * (lvl + 2);
        for (int pos = 0; pos < nch; pos++)
            for (int a = 0; a < count; a++)
                for (int b2 = a + 1; b2 < count; b2++) {
                    dt->ba[bit] = (unsigned char)(base[lvl] + a); dt->bb[bit] = (unsigned char)(base[lvl] + b2);
                    dt->bch[bit] = (unsigned char)pos;
                    bit++;
                }
    }
    dt->nbits = bit;
    return 0;
}

int build_tables(cvb_ctx *ctx, AkazeWorkspace *ws) {
    // orientation tables (scale_space_extrema.rs:233-287)
    OrientTables ot;
    memset(&ot, 0, sizeof(ot));
    static const float GAUSS25[7][7] = {
        {0.02546481f, 0.02350698f, 0.01849125f, 0.01239505f, 0.00708017f, 0.00344629f, 0.00142946f},
        {0.02350698f, 0.02169968f, 0.01706957f, 0.01144208f, 0.00653582f, 0.00318132f, 0.00131956f},
        {0.01849125f, 0.01706957f, 0.01342740f, 0.00900066f, 0.00514126f, 0.00250252f, 0.00103800f},
        {0.01239505f, 0.01144208f, 0.00900066f, 0.00603332f, 0.00344629f, 0.00167749f, 0.00069579f},
        {0.00708017f, 0.00653582f, 0.00514126f, 0.00344629f, 0.00196855f, 0.00095820f, 0.00039744f},
        {0.00344629f, 0.00318132f, 0.00250252f, 0.00167749f, 0.00095820f, 0.00046640f, 0.00019346f},
        {0.00142946f, 0.00131956f, 0.00103800f, 0.00069579f, 0.00039744f, 0.00019346f, 0.00008024f},
    };
    static const int id[13] = {6, 5, 4, 3, 2, 1, 0, 1, 2, 3, 4, 5, 6};
    int idx = 0;
    for (int j = -6; j <= 6; j++)
        for (int i = -6; i <= 6; i++)
            if (i * i + j * j < 36) {
                ot.di[idx] = (signed char)i; ot.dj[idx] = (signed char)j;
                ot.gw[idx] = GAUSS25[id[j + 6]][id[i + 6]];
                idx++;
            }
    {
        volatile float ang1 = 0.f;   // f32 accumulation exactly as the reference loop (:259-287)
        const float two_pi = 2.0f * 3.14159265358979323846f;
        int n = 0;
        while (ang1 < two_pi && n < 64) { ot.ang1[n++] = ang1; ang1 = ang1 + 0.15f; }
        ot.nwin = n;
        // upper window ends with the reference's expression, and the structure k_refine_orient relies on: the non-wrapping
        // windows come first and both ends ascend inside each group
        const float PI = 3.14159265358979323846f;
        int nn = 0;
        for (int i = 0; i < n; i++) {
            const volatile float a1 = ot.ang1[i];
            const volatile float up = a1 + PI / 3.0f, dn = a1 - 5.0f * PI / 3.0f;
            ot.ang2[i] = up > two_pi ? dn : up;
            if (ot.ang1[i] < ot.ang2[i]) nn = i + 1;
        }
        ot.nn = nn;
        bool ok = true;
        for (int i = 0; i < n; i++) {
            if ((i < nn) != (ot.ang1[i] < ot.ang2[i])) ok = false;
            if (i + 1 < n && !(ot.ang1[i] < ot.ang1[i + 1])) ok = false;
            if (i + 1 < n && i + 1 != nn && !(ot.ang2[i] < ot.ang2[i + 1])) ok = false;
        }
        if (!ok) return cvb_set_error(ctx, CVB_EUNSUPPORTED, "orientation window table is not ordered as expected");
    }
    CVB_CUDA(ctx, cudaMemcpyAsync(ws->ot, &ot, sizeof(ot), cudaMemcpyHostToDevice, ctx->stream));
    DescTables dt;
    int rc = make_desc_tables(ctx, (int)ws->cfg.descriptor_pattern_size, (int)ws->cfg.descriptor_channels, &dt);
    if (rc) return rc;
    CVB_CUDA(ctx, cudaMemcpyAsync(ws->dt, &dt, sizeof(dt), cudaMemcpyHostToDevice, ctx->stream));
    std::vector<int> oct(MAX_EVO, 0);
    for (size_t i = 0; i < ws->evo.size(); i++) oct[i] = (int)ws->evo[i].octave;
    CVB_CUDA(ctx, cudaMemcpyAsync(ws->evo_octave, oct.data(), sizeof(int) * MAX_EVO, cudaMemcpyHostToDevice, ctx->stream));
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    return 0;
}

int build_workspace(cvb_ctx *ctx, AkazeWorkspace *ws, const cvb_akaze_cfg *cfg, uint32_t batch, uint32_t w, uint32_t h, unsigned cap_out);

int ensure_workspace(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, uint32_t batch, uint32_t w, uint32_t h, unsigned cap_out) {
    AkazeWorkspace *ws = ctx->akaze;
    if (ws && same_cfg(ws->cfg, *cfg) && ws->w == w && ws->h == h && ws->batch >= batch && ws->cap_out >= cap_out) return 0;
    if (ws) { cvb_wait(ctx, ctx->stream); akaze_workspace_free(ws); ctx->akaze = nullptr; }
    if (cfg->descriptor_channels < 1 || cfg->descriptor_channels > 3) return cvb_set_error(ctx, CVB_EINVAL, "descriptor_channels must be 1..3");
    if (cfg->contrast_factor_num_bins < 1 || cfg->contrast_factor_num_bins > 8192) return cvb_set_error(ctx, CVB_EUNSUPPORTED, "contrast_factor_num_bins must be 1..8192");
    if (cfg->num_sublevels < 1) return cvb_set_error(ctx, CVB_EINVAL, "num_sublevels must be >= 1");
    if (!(cfg->base_scale_offset > 0.0)) return cvb_set_error(ctx, CVB_EINVAL, "sigma must be > 0.0");   // image.rs:384
    ws = new AkazeWorkspace();
    ws->cfg = *cfg; ws->w = w; ws->h = h; ws->batch = batch; ws->cap_out = cap_out;
    // the workspace is published on the context only when it is complete: a failed build must not satisfy the
    // fast path of the next call with identical arguments
    int rc = build_workspace(ctx, ws, cfg, batch, w, h, cap_out);
    if (rc) { cvb_wait(ctx, ctx->stream); akaze_workspace_free(ws); return rc; }
    ctx->akaze = ws;
    return 0;
}

int build_workspace(cvb_ctx *ctx, AkazeWorkspace *ws, const cvb_akaze_cfg *cfg, uint32_t batch, uint32_t w, uint32_t h, unsigned cap_out) {
    int rc = plan_evolutions(ctx, ws);
    if (rc) return rc;
    if (make_gauss_taps((float)cfg->base_scale_offset, &ws->g0)) return cvb_set_error(ctx, CVB_EUNSUPPORTED, "base_scale_offset too large");
    make_gauss_taps(1.0f, &ws->g1);
    ws->p0 = (size_t)w * h;
    // capacities for the frames of everyday threshold and texture: a frame that exceeds them makes the host calls grow them
    // (grow_keypoint_capacity) and run again; the _dev calls report it with flag 1 or 2 of cvb_akaze_dev_overflow.  A proven bound
    // (every strict 3x3 maximum needs a 2-pixel pitch: P/4 per level) would cost ~155 bytes per possible cached keypoint.
    ws->capc = (unsigned)std::min<size_t>(std::max<size_t>(ws->p0 / 8, 4096), 1u << 20);
    ws->capk = (unsigned)std::min<size_t>(std::max<size_t>(ws->p0 / 32, 4096), 1u << 17);
    const size_t B = batch, PF = ws->plane_floats, R = (size_t)std::max(ws->table.total_rows, 1);
#define DA(p, n) do { rc = dalloc(ctx, ws, &ws->p, (n)); if (rc) return rc; } while (0)
    DA(img, B * ws->p0);
    DA(Lt, B * PF); DA(Lsm, B * PF); DA(Lx, B * PF); DA(Ly, B * PF); DA(Lflow, B * PF); DA(Ldet, B * PF);
    DA(tmpA, B * ws->p0); DA(tmpB, B * ws->p0); DA(tmpC, B * ws->p0);
    DA(g2, B * ws->p0);
    DA(gmax, B); DA(hist, B * cfg->contrast_factor_num_bins); DA(npoints, B); DA(kc, B); DA(inv_k, B * MAX_EVO);
    DA(evo_octave, MAX_EVO);
    DA(rowcount, B * R); DA(rowoff, B * R); DA(ncand, B);
    DA(ncache, B); DA(nneed, B); DA(nsorted, B); DA(nvalid, B);
    DA(overflow, 1);
    if ((rc = alloc_keypoint_buffers(ctx, ws))) return rc;
    {   // scratch of the parallel duplicate suppression; bins sized for the finest class grid
        unsigned nbmax = 1;
        for (size_t i = 0; i < ws->evo.size(); i++) {
            float ratio = (float)(1u << ws->evo[i].octave), off = 0.5f * (ratio - 1.0f), size = ws->table.e[i].size;
            float cell = fmaxf(16.0f, ceilf(2.0f * size + 2.0f * off + 2.0f));
            unsigned nbx = (unsigned)((float)w / cell) + 3, nby = (unsigned)((float)h / cell) + 3;
            nbmax = std::max(nbmax, nbx * nby);
        }
        ws->sup.nbmax = nbmax;
        DA(sup.binA, B * nbmax); DA(sup.binB, B * nbmax);
        const char *env = getenv("CVB_SUPPRESS_SEQ");
        ws->suppress_seq = env && env[0] == '1';
        env = getenv("CVB_SUPPRESS_GLOBAL");
        ws->suppress_par_only = env && env[0] == '1';
        DA(sup_fallback, B);
        env = getenv("CVB_NO_GRAPH");
        ws->use_graph = !(env && env[0] == '1');
        env = getenv("CVB_NO_AUX_STREAM");
        ws->use_aux = !(env && env[0] == '1');
        env = getenv("CVB_NO_FUSE_BLUR");
        ws->fuse_blur_scharr = !(env && env[0] == '1');
        env = getenv("CVB_NO_FUSE_DET");
        ws->fuse_det = !(env && env[0] == '1');
        cudaStreamCreateWithFlags(&ws->aux, cudaStreamNonBlocking);
        for (auto &e : ws->ev_fork) cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
        cudaEventCreateWithFlags(&ws->ev_join, cudaEventDisableTiming);
        cudaFuncSetAttribute(k_suppress_smem, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SUP_SMEM);
    }
    DA(ot, 1); DA(dt, 1); DA(dt_side, 1);
    DA(tmaps, 3 * MAX_EVO);
    DA(kp_out, B * (size_t)cap_out); DA(desc_out, B * (size_t)cap_out * 64); DA(n_out, B);
#undef DA
    {   // TMA-staged tiles: per-evolution maps of the planes the derivative kernels read (CVB_TMA=0 / 1 overrides the default)
        const char *env = getenv("CVB_TMA");
        ws->use_tma = env ? env[0] == '1' : (CVB_TMA_DEFAULT != 0);
        if (const char *m = getenv("CVB_TMA_MASK")) ws->tma_mask = atoi(m);
        std::vector<CUtensorMap> hm(3 * MAX_EVO);
        memset(hm.data(), 0, sizeof(CUtensorMap) * hm.size());
        for (size_t i = 0; i < ws->evo.size() && ws->use_tma; i++) {
            const EvoHost &e = ws->evo[i];
            const int S = std::min<int>((int)e.sigma, 5);
            if ((int)e.sigma > 5) { ws->use_tma = false; break; }
            const float *src1 = (i == 0 ? ws->Lt : ws->Lsm) + e.off;
            const bool ok = make_tmap(&hm[i], src1, e.w, e.h, batch, PF, pitch3(S), SH3 + 2 * S)
                         && make_tmap(&hm[MAX_EVO + i], ws->Lx + e.off, e.w, e.h, batch, PF, pitch3(S), SH3 + 2 * S)
                         && make_tmap(&hm[2 * MAX_EVO + i], ws->Ly + e.off, e.w, e.h, batch, PF, pitch3(S), SH3 + 2 * S);
            if (!ok) ws->use_tma = false;        // e.g. a level width that is not a multiple of 4 floats: every kernel keeps the classic path
        }
        CVB_CUDA(ctx, cudaMemcpyAsync(ws->tmaps, hm.data(), sizeof(CUtensorMap) * hm.size(), cudaMemcpyHostToDevice, ctx->stream));
        CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    }
    {
        std::vector<unsigned char> te((size_t)std::max(ws->table.total_tiles, 1), 0);
        ws->deriv_v3 = true;
        for (size_t i = 0; i < ws->evo.size(); i++) {
            const int t0 = ws->table.e[i].tilebase, t1 = i + 1 < ws->evo.size() ? ws->table.e[i + 1].tilebase : ws->table.total_tiles;
            for (int t = t0; t < t1; t++) te[(size_t)t] = (unsigned char)i;
            if (ws->evo[i].sigma > 5) ws->deriv_v3 = false;
        }
        rc = dalloc(ctx, ws, &ws->tile_evo, te.size());
        if (rc) return rc;
        int words = 0;
        for (size_t i = 0; i < ws->evo.size(); i++) {
            ws->mask_layout.wordbase[i] = words;
            words += (int)(cdiv((unsigned)ws->evo[i].w, 32) * (unsigned)ws->evo[i].h);
        }
        ws->mask_layout.total_words = words;
        rc = dalloc(ctx, ws, &ws->extrema_mask, (size_t)B * std::max(words, 1));
        if (rc) return rc;
        CVB_CUDA(ctx, cudaMemcpyAsync(ws->tile_evo, te.data(), te.size(), cudaMemcpyHostToDevice, ctx->stream));
        CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    }
    CVB_CUDA(ctx, cudaMemsetAsync(ws->overflow, 0, sizeof(unsigned), ctx->stream));
    CVB_CUDA(ctx, cudaMemsetAsync(ws->inv_k, 0, sizeof(float) * B * MAX_EVO, ctx->stream));
    // opt in to large dynamic shared memory where a configuration needs it
    cudaFuncSetAttribute(k_separable, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    cudaFuncSetAttribute(k_deriv1_v3, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    cudaFuncSetAttribute(k_deriv2_v3, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    cudaFuncSetAttribute(k_deriv1<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    cudaFuncSetAttribute(k_deriv1<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    cudaFuncSetAttribute(k_deriv1<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    cudaFuncSetAttribute(k_deriv1<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    cudaFuncSetAttribute(k_deriv2_det<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    cudaFuncSetAttribute(k_deriv2_det<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    cudaFuncSetAttribute(k_deriv2_det<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    cudaFuncSetAttribute(k_deriv2_det<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    return build_tables(ctx, ws);
}

inline dim3 tile_grid(int w, int h, unsigned B) { return dim3(cdiv((unsigned)w, TW), cdiv((unsigned)h, TH), B); }

int launch_separable(cvb_ctx *ctx, const float *in, size_t in_bs, float *out, size_t out_bs, int w, int h, unsigned B,
                     const Taps &hk, const Taps &vk) {
    if (hk.ks == vk.ks && (hk.ks == 5 || hk.ks == 9) && memcmp(hk.k, vk.k, sizeof(float) * hk.ks) == 0) {
        CVB_PROF(ctx, "k_blur", 8.0 * w * h * B);
        dim3 g(cdiv((unsigned)w, SW3), cdiv((unsigned)h, SH3), B);
        CUtensorMap tm;
        const int R = hk.ks / 2;
        const int use_tma = ctx->akaze && ctx->akaze->use_tma && (ctx->akaze->tma_mask & 1) && make_tmap(&tm, in, w, h, B, in_bs, pitch3(R), SH3 + 2 * R) ? 1 : 0;
        if (!use_tma) memset(&tm, 0, sizeof(tm));
        if (hk.ks == 5) k_blur_v3<5><<<g, NT, 0, ctx->stream>>>(in, out, w, h, in_bs, out_bs, hk, tm, use_tma);
        else k_blur_v3<9><<<g, NT, 0, ctx->stream>>>(in, out, w, h, in_bs, out_bs, hk, tm, use_tma);
        CVB_LAUNCH_CHECK(ctx);
        return 0;
    }
    int rx = hk.ks / 2, ry = vk.ks / 2;
    size_t smem = sizeof(float) * ((size_t)(TH + 2 * ry) * (TW + 2 * rx) + (size_t)(TH + 2 * ry) * TW);
    { CVB_PROF(ctx, "k_separable", 8.0 * w * h * B);
    k_separable<<<tile_grid(w, h, B), NT, smem, ctx->stream>>>(in, out, w, h, in_bs, out_bs, hk, vk);
    CVB_LAUNCH_CHECK(ctx); }
    return 0;
}

int launch_deriv1(cvb_ctx *ctx, const EvoHost &e, const float *Ls, float *Lx, float *Ly, size_t bs, unsigned B) {
    int s = (int)e.sigma;
    CVB_PROF(ctx, "k_deriv1", 12.0 * e.w * e.h * B);
    size_t smem = sizeof(float) * ((size_t)(TH + 2 * s) * (TW + 2 * s) + 2 * (size_t)(TH + 2 * s) * TW);
    dim3 g = tile_grid(e.w, e.h, B);
    switch (s & 3) {
    case 0: k_deriv1<0><<<g, NT, smem, ctx->stream>>>(Ls, Lx, Ly, e.w, e.h, bs, s, e.norm, e.middle); break;
    case 1: k_deriv1<1><<<g, NT, smem, ctx->stream>>>(Ls, Lx, Ly, e.w, e.h, bs, s, e.norm, e.middle); break;
    case 2: k_deriv1<2><<<g, NT, smem, ctx->stream>>>(Ls, Lx, Ly, e.w, e.h, bs, s, e.norm, e.middle); break;
    default: k_deriv1<3><<<g, NT, smem, ctx->stream>>>(Ls, Lx, Ly, e.w, e.h, bs, s, e.norm, e.middle); break;
    }
    CVB_LAUNCH_CHECK(ctx);
    return 0;
}

int launch_deriv2(cvb_ctx *ctx, const EvoHost &e, const float *Lx, const float *Ly, float *Ldet, size_t bs, unsigned B) {
    int s = (int)e.sigma;
    CVB_PROF(ctx, "k_deriv2_det", 12.0 * e.w * e.h * B);
    size_t smem = sizeof(float) * (2 * (size_t)(TH + 2 * s) * (TW + 2 * s) + 3 * (size_t)(TH + 2 * s) * TW);
    dim3 g = tile_grid(e.w, e.h, B);
    switch (s & 3) {
    case 0: k_deriv2_det<0><<<g, NT, smem, ctx->stream>>>(Lx, Ly, Ldet, e.w, e.h, bs, s, e.norm, e.middle, e.quat); break;
    case 1: k_deriv2_det<1><<<g, NT, smem, ctx->stream>>>(Lx, Ly, Ldet, e.w, e.h, bs, s, e.norm, e.middle, e.quat); break;
    case 2: k_deriv2_det<2><<<g, NT, smem, ctx->stream>>>(Lx, Ly, Ldet, e.w, e.h, bs, s, e.norm, e.middle, e.quat); break;
    default: k_deriv2_det<3><<<g, NT, smem, ctx->stream>>>(Lx, Ly, Ldet, e.w, e.h, bs, s, e.norm, e.middle, e.quat); break;
    }
    CVB_LAUNCH_CHECK(ctx);
    return 0;
}

// ---- the extractor in three stages (lib.rs:309-339), each asynchronous on the context's stream and for B >= 1 frames of a
// workspace with at least one evolution.  run_extract_eager issues them in order; the staged calls of include/cvb200_stages.h
// issue them one at a time.

// create_nonlinear_scale_space + detector_response (lib.rs:193-258, detector_response.rs:8-85) for `B` frames already resident
// in `images` (device): every plane, and the extrema mask and per-row counts of the fused detector response
int stage_scale_space(cvb_ctx *ctx, const float *images, unsigned B) {
    AkazeWorkspace *ws = ctx->akaze;
    cudaStream_t st = ctx->stream;
    const size_t PF = ws->plane_floats, P0 = ws->p0;
    const int W = (int)ws->w, H = (int)ws->h;
    const int E = (int)ws->evo.size();
    const int nbins = (int)ws->cfg.contrast_factor_num_bins;
    int smax = 1;
    for (const EvoHost &e : ws->evo) smax = std::max(smax, (int)e.sigma);
    const bool aux_ok = ws->use_aux && !ctx->prof;
    const bool fused_det = ws->deriv_v3 && ws->fuse_det;   // the detector response writes the extrema mask itself
    const int R = ws->table.total_rows;
    const float thr = (float)ws->cfg.detector_threshold;
    bool forked = false;
    int fork_id = 0;
    // detector response (derivatives + Ldet) of evolutions [e0, e1): they only depend on Lsmooth of those evolutions
    auto issue_detector_response = [&](int e0, int e1) -> int {
        const int t0 = ws->table.e[e0].tilebase;
        const int t1 = e1 < E ? ws->table.e[e1].tilebase : ws->table.total_tiles;
        if (t1 <= t0) return 0;
        cudaStream_t ds = st;
        if (aux_ok) {
            CVB_CUDA(ctx, cudaEventRecord(ws->ev_fork[fork_id & 7], st));
            CVB_CUDA(ctx, cudaStreamWaitEvent(ws->aux, ws->ev_fork[fork_id & 7], 0));
            fork_id++;
            forked = true;
            ds = ws->aux;
        }
        double px = 0;
        for (int e = e0; e < e1; e++) px += (double)ws->evo[e].w * ws->evo[e].h;
        if (fused_det) {
            dim3 g((unsigned)(t1 - t0), 1, B);
            CVB_PROF(ctx, "k_detector_response", 16.0 * px * B);
            k_detector_response<<<g, NT, sizeof(float) * det_smem_floats(smax), ds>>>(ws->Lsm, ws->Lt, ws->Lx, ws->Ly, ws->Ldet, PF, ws->table,
                                                                                      ws->tile_evo, t0, ws->mask_layout, thr, ws->extrema_mask,
                                                                                      ws->rowcount);
            CVB_LAUNCH_CHECK(ctx);
        } else if (ws->deriv_v3) {
            const size_t region = (((size_t)pitch3(smax) * (SH3 + 2 * smax)) + 31) & ~(size_t)31;
            dim3 g((unsigned)(t1 - t0), 1, B);
            { CVB_PROF(ctx, "k_deriv1", 12.0 * px * B);
            k_deriv1_v3<<<g, NT, sizeof(float) * region + 128, ds>>>(ws->Lsm, ws->Lt, ws->Lx, ws->Ly, PF, ws->table, ws->tile_evo, t0,
                                                               ws->use_tma && (ws->tma_mask & 4) ? ws->tmaps : nullptr);
            CVB_LAUNCH_CHECK(ctx); }
            { CVB_PROF(ctx, "k_deriv2_det", 12.0 * px * B);
            k_deriv2_v3<<<g, NT, sizeof(float) * 2 * region + 128, ds>>>(ws->Lx, ws->Ly, ws->Ldet, PF, ws->table, ws->tile_evo, t0,
                                                                   ws->use_tma && (ws->tma_mask & 8) ? ws->tmaps + MAX_EVO : nullptr, ws->use_tma && (ws->tma_mask & 8) ? ws->tmaps + 2 * MAX_EVO : nullptr);
            CVB_LAUNCH_CHECK(ctx); }
        } else {   // generic two-pass tiles, one launch pair per evolution (derivative sigma > 5)
            cudaStream_t keep = ctx->stream;
            ctx->stream = ds;
            int rc2 = 0;
            for (int e = e0; e < e1 && !rc2; e++) {
                const EvoHost &ev = ws->evo[e];
                rc2 = launch_deriv1(ctx, ev, (e == 0 ? ws->Lt : ws->Lsm) + ev.off, ws->Lx + ev.off, ws->Ly + ev.off, PF, B);
                if (!rc2) rc2 = launch_deriv2(ctx, ev, ws->Lx + ev.off, ws->Ly + ev.off, ws->Ldet + ev.off, PF, B);
            }
            ctx->stream = keep;
            if (rc2) return rc2;
        }
        return 0;
    };
    int octave_first = 0;   // first evolution of the octave being built
    // ---- create_nonlinear_scale_space (lib.rs:193-258)
    // evolution 0: Lt = gaussian_blur(image, base_scale_offset); Lsmooth = Lt
    int rc = launch_separable(ctx, images, P0, ws->Lt + ws->evo[0].off, PF, W, H, B, ws->g0, ws->g0);
    if (rc) return rc;
    // (Lsmooth_0 is Lt_0 itself, lib.rs:201: the derivative kernels read Lt for evolution 0, no copy)
    // contrast factor (contrast_factor.rs:16-64)
    CVB_CUDA(ctx, cudaMemsetAsync(ws->gmax, 0, sizeof(unsigned long long) * B, st));
    CVB_CUDA(ctx, cudaMemsetAsync(ws->hist, 0, sizeof(unsigned) * B * nbins, st));
    CVB_CUDA(ctx, cudaMemsetAsync(ws->npoints, 0, sizeof(unsigned) * B, st));
    // per-row extrema counts: ordered before the first fork, the fused detector response adds to them on the auxiliary stream
    CVB_CUDA(ctx, cudaMemsetAsync(ws->rowcount, 0, sizeof(unsigned) * (size_t)B * R, st));
    rc = launch_separable(ctx, images, P0, ws->tmpA, P0, W, H, B, ws->g1, ws->g1);
    if (rc) return rc;
    { CVB_PROF(ctx, "k_contrast_grad", 4.0 * W * H * B);
    k_scharr_pm_v3<1><<<dim3(cdiv((unsigned)W, SW3), cdiv((unsigned)H, SH3), B), NT, 0, st>>>(ws->tmpA, nullptr, ws->g2, ws->gmax, W, H, P0, P0, nullptr, 0);
    CVB_LAUNCH_CHECK(ctx); }
    {
        unsigned blocks = std::min<unsigned>(cdiv((unsigned)P0, NT), (unsigned)ctx->num_sms * 8);
        { CVB_PROF(ctx, "k_contrast_hist", 4.0 * W * H * B);
        k_contrast_hist<<<dim3(blocks, 1, B), NT, sizeof(unsigned) * nbins, st>>>(ws->g2, ws->gmax, ws->hist, ws->npoints, (int)P0, P0, nbins);
        CVB_LAUNCH_CHECK(ctx); }
        { CVB_PROF(ctx, "k_contrast_final", 0);
        k_contrast_final<<<B, 32, 0, st>>>(ws->gmax, ws->hist, ws->npoints, nbins, ws->cfg.contrast_percentile, ws->evo_octave, E, ws->kc, ws->inv_k);
        CVB_LAUNCH_CHECK(ctx); }
    }
    for (int i = 1; i < E; i++) {
        const EvoHost &e = ws->evo[i];
        const EvoHost &pe = ws->evo[i - 1];
        const float *src = ws->Lt + pe.off;   // previous evolution's final Lt
        size_t src_bs = PF;
        if (e.new_octave) {
            if ((rc = issue_detector_response(octave_first, i))) return rc;
            octave_first = i;
            dim3 blk(32, 8), grd(cdiv((unsigned)e.w, 32), cdiv((unsigned)e.h, 8), B);
            { CVB_PROF(ctx, "k_half_size", 4.0 * ((double)pe.w * pe.h + (double)e.w * e.h) * B);
            k_half_size<<<grd, blk, 0, st>>>(src, ws->tmpC, pe.w, pe.h, src_bs, P0);
            CVB_LAUNCH_CHECK(ctx); }
            src = ws->tmpC; src_bs = P0;
        }
        // Lsmooth = gaussian_blur(Lt, 1.0); Lflow = pm_g2(simple_scharr_x(Lsmooth), simple_scharr_y(Lsmooth), contrast)
        if (ws->fuse_blur_scharr && ws->g1.ks == 5) {
            CVB_PROF(ctx, "k_blur_scharr", 16.0 * e.w * e.h * B);
            CUtensorMap tm;
            const int use_tma = ws->use_tma && (ws->tma_mask & 2) && make_tmap(&tm, src, e.w, e.h, B, src_bs, pitch3(3), SH3 + 6) ? 1 : 0;
            if (!use_tma) memset(&tm, 0, sizeof(tm));
            k_blur_scharr_pm<<<dim3(cdiv((unsigned)e.w, SW3), cdiv((unsigned)e.h, SH3), B), NT, 0, st>>>(
                src, ws->Lsm + e.off, ws->Lflow + e.off, e.w, e.h, src_bs, PF, PF, ws->g1, ws->inv_k + i, MAX_EVO, tm, use_tma);
            CVB_LAUNCH_CHECK(ctx);
        } else {
            rc = launch_separable(ctx, src, src_bs, ws->Lsm + e.off, PF, e.w, e.h, B, ws->g1, ws->g1);
            if (rc) return rc;
            { CVB_PROF(ctx, "k_scharr_pm", 8.0 * e.w * e.h * B);
            k_scharr_pm_v3<0><<<dim3(cdiv((unsigned)e.w, SW3), cdiv((unsigned)e.h, SH3), B), NT, 0, st>>>(ws->Lsm + e.off, ws->Lflow + e.off, nullptr, nullptr, e.w, e.h, PF, PF,
                                                                 ws->inv_k + i, MAX_EVO);
            CVB_LAUNCH_CHECK(ctx); }
        }
        // FED steps: nl launches of at most FED_SMAX fused steps (balanced split); the chain ends in Lt_i
        const int n = (int)e.tau.size();
        const int fed_fuse = fed_fuse_steps();
        const int nl = (n + fed_fuse - 1) / fed_fuse;
        if (nl == 0) {
            CVB_CUDA(ctx, cudaMemcpy2DAsync(ws->Lt + e.off, PF * sizeof(float), src, src_bs * sizeof(float),
                                            (size_t)e.w * e.h * sizeof(float), B, cudaMemcpyDeviceToDevice, st));
        }
        const float *cur = src; size_t cur_bs = src_bs;
        int done = 0;
        for (int l = 0; l < nl; l++) {
            FedSteps fs;
            fs.n = (n - done + (nl - l) - 1) / (nl - l);
            for (int t = 0; t < fs.n; t++) fs.tau[t] = (float)e.tau[(size_t)(done + t)];
            done += fs.n;
            // destinations alternate tmpA/tmpB so that the last one is Lt_i
            float *dst; size_t dst_bs;
            if (l == nl - 1) { dst = ws->Lt + e.off; dst_bs = PF; }
            else if (((nl - 1 - l) & 1) == 1) { dst = ws->tmpA; dst_bs = P0; }
            else { dst = ws->tmpB; dst_bs = P0; }
            { CVB_PROF(ctx, "k_fed", 12.0 * fs.n * e.w * e.h * B);
            const int hx = (fs.n + 3) & ~3;
            dim3 grd(cdiv((unsigned)e.w, (unsigned)(F3_W - 2 * hx)), cdiv((unsigned)e.h, (unsigned)(F3_H - 2 * fs.n)), B);
            k_fed3<<<grd, F3_H * 16, 0, st>>>(cur, ws->Lflow + e.off, dst, e.w, e.h, cur_bs, PF, dst_bs, fs);
            CVB_LAUNCH_CHECK(ctx); }
            cur = dst; cur_bs = dst_bs;
        }
    }
    if ((rc = issue_detector_response(octave_first, E))) return rc;
    // ---- detector_response (detector_response.rs:8-85) is issued per octave from inside the loop above
    if (forked) {   // join the auxiliary stream
        CVB_CUDA(ctx, cudaEventRecord(ws->ev_join, ws->aux));
        CVB_CUDA(ctx, cudaStreamWaitEvent(st, ws->ev_join, 0));
    }
    return 0;
}

// detect_keypoints (scale_space_extrema.rs): find_scale_space_extrema + do_subpixel_refinement on the planes of
// stage_scale_space; leaves ncache[b] keypoints per frame in `refined`, valid[] marking the kept ones (the reference's order)
int stage_detect(cvb_ctx *ctx, unsigned B) {
    AkazeWorkspace *ws = ctx->akaze;
    cudaStream_t st = ctx->stream;
    const size_t PF = ws->plane_floats;
    const bool fused_det = ws->deriv_v3 && ws->fuse_det;   // the detector response wrote the extrema mask itself
    const int R = ws->table.total_rows;
    const float thr = (float)ws->cfg.detector_threshold;
    {
        if (!fused_det) { CVB_PROF(ctx, "k_extrema_mask", 4.0 * ws->plane_floats * B);
        k_extrema_mask<<<dim3((unsigned)ws->table.total_tiles, 1, B), NT, 0, st>>>(ws->Ldet, PF, ws->table, ws->tile_evo, ws->mask_layout, thr,
                                                                                    ws->extrema_mask, ws->rowcount);
        CVB_LAUNCH_CHECK(ctx); }
        { CVB_PROF(ctx, "k_scan_rows", 0);
        k_scan_rows<<<B, 1024, 0, st>>>(ws->rowcount, ws->rowoff, ws->ncand, R);
        CVB_LAUNCH_CHECK(ctx); }
        { CVB_PROF(ctx, "k_extrema_emit", 0);
        k_extrema_emit<<<dim3(cdiv((unsigned)R * 32u, NT), 1, B), NT, 0, st>>>(ws->Ldet, PF, ws->table, ws->mask_layout, ws->extrema_mask, ws->rowcount,
                                                                                 ws->rowoff, ws->cand, ws->capc, ws->overflow);
        CVB_LAUNCH_CHECK(ctx); }
    }
    { CVB_PROF(ctx, "k_suppress", 0);
    if (ws->suppress_seq)
        k_suppress_seq<<<B, 1024, 0, st>>>(ws->cand, ws->ncand, ws->capc, ws->table, ws->cache, ws->ncache, ws->nneed, ws->capk,
                                           ws->overflow);
    else {
        k_suppress_smem<<<B, 1024, SUP_SMEM, st>>>(ws->cand, ws->ncand, ws->rowoff, ws->capc, ws->table, ws->sup, ws->cache,
                                                   ws->ncache, ws->nneed, ws->capk, ws->overflow, ws->sup_fallback);
        CVB_LAUNCH_CHECK(ctx);
        k_suppress_par<<<B, 1024, 0, st>>>(ws->cand, ws->ncand, ws->rowoff, ws->capc, ws->table, ws->sup, ws->cache, ws->ncache,
                                           ws->nneed, ws->capk, ws->overflow, ws->suppress_par_only ? nullptr : ws->sup_fallback);
    }
    CVB_LAUNCH_CHECK(ctx); }
    const unsigned kp_blocks = (unsigned)ctx->num_sms * 2;
    const unsigned ichunks = std::min<unsigned>(cdiv(ws->capk, NT), 64u);
    CVB_CUDA(ctx, cudaMemsetAsync(ws->keep, 1, (size_t)B * ws->capk, st));
    { CVB_PROF(ctx, "k_filter_upper", 0);
    k_filter_upper<<<dim3(ichunks, 16, B), NT, 0, st>>>(ws->cache, ws->ncache, ws->capk, ws->keep);
    CVB_LAUNCH_CHECK(ctx); }
    { CVB_PROF(ctx, "k_refine_orient", 0);
    k_refine_orient<<<dim3(kp_blocks, B), NT, 0, st>>>(ws->cache, ws->ncache, ws->capk, ws->keep, ws->table, ws->Ldet, ws->Lx, ws->Ly, PF,
                                                       ws->ot, ws->refined, ws->valid);
    CVB_LAUNCH_CHECK(ctx); }
    return 0;
}

// sort + truncate (lib.rs:326-327) and extract_descriptors (descriptors.rs:16-45) of stage_detect's keypoints, compacted into
// the caller's B x cap_out outputs
int stage_sort_describe(cvb_ctx *ctx, unsigned B, cvb_keypoint *kp_out, unsigned char *desc_out, unsigned cap_out, unsigned *n_out) {
    AkazeWorkspace *ws = ctx->akaze;
    cudaStream_t st = ctx->stream;
    const size_t PF = ws->plane_floats;
    const unsigned ichunks = std::min<unsigned>(cdiv(ws->capk, NT), 64u);
    CVB_CUDA(ctx, cudaMemsetAsync(ws->rank, 0, sizeof(unsigned) * (size_t)B * ws->capk, st));
    CVB_CUDA(ctx, cudaMemsetAsync(ws->nvalid, 0, sizeof(unsigned) * B, st));
    { CVB_PROF(ctx, "k_rank_sort", 0);
    k_rank_count<<<dim3(ichunks, 16, B), NT, 0, st>>>(ws->refined, ws->valid, ws->ncache, ws->capk, ws->rank);
    CVB_LAUNCH_CHECK(ctx);
    k_rank_scatter<<<dim3(ichunks, B), NT, 0, st>>>(ws->refined, ws->valid, ws->ncache, ws->capk, ws->rank,
                                                    (long long)ws->cfg.maximum_features, ws->sorted, ws->nvalid);
    CVB_LAUNCH_CHECK(ctx);
    k_clamp_count<<<cdiv(B, 32), 32, 0, st>>>(ws->nvalid, (long long)ws->cfg.maximum_features, ws->nsorted, (int)B);
    CVB_LAUNCH_CHECK(ctx); }
    // ---- extract_descriptors (descriptors.rs:16-45)
    { CVB_PROF(ctx, "k_descriptors", 0);
    k_descriptors<<<dim3((unsigned)ctx->num_sms * 8, B), DESC_WARPS * 32, 0, st>>>(ws->sorted, ws->nsorted, nullptr, ws->capk, ws->table, ws->Lt,
                                                     ws->Lx, ws->Ly, PF, ws->dt, (int)ws->cfg.descriptor_channels,
                                                     (int)ws->cfg.descriptor_pattern_size, ws->desc_tmp, ws->ok, ws->overflow);
    CVB_LAUNCH_CHECK(ctx); }
    { CVB_PROF(ctx, "k_compact_final", 0);
    k_compact_final<<<B, 1024, 0, st>>>(ws->sorted, ws->desc_tmp, ws->ok, ws->nsorted, ws->capk, kp_out, desc_out, cap_out, n_out,
                                        ws->overflow);
    CVB_LAUNCH_CHECK(ctx); }
    return 0;
}

// The whole extractor for `B` frames already resident in `images` (device).  Asynchronous.
int run_extract_eager(cvb_ctx *ctx, const float *images, unsigned B, cvb_keypoint *kp_out, unsigned char *desc_out,
                      unsigned cap_out, unsigned *n_out) {
    AkazeWorkspace *ws = ctx->akaze;
    if (ws->evo.empty()) {   // image too small for a single octave: the reference returns no keypoints
        CVB_CUDA(ctx, cudaMemsetAsync(n_out, 0, sizeof(unsigned) * B, ctx->stream));
        ws->has_run = true;
        return 0;
    }
    int rc = stage_scale_space(ctx, images, B);
    if (!rc) rc = stage_detect(ctx, B);
    if (!rc) rc = stage_sort_describe(ctx, B, kp_out, desc_out, cap_out, n_out);
    if (rc) return rc;
    ws->has_run = true;
    return 0;
}

// Front end: replay the whole extractor as one CUDA graph (captured once per distinct set of caller buffers);
// falls back to eager launches while profiling or when capture is unavailable.
int run_extract(cvb_ctx *ctx, const float *images, unsigned B, cvb_keypoint *kp_out, unsigned char *desc_out,
                unsigned cap_out, unsigned *n_out) {
    AkazeWorkspace *ws = ctx->akaze;
    ws->ticket = 0;   // the planes no longer hold a staged scale space
    if (!ws->use_graph || ctx->prof || ws->evo.empty()) return run_extract_eager(ctx, images, B, kp_out, desc_out, cap_out, n_out);
    for (auto &g : ws->graphs)
        if (g.img == images && g.kp == kp_out && g.desc == desc_out && g.n == n_out && g.B == B && g.cap == cap_out) {
            CVB_CUDA(ctx, cudaGraphLaunch(g.exec, ctx->stream));
            ctx->launches += ws->launches_per_graph;
            ws->has_run = true;
            return 0;
        }
    const uint64_t l0 = ctx->launches;
    cudaGraph_t graph = nullptr;
    CVB_CUDA(ctx, cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeThreadLocal));
    int rc = run_extract_eager(ctx, images, B, kp_out, desc_out, cap_out, n_out);
    cudaError_t ce = cudaStreamEndCapture(ctx->stream, &graph);
    if (rc) { if (graph) cudaGraphDestroy(graph); return rc; }
    if (ce != cudaSuccess || !graph) {   // capture not possible: run eagerly from now on
        cudaGetLastError();
        ws->use_graph = false;
        return run_extract_eager(ctx, images, B, kp_out, desc_out, cap_out, n_out);
    }
    ws->launches_per_graph = ctx->launches - l0;
    cudaGraphExec_t exec = nullptr;
    ce = cudaGraphInstantiate(&exec, graph, 0);
    cudaGraphDestroy(graph);
    if (ce != cudaSuccess) {
        cudaGetLastError();
        ws->use_graph = false;
        return run_extract_eager(ctx, images, B, kp_out, desc_out, cap_out, n_out);
    }
    if (ws->graphs.size() >= 32) { cudaGraphExecDestroy(ws->graphs.front().exec); ws->graphs.erase(ws->graphs.begin()); }
    ws->graphs.push_back({images, kp_out, desc_out, n_out, B, cap_out, exec});
    CVB_CUDA(ctx, cudaGraphLaunch(exec, ctx->stream));
    ws->has_run = true;
    return 0;
}

int check_args(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, const void *img, uint32_t batch, uint32_t w, uint32_t h) {
    if (!ctx) return CVB_EINVAL;
    if (!cfg || !img) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    if (batch == 0 || w == 0 || h == 0) return cvb_set_error(ctx, CVB_EINVAL, "empty image or batch");
    if ((uint64_t)w * h > (1ull << 28)) return cvb_set_error(ctx, CVB_EUNSUPPORTED, "image too large");
    return 0;
}


}  // namespace

extern "C" {

void cvb_akaze_default_cfg(cvb_akaze_cfg *c) {
    if (!c) return;
    c->maximum_features = -1;
    c->num_sublevels = 4; c->max_octave_evolution = 4;
    c->base_scale_offset = 1.6; c->initial_contrast = 0.001; c->contrast_percentile = 0.7;
    c->contrast_factor_num_bins = 300; c->derivative_factor = 1.5; c->detector_threshold = 0.001;
    c->descriptor_channels = 3; c->descriptor_pattern_size = 10;
}

int cvb_akaze_extract_batch_dev(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, const float *images_dev, uint32_t batch, uint32_t w,
                                uint32_t h, cvb_keypoint *kp_out_dev, uint8_t *desc_out_dev, uint32_t cap, uint32_t *n_out_dev) {
    int rc = check_args(ctx, cfg, images_dev, batch, w, h);
    if (rc) return rc;
    if (!kp_out_dev || !desc_out_dev || !n_out_dev) return cvb_set_error(ctx, CVB_EINVAL, "null output");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    rc = ensure_workspace(ctx, cfg, batch, w, h, ctx->akaze ? ctx->akaze->cap_out : 1);
    if (rc) return rc;
    return run_extract(ctx, images_dev, batch, kp_out_dev, desc_out_dev, cap, n_out_dev);
}

int cvb_akaze_dev_overflow(cvb_ctx *ctx, uint32_t *flag_out) {
    if (!ctx || !flag_out) return CVB_EINVAL;
    *flag_out = 0;
    AkazeWorkspace *ws = ctx->akaze;
    if (!ws) return 0;
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    unsigned *hs = (unsigned *)cvb_pinned(ctx, sizeof(unsigned));
    if (!hs) return cvb_set_error(ctx, CVB_ENOMEM, "page-locked scratch");
    CVB_CUDA(ctx, cudaMemcpyAsync(hs, ws->overflow, sizeof(unsigned), cudaMemcpyDeviceToHost, ctx->stream));
    CVB_CUDA(ctx, cudaMemsetAsync(ws->overflow, 0, sizeof(unsigned), ctx->stream));
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    *flag_out = hs[0];
    return 0;
}

int cvb_akaze_extract_batch(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, const float *images, uint32_t batch, uint32_t w, uint32_t h,
                            cvb_keypoint *kp_out, uint8_t *desc_out, uint32_t cap, uint32_t *n_out) {
    return akaze_extract_batch_host(ctx, cfg, images, false, batch, w, h, kp_out, desc_out, cap, n_out);
}

}  // extern "C"

// Clears the overflow flag on the context's stream, so that the flag a host call reads back belongs to that call alone.
int akaze_clear_overflow(cvb_ctx *ctx) {
    if (ctx->akaze) CVB_CUDA(ctx, cudaMemsetAsync(ctx->akaze->overflow, 0, sizeof(unsigned), ctx->stream));
    return 0;
}

// The host calls' answer to an overflow flag of their last detection (B frames): did a frame need more than capc candidates or
// capk cached keypoints?  ncand is never clamped.  nneed is exact when every candidate fit; when the candidates were clamped at
// capc the suppression saw only the first capc of them, so nneed can fall short of the frame's need and a second rerun can be
// needed.  *rerun: the capacities were grown to the need and the detection is to run again.  After MAX_CAPACITY_RERUNS reruns an
// exceeded capacity is CVB_ECAP.
int akaze_capacity_rerun(cvb_ctx *ctx, unsigned B, int attempt, bool *rerun) {
    constexpr int MAX_CAPACITY_RERUNS = 2;
    AkazeWorkspace *ws = ctx->akaze;
    cudaStream_t st = ctx->stream;
    *rerun = false;
    unsigned *hs = (unsigned *)cvb_pinned(ctx, sizeof(unsigned) * 2 * (size_t)B);
    if (!hs) return cvb_set_error(ctx, CVB_ENOMEM, "page-locked scratch");
    CVB_CUDA(ctx, cudaMemcpyAsync(hs, ws->ncand, sizeof(unsigned) * B, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(hs + B, ws->nneed, sizeof(unsigned) * B, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    size_t need_c = 0, need_k = 0;
    for (unsigned b = 0; b < B; b++) { need_c = std::max<size_t>(need_c, hs[b]); need_k = std::max<size_t>(need_k, hs[B + b]); }
    if (need_c <= ws->capc && need_k <= ws->capk) return 0;
    if (attempt >= MAX_CAPACITY_RERUNS)
        return cvb_set_error(ctx, CVB_ECAP, "internal keypoint capacity exceeded after %d reruns", MAX_CAPACITY_RERUNS);
    int rc = grow_keypoint_capacity(ctx, ws, need_c, need_k);
    if (rc) return rc;
    CVB_CUDA(ctx, cudaMemsetAsync(ws->overflow, 0, sizeof(unsigned), st));
    *rerun = true;
    return 0;
}

int akaze_extract_batch_host(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, const float *images, bool images_on_device, uint32_t batch, uint32_t w,
                             uint32_t h, cvb_keypoint *kp_out, uint8_t *desc_out, uint32_t cap, uint32_t *n_out) {
    int rc = check_args(ctx, cfg, images, batch, w, h);
    if (rc) return rc;
    if (!n_out || (cap && (!kp_out || !desc_out))) return cvb_set_error(ctx, CVB_EINVAL, "null output");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    rc = ensure_workspace(ctx, cfg, batch, w, h, std::max<uint32_t>(cap, 1));
    if (rc) return rc;
    AkazeWorkspace *ws = ctx->akaze;
    cudaStream_t st = ctx->stream;
    if (!images_on_device) CVB_CUDA(ctx, cudaMemcpyAsync(ws->img, images, sizeof(float) * ws->p0 * batch, cudaMemcpyHostToDevice, st));
    const unsigned cap_dev = ws->cap_out;
    // the frames stay resident, so a frame that exceeds the keypoint capacities is run again in a grown workspace
    if ((rc = akaze_clear_overflow(ctx))) return rc;
    bool out_full = false;
    for (int attempt = 0;; attempt++) {
        rc = run_extract(ctx, images_on_device ? images : ws->img, batch, ws->kp_out, ws->desc_out, cap_dev, ws->n_out);
        if (rc) return rc;
        unsigned *hs = (unsigned *)cvb_pinned(ctx, sizeof(unsigned) * ((size_t)batch + 1));
        if (!hs) return cvb_set_error(ctx, CVB_ENOMEM, "page-locked scratch");
        CVB_CUDA(ctx, cudaMemcpyAsync(hs, ws->n_out, sizeof(unsigned) * batch, cudaMemcpyDeviceToHost, st));
        CVB_CUDA(ctx, cudaMemcpyAsync(hs + batch, ws->overflow, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
        CVB_CUDA(ctx, cvb_wait(ctx, st));
        const unsigned ovf = hs[batch];
        for (uint32_t b = 0; b < batch; b++) n_out[b] = hs[b];
        if (!ovf) break;
        bool rerun = false;
        if ((rc = akaze_capacity_rerun(ctx, batch, attempt, &rerun))) return rc;
        if (rerun) continue;
        out_full = ovf == 3;
        CVB_CUDA(ctx, cudaMemsetAsync(ws->overflow, 0, sizeof(unsigned), st));
        break;
    }
    // the workspace's outputs may hold more than `cap` (a workspace built for a larger cap), so the counts decide too
    for (uint32_t b = 0; b < batch; b++) out_full = out_full || n_out[b] > cap;
    if (out_full) return cvb_set_error(ctx, CVB_ECAP, "output capacity %u too small", cap);
    for (uint32_t b = 0; b < batch; b++) {
        unsigned n = std::min<unsigned>(n_out[b], cap);
        if (!n) continue;
        CVB_CUDA(ctx, cudaMemcpyAsync(kp_out + (size_t)b * cap, ws->kp_out + (size_t)b * cap_dev, sizeof(cvb_keypoint) * n,
                                      cudaMemcpyDeviceToHost, st));
        CVB_CUDA(ctx, cudaMemcpyAsync(desc_out + (size_t)b * cap * 64, ws->desc_out + (size_t)b * cap_dev * 64, (size_t)n * 64,
                                      cudaMemcpyDeviceToHost, st));
    }
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    return 0;
}

// ---- staged calls: the bodies of include/cvb200_stages.h (exported by stages_abi.cu, libcvb200_stages.so) ---------------------

namespace {

std::atomic<uint64_t> g_scale_space_tickets{0};   // process-wide, so that a ticket of one context is unknown to every other

int check_ticket(cvb_ctx *ctx, uint64_t ticket) {
    if (!ctx) return CVB_EINVAL;
    if (!ticket || !ctx->akaze || ctx->akaze->ticket != ticket)
        return cvb_set_error(ctx, CVB_EINVAL, "scale space replaced: the ticket is stale or unknown to this context");
    return 0;
}

// the descriptor tables of a describe config: the workspace's own when the config matches the scale space's, else side tables
// built on demand (the scale space and its ticket stay as they are)
int desc_tables_for(cvb_ctx *ctx, AkazeWorkspace *ws, const cvb_akaze_cfg *cfg, const DescTables **out) {
    if (cfg->descriptor_channels < 1 || cfg->descriptor_channels > 3) return cvb_set_error(ctx, CVB_EINVAL, "descriptor_channels must be 1..3");
    if (cfg->descriptor_pattern_size == ws->cfg.descriptor_pattern_size && cfg->descriptor_channels == ws->cfg.descriptor_channels) {
        *out = ws->dt;
        return 0;
    }
    if (cfg->descriptor_pattern_size > (uint64_t)DESC_MAXLAT)
        return cvb_set_error(ctx, CVB_EUNSUPPORTED, "descriptor_pattern_size %llu out of range", (unsigned long long)cfg->descriptor_pattern_size);
    const int pattern = (int)cfg->descriptor_pattern_size, nch = (int)cfg->descriptor_channels;
    if (ws->dt_side_pattern != pattern || ws->dt_side_nch != nch) {
        DescTables dt;
        int rc = make_desc_tables(ctx, pattern, nch, &dt);
        if (rc) return rc;
        CVB_CUDA(ctx, cudaMemcpyAsync(ws->dt_side, &dt, sizeof(dt), cudaMemcpyHostToDevice, ctx->stream));
        CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
        ws->dt_side_pattern = pattern; ws->dt_side_nch = nch;
    }
    *out = ws->dt_side;
    return 0;
}

}  // namespace

int stages_scale_space(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, const float *images, bool on_device, uint32_t batch, uint32_t w,
                       uint32_t h, uint64_t *ticket_out) {
    int rc = check_args(ctx, cfg, images, batch, w, h);
    if (rc) return rc;
    if (!ticket_out) return cvb_set_error(ctx, CVB_EINVAL, "null output");
    *ticket_out = 0;
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    rc = ensure_workspace(ctx, cfg, batch, w, h, ctx->akaze ? ctx->akaze->cap_out : 1);
    if (rc) return rc;
    AkazeWorkspace *ws = ctx->akaze;
    ws->ticket = 0;
    if (!on_device) CVB_CUDA(ctx, cudaMemcpyAsync(ws->img, images, sizeof(float) * ws->p0 * batch, cudaMemcpyHostToDevice, ctx->stream));
    if (!ws->evo.empty()) {
        rc = stage_scale_space(ctx, on_device ? images : ws->img, batch);
        if (rc) return rc;
    }
    if (!on_device) CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    ws->ss_batch = batch;
    ws->ticket = ++g_scale_space_tickets;
    *ticket_out = ws->ticket;
    return 0;
}

int stages_evolutions(cvb_ctx *ctx, uint64_t ticket, cvb_akaze_evolution *out, uint32_t cap, uint32_t *n_out) {
    int rc = check_ticket(ctx, ticket);
    if (rc) return rc;
    if (!n_out || (cap && !out)) return cvb_set_error(ctx, CVB_EINVAL, "null output");
    const AkazeWorkspace *ws = ctx->akaze;
    *n_out = (uint32_t)ws->evo.size();
    for (size_t i = 0; i < ws->evo.size() && i < cap; i++) {
        const EvoHost &e = ws->evo[i];
        // sigma_size is EvolutionStep's `esigma.round() as u32` (evolution.rs:58; round() is half away from zero), not the
        // derivative scale of the detector response (EvoHost::sigma, detector_response.rs:13)
        out[i] = cvb_akaze_evolution{e.octave, e.sublevel, e.esigma, e.etime, (uint32_t)round(e.esigma), (uint32_t)e.w, (uint32_t)e.h,
                                     (uint32_t)e.tau.size()};
    }
    return 0;
}

int stages_find(cvb_ctx *ctx, uint64_t ticket, cvb_keypoint *kp_out, uint32_t cap, uint32_t *n_out, bool on_device) {
    int rc = check_ticket(ctx, ticket);
    if (rc) return rc;
    if (!n_out || (cap && !kp_out)) return cvb_set_error(ctx, CVB_EINVAL, "null output");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    AkazeWorkspace *ws = ctx->akaze;
    cudaStream_t st = ctx->stream;
    const unsigned B = ws->ss_batch;
    if (ws->evo.empty()) {   // no octave: no keypoints (lib.rs:268-276 over an empty evolution table)
        if (on_device) CVB_CUDA(ctx, cudaMemsetAsync(n_out, 0, sizeof(unsigned) * B, st));
        else memset(n_out, 0, sizeof(unsigned) * B);
        return 0;
    }
    // detection runs on every call, so that every _dev find reports its own capacity overflows (flags 1 and 2), and the host call
    // runs it again in a grown workspace (the planes, and so the ticket, stay).  It reads the planes and the per-row extrema counts
    // of the scale space; the unfused extrema mask adds to those counts, so they restart from 0.
    if (!on_device && (rc = akaze_clear_overflow(ctx))) return rc;   // the host call reads back this call's flag alone
    std::vector<unsigned> got(B), need(B);
    for (int attempt = 0;; attempt++) {
        if (!(ws->deriv_v3 && ws->fuse_det))
            CVB_CUDA(ctx, cudaMemsetAsync(ws->rowcount, 0, sizeof(unsigned) * (size_t)B * ws->table.total_rows, st));
        if ((rc = stage_detect(ctx, B))) return rc;
        CompactArgs A{};
        A.kp_in = ws->refined; A.keep = ws->valid; A.counts = ws->ncache; A.in_stride = ws->capk; A.cap = cap;
        A.overflow = ws->overflow;
        if (on_device) {
            A.kp_out = kp_out; A.n_out = n_out;
        } else {
            if ((rc = ws_grow(ctx, &ws->st_kp_out, &ws->st_kp_out_n, (size_t)B * cap))) return rc;
            if ((rc = ws_grow(ctx, &ws->st_n, &ws->st_n_n, B))) return rc;
            if ((rc = ws_grow(ctx, &ws->st_need, &ws->st_need_n, B))) return rc;
            A.kp_out = ws->st_kp_out; A.n_out = ws->st_n; A.need = ws->st_need;
        }
        { CVB_PROF(ctx, "k_compact_stage", 0);
        k_compact_stage<<<B, 1024, 0, st>>>(A);
        CVB_LAUNCH_CHECK(ctx); }
        if (on_device) return 0;
        unsigned *hs = (unsigned *)cvb_pinned(ctx, sizeof(unsigned) * (2 * (size_t)B + 1));
        if (!hs) return cvb_set_error(ctx, CVB_ENOMEM, "page-locked scratch");
        CVB_CUDA(ctx, cudaMemcpyAsync(hs, ws->st_n, sizeof(unsigned) * B, cudaMemcpyDeviceToHost, st));
        CVB_CUDA(ctx, cudaMemcpyAsync(hs + B, ws->st_need, sizeof(unsigned) * B, cudaMemcpyDeviceToHost, st));
        CVB_CUDA(ctx, cudaMemcpyAsync(hs + 2 * B, ws->overflow, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
        CVB_CUDA(ctx, cvb_wait(ctx, st));
        const unsigned ovf = hs[2 * B];
        got.assign(hs, hs + B); need.assign(hs + B, hs + 2 * B);
        if (!ovf) break;
        bool rerun = false;
        if ((rc = akaze_capacity_rerun(ctx, B, attempt, &rerun))) return rc;
        if (rerun) continue;
        CVB_CUDA(ctx, cudaMemsetAsync(ws->overflow, 0, sizeof(unsigned), st));
        break;   // flag 3: the output, handled below
    }
    for (unsigned b = 0; b < B; b++)
        if (need[b] > cap) {
            for (unsigned c = 0; c < B; c++) n_out[c] = need[c];
            return cvb_set_error(ctx, CVB_ECAP, "output capacity %u too small: frame %u has %u keypoints", cap, b, need[b]);
        }
    for (unsigned b = 0; b < B; b++) {
        n_out[b] = got[b];
        if (got[b])
            CVB_CUDA(ctx, cudaMemcpyAsync(kp_out + (size_t)b * cap, ws->st_kp_out + (size_t)b * cap, sizeof(cvb_keypoint) * got[b],
                                          cudaMemcpyDeviceToHost, st));
    }
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    return 0;
}

int stages_describe(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, uint64_t ticket, const cvb_keypoint *kp_in, const uint32_t *offsets,
                    uint32_t total_max, cvb_keypoint *kp_out, uint8_t *desc_out, uint32_t *n_out, bool on_device) {
    int rc = check_ticket(ctx, ticket);
    if (rc) return rc;
    if (!cfg || !offsets || !n_out) return cvb_set_error(ctx, CVB_EINVAL, "null argument");
    CVB_CUDA(ctx, cudaSetDevice(ctx->device));
    AkazeWorkspace *ws = ctx->akaze;
    cudaStream_t st = ctx->stream;
    const unsigned B = ws->ss_batch;
    const DescTables *dt = nullptr;
    if ((rc = desc_tables_for(ctx, ws, cfg, &dt))) return rc;
    size_t total = total_max;
    if (!on_device) {   // the checks the _dev kernel makes per keypoint, with the first offender named
        for (unsigned b = 0; b < B; b++)
            if (offsets[b] > offsets[b + 1]) return cvb_set_error(ctx, CVB_EINVAL, "offsets[%u] > offsets[%u]", b, b + 1);
        total = offsets[B];
        if (total > offsets[0] && !kp_in) return cvb_set_error(ctx, CVB_EINVAL, "null keypoint buffer");
        const uint32_t E = (uint32_t)ws->evo.size();
        for (size_t i = offsets[0]; i < total; i++) {
            if (kp_in[i].class_id >= E)
                return cvb_set_error(ctx, CVB_EINVAL, "keypoint %zu: class_id %u, the scale space has %u evolutions", i, kp_in[i].class_id, E);
            if (kp_in[i].octave >= 32) return cvb_set_error(ctx, CVB_EINVAL, "keypoint %zu: octave %u >= 32", i, kp_in[i].octave);
        }
    }
    if (total && (!kp_in || !kp_out || !desc_out)) return cvb_set_error(ctx, CVB_EINVAL, "null keypoint or descriptor buffer");
    if (total > 0xffffffffull) return cvb_set_error(ctx, CVB_EUNSUPPORTED, "too many keypoints");
    if ((rc = ws_grow(ctx, &ws->st_ok, &ws->st_ok_n, total))) return rc;
    if ((rc = ws_grow(ctx, &ws->st_desc, &ws->st_desc_n, total * 64))) return rc;
    CompactArgs A{};
    A.desc_in = ws->st_desc; A.keep = ws->st_ok; A.in_stride = (unsigned)total; A.overflow = ws->overflow;
    const cvb_keypoint *kin = kp_in;
    if (on_device) {
        A.offs = offsets; A.kp_out = kp_out; A.desc_out = desc_out; A.n_out = n_out;
    } else {
        if ((rc = ws_grow(ctx, &ws->st_kp, &ws->st_kp_n, total))) return rc;
        if ((rc = ws_grow(ctx, &ws->st_kp_out, &ws->st_kp_out_n, total))) return rc;
        if ((rc = ws_grow(ctx, &ws->st_desc_out, &ws->st_desc_out_n, total * 64))) return rc;
        if ((rc = ws_grow(ctx, &ws->st_off, &ws->st_off_n, (size_t)B + 1))) return rc;
        if ((rc = ws_grow(ctx, &ws->st_n, &ws->st_n_n, B))) return rc;
        if (total) CVB_CUDA(ctx, cudaMemcpyAsync(ws->st_kp, kp_in, sizeof(cvb_keypoint) * total, cudaMemcpyHostToDevice, st));
        CVB_CUDA(ctx, cudaMemcpyAsync(ws->st_off, offsets, sizeof(unsigned) * ((size_t)B + 1), cudaMemcpyHostToDevice, st));
        kin = ws->st_kp;
        A.offs = ws->st_off; A.kp_out = ws->st_kp_out; A.desc_out = ws->st_desc_out; A.n_out = ws->st_n;
    }
    A.kp_in = kin;
    { CVB_PROF(ctx, "k_descriptors", 0);
    k_descriptors<<<dim3((unsigned)ctx->num_sms * 8, B), DESC_WARPS * 32, 0, st>>>(kin, nullptr, A.offs, (unsigned)total, ws->table, ws->Lt,
                                                     ws->Lx, ws->Ly, ws->plane_floats, dt, (int)cfg->descriptor_channels,
                                                     (int)cfg->descriptor_pattern_size, ws->st_desc, ws->st_ok, ws->overflow);
    CVB_LAUNCH_CHECK(ctx); }
    { CVB_PROF(ctx, "k_compact_stage", 0);
    k_compact_stage<<<B, 1024, 0, st>>>(A);
    CVB_LAUNCH_CHECK(ctx); }
    if (on_device) return 0;
    unsigned *hs = (unsigned *)cvb_pinned(ctx, sizeof(unsigned) * B);
    if (!hs) return cvb_set_error(ctx, CVB_ENOMEM, "page-locked scratch");
    CVB_CUDA(ctx, cudaMemcpyAsync(hs, ws->st_n, sizeof(unsigned) * B, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    std::vector<unsigned> got(hs, hs + B);
    for (unsigned b = 0; b < B; b++) {
        n_out[b] = got[b];
        if (!got[b]) continue;
        const size_t o = offsets[b];
        CVB_CUDA(ctx, cudaMemcpyAsync(kp_out + o, ws->st_kp_out + o, sizeof(cvb_keypoint) * got[b], cudaMemcpyDeviceToHost, st));
        CVB_CUDA(ctx, cudaMemcpyAsync(desc_out + o * 64, ws->st_desc_out + o * 64, (size_t)got[b] * 64, cudaMemcpyDeviceToHost, st));
    }
    CVB_CUDA(ctx, cvb_wait(ctx, st));
    return 0;
}

extern "C" {

int cvb_akaze_extract(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, const float *image, uint32_t w, uint32_t h, cvb_keypoint *kp_out,
                      uint8_t *desc_out, uint32_t cap, uint32_t *n_out) {
    return cvb_akaze_extract_batch(ctx, cfg, image, 1, w, h, kp_out, desc_out, cap, n_out);
}

// ---- introspection for the parity tests ------------------------------------------------------
int cvb_akaze_debug_num_evolutions(cvb_ctx *ctx, uint32_t *n_out) {
    if (!ctx || !n_out) return CVB_EINVAL;
    if (!ctx->akaze || !ctx->akaze->has_run) return cvb_set_error(ctx, CVB_EINVAL, "no extract call yet");
    *n_out = (uint32_t)ctx->akaze->evo.size();
    return 0;
}

int cvb_akaze_debug_evolution(cvb_ctx *ctx, uint32_t i, uint32_t *w, uint32_t *h, uint32_t *octave, uint32_t *sigma_size,
                              uint32_t *n_fed_steps) {
    if (!ctx) return CVB_EINVAL;
    if (!ctx->akaze || !ctx->akaze->has_run || i >= ctx->akaze->evo.size()) return cvb_set_error(ctx, CVB_EINVAL, "bad evolution");
    const EvoHost &e = ctx->akaze->evo[i];
    if (w) *w = (uint32_t)e.w;
    if (h) *h = (uint32_t)e.h;
    if (octave) *octave = e.octave;
    if (sigma_size) *sigma_size = e.sigma;
    if (n_fed_steps) *n_fed_steps = (uint32_t)e.tau.size();
    return 0;
}

int cvb_akaze_debug_plane(cvb_ctx *ctx, uint32_t frame, uint32_t i, uint32_t plane, float *out) {
    if (!ctx || !out) return CVB_EINVAL;
    AkazeWorkspace *ws = ctx->akaze;
    if (!ws || !ws->has_run || i >= ws->evo.size() || frame >= ws->batch) return cvb_set_error(ctx, CVB_EINVAL, "bad frame/evolution");
    const float *planes[6] = {ws->Lt, ws->Lsm, ws->Lx, ws->Ly, ws->Lflow, ws->Ldet};
    if (plane >= 6) return cvb_set_error(ctx, CVB_EINVAL, "bad plane");
    const EvoHost &e = ws->evo[i];
    if (plane == 1 && i == 0) plane = 0;   // Lsmooth_0 is Lt_0 (lib.rs:201)
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    CVB_CUDA(ctx, cudaMemcpy(out, planes[plane] + (size_t)frame * ws->plane_floats + e.off, sizeof(float) * (size_t)e.w * e.h,
                             cudaMemcpyDeviceToHost));
    return 0;
}

int cvb_akaze_debug_contrast(cvb_ctx *ctx, uint32_t frame, double *k_out) {
    if (!ctx || !k_out) return CVB_EINVAL;
    AkazeWorkspace *ws = ctx->akaze;
    if (!ws || !ws->has_run || frame >= ws->batch) return cvb_set_error(ctx, CVB_EINVAL, "bad frame");
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    CVB_CUDA(ctx, cudaMemcpy(k_out, ws->kc + frame, sizeof(double), cudaMemcpyDeviceToHost));
    return 0;
}

int cvb_akaze_debug_stage(cvb_ctx *ctx, uint32_t frame, uint32_t stage, cvb_keypoint *out, uint32_t cap, uint32_t *n_out) {
    if (!ctx || !n_out) return CVB_EINVAL;
    AkazeWorkspace *ws = ctx->akaze;
    if (!ws || !ws->has_run || frame >= ws->batch) return cvb_set_error(ctx, CVB_EINVAL, "bad frame");
    CVB_CUDA(ctx, cvb_wait(ctx, ctx->stream));
    std::vector<cvb_keypoint> res;
    if (stage == 0) {
        unsigned n = 0;
        CVB_CUDA(ctx, cudaMemcpy(&n, ws->ncand + frame, sizeof(unsigned), cudaMemcpyDeviceToHost));
        n = std::min(n, ws->capc);
        std::vector<Cand> c(n);
        if (n) CVB_CUDA(ctx, cudaMemcpy(c.data(), ws->cand + (size_t)frame * ws->capc, sizeof(Cand) * n, cudaMemcpyDeviceToHost));
        for (unsigned i = 0; i < n; i++) {
            cvb_keypoint k{};
            const EvoHost &e = ws->evo[(size_t)c[i].e];
            k.x = (float)c[i].x; k.y = (float)c[i].y; k.response = fabsf(c[i].v);
            k.size = (float)(e.esigma * ws->cfg.derivative_factor); k.angle = 0.f; k.octave = e.octave; k.class_id = (uint32_t)c[i].e;
            res.push_back(k);
        }
    } else if (stage == 1 || stage == 2) {
        unsigned n = 0;
        CVB_CUDA(ctx, cudaMemcpy(&n, ws->ncache + frame, sizeof(unsigned), cudaMemcpyDeviceToHost));
        std::vector<cvb_keypoint> k(n);
        std::vector<unsigned char> f(n);
        const cvb_keypoint *src = stage == 1 ? ws->cache : ws->refined;
        const unsigned char *flg = stage == 1 ? ws->keep : ws->valid;
        if (n) {
            CVB_CUDA(ctx, cudaMemcpy(k.data(), src + (size_t)frame * ws->capk, sizeof(cvb_keypoint) * n, cudaMemcpyDeviceToHost));
            CVB_CUDA(ctx, cudaMemcpy(f.data(), flg + (size_t)frame * ws->capk, n, cudaMemcpyDeviceToHost));
        }
        for (unsigned i = 0; i < n; i++)
            if (f[i]) res.push_back(k[i]);
    } else if (stage == 3) {
        unsigned n = 0;
        CVB_CUDA(ctx, cudaMemcpy(&n, ws->nsorted + frame, sizeof(unsigned), cudaMemcpyDeviceToHost));
        res.resize(n);
        if (n) CVB_CUDA(ctx, cudaMemcpy(res.data(), ws->sorted + (size_t)frame * ws->capk, sizeof(cvb_keypoint) * n, cudaMemcpyDeviceToHost));
    } else return cvb_set_error(ctx, CVB_EINVAL, "bad stage");
    *n_out = (uint32_t)res.size();
    if (out)
        for (size_t i = 0; i < res.size() && i < cap; i++) out[i] = res[i];
    return 0;
}

}  // extern "C"
