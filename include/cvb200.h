/* include/cvb200.h -- C ABI of libcvb200.so: the H100-native drop-in for rust-cv's
 * AKAZE -> brute-force Hamming match -> RANSAC hot path.
 *
 * The reference (rust-cv/cv @ 82a25ee3) has no FFI; its boundary is the Rust-level API listed
 * below.  Each entry point here is what a thin Rust shim crate would bind with `extern "C"`
 * (see INTEGRATION.md) to keep those Rust surfaces unchanged:
 *
 *   cvb_akaze_extract*      <- akaze::Akaze::extract_from_gray_float_image   akaze/src/lib.rs:309-339
 *                              (and Akaze::extract / extract_path :295,361 after GrayFloatImage::from_dynamic)
 *   cvb_akaze_cfg           <- akaze::Akaze (11 pub fields)                   akaze/src/lib.rs:109-142
 *   cvb_keypoint            <- akaze::KeyPoint                                akaze/src/lib.rs:71-93
 *   cvb_hamming_knn*        <- space::Knn::knn on LinearKnn<Hamming, BitArray<64>>
 *                              call sites akaze/tests/estimate_pose.rs:78-97,
 *                              tutorial-code/chapter4-feature-matching/src/main.rs:91-106
 *   cvb_match_symmetric*    <- cv-sfm symmetric_matching (d0 + better_by <= d1, cross-check)
 *                              cv-sfm/src/lib.rs:3097-3133
 *
 * Conventions: every function returns 0 on success or a negative CVB_E* code and never throws
 * or aborts across the boundary; `cvb_last_error` gives the message for the last failure on a
 * context.  The caller owns every buffer.  Functions without a `_dev` suffix take HOST pointers
 * and perform the host<->device copies themselves; `_dev` variants take DEVICE pointers on the
 * context's device and are asynchronous on the context's stream until `cvb_ctx_sync`.
 * A context owns one CUDA stream and its workspaces; it is not thread-safe, distinct contexts
 * are.  There is NO CPU fallback: without a CUDA device `cvb_ctx_create` fails with CVB_ENODEV.
 */
#ifndef CVB200_H
#define CVB200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CVB_OK 0
#define CVB_EINVAL (-1)   /* bad argument */
#define CVB_ENODEV (-2)   /* no usable CUDA device */
#define CVB_ECUDA (-3)    /* CUDA runtime error (see cvb_last_error) */
#define CVB_ENOMEM (-4)   /* allocation failed */
#define CVB_ECAP (-5)     /* output capacity too small; *n_out holds the required count */
#define CVB_EUNSUPPORTED (-6)

typedef struct cvb_ctx cvb_ctx;

/* akaze::Akaze, akaze/src/lib.rs:109-142.  maximum_features < 0 means usize::MAX. */
typedef struct {
    int64_t maximum_features;
    uint32_t num_sublevels;
    uint32_t max_octave_evolution;
    double base_scale_offset;
    double initial_contrast;      /* present for layout parity; never read (lib.rs:123,176) */
    double contrast_percentile;
    uint64_t contrast_factor_num_bins;
    double derivative_factor;
    double detector_threshold;
    uint64_t descriptor_channels;
    uint64_t descriptor_pattern_size;
} cvb_akaze_cfg;

/* akaze::KeyPoint, akaze/src/lib.rs:71-93 (point.0, point.1, response, size, angle, octave, class_id) */
typedef struct {
    float x, y;
    float response;
    float size;
    float angle;
    uint32_t octave;
    uint32_t class_id;
} cvb_keypoint;

/* ---- context ---------------------------------------------------------------------------- */
int cvb_ctx_create(int device, cvb_ctx **out);
/* Same, but all work is enqueued on an existing CUDA stream (a cudaStream_t passed as void*),
 * e.g. torch.cuda.current_stream().cuda_stream, so the caller can time it with its own events. */
int cvb_ctx_create_on_stream(int device, void *cuda_stream, cvb_ctx **out);
void cvb_ctx_destroy(cvb_ctx *ctx);
/* Waits for the context's stream.  This and every other blocking call of the library SLEEPS on a blocking-sync CUDA event while the
 * GPU works (one host thread per context, several processes per box: waiting threads must not take the cores of the launching
 * ones); the environment variable CVB_SYNC=spin selects spinning waits (cudaStreamSynchronize) for a latency-critical single caller. */
int cvb_ctx_sync(cvb_ctx *ctx);
const char *cvb_last_error(const cvb_ctx *ctx);
const char *cvb_version(void);
/* kernels launched by this context since creation (the `gpu_launches` evidence in bench.py) */
uint64_t cvb_ctx_launch_count(const cvb_ctx *ctx);
/* CUDA-event timing on the context's own stream: begin/end bracket, elapsed in milliseconds. */
int cvb_ctx_timer_begin(cvb_ctx *ctx);
int cvb_ctx_timer_end(cvb_ctx *ctx, float *ms_out);

/* Optional per-kernel profiling with CUDA events on the context stream (used by bench.py for the
 * roofline line; adds event overhead, so never enabled inside a timed throughput region).
 * cvb_ctx_profile_report writes one text line per kernel: "name launches total_ms algorithmic_bytes". */
int cvb_ctx_profile(cvb_ctx *ctx, int enable);
int cvb_ctx_profile_report(cvb_ctx *ctx, char *buf, size_t cap);

/* ---- AKAZE ------------------------------------------------------------------------------ */
void cvb_akaze_default_cfg(cvb_akaze_cfg *cfg);      /* Akaze::default(), lib.rs:169-185 */

/* One frame, host buffers.  image: w*h row-major f32 in [0,1] (a GrayFloatImage).  Writes at most
 * `cap` keypoints / 64-byte descriptors, in the reference's output order (descending response,
 * out-of-bounds descriptors dropped).  *n_out = number produced. */
int cvb_akaze_extract(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, const float *image, uint32_t w, uint32_t h,
                      cvb_keypoint *kp_out, uint8_t *desc_out, uint32_t cap, uint32_t *n_out);

/* B frames of identical size in one pass (frames are independent: this is the data-parallel axis).
 * images: B contiguous w*h planes.  kp_out: B*cap, desc_out: B*cap*64, n_out: B. */
int cvb_akaze_extract_batch(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, const float *images, uint32_t batch,
                            uint32_t w, uint32_t h, cvb_keypoint *kp_out, uint8_t *desc_out, uint32_t cap,
                            uint32_t *n_out);

/* Device-resident variant: images_dev / kp_out_dev / desc_out_dev / n_out_dev are device pointers.
 * Asynchronous on the context stream.  Results stay in HBM (feed cvb_hamming_knn_dev directly). */
int cvb_akaze_extract_batch_dev(cvb_ctx *ctx, const cvb_akaze_cfg *cfg, const float *images_dev, uint32_t batch,
                                uint32_t w, uint32_t h, cvb_keypoint *kp_out_dev, uint8_t *desc_out_dev,
                                uint32_t cap, uint32_t *n_out_dev);
/* The device-resident variant cannot return CVB_ECAP (nothing is read back): n_out_dev never exceeds cap, and a truncation
 * sets a sticky flag.  This call synchronises the stream, returns the flag (0 none, 1/2 internal candidate / keypoint capacity,
 * 3 output capacity) of the extract calls since the last query and clears it.
 * Internal capacities: the context's workspace holds max(w*h/8, 4096) candidates and max(w*h/32, 4096) cached keypoints per frame
 * (fewer than a frame can need: uniform noise or a threshold near 0 exceeds them).  The host calls (cvb_akaze_extract_batch,
 * cvb_akaze_extract_dynamic_batch, cvb_akaze_find_image_keypoints, cvb_frame_features_batch and its pixel-format form) then grow
 * these capacities to what the device counted and run the frames again, at most twice, so they return the reference's keypoints;
 * the grown capacities stay with the workspace.  A host call clears the flag before it runs and leaves it clear, so a flag it reads
 * back is its own.  The _dev calls cannot run again: they return the keypoints of the clamped stages and set flag 1 or 2.  Such an
 * overflow leaves nothing behind that changes a later call: the next call runs on the capacities the workspace has (grown by any
 * host call in between).  The two-view entry of cvb200_sfm.h, cvb_two_view_frames_k1, runs the extractor as the _dev call does and
 * reads back no flag. */
int cvb_akaze_dev_overflow(cvb_ctx *ctx, uint32_t *flag_out);

/* Introspection of the last extract call (parity tests): copies one plane of one evolution of one
 * frame to host.  plane: 0 Lt, 1 Lsmooth, 2 Lx, 3 Ly, 4 Lflow, 5 Ldet.  out must hold w*h floats of
 * that evolution's level (query sizes with cvb_akaze_debug_evolution). */
int cvb_akaze_debug_num_evolutions(cvb_ctx *ctx, uint32_t *n_out);
int cvb_akaze_debug_evolution(cvb_ctx *ctx, uint32_t evolution, uint32_t *w, uint32_t *h, uint32_t *octave,
                              uint32_t *sigma_size, uint32_t *n_fed_steps);
int cvb_akaze_debug_plane(cvb_ctx *ctx, uint32_t frame, uint32_t evolution, uint32_t plane, float *out);
int cvb_akaze_debug_contrast(cvb_ctx *ctx, uint32_t frame, double *k_out);
/* stage: 0 candidates (3x3 maxima, raster order), 1 extrema (after duplicate suppression),
 * 2 refined (sub-pixel + orientation), 3 sorted.  Returns count in *n_out (<= cap written). */
int cvb_akaze_debug_stage(cvb_ctx *ctx, uint32_t frame, uint32_t stage, cvb_keypoint *out, uint32_t cap,
                          uint32_t *n_out);

/* ---- brute-force Hamming k-NN (space::LinearKnn + bitarray::Hamming) ---------------------- */
/* For each of n queries (64-byte descriptors) the k nearest of m database descriptors, ascending
 * distance, ties -> lower database index first.  idx_out/dist_out: n*k.  If m < k the missing slots
 * hold 0xffffffff.  k <= 8. */
int cvb_hamming_knn(cvb_ctx *ctx, const uint8_t *queries, uint32_t n, const uint8_t *database, uint32_t m,
                    uint32_t k, uint32_t *idx_out, uint32_t *dist_out);
int cvb_hamming_knn_dev(cvb_ctx *ctx, const uint8_t *queries_dev, uint32_t n, const uint8_t *database_dev,
                        uint32_t m, uint32_t k, uint32_t *idx_out_dev, uint32_t *dist_out_dev);
/* n and m read from device memory (e.g. the n_out_dev of cvb_akaze_extract_batch_dev); n_max/m_max
 * bound the launch.  Rows >= *n_dev are left untouched. */
int cvb_hamming_knn_dev_counts(cvb_ctx *ctx, const uint8_t *queries_dev, const uint32_t *n_dev, uint32_t n_max,
                               const uint8_t *database_dev, const uint32_t *m_dev, uint32_t m_max, uint32_t k,
                               uint32_t *idx_out_dev, uint32_t *dist_out_dev);

/* cv-sfm symmetric_matching (cv-sfm/src/lib.rs:3097-3133): forward and reverse 2-NN, keep a->b when
 * d0 + better_by <= d1 in both directions and the best matches agree.  pairs_out: up to cap (a,b)
 * index pairs in ascending a. */
int cvb_match_symmetric(cvb_ctx *ctx, const uint8_t *desc_a, uint32_t n, const uint8_t *desc_b, uint32_t m,
                        uint32_t better_by, uint32_t *pairs_out, uint32_t cap, uint32_t *n_out);

/* Device-resident variant: a_dev / b_dev are device descriptor arrays; match_out_dev[n] receives, for every a, the
 * index of its symmetric match in b or 0xffffffff.  Asynchronous on the context stream. */
int cvb_match_symmetric_dev(cvb_ctx *ctx, const uint8_t *a_dev, uint32_t n, const uint8_t *b_dev, uint32_t m,
                            uint32_t better_by, uint32_t *match_out_dev);

/* HammingHasher::<64, H>::hash_bag (external crate hamming-lsh 0.3.2; cv-sfm/src/lib.rs:205,216,672): the frame-level place-recognition
 * hash of a bag of descriptors.  Every descriptor sets the bit of its nearest codeword (Hamming distance, first minimum on ties);
 * hash bit ix = bit ix & 7 of byte ix >> 3.  codewords: ncode x 64 bytes (cv-sfm passes the 4 096 entries of cv-sfm/src/codewords.rs,
 * H = 512 bytes); hash_out: ncode / 8 bytes.  The crate source is not in the reference tree: restated from its documented behaviour,
 * parity unpinned.  The nearest-codeword search is a 1-NN query of the matcher above (same kernels). */
int cvb_hash_bag(cvb_ctx *ctx, const uint8_t *descriptors, uint32_t n, const uint8_t *codewords, uint32_t ncode, uint8_t *hash_out);
int cvb_hash_bag_dev(cvb_ctx *ctx, const uint8_t *descriptors_dev, const uint32_t *n_dev, uint32_t n_max, const uint8_t *codewords_dev,
                     uint32_t ncode, uint8_t *hash_out_dev);

/* ---- geometric verification ------------------------------------------------------------------
 * sample_consensus::{Estimator, Model, Consensus} surfaces (external crate sample-consensus 1.0.2, re-exported at
 * cv-core/src/lib.rs:82) with the solvers and residuals of the reference:
 *   cvb_eight_point_batch        <- EightPoint::estimate              eight-point/src/lib.rs:70-84 (+ essential.rs:217-231)
 *   cvb_p3p_batch                <- LambdaTwist::estimate             lambda-twist/src/lib.rs:330-347
 *   cvb_residuals_camera_to_camera <- CameraToCamera::residual        cv-core/src/pose.rs:249-296
 *   cvb_residuals_world_to_camera  <- WorldToCamera::residual         cv-core/src/pose.rs:194-202
 *   cvb_triangulate_linear_eigen <- LinearEigenTriangulator           cv-geom/src/triangulation.rs:82-130
 *   cvb_arrsac_eight_point / cvb_arrsac_p3p <- arrsac::Arrsac as Consensus<EightPoint, FeatureMatch> /
 *                                   Consensus<LambdaTwist, FeatureWorldMatch> (call sites akaze/tests/estimate_pose.rs:63-67,
 *                                   cv-sfm/src/lib.rs:1394-1406,1619-1622, vslam-sandbox/src/main.rs:105-117)
 * Data: FeatureMatch = two unit bearings (a[i*3..], b[i*3..]); FeatureWorldMatch = unit bearing + homogeneous world
 * point xyzw (xyz unit, w = 1/distance >= 0).  All pointers are HOST pointers; every model hypothesis and every
 * (hypothesis, datum) residual is evaluated on the GPU; ARRSAC's sequential bookkeeping (likelihood-ratio test, stable sort / truncate,
 * consumption of the RNG draws) also runs on the device (cv_b200/csrc/arrsac_dev.cuh), in the order of the restated reference loop
 * (oracle/ref_geom.c::ref_arrsac).  The arrsac crate's source is not available here: the control flow is a restatement, its
 * inlier-set parity with the crate is unpinned (DESIGN.md section 2); GPU and oracle agree bit for bit on inlier sets.
 * Degenerate case: the 3x3 SVD of the essential matrix returns no poses when the second singular value is <= 1e-12 * s0, where
 * nalgebra's SVD would still return four. */
typedef struct { double r[9]; double t[3]; } cvb_pose;      /* IsometryMatrix3<f64>: rotation row-major, translation */
typedef struct { int32_t kind; uint64_t s[4]; } cvb_rng;   /* kind 0: xoshiro256++ (SmallRng / Xoshiro256PlusPlus), 1: Pcg64 */
typedef struct {
    double inlier_threshold;
    uint32_t initialization_hypotheses, initialization_blocks, max_candidate_hypotheses, estimations_per_block, block_size;
    float likelihood_ratio_threshold, initial_epsilon, initial_delta;
} cvb_arrsac_cfg;

void cvb_arrsac_default_cfg(cvb_arrsac_cfg *cfg, double inlier_threshold);   /* Arrsac::new(threshold, rng) defaults */
void cvb_rng_seed_xoshiro256pp(cvb_rng *rng, uint64_t seed);                 /* Xoshiro256PlusPlus::seed_from_u64 */
void cvb_rng_seed_pcg64(cvb_rng *rng, const uint8_t seed[32]);               /* Pcg64::from_seed */
uint32_t cvb_rng_next_u32(cvb_rng *rng);

/* H minimal samples (indices into the n data): samples[h*8..] / samples[h*3..]; up to 4 poses per sample */
int cvb_eight_point_batch(cvb_ctx *ctx, const double *a, const double *b, uint32_t n, const uint32_t *samples, uint32_t H,
                          cvb_pose *poses_out, uint8_t *nposes_out);
int cvb_p3p_batch(cvb_ctx *ctx, const double *bearings, const double *world, uint32_t n, const uint32_t *samples, uint32_t H,
                  cvb_pose *poses_out, uint8_t *nposes_out);
/* NisterStewenius::estimate (nister-stewenius/src/lib.rs:303-330): samples[h*5..], up to 40 poses per sample
 * (poses_out: H*40).  eigenvector_row0 = 5 reproduces the reference, whose `fixed_rows::<4>(5)` (lib.rs:229) reads
 * the (x, y, z, 1) solution one row too early (the monomial basis has them in rows 6..9), so its essential matrices
 * violate the cubic constraints; eigenvector_row0 = 6 is the corrected solver. */
int cvb_five_point_batch(cvb_ctx *ctx, const double *a, const double *b, uint32_t n, const uint32_t *samples, uint32_t H,
                         int32_t eigenvector_row0, cvb_pose *poses_out, uint8_t *nposes_out);
/* out[m*n]: residual of pose p for datum i at out[p*n + i] */
int cvb_residuals_camera_to_camera(cvb_ctx *ctx, const cvb_pose *poses, uint32_t m, const double *a, const double *b,
                                   uint32_t n, double *out);
int cvb_residuals_world_to_camera(cvb_ctx *ctx, const cvb_pose *poses, uint32_t m, const double *bearings,
                                  const double *world, uint32_t n, double *out);
/* L landmarks; landmark l owns observations offsets[l]..offsets[l+1] of (poses, bearings). ok_out[l] = 1 -> Some(point) */
int cvb_triangulate_linear_eigen(cvb_ctx *ctx, const cvb_pose *poses, const double *bearings, const uint32_t *offsets,
                                 uint32_t L, double *xyzw_out, uint8_t *ok_out);
/* Consensus::model_inliers.  *found = 0 -> None.  inliers_out: ascending datum indices (at most cap written). */
int cvb_arrsac_eight_point(cvb_ctx *ctx, const cvb_arrsac_cfg *cfg, const double *a, const double *b, uint32_t n, cvb_rng *rng,
                           cvb_pose *model_out, uint32_t *inliers_out, uint32_t cap, uint32_t *n_inliers, int32_t *found);
int cvb_arrsac_five_point(cvb_ctx *ctx, const cvb_arrsac_cfg *cfg, const double *a, const double *b, uint32_t n, cvb_rng *rng,
                          int32_t eigenvector_row0, cvb_pose *model_out, uint32_t *inliers_out, uint32_t cap,
                          uint32_t *n_inliers, int32_t *found);
int cvb_arrsac_p3p(cvb_ctx *ctx, const cvb_arrsac_cfg *cfg, const double *bearings, const double *world, uint32_t n,
                   cvb_rng *rng, cvb_pose *model_out, uint32_t *inliers_out, uint32_t cap, uint32_t *n_inliers, int32_t *found);

/* ---- device-resident geometric verification: nothing returns to the host between enqueue and result ---------------------------
 * cv-sfm's two-view initialisation of one frame pair (cv-sfm/src/lib.rs:1375-1412): symmetric_matching (:3097-3133) -> FeatureMatch
 * bearings of the matched keypoints (CameraModel::calibrate, cv-pinhole/src/lib.rs:108-116) -> Consensus::model_inliers
 * (arrsac::Arrsac, configuration vslam-sandbox/src/main.rs:105-117).  All pointers below are DEVICE pointers unless stated; every call is
 * asynchronous on the context stream.  ARRSAC's random draws come from a stream of raw next_u32() values generated on the host from
 * *rng at call time (the generator is sequential; modulo and rejection run on the device because they need the datum count); the
 * caller's generator is advanced by the number of draws actually consumed with cvb_arrsac_commit_rng after the stream has drained. */
typedef struct { double fx, fy, cx, cy, skew; } cvb_intrinsics;   /* cv_pinhole::CameraIntrinsics (cv-pinhole/src/lib.rs:32-41), k1 = 0 */
/* (the camera with radial distortion, CameraIntrinsicsK1Distortion, and cv-sfm's frame ingestion: include/cvb200_sfm.h) */

/* counts read from device memory (the n_out_dev of cvb_akaze_extract_batch_dev); pairs_out_dev: up to cap (a, b) index pairs in
 * ascending a; *n_pairs_dev <= cap */
int cvb_match_symmetric_pairs_dev(cvb_ctx *ctx, const uint8_t *a_dev, const uint32_t *n_dev, uint32_t n_max, const uint8_t *b_dev,
                                  const uint32_t *m_dev, uint32_t m_max, uint32_t better_by, uint32_t *pairs_out_dev, uint32_t cap,
                                  uint32_t *n_pairs_dev);
/* a_out_dev[i*3..], b_out_dev[i*3..]: unit bearings of match i (keypoint pixel coordinates widened to f64, akaze/src/lib.rs:95-99) */
int cvb_pair_bearings_dev(cvb_ctx *ctx, const cvb_keypoint *kp_a_dev, const cvb_keypoint *kp_b_dev, const uint32_t *pairs_dev,
                          const uint32_t *n_pairs_dev, uint32_t cap, const cvb_intrinsics *intrinsics /* host */, double *a_out_dev,
                          double *b_out_dev);
/* Consensus::model_inliers with device data: a_dev/b_dev hold n_max rows, *n_dev of them valid.  cfg and rng are HOST pointers.
 * *found_dev = 0 -> None.  inliers_out_dev (may be NULL): ascending datum indices, at most cap written; *n_inliers_dev = their number. */
int cvb_arrsac_eight_point_dev(cvb_ctx *ctx, const cvb_arrsac_cfg *cfg, const double *a_dev, const double *b_dev, const uint32_t *n_dev,
                               uint32_t n_max, const cvb_rng *rng, cvb_pose *model_out_dev, uint32_t *inliers_out_dev, uint32_t cap,
                               uint32_t *n_inliers_dev, int32_t *found_dev);
int cvb_arrsac_p3p_dev(cvb_ctx *ctx, const cvb_arrsac_cfg *cfg, const double *bearings_dev, const double *world_dev, const uint32_t *n_dev,
                       uint32_t n_max, const cvb_rng *rng, cvb_pose *model_out_dev, uint32_t *inliers_out_dev, uint32_t cap,
                       uint32_t *n_inliers_dev, int32_t *found_dev);
/* Synchronises the context stream and advances *rng (host, may be NULL) past the draws the last cvb_arrsac_*_dev /
 * cvb_two_view_* call consumed.  stats_out (host, 16 words, may be NULL): data, valid initial models, models that passed the SPRT,
 * SPRT commit rounds, block iterations, draws consumed, inliers, found, 32-datum units scored by the two initial stages (2 words),
 * predicates the filter left to the exact evaluation, mask words the SPRT computed itself, models the SPRT walked again with their
 * exact state; three reserved words. */
int cvb_arrsac_commit_rng(cvb_ctx *ctx, cvb_rng *rng, uint32_t *stats_out);

/* One frame pair end to end on the device: symmetric match of the two descriptor sets, bearings, ARRSAC + eight-point.
 * kp/desc/n: the two frames' extraction results (device).  pairs_out_dev: cap x 2; inliers_out_dev: cap (indices into pairs). */
int cvb_two_view_pair_dev(cvb_ctx *ctx, const cvb_keypoint *kp_a_dev, const uint8_t *desc_a_dev, const uint32_t *n_a_dev,
                          const cvb_keypoint *kp_b_dev, const uint8_t *desc_b_dev, const uint32_t *n_b_dev, uint32_t n_max,
                          uint32_t better_by, const cvb_intrinsics *intrinsics, const cvb_arrsac_cfg *cfg, const cvb_rng *rng,
                          uint32_t *pairs_out_dev, uint32_t cap, uint32_t *n_pairs_dev, cvb_pose *model_out_dev,
                          uint32_t *inliers_out_dev, uint32_t *n_inliers_dev, int32_t *found_dev);
/* The same from two HOST frames (f32, w x h each, contiguous) to HOST results, one synchronisation at the end: AKAZE extract of both
 * frames (one batched pass), then cvb_two_view_pair_dev.  kp_out: 2 x cap, desc_out: 2 x cap x 64, n_out: 2, pairs_out: cap x 2,
 * inliers_out: cap.  *rng is advanced like the reference's generator.  Page-locked output buffers avoid staged copies. */
int cvb_two_view_frames(cvb_ctx *ctx, const cvb_akaze_cfg *akaze, const float *frames, uint32_t w, uint32_t h, uint32_t better_by,
                        const cvb_intrinsics *intrinsics, const cvb_arrsac_cfg *cfg, cvb_rng *rng, cvb_keypoint *kp_out, uint8_t *desc_out,
                        uint32_t cap, uint32_t *n_out, uint32_t *pairs_out, uint32_t *n_pairs, cvb_pose *model_out, uint32_t *inliers_out,
                        uint32_t *n_inliers, int32_t *found);

/* ---- post-consensus refinement and robustness checks (SURVEY.md section 8f rows 2, 3) ------------------------------
 *   cvb_single_view_optimize_l2 <- cv_optimize::single_view_simple_optimize_l2   cv-optimize/src/single_view_optimizer.rs:80-135
 *                                  (call sites cv-sfm/src/lib.rs:1655,1706; gradient cv-geom/src/epipolar.rs:193-198)
 *   cvb_three_view_optimize_l2  <- three_view_simple_optimize_l2 (adaptive = 0), three_view_adaptive_optimize_l2 (adaptive = 1,
 *                                  optimization_rate unused)                       cv-optimize/src/three_view_optimizer.rs:126-272
 *                                  (call sites cv-sfm/src/lib.rs:1131,1180,2039; gradients cv-geom/src/epipolar.rs:85-176)
 *   cvb_observation_losses      <- VSlam::observation_loss for every observation   cv-sfm/src/lib.rs:2570-2620
 *   cvb_tri_landmarks_robust    <- VSlam::is_tri_landmark_robust                   cv-sfm/src/lib.rs:1320-1360
 * B independent problems per call, problem b owns data offsets[b]..offsets[b+1]; each problem iterates to completion inside one
 * CTA (per-iteration tangent sums by a fixed reduction tree; the reference adds in landmark order, so results agree to rounding).
 * updates_out[b] = pose updates applied before the reference's patience rule or the iteration cap stopped the loop (may be NULL). */
int cvb_single_view_optimize_l2(cvb_ctx *ctx, const cvb_pose *poses, uint32_t B, double optimization_rate, uint32_t iterations,
                                const double *bearings, const double *world, const uint32_t *offsets, cvb_pose *poses_out,
                                uint32_t *updates_out);
/* poses[2*b], poses[2*b+1]: CameraToCamera centre->first, centre->second; observations[i*9..]: centre, first, second bearings */
int cvb_three_view_optimize_l2(cvb_ctx *ctx, const cvb_pose *poses, uint32_t B, int32_t adaptive, double optimization_rate,
                               uint32_t iterations, const double *observations, const uint32_t *offsets, cvb_pose *poses_out,
                               uint32_t *updates_out);
/* L landmarks with (WorldToCamera pose, bearing) observation lists as in cvb_triangulate_linear_eigen; loss_out[i] per observation:
 * 2.0 for a single observation or a failed triangulation, the epipolar loss as a cosine distance for two, else 1 - cos to the
 * triangulated point */
int cvb_observation_losses(cvb_ctx *ctx, const cvb_pose *poses, const double *bearings, const uint32_t *offsets, uint32_t L,
                           double *loss_out);
int cvb_tri_landmarks_robust(cvb_ctx *ctx, const cvb_pose *first_pose, const cvb_pose *second_pose, const double *observations,
                             uint32_t n, double maximum_cosine_distance, double incidence_minimum_cosine_distance,
                             uint8_t *robust_out);

#ifdef __cplusplus
}
#endif
#endif /* CVB200_H */
