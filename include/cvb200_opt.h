/* include/cvb200_opt.h -- C ABI of libcvb200.so for cv-optimize's L1 (Weiszfeld) pose optimizers, batched on the device.
 *
 *   cvb_single_view_optimize_l1  <- single_view_simple_optimize_l1   cv-optimize/src/single_view_optimizer.rs:16-78
 *   cvb_three_view_optimize_l1   <- three_view_simple_optimize_l1    cv-optimize/src/three_view_optimizer.rs:23-124
 *
 * The L2 optimizers are in include/cvb200.h (cvb_single_view_optimize_l2, cvb_three_view_optimize_l2); these two take the same
 * layout.  Every iteration sums, per pose, the L1 tangents `g.l1()` (each gradient normalised, a zero gradient contributing zero) and
 * the Weiszfeld weights ts = sum 1 / (|g.t| + tscale * epsilon), rs = sum 1 / (|g.r| + epsilon), then applies the delta
 * (l1sum.t * rate * (1 / ts), l1sum.r * rate * (1 / rs)).  tscale is |t| of the current pose (single view) or
 * |t0| + |t1| of the two inverted poses (three view).  The reference gives epsilon no default: the caller supplies it, and no value
 * of epsilon, rate or iterations is rejected (epsilon = 0 with an exact pose yields the reference's IEEE infinities).
 *
 * Library: libcvb200_opt.so, a module over libcvb200.so that takes its contexts (link with -lcvb200_opt -lcvb200).
 * The conventions of include/cvb200.h hold: return codes, HOST pointers, no CPU fallback (no device: no context, CVB_ENODEV).
 * B independent problems run in one launch, one CTA each.  Problem b owns landmarks offsets[b] .. offsets[b + 1] - 1 (offsets has
 * B + 1 non-decreasing entries, else CVB_EINVAL).  updates_out (B entries, may be NULL) receives the pose updates applied, i.e.
 * the iterations run before the cap or the 50-iteration patience rule ended the loop.  A problem without landmarks returns its
 * input pose(s) unchanged.  B == 0 returns CVB_OK. */
#ifndef CVB200_OPT_H
#define CVB200_OPT_H
#include "cvb200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* single_view_simple_optimize_l1 for B problems.  poses: B WorldToCamera poses; bearings: unit bearings (f64 x 3) and world:
 * homogeneous world points (f64 x 4) of the FeatureWorldMatches; landmarks whose transformed point has w == 0 are skipped
 * (landmark_delta returns None, single_view_optimizer.rs:4-14).  poses_out: B poses. */
int cvb_single_view_optimize_l1(cvb_ctx *ctx, const cvb_pose *poses, uint32_t B, double epsilon, double optimization_rate,
                                uint32_t iterations, const double *bearings, const double *world, const uint32_t *offsets,
                                cvb_pose *poses_out, uint32_t *updates_out);

/* three_view_simple_optimize_l1 for B problems.  poses: 2B CameraToCamera poses (centre -> first, centre -> second per problem);
 * observations: (centre, first, second) unit bearings, f64 x 9 per landmark.  poses_out: 2B poses. */
int cvb_three_view_optimize_l1(cvb_ctx *ctx, const cvb_pose *poses, uint32_t B, double epsilon, double optimization_rate,
                               uint32_t iterations, const double *observations, const uint32_t *offsets, cvb_pose *poses_out,
                               uint32_t *updates_out);

#ifdef __cplusplus
}
#endif
#endif /* CVB200_OPT_H */
