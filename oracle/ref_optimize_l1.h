/* oracle/ref_optimize_l1.h -- TEST INFRASTRUCTURE (CPU oracle), not product code.  The oracle of include/cvb200_opt.h: cv-optimize's
 * L1 (Weiszfeld) pose optimizers (oracle/ref_optimize_l1.c, built with ref_optimize.c's gradients by oracle/opt.mk). */
#ifndef REF_OPTIMIZE_L1_H
#define REF_OPTIMIZE_L1_H
#include <stdint.h>
#include "ref_geom.h"
#ifdef __cplusplus
extern "C" {
#endif

/* summation order of the per-iteration sums */
enum {
    REF_SUM_LANDMARK = 0,   /* landmark order, as the reference's `for` loops */
    REF_SUM_DEVICE = 1      /* the order of k_*_opt_l1 (cv_b200/csrc/geom.cu): REF_OPT_NT strided partial sums, shuffle-down tree, warps in order */
};
#define REF_OPT_NT 512

/* single_view_simple_optimize_l1 (cv-optimize/src/single_view_optimizer.rs:16-78) on *pose (WorldToCamera), in place; bearings
 * n x 3, world n x 4 (homogeneous).  Returns the pose updates applied. */
uint32_t ref_single_view_optimize_l1(ref_pose *pose, double epsilon, double rate, uint32_t iterations, const double *bearings,
                                     const double *world, uint32_t n, int order);
/* three_view_simple_optimize_l1 (cv-optimize/src/three_view_optimizer.rs:23-124) on poses[2] (CameraToCamera centre -> first /
 * second), in place; obs n x 9 (centre, first, second bearings).  Returns the pose updates applied. */
uint32_t ref_three_view_optimize_l1(ref_pose poses[2], double epsilon, double rate, uint32_t iterations, const double *obs, uint32_t n,
                                    int order);

#ifdef __cplusplus
}
#endif
#endif
