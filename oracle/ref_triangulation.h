/* oracle/ref_triangulation.h -- TEST INFRASTRUCTURE (CPU oracle), not product code.  The oracle of include/cvb200_tri.h: the
 * triangulators of cv-geom/src/triangulation.rs and cv-sfm's observation losses / tri-landmark robustness with a chosen triangulator
 * (oracle/ref_triangulation.c, built with ref_geom.c and ref_optimize.c by oracle/tri.mk). */
#ifndef REF_TRIANGULATION_H
#define REF_TRIANGULATION_H
#include <stdint.h>
#include "ref_geom.h"
#ifdef __cplusplus
extern "C" {
#endif

enum { REF_TRI_LINEAR_EIGEN = 0, REF_TRI_SINE_L1, REF_TRI_MEAN_MEAN, REF_TRI_RELATIVE_DLT, REF_TRI_ANGULAR_L1, REF_TRI_ANGULAR_LINF };
typedef struct { int32_t method; uint32_t max_iterations; double epsilon, optimization_rate; } ref_triangulator;   /* == cvb_triangulator */

void ref_triangulator_default(ref_triangulator *t, int32_t method);
/* methods 0-2; returns 1 = Some.  iterations (may be NULL): SineL1's refinement iterations, 0 for the other methods */
int ref_triangulate_observations(const ref_triangulator *t, const ref_pose *poses, const double *bearings, int n, double *out,
                                 uint32_t *iterations);
/* all six methods; P is CameraToCamera (a's camera -> b's camera); out is the CameraPoint in a's camera */
int ref_triangulate_relative(const ref_triangulator *t, const ref_pose *P, const double *a, const double *b, double *out);
/* batches in the layout of include/cvb200_tri.h (rows of failed items zeroed, ok = 0); iterations (may be NULL): L SineL1 counts */
void ref_triangulate_observations_batch(const ref_triangulator *t, const ref_pose *poses, const double *bearings, const uint32_t *offsets,
                                        uint32_t L, double *xyzw, uint8_t *ok, uint32_t *iterations);
void ref_triangulate_relative_batch(const ref_triangulator *t, const ref_pose *poses, uint32_t npose, const double *a, const double *b,
                                    uint32_t n, double *xyzw, uint8_t *ok);
/* ref_observation_losses / ref_is_tri_landmark_robust (ref_optimize.c) with the caller's triangulator (methods 0-2) */
void ref_observation_losses_tri(const ref_triangulator *tri, const ref_pose *poses, const double *bearings, uint32_t n, double *loss);
int ref_is_tri_landmark_robust_tri(const ref_triangulator *tri, const ref_pose *first, const ref_pose *second, const double *c, const double *f,
                                   const double *s, double maximum_cosine_distance, double incidence_minimum_cosine_distance);

#ifdef __cplusplus
}
#endif
#endif
