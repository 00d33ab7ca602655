/* oracle/ref_pinhole.h -- TEST INFRASTRUCTURE (CPU oracle), not product code.  The oracle of include/cvb200_pinhole.h: cv-pinhole's
 * pose reprojection error over the relative triangulators of ref_triangulation.c, and the EssentialMatrix model over the essential
 * routines of ref_geom.c (oracle/ref_pinhole.c, built with both by oracle/pinhole.mk). */
#ifndef REF_PINHOLE_H
#define REF_PINHOLE_H
#include <stdint.h>
#include "ref_geom.h"
#include "ref_triangulation.h"
#ifdef __cplusplus
extern "C" {
#endif

/* pose_reprojection_error (err: a_norm - reproject_a, b_norm - reproject_b) and average_pose_reprojection_error (avg); returns 1 = Some */
int ref_pose_reprojection_error(const ref_triangulator *t, const ref_pose *P, const double *a, const double *b, double err[4], double *avg);
/* EssentialMatrix::recondition; returns 1 = Some */
int ref_essential_recondition(const double *E, double eps, int iters, double *out);
/* batches in the layout of include/cvb200_pinhole.h: rows the reference returns None for get ok = 0 and NaN */
void ref_pose_reprojection_error_batch(const ref_triangulator *t, const ref_pose *poses, uint32_t npose, const double *a, const double *b,
                                       uint32_t n, double *err, double *avg, uint8_t *ok);
void ref_eight_point_essential_batch(const double *a, const double *b, const uint32_t *samples, uint32_t H, double eps, int iters,
                                     double *E, uint8_t *ok);
void ref_residuals_essential(const double *E, uint32_t m, const double *a, const double *b, uint32_t n, double *out);
void ref_essential_recondition_batch(const double *E, uint32_t m, double eps, int iters, double *out, uint8_t *ok);
void ref_essential_decompose_batch(const double *E, uint32_t m, double eps, int iters, double *rot_a, double *rot_b, double *t, uint8_t *ok);

#ifdef __cplusplus
}
#endif
#endif
