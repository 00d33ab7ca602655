/* oracle/ref_sfm.c -- TEST INFRASTRUCTURE: CPU restatement of the camera with radial distortion and of cv-sfm's per-frame feature
 * ingestion (include/cvb200_sfm.h).  Not product code.  Built on its own by oracle/sfm.mk into oracle/_build/libcvb_oracle_sfm.so with
 * the flags of oracle/Makefile (-ffp-contract=off: no fused multiply-add, as a default x86-64 Rust build).
 *
 * Follows (paths relative to the reference checkout):
 *   cv-pinhole/src/lib.rs:191-202,224-239   CameraIntrinsicsK1Distortion::calibrate / uncalibrate
 *   cv-sfm/src/bicubic.rs:13-68             interpolate_bicubic on an RgbImage
 *   cv-sfm/src/lib.rs:2205-2232             VSlam::kps_descriptors, per keypoint
 * and, from a crate that is NOT in the reference checkout (restated from its published source):
 *   imageproc 0.23   Clamp<f32> for u8 (definitions.rs)  -> PARITY UNPINNED beyond this restatement (as SURVEY.md Appendix A does for
 *                    the other external crates).
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>

/* cv-pinhole/src/lib.rs:191-202 calibrate: centre, divide by the focals, remove skew, divide the distorted point by 1 + k1 r^2
 * (component-wise true division, nalgebra's Vector2 / f64), then new_normalize of (x, y, 1) exactly as the undistorted camera */
void ref_calibrate_k1(double fx, double fy, double cx, double cy, double skew, double k1, double px, double py, double *bearing) {
    double y = (py - cy) / fy;
    double x = (px - cx - skew * y) / fx;
    double r2 = x * x + y * y;
    double d = 1.0 + k1 * r2;
    x = x / d; y = y / d;
    double n = sqrt(x * x + y * y + 1.0);
    bearing[0] = x / n; bearing[1] = y / n; bearing[2] = 1.0 / n;
}

/* cv-pinhole/src/lib.rs:224-239 uncalibrate.  Returns 0 (None) when z is not sign-positive.  The quadratic form is kept as written:
 * NaN when k1 * u2 == 0 (k1 = 0, or the principal point: 0 / 0) and when 4 k1 u2 > 1 (sqrt of a negative). */
int ref_uncalibrate_k1(double fx, double fy, double cx, double cy, double skew, double k1, const double *bearing, double *px) {
    if (signbit(bearing[2])) return 0;
    double ux = bearing[0] / bearing[2], uy = bearing[1] / bearing[2];
    double u2 = ux * ux + uy * uy;
    double r2_mul_k1 = -(2.0 * k1 * u2 + sqrt(1.0 - 4.0 * k1 * u2) - 1.0) / (2.0 * k1 * u2);
    double dx = ux * (1.0 + r2_mul_k1), dy = uy * (1.0 + r2_mul_k1);
    double y = dy * fy;
    double x = dx * fx + skew * dy;
    px[0] = x + cx; px[1] = y + cy;
    return 1;
}

/* imageproc 0.23 `Clamp<f32> for u8`: truncating cast inside (0, 255), saturating outside (unpinned, see above) */
static uint8_t clamp_u8(float x) { return x < 255.0f ? (x > 0.0f ? (uint8_t)x : 0) : 255; }

/* cv-sfm/src/bicubic.rs:13-31 blend_cubic, one channel, f32, the source's association order */
static float blend_cubic(float p0, float p1, float p2, float p3, float x) {
    return p1 + 0.5f * x * (p2 - p0 + x * (2.0f * p0 - 5.0f * p1 + 4.0f * p2 - p3 + x * (3.0f * (p1 - p2) + p3 - p0)));
}

/* cv-sfm/src/bicubic.rs:33-68 interpolate_bicubic on a w x h interleaved RGB8 image with default Rgb([0, 0, 0]).  Quirks kept: black
 * when right = left + 4 >= width (one column earlier than the last column read), and each row result is clamped to u8 before the column
 * blend (blend_cubic returns a Pixel of the image's type). */
void ref_bicubic_rgb8(const uint8_t *rgb, int w, int h, float x, float y, uint8_t *out) {
    float left = floorf(x) - 1.0f, right = left + 4.0f, top = floorf(y) - 1.0f, bottom = top + 4.0f;
    float x_weight = x - (left + 1.0f), y_weight = y - (top + 1.0f);
    if (left < 0.0f || right >= (float)w || top < 0.0f || bottom >= (float)h) { out[0] = out[1] = out[2] = 0; return; }
    uint8_t col[4][3];
    for (int row = (int)top; row < (int)bottom; row++) {
        const uint8_t *p = rgb + ((size_t)row * w + (size_t)left) * 3;
        for (int c = 0; c < 3; c++) col[row - (int)top][c] = clamp_u8(blend_cubic(p[c], p[3 + c], p[6 + c], p[9 + c], x_weight));
    }
    for (int c = 0; c < 3; c++) out[c] = clamp_u8(blend_cubic(col[0][c], col[1][c], col[2][c], col[3][c], y_weight));
}

/* cv-sfm/src/lib.rs:2205-2232, per keypoint of VSlam::kps_descriptors: bicubic colour and K1 bearing.  xy: n (x, y) f32 pairs;
 * K = fx, fy, cx, cy, skew, k1. */
void ref_kps_features(const float *xy, int n, const uint8_t *rgb, int w, int h, const double *K, double *bearings, uint8_t *colors) {
    for (int i = 0; i < n; i++) {
        ref_bicubic_rgb8(rgb, w, h, xy[2 * i], xy[2 * i + 1], colors + 3 * i);
        ref_calibrate_k1(K[0], K[1], K[2], K[3], K[4], K[5], (double)xy[2 * i], (double)xy[2 * i + 1], bearings + 3 * i);
    }
}
