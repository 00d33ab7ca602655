/* include/cvb200_filter.h -- C ABI of akaze::image, the akaze crate's public image module, on the device: separable correlation filters
 * of any odd length, the Gaussian kernel and blur, and the 2x2 down-sampling of the scale space.
 *
 *   cvb_horizontal_filter(_dev)   <- akaze::image::horizontal_filter                 image.rs:202-251
 *   cvb_vertical_filter(_dev)     <- akaze::image::vertical_filter                   image.rs:253-331
 *   cvb_separable_filter(_dev)    <- akaze::image::separable_filter                  image.rs:333-340
 *   cvb_gaussian_kernel           <- akaze::image::gaussian_kernel                   image.rs:349-374
 *   cvb_gaussian_blur(_dev)       <- akaze::image::gaussian_blur                     image.rs:383-389
 *   cvb_half_size(_dev)           <- akaze::image::GrayFloatImage::half_size         image.rs:154-199
 *
 * Library: libcvb200_filter.so, a module over libcvb200.so that takes its contexts (link with -lcvb200_filter -lcvb200).  The conventions
 * of include/cvb200.h hold: return codes, HOST pointers unless the name ends in _dev, asynchronous _dev variants on the context's stream,
 * no CPU fallback (no device: no context, CVB_ENODEV).  Kernel taps are always a host `const float *`; they travel to the device inside
 * the launch's parameters, so the caller may reuse them as soon as a _dev call returns.  A host form makes one upload into buffers of the
 * context (reused across calls), its launches, one download and one synchronisation.
 *
 * Planes: `batch` planes of one size, each h rows of w f32 pixels, packed, plane b at b * w * h (the layout of
 * cvb_akaze_extract_batch_dev).  Every output is a new plane of the same layout; half_size's planes are (w / 2) x (h / 2).
 *
 * Semantics (bit-exact to the reference on a default x86-64 build; the CPU restatement is oracle/ref_filter.c):
 *   - Correlation, not convolution: no kernel flip.  With half = ks / 2, output x of a row is  sum_j in[clamp(x + j - half)] * k[j],
 *     borders replicating the edge pixel; the vertical filter is the same along a column.  A kernel longer than the plane is legal.
 *   - Summation order of wide 0.7's f32x4 (no FMA target feature): lane j & 3 accumulates tap j as (pixel * k[j]) + acc from +0, two
 *     roundings; the result is reduce_add = (l0 + l2) + (l1 + l3).
 *   - Tail taps: the reference pads the kernel with zeros to 4 * ceil(ks / 4) taps, and its scratch line is
 *     [half x first][line][half x last][3 x 0.0].  Tail tap j in [ks, 4 * ceil(ks / 4)) therefore multiplies 0.0 by pixel
 *     p = x + j - half when p <= w - 1, else by pixel w - 1 when p < w + half, else by 0.0.  These taps are evaluated: on finite data
 *     they change nothing, and a NaN or +-inf under one makes the output NaN, as in the reference.
 *   - Kernel sizes: odd, 1 <= ks <= CVB_FILTER_MAX_TAPS.  An even size (0 included) is CVB_EINVAL (a debug_assert in the reference's
 *     filters, an assert in gaussian_kernel); a larger odd size is CVB_EUNSUPPORTED.
 *   - separable_filter is the horizontal then the vertical filter; the horizontal result is rounded to f32, as the reference
 *     materialises it.  The intermediate plane lives in a buffer of the context.
 *   - gaussian_kernel(r, ks) is computed on the host in f32 with the C library's expf, then divided by its sequential f32 sum.  Any r is
 *     accepted, 0 included (NaN taps, as in the reference).  Its size has no cap.
 *   - gaussian_blur(r): r > 0, otherwise CVB_EINVAL (NaN included); ks = 2 * ceil(2 r) + 1 (f32 arithmetic), the same kernel applied
 *     horizontally then vertically.  r > 255.5 needs more than CVB_FILTER_MAX_TAPS taps and is CVB_EUNSUPPORTED.
 *   - half_size: 2x2 boxes summed row by row, ((a00 + a01) + (a10 + a11)) * 0.25; an odd last row or column (1x2 / 2x1 windows) * 0.5;
 *     the corner of an odd-by-odd plane copied.  A plane 1 pixel wide or high gives an empty result: nothing is written, the call
 *     returns 0.
 *   - Errors: a null context or argument, w, h or batch = 0, and input and output buffers that overlap are CVB_EINVAL (the reference
 *     always returns a new image).  Batches whose launch grid would not fit are CVB_EUNSUPPORTED. */
#ifndef CVB200_FILTER_H
#define CVB200_FILTER_H
#include "cvb200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* the largest kernel of the device filters: 1023 taps is gaussian_blur up to r = 255.5 */
#define CVB_FILTER_MAX_TAPS 1023

/* gaussian_kernel(r, kernel_size) into out[kernel_size]; host arithmetic, no context */
int cvb_gaussian_kernel(float r, uint32_t kernel_size, float *out);

int cvb_horizontal_filter(cvb_ctx *ctx, const float *in, uint32_t batch, uint32_t w, uint32_t h, const float *kernel, uint32_t kernel_size,
                          float *out);
int cvb_horizontal_filter_dev(cvb_ctx *ctx, const float *in_dev, uint32_t batch, uint32_t w, uint32_t h, const float *kernel,
                              uint32_t kernel_size, float *out_dev);

int cvb_vertical_filter(cvb_ctx *ctx, const float *in, uint32_t batch, uint32_t w, uint32_t h, const float *kernel, uint32_t kernel_size,
                        float *out);
int cvb_vertical_filter_dev(cvb_ctx *ctx, const float *in_dev, uint32_t batch, uint32_t w, uint32_t h, const float *kernel,
                            uint32_t kernel_size, float *out_dev);

int cvb_separable_filter(cvb_ctx *ctx, const float *in, uint32_t batch, uint32_t w, uint32_t h, const float *h_kernel, uint32_t h_size,
                         const float *v_kernel, uint32_t v_size, float *out);
int cvb_separable_filter_dev(cvb_ctx *ctx, const float *in_dev, uint32_t batch, uint32_t w, uint32_t h, const float *h_kernel,
                             uint32_t h_size, const float *v_kernel, uint32_t v_size, float *out_dev);

int cvb_gaussian_blur(cvb_ctx *ctx, const float *in, uint32_t batch, uint32_t w, uint32_t h, float r, float *out);
int cvb_gaussian_blur_dev(cvb_ctx *ctx, const float *in_dev, uint32_t batch, uint32_t w, uint32_t h, float r, float *out_dev);

/* out: batch planes of (w / 2) x (h / 2) */
int cvb_half_size(cvb_ctx *ctx, const float *in, uint32_t batch, uint32_t w, uint32_t h, float *out);
int cvb_half_size_dev(cvb_ctx *ctx, const float *in_dev, uint32_t batch, uint32_t w, uint32_t h, float *out_dev);

#ifdef __cplusplus
}
#endif
#endif /* CVB200_FILTER_H */
