// cv_b200/csrc/filter_abi.cu -- libcvb200_filter.so, the module that exports the C ABI of include/cvb200_filter.h (akaze::image: the
// separable filters, gaussian_kernel / gaussian_blur and half_size).  The kernels and their host code live in filter.cu inside
// libcvb200.so; this module only gives them their C names, so that libcvb200.so's own exports stay exactly those of cvb200.h,
// cvb200_sfm.h and cvb200_tri.h.  It links libcvb200.so (rpath $ORIGIN) and takes that library's contexts.
#include "../../include/cvb200_filter.h"

int flt_gaussian_kernel(float r, uint32_t kernel_size, float *out);
int flt_filter(cvb_ctx *ctx, bool vertical, const float *in, uint32_t batch, uint32_t w, uint32_t h, const float *kernel,
               uint32_t kernel_size, float *out, bool dev);
int flt_separable_filter(cvb_ctx *ctx, const float *in, uint32_t batch, uint32_t w, uint32_t h, const float *h_kernel, uint32_t h_size,
                         const float *v_kernel, uint32_t v_size, float *out, bool dev);
int flt_gaussian_blur(cvb_ctx *ctx, const float *in, uint32_t batch, uint32_t w, uint32_t h, float r, float *out, bool dev);
int flt_half_size(cvb_ctx *ctx, const float *in, uint32_t batch, uint32_t w, uint32_t h, float *out, bool dev);

extern "C" {

int cvb_gaussian_kernel(float r, uint32_t kernel_size, float *out) { return flt_gaussian_kernel(r, kernel_size, out); }

int cvb_horizontal_filter(cvb_ctx *ctx, const float *in, uint32_t batch, uint32_t w, uint32_t h, const float *kernel, uint32_t kernel_size,
                          float *out) {
    return flt_filter(ctx, false, in, batch, w, h, kernel, kernel_size, out, false);
}

int cvb_horizontal_filter_dev(cvb_ctx *ctx, const float *in_dev, uint32_t batch, uint32_t w, uint32_t h, const float *kernel,
                              uint32_t kernel_size, float *out_dev) {
    return flt_filter(ctx, false, in_dev, batch, w, h, kernel, kernel_size, out_dev, true);
}

int cvb_vertical_filter(cvb_ctx *ctx, const float *in, uint32_t batch, uint32_t w, uint32_t h, const float *kernel, uint32_t kernel_size,
                        float *out) {
    return flt_filter(ctx, true, in, batch, w, h, kernel, kernel_size, out, false);
}

int cvb_vertical_filter_dev(cvb_ctx *ctx, const float *in_dev, uint32_t batch, uint32_t w, uint32_t h, const float *kernel,
                            uint32_t kernel_size, float *out_dev) {
    return flt_filter(ctx, true, in_dev, batch, w, h, kernel, kernel_size, out_dev, true);
}

int cvb_separable_filter(cvb_ctx *ctx, const float *in, uint32_t batch, uint32_t w, uint32_t h, const float *h_kernel, uint32_t h_size,
                         const float *v_kernel, uint32_t v_size, float *out) {
    return flt_separable_filter(ctx, in, batch, w, h, h_kernel, h_size, v_kernel, v_size, out, false);
}

int cvb_separable_filter_dev(cvb_ctx *ctx, const float *in_dev, uint32_t batch, uint32_t w, uint32_t h, const float *h_kernel,
                             uint32_t h_size, const float *v_kernel, uint32_t v_size, float *out_dev) {
    return flt_separable_filter(ctx, in_dev, batch, w, h, h_kernel, h_size, v_kernel, v_size, out_dev, true);
}

int cvb_gaussian_blur(cvb_ctx *ctx, const float *in, uint32_t batch, uint32_t w, uint32_t h, float r, float *out) {
    return flt_gaussian_blur(ctx, in, batch, w, h, r, out, false);
}

int cvb_gaussian_blur_dev(cvb_ctx *ctx, const float *in_dev, uint32_t batch, uint32_t w, uint32_t h, float r, float *out_dev) {
    return flt_gaussian_blur(ctx, in_dev, batch, w, h, r, out_dev, true);
}

int cvb_half_size(cvb_ctx *ctx, const float *in, uint32_t batch, uint32_t w, uint32_t h, float *out) {
    return flt_half_size(ctx, in, batch, w, h, out, false);
}

int cvb_half_size_dev(cvb_ctx *ctx, const float *in_dev, uint32_t batch, uint32_t w, uint32_t h, float *out_dev) {
    return flt_half_size(ctx, in_dev, batch, w, h, out_dev, true);
}

}  // extern "C"
