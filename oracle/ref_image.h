/* oracle/ref_image.h -- CPU oracle of include/cvb200_image.h (test infrastructure).  Formats are the cvb_pixel_format codes 0..7
 * (LUMA8, LUMA_A8, RGB8, RGBA8, LUMA16, LUMA_A16, RGB16, RGBA16); the functions return -1 for any other code. */
#ifndef REF_IMAGE_H
#define REF_IMAGE_H
#include <stddef.h>
#include <stdint.h>

uint32_t ref_rgb_to_luma(uint32_t r, uint32_t g, uint32_t b);
/* GrayFloatImage::from_dynamic of npx packed pixels */
int ref_from_dynamic(uint32_t format, const void *pixels, size_t npx, float *gray);
/* DynamicImage::to_rgb8() of npx packed pixels, 8-bit formats (0..3) only */
int ref_to_rgb8(uint32_t format, const void *pixels, size_t npx, uint8_t *rgb);

#endif
