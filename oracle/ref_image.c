/* oracle/ref_image.c -- CPU oracle of include/cvb200_image.h (test infrastructure): GrayFloatImage::from_dynamic
 * (akaze/src/image.rs:45-109) of the eight integer DynamicImage variants, and DynamicImage::to_rgb8() of the four 8-bit ones.
 * Frames are packed and interleaved (ImageBuffer::as_bytes(), 16-bit channels little-endian); the conversion is per pixel. */
#include <stdint.h>
#include <string.h>
#include "ref_image.h"

/* image 0.24 rgb_to_luma (color.rs; external crate, restated from its published source): integer sRGB luma coefficients over 10000,
 * u32 intermediates, truncating division.  The one oracle copy of the formula (device: rgb_to_luma in cv_b200/csrc/image.cu). */
uint32_t ref_rgb_to_luma(uint32_t r, uint32_t g, uint32_t b) { return (2126u * r + 7152u * g + 722u * b) / 10000u; }

static const int CHANNELS[8] = {1, 2, 3, 4, 1, 2, 3, 4};

static uint32_t channel(const uint8_t *p, int c, int wide) {
    if (wide) { uint16_t v; memcpy(&v, p + 2 * c, 2); return v; }
    return p[c];
}

int ref_from_dynamic(uint32_t format, const void *pixels, size_t npx, float *gray) {
    if (format > 7) return -1;
    const int ch = CHANNELS[format], wide = format >= 4, bpp = ch * (wide ? 2 : 1);
    const float div = wide ? 65535.0f : 255.0f;
    const uint8_t *src = (const uint8_t *)pixels;
    for (size_t i = 0; i < npx; i++) {
        const uint8_t *p = src + i * bpp;
        /* grayscale(): luma variants unchanged (alpha never read), RGB(A) through rgb_to_luma (alpha dropped) */
        const uint32_t y = ch >= 3 ? ref_rgb_to_luma(channel(p, 0, wide), channel(p, 1, wide), channel(p, 2, wide)) : channel(p, 0, wide);
        gray[i] = (float)y / div;     /* f32::from(v) / 255f32 or / 65535f32 (image.rs:53-86) */
    }
    return 0;
}

int ref_to_rgb8(uint32_t format, const void *pixels, size_t npx, uint8_t *rgb) {
    if (format > 3) return -1;
    const int ch = CHANNELS[format];
    const uint8_t *src = (const uint8_t *)pixels;
    for (size_t i = 0; i < npx; i++) {
        const uint8_t *p = src + i * ch;
        rgb[3 * i] = p[0];
        rgb[3 * i + 1] = ch >= 3 ? p[1] : p[0];
        rgb[3 * i + 2] = ch >= 3 ? p[2] : p[0];
    }
    return 0;
}
