//! Safe shim over include/cvb200_filter.h: akaze::image's public functions on the device, with the reference's signatures plus the
//! context.  ASSEMBLED by scripts/gen_rust_sys.py from the code block of INTEGRATION.md section 2h -- edit the document, then
//! regenerate.  A child module of the shim, so it reaches `Ctx`.
use super::*;

use cv_b200_sys::filter::*;
use ::image::{ImageBuffer, Luma};
use akaze::image::GrayFloatImage;

/// akaze::image's GrayImageBuffer (a private alias there, spelled out in its public signatures)
pub type GrayImageBuffer = ImageBuffer<Luma<f32>, Vec<f32>>;

/// One host call on `image`'s pixels into a new (out_w x out_h) buffer; panics with the context's message on an error code.
fn call(ctx: &Ctx, image: &GrayImageBuffer, out_w: u32, out_h: u32, f: impl FnOnce(*const f32, u32, u32, *mut f32) -> i32)
        -> GrayImageBuffer {
    let mut out = vec![0f32; out_w as usize * out_h as usize];
    let rc = f(image.as_raw().as_ptr(), image.width(), image.height(), out.as_mut_ptr());
    assert_eq!(rc, 0, "{}", ctx.last_error());
    GrayImageBuffer::from_raw(out_w, out_h, out).unwrap()
}

/// akaze::image::gaussian_kernel (image.rs:349-374), host arithmetic.
pub fn gaussian_kernel(r: f32, kernel_size: usize) -> Vec<f32> {
    assert!(kernel_size % 2 == 1, "kernel_size must be odd");
    let mut kernel = vec![0f32; kernel_size];
    assert_eq!(unsafe { cvb_gaussian_kernel(r, kernel_size as u32, kernel.as_mut_ptr()) }, 0);
    kernel
}

/// akaze::image::horizontal_filter (image.rs:202-251)
pub fn horizontal_filter(ctx: &Ctx, image: &GrayImageBuffer, kernel: &[f32]) -> GrayImageBuffer {
    call(ctx, image, image.width(), image.height(),
         |i, w, h, o| unsafe { cvb_horizontal_filter(ctx.0, i, 1, w, h, kernel.as_ptr(), kernel.len() as u32, o) })
}

/// akaze::image::vertical_filter (image.rs:253-331)
pub fn vertical_filter(ctx: &Ctx, image: &GrayImageBuffer, kernel: &[f32]) -> GrayImageBuffer {
    call(ctx, image, image.width(), image.height(),
         |i, w, h, o| unsafe { cvb_vertical_filter(ctx.0, i, 1, w, h, kernel.as_ptr(), kernel.len() as u32, o) })
}

/// akaze::image::separable_filter (image.rs:333-340): one call, the intermediate plane stays on the device.
pub fn separable_filter(ctx: &Ctx, image: &GrayImageBuffer, h_kernel: &[f32], v_kernel: &[f32]) -> GrayImageBuffer {
    call(ctx, image, image.width(), image.height(), |i, w, h, o| unsafe {
        cvb_separable_filter(ctx.0, i, 1, w, h, h_kernel.as_ptr(), h_kernel.len() as u32, v_kernel.as_ptr(), v_kernel.len() as u32, o)
    })
}

/// akaze::image::gaussian_blur (image.rs:383-389)
pub fn gaussian_blur(ctx: &Ctx, image: &GrayFloatImage, r: f32) -> GrayFloatImage {
    assert!(r > 0.0, "sigma must be > 0.0");
    GrayFloatImage(call(ctx, &image.0, image.0.width(), image.0.height(), |i, w, h, o| unsafe { cvb_gaussian_blur(ctx.0, i, 1, w, h, r, o) }))
}

/// GrayFloatImage::half_size (image.rs:154-199)
pub fn half_size(ctx: &Ctx, image: &GrayFloatImage) -> GrayFloatImage {
    GrayFloatImage(call(ctx, &image.0, image.0.width() / 2, image.0.height() / 2, |i, w, h, o| unsafe { cvb_half_size(ctx.0, i, 1, w, h, o) }))
}
