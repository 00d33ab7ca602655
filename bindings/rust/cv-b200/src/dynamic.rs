//! Safe shim over include/cvb200_image.h: `CudaAkaze::extract_dynamic` and `kps_descriptors_dynamic`, the reference's DynamicImage
//! input converted on the device.  ASSEMBLED by scripts/gen_rust_sys.py from the code block of INTEGRATION.md section 2g -- edit the
//! document, then regenerate.  A child module of the shim (named `dynamic` so that it does not shadow the image crate), so it reaches
//! `Ctx`, `to_c` and the private fields of `CudaAkaze`.
use super::*;

use cv_b200_sys::image::*;
use cv_core::nalgebra::{UnitVector3, Vector3};
use cv_pinhole::CameraIntrinsicsK1Distortion;

/// The variant's `cvb_pixel_format`, or None for the float variants (and any variant a later image crate adds).
pub fn pixel_format(image: &DynamicImage) -> Option<cvb_pixel_format> {
    Some(match image {
        DynamicImage::ImageLuma8(_) => CVB_PIXEL_LUMA8, DynamicImage::ImageLumaA8(_) => CVB_PIXEL_LUMA_A8,
        DynamicImage::ImageRgb8(_) => CVB_PIXEL_RGB8, DynamicImage::ImageRgba8(_) => CVB_PIXEL_RGBA8,
        DynamicImage::ImageLuma16(_) => CVB_PIXEL_LUMA16, DynamicImage::ImageLumaA16(_) => CVB_PIXEL_LUMA_A16,
        DynamicImage::ImageRgb16(_) => CVB_PIXEL_RGB16, DynamicImage::ImageRgba16(_) => CVB_PIXEL_RGBA16,
        _ => return None,
    })
}

impl CudaAkaze {
    /// Akaze::extract with the conversion on the device (`cvb_akaze_extract_dynamic_batch`): the frame's bytes are uploaded and
    /// converted as from_dynamic converts them.  The float variants take the host from_dynamic and the f32 entry point.
    pub fn extract_dynamic(&self, image: &DynamicImage) -> (Vec<akaze::KeyPoint>, Vec<BitArray<64>>) {
        let format = match pixel_format(image) { Some(f) => f, None => return self.extract(image) };
        let (w, h) = (image.width(), image.height());
        let cap = 32768u32;
        let mut kps = vec![cvb_keypoint::default(); cap as usize];
        let mut descs = vec![BitArray::<64>::zeros(); cap as usize];
        let mut n = 0u32;
        let rc = unsafe { cvb_akaze_extract_dynamic_batch(self.ctx.0, &to_c(&self.cfg), format, image.as_bytes().as_ptr() as *const _, 1,
                                                          w, h, kps.as_mut_ptr(), descs.as_mut_ptr() as *mut u8, cap, &mut n) };
        assert_eq!(rc, 0, "{}", self.ctx.last_error());
        let n = n as usize;
        (kps[..n].iter().map(|k| akaze::KeyPoint { point: (k.x, k.y), response: k.response, size: k.size, angle: k.angle,
                                                   octave: k.octave as usize, class_id: k.class_id as usize }).collect(),
         descs[..n].to_vec())
    }

    /// VSlam::kps_descriptors with both conversions on the device (`cvb_frame_features_dynamic_batch`): from_dynamic for the extractor and
    /// to_rgb8() for the colours, from the one uploaded frame.  Variants other than the four 8-bit ones take the host conversions
    /// (`kps_descriptors`).
    pub fn kps_descriptors_dynamic(&self, intrinsics: &CameraIntrinsicsK1Distortion, image: &DynamicImage)
                                   -> Vec<(BitArray<64>, FrameFeature)> {
        let format = match pixel_format(image) {
            Some(f) if f <= CVB_PIXEL_RGBA8 => f,
            _ => return self.kps_descriptors(intrinsics, image),
        };
        let (w, h) = (image.width(), image.height());
        let cap = 32768u32;
        let mut kps = vec![cvb_keypoint::default(); cap as usize];
        let mut descs = vec![BitArray::<64>::zeros(); cap as usize];
        let (mut bearings, mut colors, mut n) = (vec![0f64; 3 * cap as usize], vec![0u8; 3 * cap as usize], 0u32);
        let k = cvb_intrinsics_k1::from(intrinsics);
        let rc = unsafe { cvb_frame_features_dynamic_batch(self.ctx.0, &to_c(&self.cfg), format, image.as_bytes().as_ptr() as *const _, 1,
                                                           w, h, &k, kps.as_mut_ptr(), descs.as_mut_ptr() as *mut u8,
                                                           bearings.as_mut_ptr(), colors.as_mut_ptr(), cap, &mut n) };
        assert_eq!(rc, 0, "{}", self.ctx.last_error());
        (0..n as usize).map(|i| (descs[i].clone(), FrameFeature {
            bearing: UnitVector3::new_unchecked(Vector3::new(bearings[3 * i], bearings[3 * i + 1], bearings[3 * i + 2])),
            response: kps[i].response,
            color: [colors[3 * i], colors[3 * i + 1], colors[3 * i + 2]],
        })).collect()
    }
}
