//! Safe shim over include/cvb200_sfm.h: the reference's camera with radial distortion in the two-view entry point and cv-sfm's
//! `VSlam::kps_descriptors`.  ASSEMBLED by scripts/gen_rust_sys.py from the code block of INTEGRATION.md section 2c -- edit the
//! document, then regenerate.  A child module of the shim, so it reaches `Ctx`, `to_c` and the private fields of the parent's types.
use super::*;

use cv_core::{nalgebra::{UnitVector3, Vector3}, CameraToCamera};
use cv_pinhole::CameraIntrinsicsK1Distortion;      // cvb_intrinsics_k1::from(&camera): cv-b200-sys, feature "cv-pinhole"

impl CudaArrsac {
    /// cv-sfm's two-view initialisation of one frame pair on the device (`cvb_two_view_frames_k1`, cv-sfm/src/lib.rs:1375-1412): AKAZE
    /// on both frames, symmetric matching (`d0 + better_by <= d1`), the K1 bearings of the matches, then this object's ARRSAC +
    /// eight-point.  Both frames have one size.  Returns the pose, the matches `[a, b]` and the inliers (indices into the matches);
    /// `self.rng` advances as the reference's generator would.
    pub fn two_view_frames(&mut self, akaze: &akaze::Akaze, a: &akaze::image::GrayFloatImage, b: &akaze::image::GrayFloatImage,
                           camera: &CameraIntrinsicsK1Distortion, better_by: u32) -> Option<(CameraToCamera, Vec<[usize; 2]>, Vec<usize>)> {
        let (w, h) = (a.width() as u32, a.height() as u32);
        assert_eq!((w, h), (b.width() as u32, b.height() as u32), "both frames must have one size");
        let mut frames = Vec::with_capacity(2 * (w * h) as usize);
        frames.extend_from_slice(a.as_raw());
        frames.extend_from_slice(b.as_raw());
        let cap = 32768u32;
        let (mut kps, mut descs) = (vec![cvb_keypoint::default(); 2 * cap as usize], vec![0u8; 2 * 64 * cap as usize]);
        let (mut n, mut pairs, mut inl) = ([0u32; 2], vec![0u32; 2 * cap as usize], vec![0u32; cap as usize]);
        let (mut n_pairs, mut n_inl, mut found) = (0u32, 0u32, 0i32);
        let mut model = cvb_pose { r: [0.0; 9], t: [0.0; 3] };
        let k = cvb_intrinsics_k1::from(camera);
        let rc = unsafe { cvb_two_view_frames_k1(self.ctx.0, &to_c(akaze), frames.as_ptr(), w, h, better_by, &k, &self.cfg, &mut self.rng,
                                                 kps.as_mut_ptr(), descs.as_mut_ptr(), cap, n.as_mut_ptr(), pairs.as_mut_ptr(),
                                                 &mut n_pairs, &mut model, inl.as_mut_ptr(), &mut n_inl, &mut found) };
        assert_eq!(rc, 0, "{}", self.ctx.last_error());
        if found == 0 { return None; }
        let matches = pairs[..2 * n_pairs as usize].chunks(2).map(|p| [p[0] as usize, p[1] as usize]).collect();
        Some((CameraToCamera(pose_from_c(&model)), matches, inl[..n_inl as usize].iter().map(|&i| i as usize).collect()))
    }
}

/// cv-sfm's `Feature` (cv-sfm/src/lib.rs:61-65), field for field.
pub struct FrameFeature { pub bearing: UnitVector3<f64>, pub response: f32, pub color: [u8; 3] }

impl CudaAkaze {
    /// VSlam::kps_descriptors (cv-sfm/src/lib.rs:2195-2235) on the device (`cvb_frame_features_batch`); `self.cfg` carries cv-sfm's
    /// `maximum_features`.  The image crate converts on the host: `GrayFloatImage::from_dynamic` (i.e. `image.grayscale()`) for the
    /// extractor, `image.to_rgb8()` for the colours, so the luma stays exactly the reference's.  Features come in the reference's
    /// order (descending response, which is AKAZE's own order).
    pub fn kps_descriptors(&self, intrinsics: &CameraIntrinsicsK1Distortion, image: &DynamicImage) -> Vec<(BitArray<64>, FrameFeature)> {
        let gray = akaze::image::GrayFloatImage::from_dynamic(image);
        let rgb = image.to_rgb8();
        let (w, h) = (gray.width() as u32, gray.height() as u32);
        let cap = 32768u32;
        let mut kps = vec![cvb_keypoint::default(); cap as usize];
        let mut descs = vec![BitArray::<64>::zeros(); cap as usize];
        let (mut bearings, mut colors, mut n) = (vec![0f64; 3 * cap as usize], vec![0u8; 3 * cap as usize], 0u32);
        let k = cvb_intrinsics_k1::from(intrinsics);
        let rc = unsafe { cvb_frame_features_batch(self.ctx.0, &to_c(&self.cfg), gray.as_raw().as_ptr(), rgb.as_raw().as_ptr(), 1, w, h,
                                                   &k, kps.as_mut_ptr(), descs.as_mut_ptr() as *mut u8, bearings.as_mut_ptr(),
                                                   colors.as_mut_ptr(), cap, &mut n) };
        assert_eq!(rc, 0, "{}", self.ctx.last_error());
        (0..n as usize).map(|i| (descs[i].clone(), FrameFeature {
            bearing: UnitVector3::new_unchecked(Vector3::new(bearings[3 * i], bearings[3 * i + 1], bearings[3 * i + 2])),
            response: kps[i].response,
            color: [colors[3 * i], colors[3 * i + 1], colors[3 * i + 2]],
        })).collect()
    }
}
