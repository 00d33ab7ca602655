//! Safe shim over cv-b200-sys that keeps rust-cv's own surfaces: `akaze::Akaze::extract*`, `space::Knn`,
//! `sample_consensus::Consensus` and `cv_core::TriangulatorObservations`.  ASSEMBLED by scripts/gen_rust_sys.py from the code blocks of
//! INTEGRATION.md (sections 2 and 2b) behind this preamble -- edit the document, then regenerate.
#![allow(non_camel_case_types)]
use std::{ffi::CStr, sync::Arc};

use bitarray::{BitArray, Hamming};
use cv_b200_sys::*;
use ::image::DynamicImage;      // the image crate (the sys crate's module `image` is glob-imported above)
use space::Neighbor;

/// One library context (CUDA stream + workspaces).  Not thread-safe: keep one per worker thread; clones share the handle.
#[derive(Clone)]
pub struct Ctx(pub *mut cvb_ctx, Arc<CtxOwner>);
struct CtxOwner(*mut cvb_ctx);
impl Drop for CtxOwner { fn drop(&mut self) { unsafe { cvb_ctx_destroy(self.0) } } }
impl Ctx {
    pub fn new(device: i32) -> Result<Self, i32> {
        let mut p = std::ptr::null_mut();
        let rc = unsafe { cvb_ctx_create(device, &mut p) };
        if rc != 0 { return Err(rc); }                                   // CVB_ENODEV: there is no CPU fallback
        Ok(Ctx(p, Arc::new(CtxOwner(p))))
    }
    pub fn last_error(&self) -> String { unsafe { CStr::from_ptr(cvb_last_error(self.0)) }.to_string_lossy().into_owned() }
}

/// akaze::Akaze (akaze/src/lib.rs:109-142) -> the C configuration, field by field.
pub fn to_c(a: &akaze::Akaze) -> cvb_akaze_cfg {
    cvb_akaze_cfg { maximum_features: if a.maximum_features == usize::MAX { -1 } else { a.maximum_features as i64 },
                    num_sublevels: a.num_sublevels, max_octave_evolution: a.max_octave_evolution, base_scale_offset: a.base_scale_offset,
                    initial_contrast: a.initial_contrast, contrast_percentile: a.contrast_percentile,
                    contrast_factor_num_bins: a.contrast_factor_num_bins as u64, derivative_factor: a.derivative_factor,
                    detector_threshold: a.detector_threshold, descriptor_channels: a.descriptor_channels as u64,
                    descriptor_pattern_size: a.descriptor_pattern_size as u64 }
}

// ---- INTEGRATION.md section 2 ----
/// Drop-in for akaze::Akaze::extract_from_gray_float_image (akaze/src/lib.rs:309-339).
pub struct CudaAkaze { pub cfg: akaze::Akaze, ctx: Ctx }

impl CudaAkaze {
    pub fn extract_from_gray_float_image(&self, img: &akaze::image::GrayFloatImage) -> (Vec<akaze::KeyPoint>, Vec<BitArray<64>>) {
        let (w, h) = (img.width() as u32, img.height() as u32);
        let cap = 32768u32;
        let mut kps = vec![cvb_keypoint::default(); cap as usize];
        let mut descs = vec![BitArray::<64>::zeros(); cap as usize];        // #[repr(align(64))] [u8; 64]
        let mut n = 0u32;
        let rc = unsafe { cvb_akaze_extract(self.ctx.0, &to_c(&self.cfg), img.as_raw().as_ptr(), w, h,
                                            kps.as_mut_ptr(), descs.as_mut_ptr() as *mut u8, cap, &mut n) };
        assert_eq!(rc, 0, "{}", self.ctx.last_error());                       // the reference panics on hard errors too
        kps.truncate(n as usize); descs.truncate(n as usize);
        (kps.into_iter().map(|k| akaze::KeyPoint { point: (k.x, k.y), response: k.response, size: k.size,
                                                    octave: k.octave as usize, class_id: k.class_id as usize, angle: k.angle }).collect(), descs)
    }
    pub fn extract(&self, image: &DynamicImage) -> (Vec<akaze::KeyPoint>, Vec<BitArray<64>>) {
        self.extract_from_gray_float_image(&akaze::image::GrayFloatImage::from_dynamic(image))   // akaze/src/lib.rs:295-298
    }
}

/// space::Knn over a device-side brute force; same Neighbor order as LinearKnn (ties -> lower index).
pub struct CudaLinearKnn<'a> { pub points: &'a [BitArray<64>], ctx: Ctx }
impl<'a> space::Knn for CudaLinearKnn<'a> {
    type Ix = usize; type Metric = Hamming; type Point = BitArray<64>; type KnnIter = Vec<Neighbor<u32>>;
    fn knn(&self, query: &BitArray<64>, num: usize) -> Vec<Neighbor<u32>> {
        let (mut idx, mut dist) = (vec![0u32; num], vec![0u32; num]);
        let rc = unsafe { cvb_hamming_knn(self.ctx.0, query.as_ptr(), 1, self.points.as_ptr() as *const u8,
                                          self.points.len() as u32, num as u32, idx.as_mut_ptr(), dist.as_mut_ptr()) };
        assert_eq!(rc, 0);
        idx.into_iter().zip(dist).filter(|(i, _)| *i != u32::MAX).map(|(i, d)| Neighbor { index: i as usize, distance: d }).collect()
    }
}
// The per-query trait call is the real throughput limiter (SURVEY.md §8f-1): cv-sfm's `matching`
// (cv-sfm/src/lib.rs:3097-3114) should call `knn_batch` (one N x M launch) or `cvb_match_symmetric` directly.

// ---- INTEGRATION.md section 2b ----
use cv_core::{nalgebra::{IsometryMatrix3, Matrix3, Rotation3, Translation3, UnitVector3, Vector3},
              sample_consensus::{Consensus, Estimator}, CameraToCamera, FeatureMatch, FeatureWorldMatch, Projective,
              TriangulatorObservations, WorldPoint, WorldToCamera};

/// arrsac::Arrsac with the same builder methods; the estimator type only selects the entry point, its `estimate` is never called
/// on the host (hypotheses, residuals and ARRSAC's bookkeeping all run on the GPU).
pub struct CudaArrsac { pub cfg: cvb_arrsac_cfg, pub rng: cvb_rng, ctx: Ctx }

impl CudaArrsac {
    /// `rng`: e.g. `cvb_rng_seed_xoshiro256pp(&mut r, 0)` == `Xoshiro256PlusPlus::seed_from_u64(0)`
    pub fn new(inlier_threshold: f64, rng: cvb_rng, ctx: Ctx) -> Self {
        let mut cfg = std::mem::MaybeUninit::<cvb_arrsac_cfg>::uninit();
        unsafe { cvb_arrsac_default_cfg(cfg.as_mut_ptr(), inlier_threshold) };
        Self { cfg: unsafe { cfg.assume_init() }, rng, ctx }
    }
    pub fn initialization_hypotheses(mut self, n: usize) -> Self { self.cfg.initialization_hypotheses = n as u32; self }
    pub fn max_candidate_hypotheses(mut self, n: usize) -> Self { self.cfg.max_candidate_hypotheses = n as u32; self }
    pub fn estimations_per_block(mut self, n: usize) -> Self { self.cfg.estimations_per_block = n as u32; self }
    pub fn block_size(mut self, n: usize) -> Self { self.cfg.block_size = n as u32; self }
}

fn pose_from_c(p: &cvb_pose) -> IsometryMatrix3<f64> {
    IsometryMatrix3::from_parts(Translation3::new(p.t[0], p.t[1], p.t[2]),
                                Rotation3::from_matrix_unchecked(Matrix3::from_row_slice(&p.r)))
}
fn pose_to_c(p: &IsometryMatrix3<f64>) -> cvb_pose {
    let (m, t) = (p.rotation.matrix(), &p.translation.vector);
    cvb_pose { r: [m[(0, 0)], m[(0, 1)], m[(0, 2)], m[(1, 0)], m[(1, 1)], m[(1, 2)], m[(2, 0)], m[(2, 1)], m[(2, 2)]], t: [t.x, t.y, t.z] }
}

macro_rules! two_view_consensus {
    ($estimator:ty, $call:expr) => {
        impl Consensus<$estimator, FeatureMatch> for CudaArrsac {
            type Inliers = Vec<usize>;
            fn model<I>(&mut self, e: &$estimator, data: I) -> Option<CameraToCamera>
            where I: Iterator<Item = FeatureMatch> + Clone { self.model_inliers(e, data).map(|(m, _)| m) }
            fn model_inliers<I>(&mut self, _e: &$estimator, data: I) -> Option<(CameraToCamera, Vec<usize>)>
            where I: Iterator<Item = FeatureMatch> + Clone {
                let (mut a, mut b) = (Vec::new(), Vec::new());
                for FeatureMatch(x, y) in data { a.extend_from_slice(x.as_slice()); b.extend_from_slice(y.as_slice()); }
                let n = (a.len() / 3) as u32;
                let (mut model, mut inl) = (cvb_pose { r: [0.0; 9], t: [0.0; 3] }, vec![0u32; n as usize]);
                let (mut cnt, mut found) = (0u32, 0i32);
                let rc = unsafe { $call(self.ctx.0, &self.cfg, a.as_ptr(), b.as_ptr(), n, &mut self.rng, &mut model,
                                        inl.as_mut_ptr(), n, &mut cnt, &mut found) };
                assert_eq!(rc, 0, "{}", self.ctx.last_error());
                if found == 0 { return None; }
                inl.truncate(cnt as usize);
                Some((CameraToCamera(pose_from_c(&model)), inl.into_iter().map(|i| i as usize).collect()))   // indices follow the iterator order
            }
        }
    };
}
two_view_consensus!(eight_point::EightPoint, cvb_arrsac_eight_point);
unsafe fn five_point_ref(ctx: *mut cvb_ctx, cfg: *const cvb_arrsac_cfg, a: *const f64, b: *const f64, n: u32, rng: *mut cvb_rng,
                         model: *mut cvb_pose, inl: *mut u32, cap: u32, cnt: *mut u32, found: *mut i32) -> c_int {
    cvb_arrsac_five_point(ctx, cfg, a, b, n, rng, 5 /* the reference's rows, nister-stewenius/src/lib.rs:229 */, model, inl, cap, cnt, found)
}
two_view_consensus!(nister_stewenius::NisterStewenius, five_point_ref);

impl Consensus<lambda_twist::LambdaTwist, FeatureWorldMatch> for CudaArrsac {
    type Inliers = Vec<usize>;
    fn model<I>(&mut self, e: &lambda_twist::LambdaTwist, data: I) -> Option<WorldToCamera>
    where I: Iterator<Item = FeatureWorldMatch> + Clone { self.model_inliers(e, data).map(|(m, _)| m) }
    fn model_inliers<I>(&mut self, _e: &lambda_twist::LambdaTwist, data: I) -> Option<(WorldToCamera, Vec<usize>)>
    where I: Iterator<Item = FeatureWorldMatch> + Clone {
        let (mut bearings, mut world) = (Vec::new(), Vec::new());
        for FeatureWorldMatch(b, w) in data { bearings.extend_from_slice(b.as_slice()); world.extend_from_slice(w.homogeneous().as_slice()); }
        let n = (bearings.len() / 3) as u32;
        let (mut model, mut inl) = (cvb_pose { r: [0.0; 9], t: [0.0; 3] }, vec![0u32; n as usize]);
        let (mut cnt, mut found) = (0u32, 0i32);
        let rc = unsafe { cvb_arrsac_p3p(self.ctx.0, &self.cfg, bearings.as_ptr(), world.as_ptr(), n, &mut self.rng, &mut model,
                                         inl.as_mut_ptr(), n, &mut cnt, &mut found) };
        assert_eq!(rc, 0, "{}", self.ctx.last_error());
        if found == 0 { return None; }
        inl.truncate(cnt as usize);
        Some((WorldToCamera(pose_from_c(&model)), inl.into_iter().map(|i| i as usize).collect()))
    }
}

/// cv_geom::triangulation::LinearEigenTriangulator on the GPU.  The trait call triangulates ONE landmark; cv-sfm's hot callers
/// (`cv-sfm/src/lib.rs:1590,1679,1725,2642`) should collect their landmarks and call `triangulate_batch` once.
#[derive(Clone)]
pub struct CudaLinearEigen { ctx: Ctx }
impl CudaLinearEigen {
    pub fn triangulate_batch(&self, poses: &[cvb_pose], bearings: &[f64], offsets: &[u32]) -> Vec<Option<WorldPoint>> {
        let l = offsets.len() - 1;
        let (mut xyzw, mut ok) = (vec![0f64; 4 * l], vec![0u8; l]);
        let rc = unsafe { cvb_triangulate_linear_eigen(self.ctx.0, poses.as_ptr(), bearings.as_ptr(), offsets.as_ptr(), l as u32,
                                                       xyzw.as_mut_ptr(), ok.as_mut_ptr()) };
        assert_eq!(rc, 0, "{}", self.ctx.last_error());
        (0..l).map(|i| if ok[i] != 0 { Some(WorldPoint::from_homogeneous(cv_core::nalgebra::Vector4::from_column_slice(&xyzw[4 * i..4 * i + 4]))) } else { None }).collect()
    }
}
impl TriangulatorObservations for CudaLinearEigen {
    fn triangulate_observations(&self, pairs: impl Iterator<Item = (WorldToCamera, UnitVector3<f64>)> + Clone) -> Option<WorldPoint> {
        let (mut poses, mut bearings) = (Vec::new(), Vec::new());
        for (pose, b) in pairs { poses.push(pose_to_c(&pose.0)); bearings.extend_from_slice(b.as_slice()); }
        self.triangulate_batch(&poses, &bearings, &[0, poses.len() as u32]).pop().flatten()
    }
}


// ---- INTEGRATION.md section 2c (include/cvb200_sfm.h) ----
mod sfm;
pub use sfm::*;

// ---- INTEGRATION.md section 2d (include/cvb200_tri.h) ----
mod tri;
pub use tri::*;

// ---- INTEGRATION.md section 2e (include/cvb200_opt.h) ----
pub mod opt;

// ---- INTEGRATION.md section 2f (include/cvb200_pinhole.h) ----
pub mod pinhole;

// ---- INTEGRATION.md section 2g (include/cvb200_image.h) ----
pub mod dynamic;

// ---- INTEGRATION.md section 2h (include/cvb200_filter.h) ----
pub mod filter;

// ---- INTEGRATION.md section 2i (include/cvb200_lsh.h) ----
pub mod lsh;

// ---- INTEGRATION.md section 2j (include/cvb200_stages.h) ----
pub mod stages;

// ---- INTEGRATION.md section 2k (include/cvb200_batch.h) ----
pub mod batch;

// ---- INTEGRATION.md section 2l (include/cvb200_init.h) ----
pub mod init;

// ---- INTEGRATION.md section 2m (include/cvb200_constraints.h) ----
pub mod constraints;

// ---- INTEGRATION.md section 2n (include/cvb200_reconstruction.h) ----
pub mod reconstruction;

// ---- INTEGRATION.md section 2o (include/cvb200_export.h) ----
pub mod export;

// ---- INTEGRATION.md section 2p (include/cvb200_register.h) ----
pub mod register;

// ---- INTEGRATION.md section 2q (include/cvb200_incorporate.h) ----
pub mod incorporate;

// ---- INTEGRATION.md section 2r (include/cvb200_merge.h) ----
pub mod merge;

// ---- INTEGRATION.md section 2s (include/cvb200_try_init.h) ----
pub mod try_init;
