//! Safe shim over include/cvb200_tri.h: cv-geom's triangulators on the device behind cv-core's `TriangulatorObservations` /
//! `TriangulatorRelative`.  ASSEMBLED by scripts/gen_rust_sys.py from the code block of INTEGRATION.md section 2d -- edit the document,
//! then regenerate.  A child module of the shim, so it reaches `Ctx`.
use super::*;
use cv_b200_sys::tri::*;

use cv_core::{nalgebra::{UnitVector3, Vector4}, CameraPoint, CameraToCamera, Projective, TriangulatorObservations, TriangulatorRelative,
              WorldPoint, WorldToCamera};

fn unpack<P: Projective>(xyzw: &[f64], ok: &[u8]) -> Vec<Option<P>> {
    // the device already normalised each point as Projective::from_homogeneous does
    ok.iter().enumerate()
        .map(|(i, &k)| if k != 0 { Some(P::from_homogeneous_unchecked(Vector4::from_column_slice(&xyzw[4 * i..4 * i + 4]))) } else { None })
        .collect()
}
fn config(method: i32) -> cvb_triangulator {
    let mut cfg = cvb_triangulator::default();
    unsafe { cvb_triangulator_default(&mut cfg, method) };
    cfg
}
/// `cvb_triangulate_relative`: poses (CameraToCamera) has one entry shared by every triple, or one per triple; a, b: 3 f64 per triple.
fn relative_batch(ctx: &Ctx, cfg: &cvb_triangulator, poses: &[cvb_pose], a: &[f64], b: &[f64]) -> Vec<Option<CameraPoint>> {
    let n = a.len() / 3;
    let (mut xyzw, mut ok) = (vec![0f64; 4 * n], vec![0u8; n]);
    let rc = unsafe { cvb_triangulate_relative(ctx.0, cfg, poses.as_ptr(), poses.len() as u32, a.as_ptr(), b.as_ptr(), n as u32,
                                               xyzw.as_mut_ptr(), ok.as_mut_ptr()) };
    assert_eq!(rc, 0, "{}", ctx.last_error());
    unpack(&xyzw, &ok)
}
fn relative_one(ctx: &Ctx, cfg: &cvb_triangulator, pose: CameraToCamera, a: UnitVector3<f64>, b: UnitVector3<f64>) -> Option<CameraPoint> {
    relative_batch(ctx, cfg, &[pose_to_c(&pose.0)], a.as_slice(), b.as_slice()).pop().flatten()
}

/// LinearEigenTriangulator, SineL1Triangulator or MeanMeanTriangulator on the GPU, with their builders.  The trait call
/// triangulates ONE landmark; cv-sfm's hot callers should collect their landmarks and call `triangulate_batch` once.
#[derive(Clone)]
pub struct CudaTriangulator { pub cfg: cvb_triangulator, ctx: Ctx }
impl CudaTriangulator {
    pub fn linear_eigen(ctx: Ctx) -> Self { Self { cfg: config(CVB_TRI_LINEAR_EIGEN), ctx } }
    pub fn sine_l1(ctx: Ctx) -> Self { Self { cfg: config(CVB_TRI_SINE_L1), ctx } }
    pub fn mean_mean(ctx: Ctx) -> Self { Self { cfg: config(CVB_TRI_MEAN_MEAN), ctx } }
    pub fn epsilon(mut self, epsilon: f64) -> Self { self.cfg.epsilon = epsilon; self }
    pub fn max_iterations(mut self, n: usize) -> Self { self.cfg.max_iterations = n.min(u32::MAX as usize) as u32; self }
    pub fn optimization_rate(mut self, rate: f64) -> Self { self.cfg.optimization_rate = rate; self }
    pub fn triangulate_batch(&self, poses: &[cvb_pose], bearings: &[f64], offsets: &[u32]) -> Vec<Option<WorldPoint>> {
        let l = offsets.len() - 1;
        let (mut xyzw, mut ok) = (vec![0f64; 4 * l], vec![0u8; l]);
        let rc = unsafe { cvb_triangulate_observations(self.ctx.0, &self.cfg, poses.as_ptr(), bearings.as_ptr(), offsets.as_ptr(),
                                                       l as u32, xyzw.as_mut_ptr(), ok.as_mut_ptr()) };
        assert_eq!(rc, 0, "{}", self.ctx.last_error());
        unpack(&xyzw, &ok)
    }
    /// the blanket TriangulatorRelative impl, batched: cv-sfm's three-view initialisation (cv-sfm/src/lib.rs:1022-1031)
    pub fn triangulate_relative_batch(&self, poses: &[cvb_pose], a: &[f64], b: &[f64]) -> Vec<Option<CameraPoint>> {
        relative_batch(&self.ctx, &self.cfg, poses, a, b)
    }
}
impl TriangulatorObservations for CudaTriangulator {
    fn triangulate_observations(&self, pairs: impl Iterator<Item = (WorldToCamera, UnitVector3<f64>)> + Clone) -> Option<WorldPoint> {
        let (mut poses, mut bearings) = (Vec::new(), Vec::new());
        for (pose, b) in pairs { poses.push(pose_to_c(&pose.0)); bearings.extend_from_slice(b.as_slice()); }
        self.triangulate_batch(&poses, &bearings, &[0, poses.len() as u32]).pop().flatten()
    }
}

/// RelativeDltTriangulator, AngularL1Triangulator or AngularLInfinityTriangulator on the GPU: TriangulatorRelative only.
#[derive(Clone)]
pub struct CudaRelativeTriangulator { pub cfg: cvb_triangulator, ctx: Ctx }
impl CudaRelativeTriangulator {
    pub fn relative_dlt(ctx: Ctx) -> Self { Self { cfg: config(CVB_TRI_RELATIVE_DLT), ctx } }
    pub fn angular_l1(ctx: Ctx) -> Self { Self { cfg: config(CVB_TRI_ANGULAR_L1), ctx } }
    pub fn angular_l_infinity(ctx: Ctx) -> Self { Self { cfg: config(CVB_TRI_ANGULAR_LINF), ctx } }
    pub fn epsilon(mut self, epsilon: f64) -> Self { self.cfg.epsilon = epsilon; self }
    pub fn max_iterations(mut self, n: usize) -> Self { self.cfg.max_iterations = n.min(u32::MAX as usize) as u32; self }
    pub fn triangulate_relative_batch(&self, poses: &[cvb_pose], a: &[f64], b: &[f64]) -> Vec<Option<CameraPoint>> {
        relative_batch(&self.ctx, &self.cfg, poses, a, b)
    }
}
impl TriangulatorRelative for CudaRelativeTriangulator {
    fn triangulate_relative(&self, pose: CameraToCamera, a: UnitVector3<f64>, b: UnitVector3<f64>) -> Option<CameraPoint> {
        relative_one(&self.ctx, &self.cfg, pose, a, b)
    }
}
