//! Safe shim over include/cvb200_opt.h: cv-optimize's L1 optimizers on the device with cv-optimize's signatures (plus the context)
//! and batch forms.  ASSEMBLED by scripts/gen_rust_sys.py from the code block of INTEGRATION.md section 2e -- edit the document, then
//! regenerate.  A child module of the shim, so it reaches `Ctx`, `pose_to_c` and `pose_from_c`.
use super::*;
use cv_b200_sys::opt::*;

use cv_core::{nalgebra::UnitVector3, CameraToCamera, FeatureWorldMatch, Projective, WorldToCamera};

fn iterations_c(iterations: usize) -> u32 { iterations.min(u32::MAX as usize) as u32 }

/// single_view_simple_optimize_l1 for B problems: poses[b] with landmarks[offsets[b]..offsets[b + 1]]; returns the refined poses.
pub fn single_view_simple_optimize_l1_batch(ctx: &Ctx, poses: &[WorldToCamera], epsilon: f64, optimization_rate: f64, iterations: usize,
                                            landmarks: &[FeatureWorldMatch], offsets: &[u32]) -> Vec<WorldToCamera> {
    assert_eq!(offsets.len(), poses.len() + 1);
    let (mut bearings, mut world) = (Vec::with_capacity(3 * landmarks.len()), Vec::with_capacity(4 * landmarks.len()));
    for FeatureWorldMatch(b, w) in landmarks { bearings.extend_from_slice(b.as_slice()); world.extend_from_slice(w.homogeneous().as_slice()); }
    let input: Vec<cvb_pose> = poses.iter().map(|p| pose_to_c(&p.0)).collect();
    let mut out = vec![cvb_pose { r: [0.0; 9], t: [0.0; 3] }; poses.len()];
    let rc = unsafe { cvb_single_view_optimize_l1(ctx.0, input.as_ptr(), poses.len() as u32, epsilon, optimization_rate,
                                                  iterations_c(iterations), bearings.as_ptr(), world.as_ptr(), offsets.as_ptr(),
                                                  out.as_mut_ptr(), std::ptr::null_mut()) };
    assert_eq!(rc, 0, "{}", ctx.last_error());
    out.iter().map(|p| WorldToCamera(pose_from_c(p))).collect()
}

/// cv_optimize::single_view_simple_optimize_l1 on the GPU.
pub fn single_view_simple_optimize_l1(ctx: &Ctx, pose: WorldToCamera, epsilon: f64, optimization_rate: f64, iterations: usize,
                                      landmarks: &[FeatureWorldMatch]) -> WorldToCamera {
    if landmarks.is_empty() { return pose; }
    single_view_simple_optimize_l1_batch(ctx, &[pose], epsilon, optimization_rate, iterations, landmarks, &[0, landmarks.len() as u32])[0]
}

/// three_view_simple_optimize_l1 for B problems: poses[b] (centre -> first, centre -> second) with landmarks[offsets[b]..offsets[b + 1]].
pub fn three_view_simple_optimize_l1_batch(ctx: &Ctx, poses: &[[CameraToCamera; 2]], epsilon: f64, optimization_rate: f64,
                                           iterations: usize, landmarks: &[[UnitVector3<f64>; 3]], offsets: &[u32]) -> Vec<[CameraToCamera; 2]> {
    assert_eq!(offsets.len(), poses.len() + 1);
    let mut obs = Vec::with_capacity(9 * landmarks.len());
    for l in landmarks { for b in l { obs.extend_from_slice(b.as_slice()); } }
    let input: Vec<cvb_pose> = poses.iter().flat_map(|p| [pose_to_c(&p[0].0), pose_to_c(&p[1].0)]).collect();
    let mut out = vec![cvb_pose { r: [0.0; 9], t: [0.0; 3] }; 2 * poses.len()];
    let rc = unsafe { cvb_three_view_optimize_l1(ctx.0, input.as_ptr(), poses.len() as u32, epsilon, optimization_rate,
                                                 iterations_c(iterations), obs.as_ptr(), offsets.as_ptr(), out.as_mut_ptr(),
                                                 std::ptr::null_mut()) };
    assert_eq!(rc, 0, "{}", ctx.last_error());
    out.chunks(2).map(|p| [CameraToCamera(pose_from_c(&p[0])), CameraToCamera(pose_from_c(&p[1]))]).collect()
}

/// cv_optimize::three_view_simple_optimize_l1 on the GPU.
pub fn three_view_simple_optimize_l1(ctx: &Ctx, poses: [CameraToCamera; 2], epsilon: f64, optimization_rate: f64, iterations: usize,
                                     landmarks: &[[UnitVector3<f64>; 3]]) -> [CameraToCamera; 2] {
    if landmarks.is_empty() { return poses; }
    three_view_simple_optimize_l1_batch(ctx, &[poses], epsilon, optimization_rate, iterations, landmarks, &[0, landmarks.len() as u32])[0]
}
