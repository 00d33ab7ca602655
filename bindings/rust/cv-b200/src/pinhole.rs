//! Safe shim over include/cvb200_pinhole.h: cv-pinhole's pose reprojection error and EssentialMatrix on the device, with cv-pinhole's
//! signatures (plus the context) and batch forms.  ASSEMBLED by scripts/gen_rust_sys.py from the code block of INTEGRATION.md section 2f
//! -- edit the document, then regenerate.  A child module of the shim, so it reaches `Ctx`, `pose_to_c` and `pose_from_c`.
use super::*;
use cv_b200_sys::pinhole::*;
use cv_b200_sys::tri::cvb_triangulator;

use cv_core::{nalgebra::{Matrix3, Rotation3, Vector2, Vector3}, CameraToCamera, FeatureMatch};
use cv_pinhole::EssentialMatrix;

fn iterations_c(iterations: usize) -> u32 { iterations.min(u32::MAX as usize) as u32 }
/// nalgebra is column-major, the C ABI row-major
fn mat_to_c(m: &Matrix3<f64>) -> [f64; 9] { let mut o = [0.0; 9]; for r in 0..3 { for c in 0..3 { o[3 * r + c] = m[(r, c)]; } } o }
fn mats_to_c(essentials: &[EssentialMatrix]) -> Vec<f64> { essentials.iter().flat_map(|e| mat_to_c(&e.0)).collect() }
fn bearings(matches: &[FeatureMatch]) -> (Vec<f64>, Vec<f64>) {
    let (mut a, mut b) = (Vec::with_capacity(3 * matches.len()), Vec::with_capacity(3 * matches.len()));
    for FeatureMatch(x, y) in matches { a.extend_from_slice(x.as_slice()); b.extend_from_slice(y.as_slice()); }
    (a, b)
}

/// pose_reprojection_error and average_pose_reprojection_error of every match; `poses` has one entry for every match or one per match.
pub fn pose_reprojection_error_batch(ctx: &Ctx, cfg: &cvb_triangulator, poses: &[CameraToCamera], matches: &[FeatureMatch])
                                     -> Vec<Option<([Vector2<f64>; 2], f64)>> {
    let n = matches.len();
    let (a, b) = bearings(matches);
    let p: Vec<cvb_pose> = poses.iter().map(|p| pose_to_c(&p.0)).collect();
    let (mut err, mut avg, mut ok) = (vec![0f64; 4 * n], vec![0f64; n], vec![0u8; n]);
    let rc = unsafe { cvb_pose_reprojection_error(ctx.0, cfg, p.as_ptr(), p.len() as u32, a.as_ptr(), b.as_ptr(), n as u32,
                                                  err.as_mut_ptr(), avg.as_mut_ptr(), ok.as_mut_ptr()) };
    assert_eq!(rc, 0, "{}", ctx.last_error());
    (0..n).map(|i| (ok[i] != 0).then(|| ([Vector2::new(err[4 * i], err[4 * i + 1]), Vector2::new(err[4 * i + 2], err[4 * i + 3])], avg[i])))
        .collect()
}

/// cv_pinhole::pose_reprojection_error on the GPU.
pub fn pose_reprojection_error(ctx: &Ctx, cfg: &cvb_triangulator, pose: CameraToCamera, m: FeatureMatch) -> Option<[Vector2<f64>; 2]> {
    pose_reprojection_error_batch(ctx, cfg, &[pose], &[m]).pop().flatten().map(|(e, _)| e)
}

/// cv_pinhole::average_pose_reprojection_error on the GPU.
pub fn average_pose_reprojection_error(ctx: &Ctx, cfg: &cvb_triangulator, pose: CameraToCamera, m: FeatureMatch) -> Option<f64> {
    pose_reprojection_error_batch(ctx, cfg, &[pose], &[m]).pop().flatten().map(|(_, avg)| avg)
}

/// EightPoint { epsilon, iterations }::from_matches for every sample of 8 indices into `matches`.
pub fn from_matches_batch(ctx: &Ctx, epsilon: f64, iterations: usize, matches: &[FeatureMatch], samples: &[[u32; 8]])
                          -> Vec<Option<EssentialMatrix>> {
    let (a, b) = bearings(matches);
    let h = samples.len();
    let (mut e, mut ok) = (vec![0f64; 9 * h], vec![0u8; h]);
    let rc = unsafe { cvb_eight_point_essential_batch(ctx.0, epsilon, iterations_c(iterations), a.as_ptr(), b.as_ptr(), matches.len() as u32,
                                                      samples.as_ptr() as *const u32, h as u32, e.as_mut_ptr(), ok.as_mut_ptr()) };
    assert_eq!(rc, 0, "{}", ctx.last_error());
    (0..h).map(|k| (ok[k] != 0).then(|| EssentialMatrix(Matrix3::from_row_slice(&e[9 * k..9 * k + 9])))).collect()
}

/// Model::residual of every (essential matrix, match): essentials.len() rows of matches.len() residuals.
pub fn residuals_batch(ctx: &Ctx, essentials: &[EssentialMatrix], matches: &[FeatureMatch]) -> Vec<f64> {
    let (a, b) = bearings(matches);
    let e = mats_to_c(essentials);
    let mut out = vec![0f64; essentials.len() * matches.len()];
    let rc = unsafe { cvb_residuals_essential(ctx.0, e.as_ptr(), essentials.len() as u32, a.as_ptr(), b.as_ptr(), matches.len() as u32,
                                              out.as_mut_ptr()) };
    assert_eq!(rc, 0, "{}", ctx.last_error());
    out
}

/// EssentialMatrix::recondition of every matrix.
pub fn recondition_batch(ctx: &Ctx, essentials: &[EssentialMatrix], epsilon: f64, max_iterations: usize) -> Vec<Option<EssentialMatrix>> {
    let m = essentials.len();
    let e = mats_to_c(essentials);
    let (mut out, mut ok) = (vec![0f64; 9 * m], vec![0u8; m]);
    let rc = unsafe { cvb_essential_recondition(ctx.0, e.as_ptr(), m as u32, epsilon, iterations_c(max_iterations), out.as_mut_ptr(),
                                                ok.as_mut_ptr()) };
    assert_eq!(rc, 0, "{}", ctx.last_error());
    (0..m).map(|k| (ok[k] != 0).then(|| EssentialMatrix(Matrix3::from_row_slice(&out[9 * k..9 * k + 9])))).collect()
}

/// EssentialMatrix::possible_rotations_unscaled_translation of every matrix.
pub fn possible_rotations_unscaled_translation_batch(ctx: &Ctx, essentials: &[EssentialMatrix], epsilon: f64, max_iterations: usize)
                                                     -> Vec<Option<(Rotation3<f64>, Rotation3<f64>, Vector3<f64>)>> {
    let m = essentials.len();
    let e = mats_to_c(essentials);
    let (mut ra, mut rb, mut t, mut ok) = (vec![0f64; 9 * m], vec![0f64; 9 * m], vec![0f64; 3 * m], vec![0u8; m]);
    let rc = unsafe { cvb_essential_decompose(ctx.0, e.as_ptr(), m as u32, epsilon, iterations_c(max_iterations), ra.as_mut_ptr(),
                                              rb.as_mut_ptr(), t.as_mut_ptr(), ok.as_mut_ptr()) };
    assert_eq!(rc, 0, "{}", ctx.last_error());
    (0..m).map(|k| (ok[k] != 0).then(|| (Rotation3::from_matrix_unchecked(Matrix3::from_row_slice(&ra[9 * k..9 * k + 9])),
                                          Rotation3::from_matrix_unchecked(Matrix3::from_row_slice(&rb[9 * k..9 * k + 9])),
                                          Vector3::from_column_slice(&t[3 * k..3 * k + 3]))))
        .collect()
}

/// EssentialMatrix::possible_rotations of every matrix.
pub fn possible_rotations_batch(ctx: &Ctx, essentials: &[EssentialMatrix], epsilon: f64, max_iterations: usize) -> Vec<Option<[Rotation3<f64>; 2]>> {
    possible_rotations_unscaled_translation_batch(ctx, essentials, epsilon, max_iterations).into_iter()
        .map(|r| r.map(|(a, b, _)| [a, b])).collect()
}

/// EssentialMatrix::possible_unscaled_poses of every matrix: (t, Ra), (t, Rb), (-t, Ra), (-t, Rb).
pub fn possible_unscaled_poses_batch(ctx: &Ctx, essentials: &[EssentialMatrix], epsilon: f64, max_iterations: usize)
                                     -> Vec<Option<[CameraToCamera; 4]>> {
    possible_rotations_unscaled_translation_batch(ctx, essentials, epsilon, max_iterations).into_iter()
        .map(|r| r.map(|(a, b, t)| [CameraToCamera::from_parts(t, a), CameraToCamera::from_parts(t, b),
                                    CameraToCamera::from_parts(-t, a), CameraToCamera::from_parts(-t, b)]))
        .collect()
}

/// EssentialMatrix::possible_unscaled_poses_bearing of every matrix: (t, Ra), (t, Rb).
pub fn possible_unscaled_poses_bearing_batch(ctx: &Ctx, essentials: &[EssentialMatrix], epsilon: f64, max_iterations: usize)
                                             -> Vec<Option<[CameraToCamera; 2]>> {
    possible_rotations_unscaled_translation_batch(ctx, essentials, epsilon, max_iterations).into_iter()
        .map(|r| r.map(|(a, b, t)| [CameraToCamera::from_parts(t, a), CameraToCamera::from_parts(t, b)]))
        .collect()
}
