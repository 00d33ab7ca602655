//! Safe shim over include/cvb200_export.h: cv-sfm's reconstruction export on the device.
//! ASSEMBLED by scripts/gen_rust_sys.py from the code block of INTEGRATION.md section 2o -- edit the document, then regenerate.  A child
//! module of the shim, so it reaches `Ctx`.
use super::*;

use cv_b200_sys::constraints::cvb_view_constraint;
use cv_b200_sys::export::*;
use cv_b200_sys::tri::cvb_triangulator;
use crate::constraints::Snapshot;

/// cv-sfm's defaults of the settings the export reads (cv-sfm/src/settings.rs).
pub fn export_cfg_default() -> cvb_export_cfg {
    let mut c = cvb_export_cfg::default();
    unsafe { cvb_export_cfg_default(&mut c) };
    c
}

/// `normalize_reconstruction` of one snapshot; `first_view` is the view the reconstruction's slot map yields first.  Returns the result,
/// the poses and the constraints (the inputs unchanged when `result.normalized` is 0).
pub fn normalize_reconstruction(ctx: &Ctx, cfg: &cvb_export_cfg, tri: &cvb_triangulator, s: &Snapshot, constraints: &[cvb_view_constraint],
                                first_view: u32) -> Result<(cvb_normalize_result, Vec<cvb_pose>, Vec<cvb_view_constraint>), String> {
    let v = s.poses.len();
    let mut res = cvb_normalize_result::default();
    let mut poses = vec![cvb_pose::default(); v.max(1)];
    let mut cons = vec![cvb_view_constraint::default(); constraints.len().max(1)];
    let rc = unsafe {
        cvb_normalize_reconstruction(ctx.0, cfg, tri, v as u32, s.poses.as_ptr(), s.view_offsets.as_ptr(), s.view_landmarks.as_ptr(),
                                     s.bearings.as_ptr() as *const f64, (s.landmark_offsets.len() - 1) as u32, s.landmark_offsets.as_ptr(),
                                     s.observations.as_ptr() as *const u32, constraints.as_ptr(), constraints.len() as u32, first_view,
                                     poses.as_mut_ptr(), cons.as_mut_ptr(), &mut res)
    };
    if rc != 0 { return Err(ctx.last_error()); }
    poses.truncate(v);
    cons.truncate(constraints.len());
    Ok((res, poses, cons))
}

/// What `export_reconstruction` writes: the points with their colours, and the cameras in view order.
pub struct Exported { pub points: Vec<[f64; 3]>, pub colors: Vec<[u8; 3]>, pub cameras: Vec<cvb_export_camera> }

/// `export_reconstruction` of one snapshot without the file; `colors` are the features' colours on the view CSR.
pub fn export_reconstruction(ctx: &Ctx, cfg: &cvb_export_cfg, tri: &cvb_triangulator, s: &Snapshot, colors: &[[u8; 3]])
                             -> Result<Exported, String> {
    let v = s.poses.len();
    let l = s.landmark_offsets.len() - 1;
    let mut n = 0u32;
    let mut e = Exported { points: vec![[0.0; 3]; l.max(1)], colors: vec![[0; 3]; l.max(1)], cameras: vec![cvb_export_camera::default(); v.max(1)] };
    let rc = unsafe {
        cvb_export_reconstruction(ctx.0, cfg, tri, v as u32, s.poses.as_ptr(), s.view_offsets.as_ptr(), s.view_landmarks.as_ptr(),
                                  s.bearings.as_ptr() as *const f64, colors.as_ptr() as *const u8, l as u32, s.landmark_offsets.as_ptr(),
                                  s.observations.as_ptr() as *const u32, e.points.as_mut_ptr() as *mut f64, e.colors.as_mut_ptr() as *mut u8,
                                  &mut n, e.cameras.as_mut_ptr(), std::ptr::null_mut())
    };
    if rc != 0 { return Err(ctx.last_error()); }
    e.points.truncate(n as usize);
    e.colors.truncate(n as usize);
    e.cameras.truncate(v);
    Ok(e)
}
