//! Safe shim over include/cvb200_register.h: cv-sfm's frame registration on the device.
//! ASSEMBLED by scripts/gen_rust_sys.py from the code block of INTEGRATION.md section 2p -- edit the document, then regenerate.  A child
//! module of the shim, so it reaches `Ctx`.
use super::*;

use cv_b200_sys::register::*;
use cv_b200_sys::tri::cvb_triangulator;
use crate::constraints::Snapshot;

/// cv-sfm's defaults of the settings register_frame reads (cv-sfm/src/settings.rs).
pub fn register_cfg_default() -> cvb_register_cfg {
    let mut c = cvb_register_cfg::default();
    unsafe { cvb_register_cfg_default(&mut c) };
    c
}

/// `register_frame` of one new frame against one snapshot: `descriptors` on the snapshot's view CSR, the new frame's descriptors and
/// bearings, the views to match against.  `arrsac` and `rng` are VSlam's `single_view_consensus`; `rng` advances as the reference's does.
/// `Ok(Some((pose, matches)))` is the reference's `Some` (the matches ascending by feature, `landmark_b` = `CVB_REGISTER_NONE` for a
/// single landmark), `Ok(None)` its `None`, and the reference's panic is an `Err`.
pub fn register_frame(ctx: &Ctx, cfg: &cvb_register_cfg, tri: &cvb_triangulator, arrsac: &cvb_arrsac_cfg, rng: &mut cvb_rng,
                      s: &Snapshot, descriptors: &[[u8; 64]], new_descriptors: &[[u8; 64]], new_bearings: &[[f64; 3]],
                      view_matches: &[u32]) -> Result<Option<(cvb_pose, Vec<cvb_register_match>)>, String> {
    if new_descriptors.len() != new_bearings.len() { return Err("one bearing per new descriptor".into()); }
    let n = new_descriptors.len();
    let mut res = cvb_register_result::default();
    let mut matches = vec![cvb_register_match::default(); n.max(1)];
    let rc = unsafe {
        cvb_register_frame(ctx.0, cfg, tri, arrsac, rng, s.poses.len() as u32, s.poses.as_ptr(), s.view_offsets.as_ptr(),
                           s.view_landmarks.as_ptr(), s.bearings.as_ptr() as *const f64, descriptors.as_ptr() as *const u8,
                           (s.landmark_offsets.len() - 1) as u32, s.landmark_offsets.as_ptr(), s.observations.as_ptr() as *const u32,
                           new_descriptors.as_ptr() as *const u8, new_bearings.as_ptr() as *const f64, n as u32, view_matches.as_ptr(),
                           view_matches.len() as u32, &mut res, matches.as_mut_ptr(), std::ptr::null_mut(), std::ptr::null_mut())
    };
    if rc != 0 { return Err(ctx.last_error()); }
    match res.status as u32 {
        CVB_REGISTER_OK => { matches.truncate(res.n_matches as usize); Ok(Some((res.pose, matches))) }
        CVB_REGISTER_PANIC => Err("register_frame: a feature has fewer than three distinct candidate landmarks".into()),
        _ => Ok(None),
    }
}
