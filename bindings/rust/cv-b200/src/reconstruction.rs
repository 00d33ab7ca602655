//! Safe shim over include/cvb200_reconstruction.h: cv-sfm's reconstruction optimisation on the device.
//! ASSEMBLED by scripts/gen_rust_sys.py from the code block of INTEGRATION.md section 2n -- edit the document, then regenerate.  A child
//! module of the shim, so it reaches `Ctx`.
use super::*;

use cv_b200_sys::constraints::cvb_view_constraint;
use cv_b200_sys::reconstruction::*;
use cv_b200_sys::tri::cvb_triangulator;
use crate::constraints::Snapshot;

/// cv-sfm's defaults of the settings optimize_reconstruction reads (cv-sfm/src/settings.rs).
pub fn recon_cfg_default() -> cvb_recon_cfg {
    let mut c = cvb_recon_cfg::default();
    unsafe { cvb_recon_cfg_default(&mut c) };
    c
}

/// The outcome of `optimize_reconstruction`: the result header, the final poses, a state per view and a state per observation.
pub struct Optimized {
    pub result: cvb_recon_result, pub poses: Vec<cvb_pose>, pub view_state: Vec<u8>, pub obs_state: Vec<u8>,
}

/// `optimize_reconstruction` of one snapshot with its constraints, in the reconstruction's order.
pub fn optimize_reconstruction(ctx: &Ctx, cfg: &cvb_recon_cfg, tri: &cvb_triangulator, s: &Snapshot, constraints: &[cvb_view_constraint])
                               -> Result<Optimized, String> {
    let v = s.poses.len();
    let n_obs = s.observations.len();
    let mut o = Optimized { result: cvb_recon_result::default(), poses: vec![cvb_pose::default(); v.max(1)], view_state: vec![0; v.max(1)],
                            obs_state: vec![0; n_obs.max(1)] };
    let rc = unsafe {
        cvb_optimize_reconstruction(ctx.0, cfg, tri, v as u32, s.poses.as_ptr(), s.view_offsets.as_ptr(), s.view_landmarks.as_ptr(),
                                    s.bearings.as_ptr() as *const f64, (s.landmark_offsets.len() - 1) as u32, s.landmark_offsets.as_ptr(),
                                    s.observations.as_ptr() as *const u32, constraints.as_ptr(), constraints.len() as u32, &mut o.result,
                                    o.poses.as_mut_ptr(), o.view_state.as_mut_ptr(), o.obs_state.as_mut_ptr())
    };
    if rc != 0 { return Err(ctx.last_error()); }
    o.poses.truncate(v);
    o.view_state.truncate(v);
    o.obs_state.truncate(n_obs);
    Ok(o)
}
