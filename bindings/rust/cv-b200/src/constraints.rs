//! Safe shim over include/cvb200_constraints.h: cv-sfm's three-view constraints of many views of a reconstruction on the device.
//! ASSEMBLED by scripts/gen_rust_sys.py from the code block of INTEGRATION.md section 2m -- edit the document, then regenerate.  A child
//! module of the shim, so it reaches `Ctx`.
use super::*;

use cv_b200_sys::constraints::*;
use cv_b200_sys::tri::cvb_triangulator;

/// cv-sfm's defaults of the settings generate_view_constraints and record_view_constraints read (cv-sfm/src/settings.rs).
pub fn constraints_cfg_default() -> cvb_constraints_cfg {
    let mut c = cvb_constraints_cfg::default();
    unsafe { cvb_constraints_cfg_default(&mut c) };
    c
}

/// One reconstruction snapshot on the host, views in ascending ViewKey order (include/cvb200_constraints.h).
pub struct Snapshot<'a> {
    pub poses: &'a [cvb_pose], pub view_offsets: &'a [u32], pub view_landmarks: &'a [u32], pub bearings: &'a [[f64; 3]],
    pub landmark_offsets: &'a [u32], pub observations: &'a [[u32; 2]],
}

/// `generate_view_constraints` and `record_view_constraints`' acceptance for every view in `queries`: per query its constraints in the
/// reference's evaluation order and whether the reference would record them.
pub fn view_constraints(ctx: &Ctx, cfg: &cvb_constraints_cfg, tri: &cvb_triangulator, s: &Snapshot, queries: &[u32])
                        -> Result<Vec<(Vec<cvb_view_constraint>, bool)>, String> {
    let maxc = cfg.optimization_maximum_three_view_constraints as usize;
    let q = queries.len();
    let mut out = vec![cvb_view_constraint::default(); (q * maxc).max(1)];
    let mut res = vec![cvb_view_constraints_result::default(); q.max(1)];
    let rc = unsafe {
        cvb_view_constraints(ctx.0, cfg, tri, s.poses.len() as u32, s.poses.as_ptr(), s.view_offsets.as_ptr(), s.view_landmarks.as_ptr(),
                             s.bearings.as_ptr() as *const f64, (s.landmark_offsets.len() - 1) as u32, s.landmark_offsets.as_ptr(),
                             s.observations.as_ptr() as *const u32, queries.as_ptr(), q as u32, out.as_mut_ptr(), res.as_mut_ptr(),
                             std::ptr::null_mut())
    };
    if rc != 0 { return Err(ctx.last_error()); }
    Ok((0..q).map(|i| (out[i * maxc..i * maxc + res[i].n_constraints as usize].to_vec(), res[i].accepted != 0)).collect())
}
