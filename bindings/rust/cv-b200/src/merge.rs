//! Safe shim over include/cvb200_merge.h: cv-sfm's reconstruction merging on the device.
//! ASSEMBLED by scripts/gen_rust_sys.py from the code block of INTEGRATION.md section 2r -- edit the document, then regenerate.  A child
//! module of the shim, so it reaches `Ctx`.
use super::*;

use cv_b200_sys::constraints::{cvb_constraints_cfg, cvb_view_constraints_result};
use cv_b200_sys::merge::*;
use cv_b200_sys::reconstruction::cvb_recon_cfg;
use cv_b200_sys::register::cvb_register_cfg;
use cv_b200_sys::tri::cvb_triangulator;
use cv_b200_sys::incorporate::cvb_incorporate_counts;
use cv_b200_sys::constraints::cvb_view_constraint;
use crate::incorporate::OwnedSnapshot;

fn opt_ptr<T>(v: &[T]) -> *const u8 { if v.is_empty() { std::ptr::null() } else { v.as_ptr() as *const u8 } }
fn opt_mut<T>(v: &mut [T]) -> *mut u8 { if v.is_empty() { std::ptr::null_mut() } else { v.as_mut_ptr() as *mut u8 } }

fn sized(v: usize, nf: usize, l: usize, no: usize, c: usize, colors: bool) -> OwnedSnapshot {
    OwnedSnapshot { poses: vec![cvb_pose::default(); v.max(1)], view_offsets: vec![0; v + 1], view_landmarks: vec![0; nf.max(1)],
                    bearings: vec![[0.0; 3]; nf.max(1)], descriptors: vec![[0; 64]; nf.max(1)],
                    colors: if colors { vec![[0; 3]; nf.max(1)] } else { Vec::new() }, landmark_offsets: vec![0; l + 1],
                    observations: vec![[0; 2]; no.max(1)], constraints: vec![cvb_view_constraint::default(); c.max(1)] }
}
fn trim(o: &mut OwnedSnapshot, c: &cvb_incorporate_counts) {
    let nf = c.n_features as usize;
    o.poses.truncate(c.V as usize);
    o.view_offsets.truncate(c.V as usize + 1);
    o.view_landmarks.truncate(nf);
    o.bearings.truncate(nf);
    o.descriptors.truncate(nf);
    if !o.colors.is_empty() { o.colors.truncate(nf); }
    o.landmark_offsets.truncate(c.L as usize + 1);
    o.observations.truncate(c.n_observations as usize);
    o.constraints.truncate(c.C as usize);
}

/// What `merge_reconstructions` returns: the result header, the merged snapshot when one exists (merged, rejected, or D when the frame
/// was not registered), and the maps from both inputs' views and landmarks to the output's.
pub struct Merged {
    pub result: cvb_merge_result, pub snapshot: Option<OwnedSnapshot>, pub dest_view_map: Vec<u32>, pub dest_landmark_map: Vec<u32>,
    pub src_view_map: Vec<u32>, pub src_landmark_map: Vec<u32>, pub con_results: Vec<cvb_view_constraints_result>,
}

/// `try_merge_reconstructions(src, s_view, dest, dest_view_matches)` followed by `optimize_reconstruction(dest)`.  `arrsac` and `rng`
/// are VSlam's `single_view_consensus`; `rng` advances as `register_frame`'s does.  Both snapshots carry descriptors, and colours on both
/// sides or on neither.
pub fn merge_reconstructions(ctx: &Ctx, reg: &cvb_register_cfg, con: &cvb_constraints_cfg, rec: &cvb_recon_cfg, tri: &cvb_triangulator,
                             arrsac: &cvb_arrsac_cfg, rng: &mut cvb_rng, dest: &OwnedSnapshot, src: &OwnedSnapshot, s_view: u32,
                             dest_view_matches: &[u32]) -> Result<Merged, String> {
    let (v, l, nf, no, c) = (dest.poses.len(), dest.landmark_offsets.len() - 1, dest.view_landmarks.len(), dest.observations.len(),
                             dest.constraints.len());
    let (vs, ls, nfs) = (src.poses.len(), src.landmark_offsets.len() - 1, src.view_landmarks.len());
    let maxc = con.optimization_maximum_three_view_constraints as usize;
    let mut o = sized(v + vs, nf + nfs, l + no + 4 * nfs, no + 2 * nfs, c + (vs + 1) * maxc, !dest.colors.is_empty());
    let mut r = Merged { result: cvb_merge_result::default(), snapshot: None, dest_view_map: vec![0; v.max(1)],
                         dest_landmark_map: vec![0; l.max(1)], src_view_map: vec![0; vs.max(1)], src_landmark_map: vec![0; ls.max(1)],
                         con_results: vec![cvb_view_constraints_result::default(); vs.max(1)] };
    let rc = unsafe {
        cvb_merge_reconstructions(ctx.0, reg, con, rec, tri, arrsac, rng, v as u32, dest.poses.as_ptr(), dest.view_offsets.as_ptr(),
                                  dest.view_landmarks.as_ptr(), dest.bearings.as_ptr() as *const f64,
                                  dest.descriptors.as_ptr() as *const u8, opt_ptr(&dest.colors), l as u32, dest.landmark_offsets.as_ptr(),
                                  dest.observations.as_ptr() as *const u32, dest.constraints.as_ptr(), c as u32, vs as u32,
                                  src.poses.as_ptr(), src.view_offsets.as_ptr(), src.view_landmarks.as_ptr(),
                                  src.bearings.as_ptr() as *const f64, src.descriptors.as_ptr() as *const u8, opt_ptr(&src.colors),
                                  ls as u32, src.landmark_offsets.as_ptr(), src.observations.as_ptr() as *const u32, s_view,
                                  dest_view_matches.as_ptr(), dest_view_matches.len() as u32, o.poses.as_mut_ptr(),
                                  o.view_offsets.as_mut_ptr(), o.view_landmarks.as_mut_ptr(), o.bearings.as_mut_ptr() as *mut f64,
                                  o.descriptors.as_mut_ptr() as *mut u8, opt_mut(&mut o.colors), o.landmark_offsets.as_mut_ptr(),
                                  o.observations.as_mut_ptr() as *mut u32, o.constraints.as_mut_ptr(), r.dest_view_map.as_mut_ptr(),
                                  r.dest_landmark_map.as_mut_ptr(), r.src_view_map.as_mut_ptr(), r.src_landmark_map.as_mut_ptr(),
                                  r.con_results.as_mut_ptr(), &mut r.result)
    };
    if rc != 0 { return Err(ctx.last_error()); }
    let st = r.result.status as u32;
    if st == CVB_MERGE_MERGED || st == CVB_MERGE_REJECTED || st == CVB_MERGE_NOT_REGISTERED {
        trim(&mut o, &r.result.counts);
        r.snapshot = Some(o);
    }
    r.dest_view_map.truncate(v);
    r.dest_landmark_map.truncate(l);
    r.src_view_map.truncate(vs);
    r.src_landmark_map.truncate(ls);
    r.con_results.truncate(vs);
    Ok(r)
}
