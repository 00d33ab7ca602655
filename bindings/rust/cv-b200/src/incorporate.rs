//! Safe shim over include/cvb200_incorporate.h: cv-sfm's frame incorporation on the device.
//! ASSEMBLED by scripts/gen_rust_sys.py from the code block of INTEGRATION.md section 2q -- edit the document, then regenerate.  A child
//! module of the shim, so it reaches `Ctx`.
use super::*;

use cv_b200_sys::constraints::{cvb_constraints_cfg, cvb_view_constraint};
use cv_b200_sys::incorporate::*;
use cv_b200_sys::reconstruction::cvb_recon_cfg;
use cv_b200_sys::register::{cvb_register_cfg, cvb_register_match};
use cv_b200_sys::tri::cvb_triangulator;
use crate::constraints::Snapshot;

/// A snapshot that owns its rows: the layout of §2m plus the descriptors, colours and constraints.
#[derive(Clone, Default)]
pub struct OwnedSnapshot {
    pub poses: Vec<cvb_pose>, pub view_offsets: Vec<u32>, pub view_landmarks: Vec<u32>, pub bearings: Vec<[f64; 3]>,
    pub descriptors: Vec<[u8; 64]>, pub colors: Vec<[u8; 3]>, pub landmark_offsets: Vec<u32>, pub observations: Vec<[u32; 2]>,
    pub constraints: Vec<cvb_view_constraint>,
}
impl OwnedSnapshot {
    pub fn view(&self) -> Snapshot<'_> {
        Snapshot { poses: &self.poses, view_offsets: &self.view_offsets, view_landmarks: &self.view_landmarks, bearings: &self.bearings,
                   landmark_offsets: &self.landmark_offsets, observations: &self.observations }
    }
    fn with_capacity(v: usize, nf: usize, l: usize, no: usize, c: usize, colors: bool) -> Self {
        OwnedSnapshot { poses: vec![cvb_pose::default(); v.max(1)], view_offsets: vec![0; v + 1], view_landmarks: vec![0; nf.max(1)],
                        bearings: vec![[0.0; 3]; nf.max(1)], descriptors: vec![[0; 64]; nf.max(1)],
                        colors: if colors { vec![[0; 3]; nf.max(1)] } else { Vec::new() }, landmark_offsets: vec![0; l + 1],
                        observations: vec![[0; 2]; no.max(1)], constraints: vec![cvb_view_constraint::default(); c.max(1)] }
    }
    fn truncate(&mut self, c: &cvb_incorporate_counts) {
        let nf = c.n_features as usize;
        self.poses.truncate(c.V as usize);
        self.view_offsets.truncate(c.V as usize + 1);
        self.view_landmarks.truncate(nf);
        self.bearings.truncate(nf);
        self.descriptors.truncate(nf);
        if !self.colors.is_empty() { self.colors.truncate(nf); }
        self.landmark_offsets.truncate(c.L as usize + 1);
        self.observations.truncate(c.n_observations as usize);
        self.constraints.truncate(c.C as usize);
    }
}
fn opt_ptr<T>(v: &[T]) -> *const u8 { if v.is_empty() { std::ptr::null() } else { v.as_ptr() as *const u8 } }
fn opt_mut<T>(v: &mut [T]) -> *mut u8 { if v.is_empty() { std::ptr::null_mut() } else { v.as_mut_ptr() as *mut u8 } }

/// What `incorporate_frame` returns: the result header (status, the stages' results, the output counts), the snapshot when one exists
/// (kept, rejected, or the input when the frame was not registered), the maps from the input's views and landmarks to the output's, and
/// the registration's matches.
pub struct Incorporated {
    pub result: cvb_incorporate_result, pub snapshot: Option<OwnedSnapshot>, pub view_map: Vec<u32>, pub landmark_map: Vec<u32>,
    pub matches: Vec<cvb_register_match>,
}

/// `incorporate_frame` followed by `optimize_reconstruction` of one new frame against one snapshot.  `arrsac` and `rng` are VSlam's
/// `single_view_consensus`; `rng` advances as `register_frame`'s does.  `new_colors` is empty exactly when `s.colors` is.
pub fn incorporate_frame(ctx: &Ctx, reg: &cvb_register_cfg, con: &cvb_constraints_cfg, rec: &cvb_recon_cfg, tri: &cvb_triangulator,
                         arrsac: &cvb_arrsac_cfg, rng: &mut cvb_rng, s: &OwnedSnapshot, new_descriptors: &[[u8; 64]],
                         new_bearings: &[[f64; 3]], new_colors: &[[u8; 3]], view_matches: &[u32]) -> Result<Incorporated, String> {
    if new_descriptors.len() != new_bearings.len() { return Err("one bearing per new descriptor".into()); }
    let (v, l, n) = (s.poses.len(), s.landmark_offsets.len() - 1, new_descriptors.len());
    let (nf, no, c) = (s.view_landmarks.len(), s.observations.len(), s.constraints.len());
    let mut o = OwnedSnapshot::with_capacity(v + 1, nf + n, l + n + no + n, no + n,
                                             c + con.optimization_maximum_three_view_constraints as usize, !s.colors.is_empty());
    let mut r = Incorporated { result: cvb_incorporate_result::default(), snapshot: None, view_map: vec![0; v.max(1)],
                               landmark_map: vec![0; l.max(1)], matches: vec![cvb_register_match::default(); n.max(1)] };
    let rc = unsafe {
        cvb_incorporate_frame(ctx.0, reg, con, rec, tri, arrsac, rng, v as u32, s.poses.as_ptr(), s.view_offsets.as_ptr(),
                              s.view_landmarks.as_ptr(), s.bearings.as_ptr() as *const f64, s.descriptors.as_ptr() as *const u8,
                              opt_ptr(&s.colors), l as u32, s.landmark_offsets.as_ptr(), s.observations.as_ptr() as *const u32,
                              s.constraints.as_ptr(), c as u32, new_descriptors.as_ptr() as *const u8, new_bearings.as_ptr() as *const f64,
                              opt_ptr(new_colors), n as u32, view_matches.as_ptr(), view_matches.len() as u32, o.poses.as_mut_ptr(),
                              o.view_offsets.as_mut_ptr(), o.view_landmarks.as_mut_ptr(), o.bearings.as_mut_ptr() as *mut f64,
                              o.descriptors.as_mut_ptr() as *mut u8, opt_mut(&mut o.colors), o.landmark_offsets.as_mut_ptr(),
                              o.observations.as_mut_ptr() as *mut u32, o.constraints.as_mut_ptr(), r.view_map.as_mut_ptr(),
                              r.landmark_map.as_mut_ptr(), r.matches.as_mut_ptr(), &mut r.result)
    };
    if rc != 0 { return Err(ctx.last_error()); }
    let st = r.result.status as u32;
    if st == CVB_INCORPORATE_KEPT || st == CVB_INCORPORATE_REJECTED || st == CVB_INCORPORATE_NOT_REGISTERED {
        o.truncate(&r.result.counts);
        r.snapshot = Some(o);
    }
    r.view_map.truncate(v);
    r.landmark_map.truncate(l);
    r.matches.truncate(if r.result.reg.status == 0 { r.result.reg.n_matches as usize } else { 0 });
    Ok(r)
}

/// The edits of `optimize_reconstruction` (§2n) on the snapshot: `poses`, `view_state` and `obs_state` are its outputs (status kept).
/// Returns the new snapshot and the view and landmark maps.
pub fn apply_optimization(ctx: &Ctx, s: &OwnedSnapshot, poses: &[cvb_pose], view_state: &[u8], obs_state: &[u8])
                          -> Result<(OwnedSnapshot, Vec<u32>, Vec<u32>), String> {
    let (v, l, nf, no, c) = (s.poses.len(), s.landmark_offsets.len() - 1, s.view_landmarks.len(), s.observations.len(), s.constraints.len());
    let mut o = OwnedSnapshot::with_capacity(v, nf, l + no, no, c, !s.colors.is_empty());
    let (mut vmap, mut lmap) = (vec![0u32; v.max(1)], vec![0u32; l.max(1)]);
    let mut counts = cvb_incorporate_counts::default();
    let rc = unsafe {
        cvb_apply_optimization(ctx.0, v as u32, poses.as_ptr(), s.view_offsets.as_ptr(), s.view_landmarks.as_ptr(),
                               s.bearings.as_ptr() as *const f64, opt_ptr(&s.descriptors), opt_ptr(&s.colors), l as u32,
                               s.landmark_offsets.as_ptr(), s.observations.as_ptr() as *const u32, s.constraints.as_ptr(), c as u32,
                               view_state.as_ptr(), obs_state.as_ptr(), o.poses.as_mut_ptr(), o.view_offsets.as_mut_ptr(),
                               o.view_landmarks.as_mut_ptr(), o.bearings.as_mut_ptr() as *mut f64,
                               if s.descriptors.is_empty() { std::ptr::null_mut() } else { o.descriptors.as_mut_ptr() as *mut u8 },
                               opt_mut(&mut o.colors), o.landmark_offsets.as_mut_ptr(), o.observations.as_mut_ptr() as *mut u32,
                               o.constraints.as_mut_ptr(), vmap.as_mut_ptr(), lmap.as_mut_ptr(), &mut counts)
    };
    if rc != 0 { return Err(ctx.last_error()); }
    o.truncate(&counts);
    if s.descriptors.is_empty() { o.descriptors.clear(); }
    vmap.truncate(v);
    lmap.truncate(l);
    Ok((o, vmap, lmap))
}
