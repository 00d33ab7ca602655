//! Safe shim over include/cvb200_try_init.h: cv-sfm's reconstruction creation on the device.
//! ASSEMBLED by scripts/gen_rust_sys.py from the code block of INTEGRATION.md section 2s -- edit the document, then regenerate.  A child
//! module of the shim, so it reaches `Ctx`.
use super::*;

use cv_b200_sys::constraints::cvb_view_constraint;
use cv_b200_sys::init::cvb_init_cfg;
use cv_b200_sys::tri::cvb_triangulator;
use cv_b200_sys::try_init::*;
use crate::incorporate::OwnedSnapshot;

/// A frame store as `cvb_frame_features_batch_dev` lays it out: frame b owns rows b * cap .. (b + 1) * cap; colours may be empty.
pub struct FrameStore<'a> {
    pub cap: usize, pub counts: &'a [u32], pub descriptors: &'a [[u8; 64]], pub bearings: &'a [[f64; 3]], pub colors: &'a [[u8; 3]],
}

/// What `try_init` returns: the result record (status, the three frames, the init's result, the counts) and the snapshot when created.
pub struct Created { pub result: cvb_try_init_result, pub snapshot: Option<OwnedSnapshot> }

/// `try_init(center, options)`: the two-view options with generator `rngs[f]` for option f (all advanced), the three-view
/// initialisation and, when accepted, `add_reconstruction`.
pub fn try_init(ctx: &Ctx, init: &cvb_init_cfg, tri: &cvb_triangulator, arrsac: &cvb_arrsac_cfg, rngs: &mut [cvb_rng], better_by: u32,
                store: &FrameStore, center: u32, options: &[u32]) -> Result<Created, String> {
    if options.len() != rngs.len() { return Err("one generator per option".into()); }
    let (cap, frames) = (store.cap, store.counts.len());
    let n = 3 * cap;
    let colors = !store.colors.is_empty();
    let mut o = OwnedSnapshot { poses: vec![cvb_pose::default(); 3], view_offsets: vec![0; 4], view_landmarks: vec![0; n],
                                bearings: vec![[0.0; 3]; n], descriptors: vec![[0; 64]; n],
                                colors: if colors { vec![[0; 3]; n] } else { Vec::new() }, landmark_offsets: vec![0; n + 1],
                                observations: vec![[0; 2]; n], constraints: vec![cvb_view_constraint::default(); 1] };
    let mut r = Created { result: cvb_try_init_result::default(), snapshot: None };
    let col_in = if colors { store.colors.as_ptr() as *const u8 } else { std::ptr::null() };
    let col_out = if colors { o.colors.as_mut_ptr() as *mut u8 } else { std::ptr::null_mut() };
    let rc = unsafe {
        cvb_try_init(ctx.0, init, tri, arrsac, rngs.as_mut_ptr(), better_by, store.descriptors.as_ptr() as *const u8, store.counts.as_ptr(),
                     store.bearings.as_ptr() as *const f64, col_in, frames as u32, cap as u32, center, options.as_ptr(), options.len() as u32,
                     o.poses.as_mut_ptr(), o.view_offsets.as_mut_ptr(), o.view_landmarks.as_mut_ptr(), o.bearings.as_mut_ptr() as *mut f64,
                     o.descriptors.as_mut_ptr() as *mut u8, col_out, o.landmark_offsets.as_mut_ptr(), o.observations.as_mut_ptr() as *mut u32,
                     o.constraints.as_mut_ptr(), &mut r.result)
    };
    if rc != 0 { return Err(ctx.last_error()); }
    if r.result.status as u32 == CVB_TRY_INIT_CREATED {
        let c = &r.result.counts;
        let nf = c.n_features as usize;
        o.view_landmarks.truncate(nf);
        o.bearings.truncate(nf);
        o.descriptors.truncate(nf);
        if colors { o.colors.truncate(nf); }
        o.landmark_offsets.truncate(c.L as usize + 1);
        o.observations.truncate(c.n_observations as usize);
        r.snapshot = Some(o);
    }
    Ok(r)
}
