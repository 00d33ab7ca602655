//! Safe shim over include/cvb200_init.h: cv-sfm's three-view initialisation over the two-view options on the device.
//! ASSEMBLED by scripts/gen_rust_sys.py from the code block of INTEGRATION.md section 2l -- edit the document, then regenerate.  A child
//! module of the shim, so it reaches `Ctx`.
use super::*;

use cv_b200_sys::init::*;
use cv_b200_sys::tri::cvb_triangulator;

/// cv-sfm's defaults of the settings init_reconstruction reads (cv-sfm/src/settings.rs).
pub fn init_cfg_default() -> cvb_init_cfg {
    let mut c = cvb_init_cfg::default();
    unsafe { cvb_init_cfg_default(&mut c) };
    c
}

/// Device buffers of one `cvb_init_reconstruction_dev` call: the outputs of `cvb_two_view_options_dev` for `options` (device
/// pointers, F = options.len()) and room for the result.
pub struct InitDeviceBuffers {
    pub bearings: *const f64, pub frames: u32, pub cap: u32,
    pub pairs: *const u32, pub n_pairs: *const u32, pub model: *const cvb_pose, pub inliers: *const u32, pub n_inliers: *const u32,
    pub found: *const i32,
    pub result: *mut cvb_init_result, pub combined: *mut u32, pub first_matches: *mut u32, pub second_matches: *mut u32,
    pub stats: *mut cvb_init_pair_stats,
}

/// `VSlam::init_reconstruction`'s choice of the three-view initialisation of `center` over `options` on the device.  The result
/// (`cvb_init_result`, lists) is left in the device buffers; the call returns once the decision is known.
///
/// # Safety
/// Every pointer in `b` must be a device allocation of the size include/cvb200_init.h gives, on `ctx`'s device.
pub unsafe fn init_reconstruction_dev(ctx: &Ctx, cfg: &cvb_init_cfg, tri: &cvb_triangulator, center: u32, options: &[u32],
                                      b: &InitDeviceBuffers) -> Result<(), String> {
    let rc = cvb_init_reconstruction_dev(ctx.0, cfg, tri, b.bearings, b.frames, b.cap, center, options.as_ptr(), options.len() as u32,
                                         b.pairs, b.n_pairs, b.model, b.inliers, b.n_inliers, b.found, b.result, b.combined,
                                         b.first_matches, b.second_matches, b.stats);
    if rc == 0 { Ok(()) } else { Err(ctx.last_error()) }
}
