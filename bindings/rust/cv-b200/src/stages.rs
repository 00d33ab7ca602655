//! Safe shim over include/cvb200_stages.h: `CudaEvolutions` and the staged methods of `CudaAkaze` with the reference's signatures.
//! ASSEMBLED by scripts/gen_rust_sys.py from the code block of INTEGRATION.md section 2j -- edit the document, then regenerate.  A child
//! module of the shim, so it reaches `Ctx`, `to_c` and the private fields of `CudaAkaze`.
use super::*;

use cv_b200_sys::stages::*;

/// A scale space resident in a context (the device-side counterpart of akaze's Vec<EvolutionStep>): its ticket, the context that holds
/// it, the EvolutionStep scalars and the config it was built with.  A later extract or scale space on the same context replaces it.
pub struct CudaEvolutions { pub ticket: u64, pub ctx: Ctx, pub evolutions: Vec<cvb_akaze_evolution>, batch: u32, cfg: cvb_akaze_cfg }

/// The fields detection depends on: all but maximum_features (ignored by find), the descriptor fields and initial_contrast (never read).
fn same_detector(a: &cvb_akaze_cfg, b: &cvb_akaze_cfg) -> bool {
    a.num_sublevels == b.num_sublevels && a.max_octave_evolution == b.max_octave_evolution && a.base_scale_offset == b.base_scale_offset
        && a.contrast_percentile == b.contrast_percentile && a.contrast_factor_num_bins == b.contrast_factor_num_bins
        && a.derivative_factor == b.derivative_factor && a.detector_threshold == b.detector_threshold
}

fn kp_to_c(k: &akaze::KeyPoint) -> cvb_keypoint {
    cvb_keypoint { x: k.point.0, y: k.point.1, response: k.response, size: k.size, angle: k.angle,
                   octave: u32::try_from(k.octave).unwrap_or(u32::MAX), class_id: u32::try_from(k.class_id).unwrap_or(u32::MAX) }
}

fn kp_from_c(k: &cvb_keypoint) -> akaze::KeyPoint {
    akaze::KeyPoint { point: (k.x, k.y), response: k.response, size: k.size, octave: k.octave as usize, class_id: k.class_id as usize,
                      angle: k.angle }
}

impl CudaAkaze {
    /// allocate_evolutions + create_nonlinear_scale_space + detector_response (akaze/src/lib.rs:309-323) on the device.
    pub fn create_scale_space(&self, img: &akaze::image::GrayFloatImage) -> CudaEvolutions {
        let mut ticket = 0u64;
        let rc = unsafe { cvb_akaze_scale_space(self.ctx.0, &to_c(&self.cfg), img.as_raw().as_ptr(), 1, img.width() as u32,
                                                img.height() as u32, &mut ticket) };
        assert_eq!(rc, 0, "{}", self.ctx.last_error());
        let mut n = 0u32;
        let rc = unsafe { cvb_akaze_evolutions(self.ctx.0, ticket, std::ptr::null_mut(), 0, &mut n) };
        assert_eq!(rc, 0, "{}", self.ctx.last_error());
        let mut evolutions = vec![cvb_akaze_evolution::default(); n as usize];
        let rc = unsafe { cvb_akaze_evolutions(self.ctx.0, ticket, evolutions.as_mut_ptr(), n, &mut n) };
        assert_eq!(rc, 0, "{}", self.ctx.last_error());
        CudaEvolutions { ticket, ctx: self.ctx.clone(), evolutions, batch: 1, cfg: to_c(&self.cfg) }
    }

    /// Akaze::find_image_keypoints (akaze/src/lib.rs:268-276): unsorted, untruncated, in the reference's order.  Detection runs
    /// with the config the scale space was built with, whose detector response already depends on it: panics when this Akaze's
    /// detector fields differ from it (maximum_features and the descriptor fields may differ).
    pub fn find_image_keypoints(&self, evolutions: &mut CudaEvolutions) -> Vec<akaze::KeyPoint> {
        assert!(same_detector(&to_c(&self.cfg), &evolutions.cfg), "build the scale space with the Akaze that detects on it");
        let mut cap = 32768u32;
        loop {
            let mut kps = vec![cvb_keypoint::default(); cap as usize * evolutions.batch as usize];
            let mut n = vec![0u32; evolutions.batch as usize];
            let rc = unsafe { cvb_akaze_find_image_keypoints(evolutions.ctx.0, evolutions.ticket, kps.as_mut_ptr(), cap, n.as_mut_ptr()) };
            if rc == CVB_ECAP && n[0] > cap { cap = n[0]; continue; }
            assert_eq!(rc, 0, "{}", evolutions.ctx.last_error());
            return kps[..n[0] as usize].iter().map(kp_from_c).collect();
        }
    }

    /// Akaze::extract_descriptors (akaze/src/descriptors.rs:16-45); panics on a keypoint the reference would panic on.
    pub fn extract_descriptors(&self, evolutions: &CudaEvolutions, keypoints: &[akaze::KeyPoint]) -> (Vec<akaze::KeyPoint>, Vec<BitArray<64>>) {
        let kin: Vec<cvb_keypoint> = keypoints.iter().map(kp_to_c).collect();
        let offsets = [0u32, kin.len() as u32];
        let mut kout = vec![cvb_keypoint::default(); kin.len()];
        let mut descs = vec![BitArray::<64>::zeros(); kin.len()];
        let mut n = 0u32;
        let rc = unsafe { cvb_akaze_extract_descriptors(evolutions.ctx.0, &to_c(&self.cfg), evolutions.ticket, kin.as_ptr(), offsets.as_ptr(),
                                                        kout.as_mut_ptr(), descs.as_mut_ptr() as *mut u8, &mut n) };
        assert_eq!(rc, 0, "{}", evolutions.ctx.last_error());
        kout.truncate(n as usize); descs.truncate(n as usize);
        (kout.iter().map(kp_from_c).collect(), descs)
    }
}
