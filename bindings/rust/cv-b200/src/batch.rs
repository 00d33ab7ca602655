//! Safe shim over include/cvb200_batch.h: `CudaArrsac::model_inliers_batch`, many independent consensus problems in one device run.
//! ASSEMBLED by scripts/gen_rust_sys.py from the code block of INTEGRATION.md section 2k -- edit the document, then regenerate.  A child
//! module of the shim, so it reaches `Ctx`, `pose_from_c` and the private fields of `CudaArrsac`.
use super::*;

use cv_b200_sys::batch::*;

impl CudaArrsac {
    /// `Consensus::<EightPoint, FeatureMatch>::model_inliers` of every problem in one batched device run: problem i with generator
    /// `rngs[i]`, advanced as model_inliers would advance it (`self.rng` is not used).  Problem i's result is bit for bit that of
    /// `model_inliers` with `rngs[i]`; inlier indices follow problem i's order.  At most CVB_ARRSAC_BATCH_MAX problems.  cv-sfm runs
    /// such problems on ONE shared generator: parity with that sequence is unpinned.
    pub fn model_inliers_batch(&mut self, _e: &eight_point::EightPoint, problems: &[Vec<FeatureMatch>], rngs: &mut [cvb_rng])
        -> Vec<Option<(CameraToCamera, Vec<usize>)>> {
        assert_eq!(problems.len(), rngs.len(), "one generator per problem");
        assert!(problems.len() <= CVB_ARRSAC_BATCH_MAX as usize, "at most {} problems per batch", CVB_ARRSAC_BATCH_MAX);
        let nb = problems.len();
        let (mut a, mut b, mut offsets) = (Vec::new(), Vec::new(), vec![0u32]);
        for p in problems {
            for FeatureMatch(x, y) in p { a.extend_from_slice(x.as_slice()); b.extend_from_slice(y.as_slice()); }
            offsets.push((a.len() / 3) as u32);
        }
        let mut models = vec![cvb_pose { r: [0.0; 9], t: [0.0; 3] }; nb];
        let mut inl = vec![0u32; (a.len() / 3).max(1)];
        let (mut cnt, mut found) = (vec![0u32; nb], vec![0i32; nb]);
        let rc = unsafe { cvb_arrsac_batch(self.ctx.0, &self.cfg, 0, 5, a.as_ptr(), b.as_ptr(), offsets.as_ptr(), nb as u32,
                                           rngs.as_mut_ptr(), models.as_mut_ptr(), inl.as_mut_ptr(), cnt.as_mut_ptr(),
                                           found.as_mut_ptr()) };
        assert_eq!(rc, 0, "{}", self.ctx.last_error());
        (0..nb).map(|i| {
            if found[i] == 0 { return None; }
            let o = offsets[i] as usize;
            Some((CameraToCamera(pose_from_c(&models[i])), inl[o..o + cnt[i] as usize].iter().map(|&j| j as usize).collect()))
        }).collect()
    }
}
