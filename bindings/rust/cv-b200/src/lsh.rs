//! Safe shim over include/cvb200_lsh.h: `CudaFrameIndex`, a drop-in for cv-sfm's `lsh_to_frame` with the reference's method names.
//! ASSEMBLED by scripts/gen_rust_sys.py from the code block of INTEGRATION.md section 2i -- edit the document, then regenerate.  A child
//! module of the shim, so it reaches `Ctx`.
use super::*;

use cv_b200_sys::lsh::*;

/// cv-sfm's `lsh_to_frame` (HggLite<Hamming, BitArray<512>, FrameKey>, cv-sfm/src/lib.rs:207) answered exactly on the device:
/// `knn_values` lists (distance, &value), nearest first, equal distances in insertion order.
pub struct CudaFrameIndex<V> { hashes: Vec<BitArray<512>>, values: Vec<V>, ctx: Ctx }

impl<V> CudaFrameIndex<V> {
    pub fn new(ctx: Ctx) -> Self { CudaFrameIndex { hashes: Vec::new(), values: Vec::new(), ctx } }
    pub fn len(&self) -> usize { self.values.len() }
    pub fn is_empty(&self) -> bool { self.values.is_empty() }

    /// HggLite::insert (cv-sfm/src/lib.rs:684)
    pub fn insert(&mut self, key: BitArray<512>, value: V) {
        self.hashes.push(key);
        self.values.push(value);
    }

    /// HggLite::knn_values (cv-sfm/src/lib.rs:623-624); num is at most CVB_LSH_MAX_K.
    pub fn knn_values(&self, query: &BitArray<512>, num: usize) -> Vec<(u32, &V)> {
        let (mut idx, mut dist) = (vec![0u32; num], vec![0u32; num]);
        let rc = unsafe { cvb_hash_knn(self.ctx.0, 128, query.as_ptr(), 1, self.hashes.as_ptr() as *const u8, self.hashes.len() as u32,
                                       num as u32, idx.as_mut_ptr(), dist.as_mut_ptr()) };
        assert_eq!(rc, 0, "{}", self.ctx.last_error());
        idx.into_iter().zip(dist).filter(|(i, _)| *i != u32::MAX).map(|(i, d)| (d, &self.values[i as usize])).collect()
    }
}
