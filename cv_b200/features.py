"""cv-sfm's per-frame feature ingestion, VSlam::kps_descriptors (cv-sfm/src/lib.rs:2195-2235), for B frames in one call
(include/cvb200.h: cvb_frame_features_batch): AKAZE, the bicubic colour of every keypoint and its calibrated bearing, on the device."""
import ctypes as C

import numpy as np

from ._lib import KP_DTYPE
from .image import is_dynamic
from .image import lib as _image_lib
from .image import stack as _stack_frames
from .pair import IntrinsicsK1, bind


def frame_features(akaze, gray_frames, rgb_frames=None, camera=None):
    """frame_features(akaze, images, camera): images is a DynamicImage (or a list of them, one size and format) of an 8-bit format;
    both the extractor's plane and the colour plane are made from it on the device (include/cvb200_image.h), as kps_descriptors makes
    them from one DynamicImage (from_dynamic and to_rgb8()).

    frame_features(akaze, gray_frames, rgb_frames, camera): gray_frames: [B, H, W] float32 luma in [0, 1] (what Akaze.extract_batch takes).  rgb_frames: [B, H, W, 3] uint8 (an RgbImage per
    frame), or [B, H, W] uint8 grayscale, whose channel is replicated as DynamicImage::to_rgb8() does for a Luma8 image.
    camera: cv_b200.CameraIntrinsicsK1Distortion (or CameraIntrinsics, i.e. k1 = 0).

    Returns one dict per frame: keypoints and descriptors (exactly Akaze.extract_batch's), bearings [n, 3] f64, responses [n] f32 and
    colors [n, 3] u8 -- the arrays cv_b200.checkpoint.features_to_bytes takes -- in the reference's feature order (descending
    response, which is AKAZE's own order)."""
    if is_dynamic(gray_frames):
        return _frame_features_dynamic(akaze, gray_frames, camera if camera is not None else rgb_frames)
    gray = np.ascontiguousarray(gray_frames, np.float32)
    if gray.ndim != 3:
        raise ValueError("gray_frames must be [B, H, W] float32")
    B, H, W = gray.shape
    rgb = np.asarray(rgb_frames)
    if rgb.dtype != np.uint8:
        raise TypeError("rgb_frames must be uint8")
    if rgb.shape == (B, H, W):
        rgb = np.repeat(rgb[..., None], 3, axis=3)
    if rgb.shape != (B, H, W, 3):
        raise ValueError(f"rgb_frames must be [B, H, W, 3] or [B, H, W] uint8 matching gray_frames {gray.shape}")
    rgb = np.ascontiguousarray(rgb)
    ctx = akaze._ctx()
    L = ctx.lib
    bind(L)
    cap = akaze.max_keypoints
    kp = np.zeros((B, cap), KP_DTYPE)
    desc = np.zeros((B, cap, 64), np.uint8)
    bear = np.zeros((B, cap, 3), np.float64)
    col = np.zeros((B, cap, 3), np.uint8)
    n = np.zeros(B, np.uint32)
    cfg = akaze.config.to_c()
    K = IntrinsicsK1.from_camera(camera)
    ctx.check(L.cvb_frame_features_batch(ctx.handle, C.byref(cfg), gray.ctypes.data, rgb.ctypes.data, B, W, H, C.byref(K), kp.ctypes.data,
                                         desc.ctypes.data, bear.ctypes.data, col.ctypes.data, cap, n.ctypes.data))
    return _per_frame(kp, desc, bear, col, n)


def _frame_features_dynamic(akaze, images, camera):
    if camera is None:
        raise TypeError("frame_features(akaze, images, camera): camera missing")
    fmt, pixels, W, H = _stack_frames(images)
    B = pixels.shape[0]
    ctx = akaze._ctx()
    L = _image_lib()
    cap = akaze.max_keypoints
    kp = np.zeros((B, cap), KP_DTYPE)
    desc = np.zeros((B, cap, 64), np.uint8)
    bear = np.zeros((B, cap, 3), np.float64)
    col = np.zeros((B, cap, 3), np.uint8)
    n = np.zeros(B, np.uint32)
    cfg = akaze.config.to_c()
    K = IntrinsicsK1.from_camera(camera)
    ctx.check(L.cvb_frame_features_dynamic_batch(ctx.handle, C.addressof(cfg), fmt, pixels.ctypes.data, B, W, H, C.addressof(K),
                                                 kp.ctypes.data, desc.ctypes.data, bear.ctypes.data, col.ctypes.data, cap, n.ctypes.data))
    return _per_frame(kp, desc, bear, col, n)


def _per_frame(kp, desc, bear, col, n):
    out = []
    for b in range(len(n)):
        k = kp[b, :n[b]].copy()
        out.append(dict(keypoints=k, descriptors=desc[b, :n[b]].copy(), bearings=bear[b, :n[b]].copy(), responses=k["response"].copy(),
                        colors=col[b, :n[b]].copy()))
    return out
