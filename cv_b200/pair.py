"""cv-sfm's two-view initialisation of one frame pair as ONE call (cv-sfm/src/lib.rs:1375-1412, extraction at :2200-2204):
AKAZE extract of both frames -> symmetric_matching -> FeatureMatch bearings -> Arrsac + EightPoint, everything on the device,
one synchronisation at the end (include/cvb200.h: cvb_two_view_frames)."""
import ctypes as C

import numpy as np

from ._lib import KP_DTYPE, default_context
from .geom import Arrsac, Pose, _lib as _geom_lib
from .image import is_dynamic
from .image import lib as _image_lib
from .image import stack as _stack_frames
from .pinhole import CameraIntrinsicsK1Distortion


class Intrinsics(C.Structure):
    """cvb_intrinsics == cv_pinhole::CameraIntrinsics without distortion"""
    _fields_ = [("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double), ("skew", C.c_double)]

    @classmethod
    def from_camera(cls, cam):
        return cls(cam.focals[0], cam.focals[1], cam.principal_point[0], cam.principal_point[1], cam.skew)


class IntrinsicsK1(C.Structure):
    """cvb_intrinsics_k1 == cv_pinhole::CameraIntrinsicsK1Distortion (simple intrinsics + k1)"""
    _fields_ = Intrinsics._fields_ + [("k1", C.c_double)]

    @classmethod
    def from_camera(cls, cam):
        """a CameraIntrinsicsK1Distortion, or a CameraIntrinsics (k1 = 0: the same bearings bit for bit)"""
        k1 = getattr(cam, "k1", None)
        s = cam.simple_intrinsics if k1 is not None else cam
        return cls(s.focals[0], s.focals[1], s.principal_point[0], s.principal_point[1], s.skew, 0.0 if k1 is None else k1)


def bind(L):
    if getattr(L, "_pair_bound", False):
        return
    vp, u32 = C.c_void_p, C.c_uint32
    L.cvb_match_symmetric_pairs_dev.argtypes = [vp, vp, vp, u32, vp, vp, u32, u32, vp, u32, vp]
    L.cvb_pair_bearings_dev.argtypes = [vp, vp, vp, vp, vp, u32, C.POINTER(Intrinsics), vp, vp]
    L.cvb_arrsac_eight_point_dev.argtypes = [vp, vp, vp, vp, vp, u32, vp, vp, vp, u32, vp, vp]
    L.cvb_arrsac_p3p_dev.argtypes = L.cvb_arrsac_eight_point_dev.argtypes
    L.cvb_arrsac_commit_rng.argtypes = [vp, vp, vp]
    L.cvb_two_view_pair_dev.argtypes = [vp, vp, vp, vp, vp, vp, vp, u32, u32, C.POINTER(Intrinsics), vp, vp, vp, u32, vp, vp, vp, vp, vp]
    L.cvb_two_view_frames.argtypes = [vp, vp, vp, u32, u32, u32, C.POINTER(Intrinsics), vp, vp, vp, vp, u32, vp, vp, vp, vp, vp, vp, vp]
    L.cvb_pair_bearings_k1_dev.argtypes = [vp, vp, vp, vp, vp, u32, C.POINTER(IntrinsicsK1), vp, vp]
    L.cvb_two_view_pair_k1_dev.argtypes = [vp, vp, vp, vp, vp, vp, vp, u32, u32, C.POINTER(IntrinsicsK1), vp, vp, vp, u32, vp, vp, vp, vp, vp]
    L.cvb_two_view_frames_k1.argtypes = [vp, vp, vp, u32, u32, u32, C.POINTER(IntrinsicsK1), vp, vp, vp, vp, u32, vp, vp, vp, vp, vp, vp, vp]
    L.cvb_frame_features_batch.argtypes = [vp, vp, vp, vp, u32, u32, u32, C.POINTER(IntrinsicsK1), vp, vp, vp, vp, u32, vp]
    L.cvb_frame_features_batch_dev.argtypes = [vp, vp, vp, u32, u32, vp, u32, u32, C.POINTER(IntrinsicsK1), vp, vp]
    L._pair_bound = True


class TwoViewBuffers:
    """Host result buffers of cvb_two_view_frames for frames with up to `cap` keypoints (numpy; pass `pinned=True` arrays made
    with torch for page-locked memory in throughput code)."""

    def __init__(self, cap):
        self.cap = cap
        self.kp = np.zeros((2, cap), KP_DTYPE)
        self.desc = np.zeros((2, cap, 64), np.uint8)
        self.n = np.zeros(2, np.uint32)
        self.pairs = np.zeros((cap, 2), np.uint32)
        self.inliers = np.zeros(cap, np.uint32)
        self.n_pairs, self.n_inliers, self.found = C.c_uint32(), C.c_uint32(), C.c_int32()
        self.model = Pose()


def two_view_frames(akaze, frames, camera, arrsac, better_by=24, cap=8192, buffers=None):
    """frames: [2, H, W] float32, or two DynamicImage of one size and format (cvb_two_view_frames_dynamic_k1: uploaded as they are and
    converted on the device; a CameraIntrinsics goes in as k1 = 0).  akaze: cv_b200.Akaze; camera: cv_b200.CameraIntrinsics
    (cvb_two_view_frames) or cv_b200.CameraIntrinsicsK1Distortion (cvb_two_view_frames_k1); arrsac: cv_b200.Arrsac (its generator
    advances as the reference's would).  Returns dict(keypoints, descriptors, matches [[a, b], ...], pose (R, t) or None,
    inliers (indices into matches))."""
    dynamic = is_dynamic(frames)
    if dynamic:
        if isinstance(frames, (list, tuple)) and len(frames) != 2:
            raise ValueError("frames must be two DynamicImage")
        fmt, pixels, W, H = _stack_frames(frames)
        if pixels.shape[0] != 2:
            raise ValueError("frames must be two DynamicImage")
    else:
        frames = np.ascontiguousarray(frames, np.float32)
        if frames.ndim != 3 or frames.shape[0] != 2:
            raise ValueError("frames must be [2, H, W] float32")
        pixels, H, W = frames, frames.shape[1], frames.shape[2]
    ctx = akaze._ctx()
    _geom_lib(ctx)
    L = ctx.lib
    bind(L)
    b = buffers or TwoViewBuffers(cap)
    cfg = akaze.config.to_c()
    if dynamic:
        K, IL = IntrinsicsK1.from_camera(camera), _image_lib()
        entry = lambda *a: IL.cvb_two_view_frames_dynamic_k1(a[0], a[1], fmt, *a[2:])   # noqa: E731
    elif isinstance(camera, CameraIntrinsicsK1Distortion):
        K, entry = IntrinsicsK1.from_camera(camera), L.cvb_two_view_frames_k1
    else:
        K, entry = Intrinsics.from_camera(camera), L.cvb_two_view_frames
    ctx.check(entry(ctx.handle, C.addressof(cfg), pixels.ctypes.data, W, H, better_by, C.byref(K),
                    C.addressof(arrsac.cfg), C.addressof(arrsac.rng.state), b.kp.ctypes.data, b.desc.ctypes.data, b.cap,
                    b.n.ctypes.data, b.pairs.ctypes.data, C.addressof(b.n_pairs), C.addressof(b.model), b.inliers.ctypes.data,
                    C.addressof(b.n_inliers), C.addressof(b.found)))
    kps = [b.kp[f, :b.n[f]].copy() for f in range(2)]
    descs = [b.desc[f, :b.n[f]].copy() for f in range(2)]
    pose = (np.array(b.model.r).reshape(3, 3), np.array(b.model.t)) if b.found.value else None
    return dict(keypoints=kps, descriptors=descs, matches=b.pairs[:b.n_pairs.value].astype(np.int64), pose=pose,
                inliers=b.inliers[:b.n_inliers.value].copy() if b.found.value else np.zeros(0, np.uint32))
