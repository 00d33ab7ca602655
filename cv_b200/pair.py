"""cv-sfm's two-view initialisation of one frame pair as ONE call (cv-sfm/src/lib.rs:1375-1412, extraction at :2200-2204):
AKAZE extract of both frames -> symmetric_matching -> FeatureMatch bearings -> Arrsac + EightPoint, everything on the device,
one synchronisation at the end (include/cvb200.h: cvb_two_view_frames).  init_two_view_options: the same initialisation of one frame
against many candidate frames, with one batched consensus run (include/cvb200_batch.h: cvb_two_view_options_dev).  init_reconstruction:
cv-sfm's three-view initialisation over those options, chained on the device (include/cvb200_init.h: cvb_init_reconstruction_dev)."""
import ctypes as C

import numpy as np

from ._lib import KP_DTYPE, default_context
from .geom import Arrsac, Pose, Rng, _lib as _geom_lib
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


# cv-sfm's default two_view_minimum_robust_matches (cv-sfm/src/settings.rs:393-395)
TWO_VIEW_MINIMUM_ROBUST_MATCHES = 1 << 8


def two_view_option_result(pairs, n_pairs, model_r, model_t, inliers, n_inliers, found, minimum_robust_matches):
    """One option of init_two_view_options from its device outputs (host copies): None when consensus found nothing or kept fewer
    than minimum_robust_matches inlier matches (cv-sfm/src/lib.rs:1417-1424), else (R, t, matches), matches = the inlier matches as
    [center feature, option feature] rows in inlier order (lib.rs:1414)."""
    if not found or n_inliers < minimum_robust_matches:
        return None
    pairs = np.asarray(pairs, np.int64).reshape(-1, 2)[:n_pairs]
    inl = np.asarray(inliers, np.int64)[:n_inliers]
    return np.asarray(model_r, np.float64).reshape(3, 3).copy(), np.asarray(model_t, np.float64).copy(), pairs[inl]


def _two_view_options_dev(features, center, options, arrsac, rngs, better_by):
    """The checks and the device call shared by init_two_view_options and init_reconstruction: runs cvb_two_view_options_dev, commits
    the generators, and returns (frames, cap, opts, device outputs dict) -- the outputs stay on the device.  None when F = 0."""
    from ._lib import ARRSAC_BATCH_MAX, load_batch_library
    import torch
    desc, cnt, bear = features["descriptors"], features["counts"], features["bearings"]
    if desc.dtype != torch.uint8 or desc.dim() != 3 or desc.shape[2] != 64 or not desc.is_cuda or not desc.is_contiguous():
        raise ValueError("descriptors must be a contiguous CUDA uint8 tensor [frames, cap, 64]")
    frames, cap = desc.shape[0], desc.shape[1]
    if bear.dtype != torch.float64 or tuple(bear.shape) != (frames, cap, 3) or not bear.is_cuda or not bear.is_contiguous():
        raise ValueError("bearings must be a contiguous CUDA float64 tensor [frames, cap, 3]")
    if cnt.dtype not in (torch.int32, torch.uint32) or tuple(cnt.shape) != (frames,) or not cnt.is_cuda:
        raise ValueError("counts must be a CUDA int32 tensor [frames]")
    opts = np.ascontiguousarray(options, np.uint32)
    F = len(opts)
    if len(rngs) != F:
        raise ValueError(f"one generator per option ({len(rngs)} != {F})")
    if F > ARRSAC_BATCH_MAX:
        raise ValueError(f"at most {ARRSAC_BATCH_MAX} options per call")
    if F == 0:
        return frames, cap, opts, None
    ctx = arrsac.ctx
    BL = load_batch_library()
    dev = desc.device
    out = dict(pairs=torch.zeros((F, cap, 2), dtype=torch.int32, device=dev), n_pairs=torch.zeros(F, dtype=torch.int32, device=dev),
               model=torch.zeros((F, 12), dtype=torch.float64, device=dev), inliers=torch.zeros((F, cap), dtype=torch.int32, device=dev),
               n_inliers=torch.zeros(F, dtype=torch.int32, device=dev), found=torch.zeros(F, dtype=torch.int32, device=dev))
    states = (Rng * F)(*[r.state for r in rngs])
    torch.cuda.synchronize(dev)
    ctx.check(BL.cvb_two_view_options_dev(ctx.handle, desc.data_ptr(), cnt.data_ptr(), bear.data_ptr(), frames, cap, int(center),
                                          opts.ctypes.data, F, better_by, C.addressof(arrsac.cfg), C.addressof(states),
                                          out["pairs"].data_ptr(), out["n_pairs"].data_ptr(), out["model"].data_ptr(),
                                          out["inliers"].data_ptr(), out["n_inliers"].data_ptr(), out["found"].data_ptr()))
    ctx.check(BL.cvb_arrsac_commit_rng_batch(ctx.handle, C.addressof(states), F, None))
    for f in range(F):
        C.memmove(C.addressof(rngs[f].state), C.addressof(states[f]), C.sizeof(Rng))
    return frames, cap, opts, out


def init_two_view_options(features, center, options, arrsac, rngs, better_by=24,
                          minimum_robust_matches=TWO_VIEW_MINIMUM_ROBUST_MATCHES):
    """cv-sfm's init_two_view(center, option) for every option frame (VSlam::init_reconstruction, cv-sfm/src/lib.rs:966-985 and
    1365-1432) in one call: F symmetric matches, one gather of the matched bearings, one batched ARRSAC + EightPoint.

    features: device tensors of the frames, as cvb_frame_features_batch_dev leaves them -- "descriptors" [frames, cap, 64] uint8,
    "counts" [frames] int32 / uint32, "bearings" [frames, cap, 3] float64 (torch CUDA tensors on the context's device).  center, options:
    frame indices.  arrsac: cv_b200.Arrsac (its configuration; its own generator is not used); rngs: one generator per option, each
    advanced as model_inliers would advance it.  Returns one result per option: None, or (R, t, matches) with matches the inlier
    [center feature, option feature] pairs.  Option f equals cvb_two_view_pair_k1_dev on the same frames with rngs[f].  The reference
    runs the options on one shared generator and shuffles the matches first; parity with that is unpinned."""
    _, _, opts, out = _two_view_options_dev(features, center, options, arrsac, rngs, better_by)
    if out is None:
        return []
    pairs, n_pairs, model = out["pairs"].cpu().numpy(), out["n_pairs"].cpu().numpy(), out["model"].cpu().numpy()
    inl, n_inl, found = out["inliers"].cpu().numpy(), out["n_inliers"].cpu().numpy(), out["found"].cpu().numpy()
    return [two_view_option_result(pairs[f], int(n_pairs[f]), model[f, :9], model[f, 9:], inl[f], int(n_inl[f]), int(found[f]),
                                   minimum_robust_matches) for f in range(len(opts))]


class InitSettings(C.Structure):
    """cvb_init_cfg: the cv-sfm settings init_reconstruction reads, with their defaults (cv-sfm/src/settings.rs:320-428)."""
    _fields_ = [("robust_observation_incidence_minimum_cosine_distance", C.c_double),
                ("robust_view_bearing_pair_minimum_cosine_distance", C.c_double), ("maximum_cosine_distance", C.c_double),
                ("maximum_sine_distance", C.c_double), ("two_view_minimum_robust_matches", C.c_uint32),
                ("three_view_minimum_relative_scales", C.c_uint32), ("three_view_optimization_landmarks", C.c_uint32),
                ("robust_view_num_robust_bearing_pair", C.c_uint32), ("three_view_filter_loop_iterations", C.c_uint32),
                ("three_view_patience", C.c_uint32), ("three_view_minimum_robust_matches", C.c_uint32), ("reserved", C.c_uint32)]

    def __init__(self, **kw):
        d = dict(robust_observation_incidence_minimum_cosine_distance=1e-3, robust_view_bearing_pair_minimum_cosine_distance=1e-2,
                 maximum_cosine_distance=1e-5, maximum_sine_distance=0.1, two_view_minimum_robust_matches=TWO_VIEW_MINIMUM_ROBUST_MATCHES,
                 three_view_minimum_relative_scales=16, three_view_optimization_landmarks=1024, robust_view_num_robust_bearing_pair=3,
                 three_view_filter_loop_iterations=8, three_view_patience=1 << 16, three_view_minimum_robust_matches=32)
        d.update(kw)
        super().__init__(**d)


POSE_DTYPE = np.dtype([("r", "<f8", (9,)), ("t", "<f8", (3,))])
# cvb_init_result and cvb_init_pair_stats (include/cvb200_init.h)
INIT_RESULT_DTYPE = np.dtype([("status", "<i4"), ("pair", "<u4"), ("first", "<u4"), ("second", "<u4"), ("n_pairs", "<u4"),
                              ("n_combined", "<u4"), ("n_first_matches", "<u4"), ("n_second_matches", "<u4"), ("first_pose", POSE_DTYPE),
                              ("second_pose", POSE_DTYPE)])
INIT_PAIR_STATS_DTYPE = np.dtype([("outcome", "<i4"), ("first", "<u4"), ("second", "<u4"), ("scales", "<u4"), ("median_scale", "<f8"),
                                  ("bearing_pairs", "<u8"), ("common", "<u4"), ("opti", "<u4"), ("updates", "<u4"), ("robust", "<u4")])


def init_reconstruction_dev(ctx, features_bearings, center, options, two_view, settings=None, triangulator=None, stats=False):
    """cvb_init_reconstruction_dev on device tensors: features_bearings [frames, cap, 3] float64 (CUDA), two_view: the device outputs of
    cvb_two_view_options_dev for the same center / options (dict pairs, n_pairs, model, inliers, n_inliers, found).  Returns host copies:
    dict(result (INIT_RESULT_DTYPE record), combined [n, 3], first_matches [n, 2], second_matches [n, 2], stats (or None))."""
    from ._lib import load_init_library
    from .triangulation import LinearEigenTriangulator
    import torch
    bear = features_bearings
    if bear.dtype != torch.float64 or bear.dim() != 3 or bear.shape[2] != 3 or not bear.is_cuda or not bear.is_contiguous():
        raise ValueError("bearings must be a contiguous CUDA float64 tensor [frames, cap, 3]")
    frames, cap = bear.shape[0], bear.shape[1]
    opts = np.ascontiguousarray(options, np.uint32)
    F = len(opts)
    settings = settings if settings is not None else InitSettings()
    tri = triangulator if triangulator is not None else LinearEigenTriangulator()
    dev = bear.device
    res = torch.zeros(INIT_RESULT_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    comb = torch.zeros((cap, 3), dtype=torch.int32, device=dev)
    fm = torch.zeros((cap, 2), dtype=torch.int32, device=dev)
    sm = torch.zeros((cap, 2), dtype=torch.int32, device=dev)
    npairs = F * (F - 1) // 2
    st = torch.zeros(max(npairs, 1) * INIT_PAIR_STATS_DTYPE.itemsize, dtype=torch.uint8, device=dev) if stats else None
    if two_view is None:
        z = torch.zeros(max(F, 1) * cap * 2, dtype=torch.int32, device=dev)
        two_view = dict(pairs=z, n_pairs=z, model=torch.zeros((1, 12), dtype=torch.float64, device=dev), inliers=z, n_inliers=z, found=z)
    IL = load_init_library()
    torch.cuda.synchronize(dev)
    ctx.check(IL.cvb_init_reconstruction_dev(ctx.handle, C.addressof(settings), C.addressof(tri.cfg), bear.data_ptr(), frames, cap, int(center),
                                             opts.ctypes.data if F else None, F, two_view["pairs"].data_ptr(), two_view["n_pairs"].data_ptr(),
                                             two_view["model"].data_ptr(), two_view["inliers"].data_ptr(), two_view["n_inliers"].data_ptr(),
                                             two_view["found"].data_ptr(), res.data_ptr(), comb.data_ptr(), fm.data_ptr(), sm.data_ptr(),
                                             st.data_ptr() if st is not None else None))
    torch.cuda.synchronize(dev)
    r = np.frombuffer(res.cpu().numpy().tobytes(), INIT_RESULT_DTYPE)[0]
    return dict(result=r, combined=comb[:int(r["n_combined"])].cpu().numpy().astype(np.int64),
                first_matches=fm[:int(r["n_first_matches"])].cpu().numpy().astype(np.int64),
                second_matches=sm[:int(r["n_second_matches"])].cpu().numpy().astype(np.int64),
                stats=np.frombuffer(st.cpu().numpy().tobytes(), INIT_PAIR_STATS_DTYPE)[:npairs].copy() if st is not None else None)


def init_reconstruction(features, center, options, arrsac, rngs, settings=None, triangulator=None, better_by=24):
    """cv-sfm's VSlam::init_reconstruction (cv-sfm/src/lib.rs:966-1303) of frame `center` against the option frames, on the device:
    init_two_view against every option (init_two_view_options) and the choice of the three-view initialisation over every pair of the
    options that pass (include/cvb200_init.h), with no host copy between them.

    features, center, options, arrsac, rngs, better_by: as init_two_view_options.  settings: InitSettings (cv-sfm's defaults);
    triangulator: a TriangulatorObservations (LinearEigenTriangulator, SineL1Triangulator or MeanMeanTriangulator; default
    LinearEigen).  Returns None, or dict(first, first_pose, second, second_pose, combined, first_matches, second_matches) with first /
    second the chosen frames, poses (R, t) CameraToCamera center -> frame, combined [n, 3] (center, first, second feature) and the two
    [n, 2] (center, option feature) lists.  Unpinned: the reference shuffles the common matches (lib.rs:999) and the matches in front of
    consensus with one shared generator; here they keep their order, and each option has its own generator."""
    settings = settings if settings is not None else InitSettings()
    if triangulator is not None and getattr(triangulator, "method", None) not in (0, 1, 2):
        raise ValueError("init_reconstruction takes a TriangulatorObservations: LinearEigen, SineL1 or MeanMean")
    frames, cap, opts, out = _two_view_options_dev(features, center, options, arrsac, rngs, better_by)
    r = init_reconstruction_dev(arrsac.ctx, features["bearings"], center, opts, out, settings, triangulator)
    res = r["result"]
    if res["status"] != 1:
        return None

    def pose(p):
        return np.array(p["r"]).reshape(3, 3), np.array(p["t"])
    return dict(first=int(opts[res["first"]]), first_pose=pose(res["first_pose"]), second=int(opts[res["second"]]),
                second_pose=pose(res["second_pose"]), combined=r["combined"], first_matches=r["first_matches"],
                second_matches=r["second_matches"])
