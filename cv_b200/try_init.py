"""cv-sfm's reconstruction creation on the device (include/cvb200_try_init.h): VSlamData::add_reconstruction (cv-sfm/src/lib.rs:377-427),
the first snapshot of a reconstruction from three frames and init_reconstruction's match lists, and VSlam::try_init (lib.rs:814-839), the
two-view options, the three-view initialisation and add_reconstruction of a frame against its free frames.

The frame store is cvb_frame_features_batch_dev's: a dict with "descriptors" [frames, cap, 64] uint8, "counts" [frames], "bearings"
[frames, cap, 3] float64 and optional "colors" [frames, cap, 3] uint8 -- numpy arrays for the host forms, torch CUDA tensors for the
*_dev forms.  The snapshot is cv_b200.incorporate's (SNAP_KEYS): view i is frames[i], landmark index = slot-map insertion order, and the
*_dev forms return the device dict that cv_b200.incorporate.incorporate_frame_dev takes."""
import ctypes as C

import numpy as np

from ._lib import ARRSAC_BATCH_MAX, load_try_init_library
from .constraints import _u32
from .geom import Rng
from .incorporate import COUNTS_DTYPE, _counts, _dev_out, _dev_trim, _out, _trim
from .pair import INIT_RESULT_DTYPE, InitSettings

NO_FRAME = 0xFFFFFFFF
# statuses of include/cvb200_try_init.h
STATUS_NAMES = ["created", "none", "none_bearing_pairs"]
RESULT_DTYPE = np.dtype([("status", "<i4"), ("frames", "<u4", (3,)), ("init", INIT_RESULT_DTYPE), ("counts", COUNTS_DTYPE)])


def _p(a):
    return a.ctypes.data if a is not None and a.size else None


def _dp(x):
    return x.data_ptr() if x is not None and x.numel() else None


def _list(a, k):
    return np.ascontiguousarray(np.asarray(a, np.uint32).reshape(-1, k))


def _pose12(p):
    if isinstance(p, tuple):
        return np.concatenate([np.asarray(p[0], np.float64).reshape(9), np.asarray(p[1], np.float64).reshape(3)])
    return np.ascontiguousarray(p, np.float64).reshape(12)


def _capacities(cap, col):
    """the output capacities of include/cvb200_try_init.h's table, as cv_b200.incorporate's _out arguments"""
    return 3, 3 * cap, 3 * cap, 3 * cap, 1, True, col


def _store(features):
    d = np.ascontiguousarray(features["descriptors"], np.uint8)
    frames, cap = d.shape[0], d.shape[1]
    b = np.ascontiguousarray(features["bearings"], np.float64).reshape(frames, cap, 3)
    n = _u32(features["counts"]).reshape(frames)
    c = features.get("colors")
    c = None if c is None else np.ascontiguousarray(c, np.uint8).reshape(frames, cap, 3)
    return d, n, b, c, frames, cap


def check_try_init(n_center, n_first, n_second, combined, first_matches, second_matches, frames=(0, 1, 2)):
    """cvb_try_init_check on the host (no device): 0, or CVB_EINVAL."""
    comb, fm, sm = _list(combined, 3), _list(first_matches, 2), _list(second_matches, 2)
    return load_try_init_library().cvb_try_init_check(int(n_center), int(n_first), int(n_second), *[int(f) for f in frames], _p(comb), len(comb),
                                                      _p(fm), len(fm), _p(sm), len(sm))


def add_reconstruction(ctx, features, center, first, second, first_pose, second_pose, combined, first_matches, second_matches):
    """cv-sfm's add_reconstruction (cvb_add_reconstruction) on a host frame store: poses (R, t) or [12] are init's CameraToCamera poses
    center -> first / second, combined [n, 3], first_matches / second_matches [n, 2].  Returns (snapshot, counts record)."""
    d, n, b, c, frames, cap = _store(features)
    comb, fm, sm = _list(combined, 3), _list(first_matches, 2), _list(second_matches, 2)
    ir = np.zeros(1, INIT_RESULT_DTYPE)
    ir["status"] = 1
    ir["n_combined"], ir["n_first_matches"], ir["n_second_matches"] = len(comb), len(fm), len(sm)
    for k, p in (("first_pose", first_pose), ("second_pose", second_pose)):
        p = _pose12(p)
        ir[k]["r"], ir[k]["t"] = p[:9], p[9:]
    o = _out(*_capacities(cap, c is not None))
    cnt = np.zeros(1, COUNTS_DTYPE)
    ctx.check(load_try_init_library().cvb_add_reconstruction(
        ctx.handle, _p(d), _p(n), _p(b), _p(c), frames, cap, int(center), int(first), int(second), ir.ctypes.data, _p(comb), _p(fm), _p(sm),
        o["poses"].ctypes.data, o["view_offsets"].ctypes.data, o["view_landmarks"].ctypes.data, o["bearings"].ctypes.data,
        o["descriptors"].ctypes.data, _p(o["colors"]), o["landmark_offsets"].ctypes.data, o["observations"].ctypes.data,
        o["constraints"].ctypes.data, cnt.ctypes.data))
    return _trim(o, cnt[0]), cnt[0]


def _rngs(rngs, F):
    if len(rngs) != F:
        raise ValueError(f"one generator per option ({len(rngs)} != {F})")
    if F > ARRSAC_BATCH_MAX:
        raise ValueError(f"at most {ARRSAC_BATCH_MAX} options per call")
    return (Rng * max(F, 1))(*[r.state for r in rngs])


def _advance(rngs, states):
    for f, r in enumerate(rngs):
        C.memmove(C.addressof(r.state), C.addressof(states[f]), C.sizeof(Rng))


def _settings(settings, triangulator):
    from .triangulation import LinearEigenTriangulator
    return settings if settings is not None else InitSettings(), triangulator if triangulator is not None else LinearEigenTriangulator()


def try_init(features, center, options, arrsac, rngs, settings=None, triangulator=None, better_by=24):
    """cv-sfm's try_init (cvb_try_init) on a host frame store: init_two_view against every option with generator rngs[f] (advanced),
    init_reconstruction (InitSettings, a TriangulatorObservations) and, when accepted, add_reconstruction.  arrsac: a cv_b200.Arrsac (its
    configuration and context).  Returns dict(status name, result RESULT_DTYPE record, frames [3] (or None for the pair's frames when no
    pair was decided), snapshot (or None))."""
    d, n, b, c, frames, cap = _store(features)
    opts = np.ascontiguousarray(options, np.uint32)
    F = len(opts)
    states = _rngs(rngs, F)
    cfg, tri = _settings(settings, triangulator)
    o = _out(*_capacities(cap, c is not None))
    res = np.zeros(1, RESULT_DTYPE)
    ctx = arrsac.ctx
    ctx.check(load_try_init_library().cvb_try_init(
        ctx.handle, C.addressof(cfg), C.addressof(tri.cfg), C.addressof(arrsac.cfg), C.addressof(states), better_by, _p(d), _p(n), _p(b), _p(c),
        frames, cap, int(center), _p(opts), F, o["poses"].ctypes.data, o["view_offsets"].ctypes.data, o["view_landmarks"].ctypes.data,
        o["bearings"].ctypes.data, o["descriptors"].ctypes.data, _p(o["colors"]), o["landmark_offsets"].ctypes.data, o["observations"].ctypes.data,
        o["constraints"].ctypes.data, res.ctypes.data))
    _advance(rngs, states)
    r = res[0]
    status = STATUS_NAMES[int(r["status"])]
    return dict(status=status, result=r, frames=[None if f == NO_FRAME else int(f) for f in r["frames"]],
                snapshot=_trim(o, r["counts"]) if status == "created" else None)


# ---- torch CUDA forms ------------------------------------------------------------------------------------------------------------------
def _dev_store(features):
    import torch
    d, n, b = features["descriptors"], features["counts"], features["bearings"]
    if d.dtype != torch.uint8 or d.dim() != 3 or d.shape[2] != 64 or not d.is_cuda or not d.is_contiguous():
        raise ValueError("descriptors must be a contiguous CUDA uint8 tensor [frames, cap, 64]")
    frames, cap = d.shape[0], d.shape[1]
    if b.dtype != torch.float64 or tuple(b.shape) != (frames, cap, 3) or not b.is_cuda or not b.is_contiguous():
        raise ValueError("bearings must be a contiguous CUDA float64 tensor [frames, cap, 3]")
    if n.dtype not in (torch.int32, torch.uint32) or tuple(n.shape) != (frames,) or not n.is_cuda:
        raise ValueError("counts must be a CUDA int32 tensor [frames]")
    c = features.get("colors")
    if c is not None and (c.dtype != torch.uint8 or tuple(c.shape) != (frames, cap, 3) or not c.is_cuda or not c.is_contiguous()):
        raise ValueError("colors must be a contiguous CUDA uint8 tensor [frames, cap, 3]")
    return d, n, b, c, frames, cap


def add_reconstruction_dev(ctx, features, center, first, second, init_result, combined, first_matches, second_matches):
    """add_reconstruction on torch CUDA tensors (cvb_add_reconstruction_dev): a device frame store, init_result uint8
    [INIT_RESULT_DTYPE.itemsize] and the lists int32 [cap, 3] / [cap, 2] / [cap, 2] as cvb_init_reconstruction_dev writes them (lengths
    and poses are read from init_result on the device).  Returns (device snapshot, counts record)."""
    import torch
    d, n, b, c, frames, cap = _dev_store(features)
    dev = d.device
    o = _dev_out(*_capacities(cap, c is not None), dev)
    cnt = torch.zeros(COUNTS_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    torch.cuda.current_stream(dev).synchronize()     # the inputs come from torch's stream, the call runs on the context's
    ctx.check(load_try_init_library().cvb_add_reconstruction_dev(
        ctx.handle, _dp(d), _dp(n), _dp(b), _dp(c), frames, cap, int(center), int(first), int(second), _dp(init_result), _dp(combined),
        _dp(first_matches), _dp(second_matches), _dp(o["poses"]), _dp(o["view_offsets"]), _dp(o["view_landmarks"]), _dp(o["bearings"]),
        _dp(o["descriptors"]), _dp(o["colors"]), _dp(o["landmark_offsets"]), _dp(o["observations"]), _dp(o["constraints"]), _dp(cnt)))
    k = _counts(cnt)
    return _dev_trim(o, k), k


def try_init_dev(features, center, options, arrsac, rngs, settings=None, triangulator=None, better_by=24):
    """try_init on a device frame store (cvb_try_init_dev): arguments as try_init.  Returns the dict of try_init with the snapshot as
    device tensors (the dict cv_b200.incorporate.incorporate_frame_dev takes), or None."""
    import torch
    d, n, b, c, frames, cap = _dev_store(features)
    opts = np.ascontiguousarray(options, np.uint32)
    F = len(opts)
    states = _rngs(rngs, F)
    cfg, tri = _settings(settings, triangulator)
    dev = d.device
    o = _dev_out(*_capacities(cap, c is not None), dev)
    res = torch.zeros(RESULT_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    ctx = arrsac.ctx
    torch.cuda.current_stream(dev).synchronize()
    ctx.check(load_try_init_library().cvb_try_init_dev(
        ctx.handle, C.addressof(cfg), C.addressof(tri.cfg), C.addressof(arrsac.cfg), C.addressof(states), better_by, _dp(d), _dp(n), _dp(b),
        _dp(c), frames, cap, int(center), _p(opts), F, _dp(o["poses"]), _dp(o["view_offsets"]), _dp(o["view_landmarks"]), _dp(o["bearings"]),
        _dp(o["descriptors"]), _dp(o["colors"]), _dp(o["landmark_offsets"]), _dp(o["observations"]), _dp(o["constraints"]), _dp(res)))
    _advance(rngs, states)
    r = np.frombuffer(res.cpu().numpy().tobytes(), RESULT_DTYPE)[0]
    status = STATUS_NAMES[int(r["status"])]
    return dict(status=status, result=r, frames=[None if f == NO_FRAME else int(f) for f in r["frames"]],
                snapshot=_dev_trim(o, r["counts"]) if status == "created" else None)


__all__ = ["add_reconstruction", "try_init", "add_reconstruction_dev", "try_init_dev", "check_try_init", "STATUS_NAMES", "RESULT_DTYPE",
           "NO_FRAME"]
