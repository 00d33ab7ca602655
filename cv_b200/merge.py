"""cv-sfm's reconstruction merging on the device (include/cvb200_merge.h): incorporate_reconstruction (cv-sfm/src/lib.rs:1817-1887), which
moves every view of a source reconstruction S into a destination D, and try_merge_reconstructions (lib.rs:2116-2193) followed by
optimize_reconstruction, as pure functions from two reconstruction snapshots to one.

Snapshots are those of cv_b200.incorporate (SNAP_KEYS); S's constraints are never read.  The host forms take and return numpy arrays; the
*_dev forms take and return torch CUDA tensors in the layout of cv_b200.incorporate.snapshot_to_device."""
import ctypes as C

import numpy as np

from ._lib import load_merge_library
from .constraints import RESULT_DTYPE as CON_RESULT_DTYPE, _u32
from .incorporate import (COUNTS_DTYPE, NONE, _dev_out, _dev_trim, _dp, _host, _out, _ptr, _settings, _sizes, _trim)
from .reconstruction import RESULT_DTYPE as RECON_RESULT_DTYPE
from .register import RESULT_DTYPE as REG_RESULT_DTYPE, STATS_DTYPE as REG_STATS_DTYPE

# statuses of include/cvb200_merge.h
STATUS_NAMES = ["merged", "not_registered", "register_panic", "rejected", "removed_constraints", "removed_filter", "recon_panic"]
MOVE_DTYPE = np.dtype([("counts", COUNTS_DTYPE), ("moved_views", "<u4"), ("refused_views", "<u4"), ("created_landmarks", "<u4"),
                       ("constraint_calls", "<u4")])
RESULT_DTYPE = np.dtype([("status", "<i4"), ("dest_view", "<u4"), ("counts", COUNTS_DTYPE), ("reg", REG_RESULT_DTYPE),
                         ("reg_stats", REG_STATS_DTYPE), ("con", CON_RESULT_DTYPE), ("move", MOVE_DTYPE), ("recon", RECON_RESULT_DTYPE)])


def _pose12(p):
    if isinstance(p, tuple):
        return np.concatenate([np.asarray(p[0], np.float64).reshape(9), np.asarray(p[1], np.float64).reshape(3)])
    return np.ascontiguousarray(p, np.float64).reshape(12)


def check_merge(dest, src, view=NONE, landmark_map=None):
    """cvb_merge_check on the host (no device): 0, or CVB_EINVAL.  view: s_view or skip_view of src."""
    P, vo, vl, bear, d, col, lo, ob, cons = _host(dest)
    Ps, vos, vls, bs, ds, cs, los, obs_s, _ = _host(src)
    lm = None if landmark_map is None else _u32(landmark_map).reshape(-1)
    return load_merge_library().cvb_merge_check(
        len(vo) - 1, _ptr(vo), _ptr(vl), len(lo) - 1, _ptr(lo), _ptr(ob), _ptr(cons), len(cons), len(vos) - 1, _ptr(vos), _ptr(vls), len(los) - 1,
        _ptr(los), _ptr(obs_s), int(view), (lm.ctypes.data if lm is not None else None), int(col is not None), int(cs is not None))


def incorporate_reconstruction(ctx, dest, src, world_transform, landmark_map, skip_view=None, constraint_settings=None, triangulator=None):
    """cv-sfm's incorporate_reconstruction (cvb_incorporate_reconstruction): src's views (without skip_view) moved into dest under
    world_transform ((R, t) or [12], a WorldToWorld), landmark_map uint32 [L_S] (NONE for unmapped).  Returns dict(snapshot,
    src_view_map [V_S], src_landmark_map [L_S], con_results (per src view), result MOVE_DTYPE record)."""
    _, cs, _, tri = _settings(None, constraint_settings, None, triangulator)
    P, vo, vl, bear, d, col, lo, ob, cons = _host(dest)
    Ps, vos, vls, bs, ds, cls, los, obs_s, _ = _host(src)
    lm = _u32(landmark_map).reshape(-1)
    wt = _pose12(world_transform)
    V, Lm, nf, no, VS, LS, nfs = len(vo) - 1, len(lo) - 1, int(vo[-1]), int(lo[-1]), len(vos) - 1, len(los) - 1, int(vos[-1])
    if len(lm) != LS:
        raise ValueError("one landmark_map entry per source landmark expected")
    skip = NONE if skip_view is None else int(skip_view)
    hd = d is not None or ds is not None
    o = _out(V + VS, nf + nfs, Lm + nfs, no + nfs, len(cons) + VS * cs.optimization_maximum_three_view_constraints, hd, col is not None)
    svm, slm = np.zeros(max(VS, 1), np.uint32), np.zeros(max(LS, 1), np.uint32)
    cres = np.zeros(max(VS, 1), CON_RESULT_DTYPE)
    res = np.zeros(1, MOVE_DTYPE)
    ctx.check(load_merge_library().cvb_incorporate_reconstruction(
        ctx.handle, C.addressof(cs), C.addressof(tri.cfg), V, _ptr(P), _ptr(vo), _ptr(vl), _ptr(bear), _ptr(d), _ptr(col), Lm, _ptr(lo), _ptr(ob),
        _ptr(cons), len(cons), VS, _ptr(Ps), _ptr(vos), _ptr(vls), _ptr(bs), _ptr(ds), _ptr(cls), LS, _ptr(los), _ptr(obs_s), skip, wt.ctypes.data,
        _ptr(lm), o["poses"].ctypes.data, o["view_offsets"].ctypes.data, o["view_landmarks"].ctypes.data, o["bearings"].ctypes.data,
        _ptr(o["descriptors"]), _ptr(o["colors"]), o["landmark_offsets"].ctypes.data, o["observations"].ctypes.data, o["constraints"].ctypes.data,
        svm.ctypes.data, slm.ctypes.data, cres.ctypes.data, res.ctypes.data))
    r = res[0]
    return dict(snapshot=_trim(o, r["counts"]), src_view_map=svm[:VS].copy(), src_landmark_map=slm[:LS].copy(), con_results=cres[:VS].copy(),
                result=r)


def _merge_out(V, nf, Lm, no, C_, VS, nfs, cs, col):
    return V + VS, nf + nfs, Lm + no + 4 * nfs, no + 2 * nfs, C_ + (VS + 1) * cs.optimization_maximum_three_view_constraints, True, col


def merge_reconstructions(ctx, dest, src, s_view, dest_view_matches, arrsac, register_settings=None, constraint_settings=None,
                          reconstruction_settings=None, triangulator=None):
    """cv-sfm's try_merge_reconstructions followed by optimize_reconstruction (cvb_merge_reconstructions): s_view's frame of src registered
    against dest with dest_view_matches, then every other view of src moved in.  Both snapshots need their descriptors (and both or
    neither their colours); arrsac: a cv_b200.Arrsac, advanced as register_frame advances it.  Returns dict(status name, result RESULT_DTYPE
    record, snapshot (None for register_panic, removed_* and recon_panic), dest_view_map [V], dest_landmark_map [L], src_view_map [V_S],
    src_landmark_map [L_S], con_results [V_S], dest_view (index or None))."""
    rs, cs, os_, tri = _settings(register_settings, constraint_settings, reconstruction_settings, triangulator)
    P, vo, vl, bear, d, col, lo, ob, cons = _host(dest, need_desc=True)
    Ps, vos, vls, bs, ds, cls, los, obs_s, _ = _host(src, need_desc=True)
    vm = _u32(dest_view_matches).reshape(-1)
    V, Lm, nf, no, VS, LS, nfs = len(vo) - 1, len(lo) - 1, int(vo[-1]), int(lo[-1]), len(vos) - 1, len(los) - 1, int(vos[-1])
    o = _out(*_merge_out(V, nf, Lm, no, len(cons), VS, nfs, cs, col is not None))
    dvm, dlm = np.zeros(max(V, 1), np.uint32), np.zeros(max(Lm, 1), np.uint32)
    svm, slm = np.zeros(max(VS, 1), np.uint32), np.zeros(max(LS, 1), np.uint32)
    cres = np.zeros(max(VS, 1), CON_RESULT_DTYPE)
    res = np.zeros(1, RESULT_DTYPE)
    ctx.check(load_merge_library().cvb_merge_reconstructions(
        ctx.handle, C.addressof(rs), C.addressof(cs), C.addressof(os_), C.addressof(tri.cfg), C.addressof(arrsac.cfg), C.addressof(arrsac.rng.state),
        V, _ptr(P), _ptr(vo), _ptr(vl), _ptr(bear), _ptr(d), _ptr(col), Lm, _ptr(lo), _ptr(ob), _ptr(cons), len(cons), VS, _ptr(Ps), _ptr(vos),
        _ptr(vls), _ptr(bs), _ptr(ds), _ptr(cls), LS, _ptr(los), _ptr(obs_s), int(s_view), _ptr(vm), len(vm), o["poses"].ctypes.data,
        o["view_offsets"].ctypes.data, o["view_landmarks"].ctypes.data, o["bearings"].ctypes.data, _ptr(o["descriptors"]), _ptr(o["colors"]),
        o["landmark_offsets"].ctypes.data, o["observations"].ctypes.data, o["constraints"].ctypes.data, dvm.ctypes.data, dlm.ctypes.data,
        svm.ctypes.data, slm.ctypes.data, cres.ctypes.data, res.ctypes.data))
    r = res[0]
    status = STATUS_NAMES[int(r["status"])]
    have = status in ("merged", "rejected", "not_registered")
    return dict(status=status, result=r, snapshot=_trim(o, r["counts"]) if have else None, dest_view_map=dvm[:V].copy(),
                dest_landmark_map=dlm[:Lm].copy(), src_view_map=svm[:VS].copy(), src_landmark_map=slm[:LS].copy(), con_results=cres[:VS].copy(),
                dest_view=None if int(r["dest_view"]) == NONE else int(r["dest_view"]))


# ---- torch CUDA forms ------------------------------------------------------------------------------------------------------------------
def _rec(t, dtype):
    return np.frombuffer(t.cpu().numpy().tobytes(), dtype)


def incorporate_reconstruction_dev(ctx, dd, sd, world_transform, landmark_map, skip_view=None, constraint_settings=None, triangulator=None):
    """incorporate_reconstruction on torch CUDA tensors (cvb_incorporate_reconstruction_dev): dd / sd device snapshots, world_transform
    float64 [12] and landmark_map int32 [L_S] on the device.  Returns the dict of incorporate_reconstruction with device tensors."""
    import torch
    _, cs, _, tri = _settings(None, constraint_settings, None, triangulator)
    V, nf, Lm, no, C_ = _sizes(dd)
    VS, nfs, LS, nos, _ = _sizes(sd)
    dev = dd["poses"].device
    skip = NONE if skip_view is None else int(skip_view)
    hd = dd["descriptors"] is not None or sd["descriptors"] is not None
    o = _dev_out(V + VS, nf + nfs, Lm + nfs, no + nfs, C_ + VS * cs.optimization_maximum_three_view_constraints, hd, dd["colors"] is not None, dev)
    z = lambda n, dt=torch.int32: torch.zeros(n, dtype=dt, device=dev)
    svm, slm = z(max(VS, 1)), z(max(LS, 1))
    cres, res = z(max(VS, 1) * CON_RESULT_DTYPE.itemsize, torch.uint8), z(MOVE_DTYPE.itemsize, torch.uint8)
    torch.cuda.current_stream(dev).synchronize()     # the inputs come from torch's stream, the call runs on the context's
    ctx.check(load_merge_library().cvb_incorporate_reconstruction_dev(
        ctx.handle, C.addressof(cs), C.addressof(tri.cfg), V, _dp(dd["poses"]), _dp(dd["view_offsets"]), _dp(dd["view_landmarks"]),
        _dp(dd["bearings"]), _dp(dd["descriptors"]), _dp(dd["colors"]), nf, Lm, _dp(dd["landmark_offsets"]), _dp(dd["observations"]), no,
        _dp(dd["constraints"]), C_, VS, _dp(sd["poses"]), _dp(sd["view_offsets"]), _dp(sd["view_landmarks"]), _dp(sd["bearings"]),
        _dp(sd["descriptors"]), _dp(sd["colors"]), nfs, LS, _dp(sd["landmark_offsets"]), _dp(sd["observations"]), nos, skip, _dp(world_transform),
        _dp(landmark_map), _dp(o["poses"]), _dp(o["view_offsets"]), _dp(o["view_landmarks"]), _dp(o["bearings"]), _dp(o["descriptors"]),
        _dp(o["colors"]), _dp(o["landmark_offsets"]), _dp(o["observations"]), _dp(o["constraints"]), _dp(svm), _dp(slm), _dp(cres), _dp(res)))
    r = _rec(res, MOVE_DTYPE)[0]
    return dict(snapshot=_dev_trim(o, r["counts"]), src_view_map=svm[:VS], src_landmark_map=slm[:LS],
                con_results=_rec(cres, CON_RESULT_DTYPE)[:VS].copy(), result=r)


def merge_reconstructions_dev(ctx, dd, sd, s_view, dest_view_matches, arrsac, register_settings=None, constraint_settings=None,
                              reconstruction_settings=None, triangulator=None):
    """merge_reconstructions on torch CUDA tensors (cvb_merge_reconstructions_dev): dd / sd device snapshots with descriptors,
    dest_view_matches on the host.  Returns the dict of merge_reconstructions with device tensors."""
    import torch
    rs, cs, os_, tri = _settings(register_settings, constraint_settings, reconstruction_settings, triangulator)
    V, nf, Lm, no, C_ = _sizes(dd)
    VS, nfs, LS, nos, _ = _sizes(sd)
    dev = dd["poses"].device
    vm = _u32(dest_view_matches).reshape(-1)
    o = _dev_out(*_merge_out(V, nf, Lm, no, C_, VS, nfs, cs, dd["colors"] is not None), dev)
    z = lambda n, dt=torch.int32: torch.zeros(n, dtype=dt, device=dev)
    dvm, dlm, svm, slm = z(max(V, 1)), z(max(Lm, 1)), z(max(VS, 1)), z(max(LS, 1))
    cres, res = z(max(VS, 1) * CON_RESULT_DTYPE.itemsize, torch.uint8), z(RESULT_DTYPE.itemsize, torch.uint8)
    torch.cuda.current_stream(dev).synchronize()
    ctx.check(load_merge_library().cvb_merge_reconstructions_dev(
        ctx.handle, C.addressof(rs), C.addressof(cs), C.addressof(os_), C.addressof(tri.cfg), C.addressof(arrsac.cfg), C.addressof(arrsac.rng.state),
        V, _dp(dd["poses"]), _dp(dd["view_offsets"]), _dp(dd["view_landmarks"]), _dp(dd["bearings"]), _dp(dd["descriptors"]), _dp(dd["colors"]),
        nf, Lm, _dp(dd["landmark_offsets"]), _dp(dd["observations"]), no, _dp(dd["constraints"]), C_, VS, _dp(sd["poses"]), _dp(sd["view_offsets"]),
        _dp(sd["view_landmarks"]), _dp(sd["bearings"]), _dp(sd["descriptors"]), _dp(sd["colors"]), nfs, LS, _dp(sd["landmark_offsets"]),
        _dp(sd["observations"]), nos, int(s_view), _ptr(vm), len(vm), _dp(o["poses"]), _dp(o["view_offsets"]), _dp(o["view_landmarks"]),
        _dp(o["bearings"]), _dp(o["descriptors"]), _dp(o["colors"]), _dp(o["landmark_offsets"]), _dp(o["observations"]), _dp(o["constraints"]),
        _dp(dvm), _dp(dlm), _dp(svm), _dp(slm), _dp(cres), _dp(res)))
    r = _rec(res, RESULT_DTYPE)[0]
    status = STATUS_NAMES[int(r["status"])]
    have = status in ("merged", "rejected", "not_registered")
    return dict(status=status, result=r, snapshot=_dev_trim(o, r["counts"]) if have else None, dest_view_map=dvm[:V], dest_landmark_map=dlm[:Lm],
                src_view_map=svm[:VS], src_landmark_map=slm[:LS], con_results=_rec(cres, CON_RESULT_DTYPE)[:VS].copy(),
                dest_view=None if int(r["dest_view"]) == NONE else int(r["dest_view"]))


__all__ = ["incorporate_reconstruction", "merge_reconstructions", "incorporate_reconstruction_dev", "merge_reconstructions_dev", "check_merge",
           "STATUS_NAMES", "RESULT_DTYPE", "MOVE_DTYPE", "NONE"]
