"""cv-sfm's frame incorporation on the device (include/cvb200_incorporate.h): add_view with merge_landmarks (cv-sfm/src/lib.rs:432-483,
699-721), the replay of optimize_reconstruction's edits (remove_view, split_landmark, split_observation, lib.rs:517-588), and
incorporate_frame (lib.rs:2067-2087) followed by optimize_reconstruction, as pure functions from one reconstruction snapshot to the next.

A snapshot is a dict with the keys of SNAP_KEYS: poses [V, 12] float64 (WorldToCamera), view_offsets [V + 1], view_landmarks
[n_features], bearings [n_features, 3], descriptors uint8 [n_features, 64] (or None), colors uint8 [n_features, 3] (or None),
landmark_offsets [L + 1], observations [n_observations, 2] of (view, feature), constraints CONSTRAINT_DTYPE [C].  The host forms take and
return numpy arrays; the *_dev forms take and return torch CUDA tensors (int32 for the index arrays, uint8 [C, CONSTRAINT_DTYPE.itemsize]
for the constraints), so that a loop over frames never copies the snapshot to the host."""
import ctypes as C

import numpy as np

from ._lib import load_incorporate_library
from .constraints import CONSTRAINT_DTYPE, ConstraintSettings, RESULT_DTYPE as CON_RESULT_DTYPE, _poses, _u32
from .reconstruction import RESULT_DTYPE as RECON_RESULT_DTYPE, ReconstructionSettings
from .register import MATCH_DTYPE, RESULT_DTYPE as REG_RESULT_DTYPE, STATS_DTYPE as REG_STATS_DTYPE, RegisterSettings

NONE = 0xFFFFFFFF
SNAP_KEYS = ("poses", "view_offsets", "view_landmarks", "bearings", "descriptors", "colors", "landmark_offsets", "observations", "constraints")
# statuses of include/cvb200_incorporate.h
STATUS_NAMES = ["kept", "not_registered", "register_panic", "rejected", "removed_constraints", "removed_filter", "recon_panic"]
COUNTS_DTYPE = np.dtype([("V", "<u4"), ("n_features", "<u4"), ("L", "<u4"), ("n_observations", "<u4"), ("C", "<u4"), ("merges", "<u4")])
RESULT_DTYPE = np.dtype([("status", "<i4"), ("new_view", "<u4"), ("counts", COUNTS_DTYPE), ("reg", REG_RESULT_DTYPE),
                         ("reg_stats", REG_STATS_DTYPE), ("con", CON_RESULT_DTYPE), ("recon", RECON_RESULT_DTYPE), ("reserved", "<u4", (2,))])


def _ptr(a):
    return a.ctypes.data if a is not None and a.size else None


def _host(snap, need_desc=False):
    """the snapshot's arrays in the layout of the C calls"""
    P = _poses(snap["poses"])
    vo, vl, lo = _u32(snap["view_offsets"]).reshape(-1), _u32(snap["view_landmarks"]).reshape(-1), _u32(snap["landmark_offsets"]).reshape(-1)
    ob = _u32(snap["observations"]).reshape(-1)
    bear = np.ascontiguousarray(snap["bearings"], np.float64).reshape(-1, 3)
    d = snap.get("descriptors")
    d = None if d is None else np.ascontiguousarray(d, np.uint8).reshape(-1, 64)
    if need_desc and d is None:
        raise ValueError("the snapshot needs its descriptors")
    col = snap.get("colors")
    col = None if col is None else np.ascontiguousarray(col, np.uint8).reshape(-1, 3)
    cons = snap.get("constraints")
    cons = np.ascontiguousarray(cons if cons is not None else np.zeros(0, CONSTRAINT_DTYPE), CONSTRAINT_DTYPE).reshape(-1)
    return P, vo, vl, bear, d, col, lo, ob, cons


def _out(V, nf, L, no, C_, desc, col):
    return dict(poses=np.zeros((max(V, 1), 12)), view_offsets=np.zeros(V + 1, np.uint32), view_landmarks=np.zeros(max(nf, 1), np.uint32),
                bearings=np.zeros((max(nf, 1), 3)), descriptors=np.zeros((max(nf, 1), 64), np.uint8) if desc else None,
                colors=np.zeros((max(nf, 1), 3), np.uint8) if col else None, landmark_offsets=np.zeros(L + 1, np.uint32),
                observations=np.zeros((max(no, 1), 2), np.uint32), constraints=np.zeros(max(C_, 1), CONSTRAINT_DTYPE))


def _trim(o, c):
    V, nf, L, no, C_ = int(c["V"]), int(c["n_features"]), int(c["L"]), int(c["n_observations"]), int(c["C"])
    return dict(poses=o["poses"][:V].copy(), view_offsets=o["view_offsets"][:V + 1].copy(), view_landmarks=o["view_landmarks"][:nf].copy(),
                bearings=o["bearings"][:nf].copy(), descriptors=None if o["descriptors"] is None else o["descriptors"][:nf].copy(),
                colors=None if o["colors"] is None else o["colors"][:nf].copy(), landmark_offsets=o["landmark_offsets"][:L + 1].copy(),
                observations=o["observations"][:no].copy(), constraints=o["constraints"][:C_].copy())


def check_incorporate(snap, N=0, matches=None, view_state=None, obs_state=None):
    """cvb_incorporate_check on the host (no device): 0, or CVB_EINVAL.  With matches (MATCH_DTYPE) an add_view of N features is checked;
    with view_state / obs_state an apply_optimization."""
    P, vo, vl, bear, d, col, lo, ob, cons = _host(snap)
    m = None if matches is None else np.ascontiguousarray(matches, MATCH_DTYPE).reshape(-1)
    vs = None if view_state is None else np.ascontiguousarray(view_state, np.uint8).reshape(-1)
    os_ = None if obs_state is None else np.ascontiguousarray(obs_state, np.uint8).reshape(-1)
    return load_incorporate_library().cvb_incorporate_check(
        max(len(vo) - 1, 0), _ptr(vo), _ptr(vl), max(len(lo) - 1, 0), _ptr(lo), _ptr(ob), _ptr(cons), len(cons), int(N),
        m.ctypes.data if m is not None else None, 0 if m is None else len(m), vs.ctypes.data if vs is not None else None,
        0 if vs is None else len(vs), os_.ctypes.data if os_ is not None else None, 0 if os_ is None else len(os_))


def add_view(ctx, snap, pose, new_bearings, matches, new_descriptors=None, new_colors=None):
    """cv-sfm's add_view with merge_landmarks (cvb_add_view): the new view V with pose (R [3, 3], t [3]) or [12], its N features'
    bearings (and descriptors / colours when the snapshot has them), and register_frame's matches (MATCH_DTYPE, ascending by feature).
    Returns the new snapshot (constraints unchanged) plus landmark_map uint32 [L] and merges."""
    P, vo, vl, bear, d, col, lo, ob, cons = _host(snap)
    pose = np.concatenate([np.asarray(pose[0], np.float64).reshape(9), np.asarray(pose[1], np.float64).reshape(3)]) \
        if isinstance(pose, tuple) else np.ascontiguousarray(pose, np.float64).reshape(12)
    nb = np.ascontiguousarray(new_bearings, np.float64).reshape(-1, 3)
    N = len(nb)
    nd = None if new_descriptors is None else np.ascontiguousarray(new_descriptors, np.uint8).reshape(-1, 64)
    nc = None if new_colors is None else np.ascontiguousarray(new_colors, np.uint8).reshape(-1, 3)
    m = np.ascontiguousarray(matches, MATCH_DTYPE).reshape(-1)
    V, Lm, nf, no = len(vo) - 1, len(lo) - 1, int(vo[-1]), int(lo[-1])
    o = _out(V + 1, nf + N, Lm + N, no + N, 0, d is not None, col is not None)
    lmap = np.zeros(max(Lm, 1), np.uint32)
    cnt = np.zeros(1, COUNTS_DTYPE)
    ctx.check(load_incorporate_library().cvb_add_view(
        ctx.handle, V, _ptr(P), _ptr(vo), _ptr(vl), _ptr(bear), _ptr(d), _ptr(col), Lm, _ptr(lo), _ptr(ob), pose.ctypes.data, _ptr(nb), _ptr(nd),
        _ptr(nc), N, _ptr(m), len(m), o["poses"].ctypes.data, o["view_offsets"].ctypes.data, o["view_landmarks"].ctypes.data,
        o["bearings"].ctypes.data, _ptr(o["descriptors"]), _ptr(o["colors"]), o["landmark_offsets"].ctypes.data, o["observations"].ctypes.data,
        lmap.ctypes.data, cnt.ctypes.data))
    c = cnt[0].copy()
    c["C"] = len(cons)
    out = _trim(o, c)
    out["constraints"] = cons.copy()
    out.update(landmark_map=lmap[:Lm].copy(), merges=int(c["merges"]))
    return out


def apply_optimization(ctx, snap, poses, view_state, obs_state):
    """The edits of optimize_reconstruction replayed (cvb_apply_optimization): poses, view_state and obs_state are
    cv_b200.optimize_reconstruction's (status KEPT) on this snapshot.  Returns the new snapshot plus view_map [V] and landmark_map [L]."""
    P, vo, vl, bear, d, col, lo, ob, cons = _host(snap)
    P = _poses(poses)
    vs, os_ = np.ascontiguousarray(view_state, np.uint8).reshape(-1), np.ascontiguousarray(obs_state, np.uint8).reshape(-1)
    V, Lm, nf, no = len(vo) - 1, len(lo) - 1, int(vo[-1]), int(lo[-1])
    o = _out(V, nf, Lm + no, no, len(cons), d is not None, col is not None)
    vmap, lmap = np.zeros(max(V, 1), np.uint32), np.zeros(max(Lm, 1), np.uint32)
    cnt = np.zeros(1, COUNTS_DTYPE)
    ctx.check(load_incorporate_library().cvb_apply_optimization(
        ctx.handle, V, _ptr(P), _ptr(vo), _ptr(vl), _ptr(bear), _ptr(d), _ptr(col), Lm, _ptr(lo), _ptr(ob), _ptr(cons), len(cons), _ptr(vs),
        _ptr(os_), o["poses"].ctypes.data, o["view_offsets"].ctypes.data, o["view_landmarks"].ctypes.data, o["bearings"].ctypes.data,
        _ptr(o["descriptors"]), _ptr(o["colors"]), o["landmark_offsets"].ctypes.data, o["observations"].ctypes.data,
        o["constraints"].ctypes.data, vmap.ctypes.data, lmap.ctypes.data, cnt.ctypes.data))
    out = _trim(o, cnt[0])
    out.update(view_map=vmap[:V].copy(), landmark_map=lmap[:Lm].copy())
    return out


def _settings(register_settings, constraint_settings, reconstruction_settings, triangulator):
    from .triangulation import LinearEigenTriangulator
    return (register_settings if register_settings is not None else RegisterSettings(),
            constraint_settings if constraint_settings is not None else ConstraintSettings(),
            reconstruction_settings if reconstruction_settings is not None else ReconstructionSettings(),
            triangulator if triangulator is not None else LinearEigenTriangulator())


def incorporate_frame(ctx, snap, new_descriptors, new_bearings, view_matches, arrsac, new_colors=None, register_settings=None,
                      constraint_settings=None, reconstruction_settings=None, triangulator=None):
    """cv-sfm's incorporate_frame followed by optimize_reconstruction (cvb_incorporate_frame).  snap needs its descriptors (and colours
    when new_colors is given); arrsac: a cv_b200.Arrsac (VSlam's single_view_consensus), advanced as register_frame advances it.
    Returns dict(status name, result RESULT_DTYPE record, snapshot (None for register_panic, removed_* and recon_panic), view_map [V],
    landmark_map [L], new_view (index or None), matches MATCH_DTYPE [n])."""
    rs, cs, os_, tri = _settings(register_settings, constraint_settings, reconstruction_settings, triangulator)
    P, vo, vl, bear, d, col, lo, ob, cons = _host(snap, need_desc=True)
    nd = np.ascontiguousarray(new_descriptors, np.uint8).reshape(-1, 64)
    nb = np.ascontiguousarray(new_bearings, np.float64).reshape(-1, 3)
    if len(nd) != len(nb):
        raise ValueError("one bearing per new descriptor expected")
    nc = None if new_colors is None else np.ascontiguousarray(new_colors, np.uint8).reshape(-1, 3)
    vm = _u32(view_matches).reshape(-1)
    V, Lm, nf, no, N = len(vo) - 1, len(lo) - 1, int(vo[-1]), int(lo[-1]), len(nd)
    o = _out(V + 1, nf + N, Lm + N + no + N, no + N, len(cons) + cs.optimization_maximum_three_view_constraints, True, col is not None)
    vmap, lmap = np.zeros(max(V, 1), np.uint32), np.zeros(max(Lm, 1), np.uint32)
    matches = np.zeros(max(N, 1), MATCH_DTYPE)
    res = np.zeros(1, RESULT_DTYPE)
    ctx.check(load_incorporate_library().cvb_incorporate_frame(
        ctx.handle, C.addressof(rs), C.addressof(cs), C.addressof(os_), C.addressof(tri.cfg), C.addressof(arrsac.cfg),
        C.addressof(arrsac.rng.state), V, _ptr(P), _ptr(vo), _ptr(vl), _ptr(bear), _ptr(d), _ptr(col), Lm, _ptr(lo), _ptr(ob), _ptr(cons),
        len(cons), _ptr(nd), _ptr(nb), _ptr(nc), N, _ptr(vm), len(vm), o["poses"].ctypes.data, o["view_offsets"].ctypes.data,
        o["view_landmarks"].ctypes.data, o["bearings"].ctypes.data, _ptr(o["descriptors"]), _ptr(o["colors"]), o["landmark_offsets"].ctypes.data,
        o["observations"].ctypes.data, o["constraints"].ctypes.data, vmap.ctypes.data, lmap.ctypes.data, matches.ctypes.data, res.ctypes.data))
    r = res[0]
    status = STATUS_NAMES[int(r["status"])]
    have = status in ("kept", "rejected", "not_registered")
    nm = int(r["reg"]["n_matches"]) if int(r["reg"]["status"]) == 0 else 0
    return dict(status=status, result=r, snapshot=_trim(o, r["counts"]) if have else None, view_map=vmap[:V].copy(),
                landmark_map=lmap[:Lm].copy(), new_view=None if int(r["new_view"]) == NONE else int(r["new_view"]),
                matches=matches[:nm].copy())


# ---- torch CUDA forms ------------------------------------------------------------------------------------------------------------------
def snapshot_to_device(snap, device="cuda"):
    """A host snapshot as torch CUDA tensors in the layout of the *_dev forms."""
    import torch
    P, vo, vl, bear, d, col, lo, ob, cons = _host(snap)
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(device)
    return dict(poses=t(P), view_offsets=t(vo.view(np.int32)), view_landmarks=t(vl.view(np.int32)), bearings=t(bear), descriptors=t(d),
                colors=t(col), landmark_offsets=t(lo.view(np.int32)), observations=t(ob.view(np.int32).reshape(-1, 2)),
                constraints=t(cons.view(np.uint8).reshape(-1, CONSTRAINT_DTYPE.itemsize)))


def snapshot_to_host(sd):
    """The inverse of snapshot_to_device."""
    h = lambda x: None if x is None else x.cpu().numpy()
    return dict(poses=h(sd["poses"]), view_offsets=h(sd["view_offsets"]).view(np.uint32), view_landmarks=h(sd["view_landmarks"]).view(np.uint32),
                bearings=h(sd["bearings"]), descriptors=h(sd["descriptors"]), colors=h(sd["colors"]),
                landmark_offsets=h(sd["landmark_offsets"]).view(np.uint32), observations=h(sd["observations"]).view(np.uint32),
                constraints=np.ascontiguousarray(h(sd["constraints"])).reshape(-1).view(CONSTRAINT_DTYPE))


def _dp(x):
    return x.data_ptr() if x is not None and x.numel() else None


def _sizes(sd):
    return (sd["view_offsets"].numel() - 1, sd["view_landmarks"].numel(), sd["landmark_offsets"].numel() - 1, sd["observations"].shape[0],
            sd["constraints"].shape[0])


def _dev_out(V, nf, L, no, C_, desc, col, dev):
    import torch
    z = lambda *s, dt: torch.zeros(*s, dtype=dt, device=dev)
    return dict(poses=z(max(V, 1), 12, dt=torch.float64), view_offsets=z(V + 1, dt=torch.int32), view_landmarks=z(max(nf, 1), dt=torch.int32),
                bearings=z(max(nf, 1), 3, dt=torch.float64), descriptors=z(max(nf, 1), 64, dt=torch.uint8) if desc else None,
                colors=z(max(nf, 1), 3, dt=torch.uint8) if col else None, landmark_offsets=z(L + 1, dt=torch.int32),
                observations=z(max(no, 1), 2, dt=torch.int32), constraints=z(max(C_, 1), CONSTRAINT_DTYPE.itemsize, dt=torch.uint8))


def _dev_trim(o, c):
    V, nf, L, no, C_ = int(c["V"]), int(c["n_features"]), int(c["L"]), int(c["n_observations"]), int(c["C"])
    return dict(poses=o["poses"][:V], view_offsets=o["view_offsets"][:V + 1], view_landmarks=o["view_landmarks"][:nf],
                bearings=o["bearings"][:nf], descriptors=None if o["descriptors"] is None else o["descriptors"][:nf],
                colors=None if o["colors"] is None else o["colors"][:nf], landmark_offsets=o["landmark_offsets"][:L + 1],
                observations=o["observations"][:no], constraints=o["constraints"][:C_])


def _counts(t):
    return np.frombuffer(t.cpu().numpy().tobytes(), COUNTS_DTYPE)[0]


def add_view_dev(ctx, sd, pose, new_bearings, matches, new_descriptors=None, new_colors=None):
    """add_view on torch CUDA tensors (cvb_add_view_dev): sd a device snapshot, pose float64 [12], new_bearings [N, 3], matches uint8
    [M, 12] (MATCH_DTYPE rows) on the device.  Returns the device snapshot (constraints unchanged), landmark_map int32 [L] and the counts."""
    import torch
    V, nf, Lm, no, C_ = _sizes(sd)
    N, M = new_bearings.shape[0], matches.shape[0]
    dev = sd["poses"].device
    o = _dev_out(V + 1, nf + N, Lm + N, no + N, 0, sd["descriptors"] is not None, sd["colors"] is not None, dev)
    lmap = torch.zeros(max(Lm, 1), dtype=torch.int32, device=dev)
    cnt = torch.zeros(COUNTS_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    torch.cuda.current_stream(dev).synchronize()     # the inputs come from torch's stream, the call runs on the context's
    ctx.check(load_incorporate_library().cvb_add_view_dev(
        ctx.handle, V, _dp(sd["poses"]), _dp(sd["view_offsets"]), _dp(sd["view_landmarks"]), _dp(sd["bearings"]), _dp(sd["descriptors"]),
        _dp(sd["colors"]), nf, Lm, _dp(sd["landmark_offsets"]), _dp(sd["observations"]), no, _dp(pose), _dp(new_bearings),
        _dp(new_descriptors), _dp(new_colors), N, _dp(matches), M, _dp(o["poses"]), _dp(o["view_offsets"]), _dp(o["view_landmarks"]),
        _dp(o["bearings"]), _dp(o["descriptors"]), _dp(o["colors"]), _dp(o["landmark_offsets"]), _dp(o["observations"]), _dp(lmap),
        _dp(cnt)))
    c = _counts(cnt)
    out = _dev_trim(o, c)
    out["constraints"] = sd["constraints"]
    return out, lmap[:Lm], c


def apply_optimization_dev(ctx, sd, poses, view_state, obs_state):
    """apply_optimization on torch CUDA tensors (cvb_apply_optimization_dev): poses float64 [V, 12], view_state / obs_state uint8.
    Returns the device snapshot, view_map int32 [V], landmark_map int32 [L] and the counts."""
    import torch
    V, nf, Lm, no, C_ = _sizes(sd)
    dev = sd["poses"].device
    o = _dev_out(V, nf, Lm + no, no, C_, sd["descriptors"] is not None, sd["colors"] is not None, dev)
    vmap = torch.zeros(max(V, 1), dtype=torch.int32, device=dev)
    lmap = torch.zeros(max(Lm, 1), dtype=torch.int32, device=dev)
    cnt = torch.zeros(COUNTS_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    torch.cuda.current_stream(dev).synchronize()
    ctx.check(load_incorporate_library().cvb_apply_optimization_dev(
        ctx.handle, V, _dp(poses), _dp(sd["view_offsets"]), _dp(sd["view_landmarks"]), _dp(sd["bearings"]), _dp(sd["descriptors"]),
        _dp(sd["colors"]), nf, Lm, _dp(sd["landmark_offsets"]), _dp(sd["observations"]), no, _dp(sd["constraints"]), C_, _dp(view_state),
        _dp(obs_state), _dp(o["poses"]), _dp(o["view_offsets"]), _dp(o["view_landmarks"]), _dp(o["bearings"]), _dp(o["descriptors"]),
        _dp(o["colors"]), _dp(o["landmark_offsets"]), _dp(o["observations"]), _dp(o["constraints"]), _dp(vmap), _dp(lmap), _dp(cnt)))
    c = _counts(cnt)
    return _dev_trim(o, c), vmap[:V], lmap[:Lm], c


def incorporate_frame_dev(ctx, sd, new_descriptors, new_bearings, view_matches, arrsac, new_colors=None, register_settings=None,
                          constraint_settings=None, reconstruction_settings=None, triangulator=None):
    """incorporate_frame on torch CUDA tensors (cvb_incorporate_frame_dev): sd a device snapshot with descriptors, the new frame's
    tensors on the device, view_matches on the host.  Returns dict(status, result, snapshot (device tensors, or None), view_map int32 [V],
    landmark_map int32 [L], new_view, matches uint8 [n, 12])."""
    import torch
    rs, cs, os_, tri = _settings(register_settings, constraint_settings, reconstruction_settings, triangulator)
    V, nf, Lm, no, C_ = _sizes(sd)
    N = new_bearings.shape[0]
    dev = sd["poses"].device
    vm = _u32(view_matches).reshape(-1)
    o = _dev_out(V + 1, nf + N, Lm + N + no + N, no + N, C_ + cs.optimization_maximum_three_view_constraints, True, sd["colors"] is not None,
                 dev)
    vmap = torch.zeros(max(V, 1), dtype=torch.int32, device=dev)
    lmap = torch.zeros(max(Lm, 1), dtype=torch.int32, device=dev)
    matches = torch.zeros(max(N, 1), MATCH_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    res = torch.zeros(RESULT_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    torch.cuda.current_stream(dev).synchronize()
    ctx.check(load_incorporate_library().cvb_incorporate_frame_dev(
        ctx.handle, C.addressof(rs), C.addressof(cs), C.addressof(os_), C.addressof(tri.cfg), C.addressof(arrsac.cfg),
        C.addressof(arrsac.rng.state), V, _dp(sd["poses"]), _dp(sd["view_offsets"]), _dp(sd["view_landmarks"]), _dp(sd["bearings"]),
        _dp(sd["descriptors"]), _dp(sd["colors"]), nf, Lm, _dp(sd["landmark_offsets"]), _dp(sd["observations"]), no, _dp(sd["constraints"]),
        C_, _dp(new_descriptors), _dp(new_bearings), _dp(new_colors), N, _ptr(vm), len(vm), _dp(o["poses"]), _dp(o["view_offsets"]),
        _dp(o["view_landmarks"]), _dp(o["bearings"]), _dp(o["descriptors"]), _dp(o["colors"]), _dp(o["landmark_offsets"]),
        _dp(o["observations"]), _dp(o["constraints"]), _dp(vmap), _dp(lmap), _dp(matches), _dp(res)))
    r = np.frombuffer(res.cpu().numpy().tobytes(), RESULT_DTYPE)[0]
    status = STATUS_NAMES[int(r["status"])]
    have = status in ("kept", "rejected", "not_registered")
    nm = int(r["reg"]["n_matches"]) if int(r["reg"]["status"]) == 0 else 0
    return dict(status=status, result=r, snapshot=_dev_trim(o, r["counts"]) if have else None, view_map=vmap[:V], landmark_map=lmap[:Lm],
                new_view=None if int(r["new_view"]) == NONE else int(r["new_view"]), matches=matches[:nm])


__all__ = ["add_view", "apply_optimization", "incorporate_frame", "add_view_dev", "apply_optimization_dev", "incorporate_frame_dev",
           "check_incorporate", "snapshot_to_device", "snapshot_to_host", "SNAP_KEYS", "STATUS_NAMES", "RESULT_DTYPE", "COUNTS_DTYPE", "NONE"]
