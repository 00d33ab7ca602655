"""ctypes binding of the CPU oracle of include/cvb200_try_init.h (oracle/ref_try_init.c in oracle/_build/libcvb_oracle_try_init.so, built by
oracle/try_init.mk): add_reconstruction restated on slot maps, with the row gathers of bearings, descriptors and colours done here; and
try_init as the init oracle (oracle/pyoracle_init.py) followed by that restatement.

TEST INFRASTRUCTURE ONLY, like oracle/pyoracle.py.  The frame store is host copies of cvb_frame_features_batch_dev's arrays: descriptors
[frames, cap, 64], counts [frames], bearings [frames, cap, 3], colours [frames, cap, 3] or None.  Snapshots are dicts with the keys of
cv_b200.incorporate.SNAP_KEYS (host arrays)."""
import ctypes as C
import os
import subprocess

import numpy as np

from . import pyoracle_init as OINIT
from .pyoracle_constraints import CONSTRAINT_DTYPE

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "libcvb_oracle_try_init.so")

CREATED, NONE, NONE_BEARING_PAIRS = 0, 1, 2
NO_FRAME = 0xFFFFFFFF
_L = None


def build(force=False):
    srcs = [os.path.join(_HERE, f) for f in ("ref_try_init.c", "try_init.mk")]
    if not force and os.path.exists(_LIB_PATH) and all(os.path.getmtime(_LIB_PATH) >= os.path.getmtime(s) for s in srcs):
        return _LIB_PATH
    subprocess.check_call(["make", "-s", "-C", _HERE, "-f", "try_init.mk"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


def _lib():
    global _L
    if _L is None:
        build()
        L = C.CDLL(_LIB_PATH)
        vp, u32 = C.c_void_p, C.c_uint32
        L.ref_add_reconstruction.argtypes = [u32, u32, u32, vp, u32, vp, u32, vp, u32, vp, vp, vp, vp, vp]
        L.ref_add_reconstruction.restype = C.c_int
        _L = L
    return _L


def _list(a, k):
    return np.ascontiguousarray(np.asarray(a, np.uint32).reshape(-1, k))


def _pose12(p):
    if isinstance(p, tuple):
        return np.concatenate([np.asarray(p[0], np.float64).reshape(9), np.asarray(p[1], np.float64).reshape(3)])
    if isinstance(p, np.void):
        return np.concatenate([np.asarray(p["r"], np.float64).reshape(9), np.asarray(p["t"], np.float64).reshape(3)])
    return np.ascontiguousarray(p, np.float64).reshape(12)


def add_reconstruction(descriptors, counts, bearings, colors, center, first, second, first_pose, second_pose, combined, first_matches,
                       second_matches):
    """The snapshot add_reconstruction builds (views center, first, second), as a host snapshot dict.  Raises ValueError where the
    reference would index out of bounds."""
    cap = np.asarray(bearings).shape[1]
    fr = (int(center), int(first), int(second))
    n = [min(int(counts[f]), cap) for f in fr]
    comb, fm, sm = _list(combined, 3), _list(first_matches, 2), _list(second_matches, 2)
    N = sum(n)
    vo, vl = np.zeros(4, np.uint32), np.zeros(max(N, 1), np.uint32)
    lo, obs, cnt = np.zeros(N + 1, np.uint32), np.zeros((max(N, 1), 2), np.uint32), np.zeros(4, np.uint32)
    p = lambda a: a.ctypes.data if a.size else None
    if _lib().ref_add_reconstruction(n[0], n[1], n[2], p(comb), len(comb), p(fm), len(fm), p(sm), len(sm), vo.ctypes.data, vl.ctypes.data,
                                     lo.ctypes.data, obs.ctypes.data, cnt.ctypes.data):
        raise ValueError("a match list entry is out of range of its frame's features")
    L, no = int(cnt[1]), int(cnt[2])
    rows = lambda a: np.concatenate([np.asarray(a)[f, :k] for f, k in zip(fr, n)])
    cons = np.zeros(1, CONSTRAINT_DTYPE)
    cons["views"] = (0, 1, 2)
    p1, p2 = _pose12(first_pose), _pose12(second_pose)
    cons["poses"][0, 0] = (p1[:9], p1[9:])
    cons["poses"][0, 1] = (p2[:9], p2[9:])
    return dict(poses=np.stack([np.concatenate([np.eye(3).reshape(9), np.zeros(3)]), p1, p2]), view_offsets=vo, view_landmarks=vl[:N].copy(),
                bearings=rows(bearings).astype(np.float64), descriptors=rows(descriptors).astype(np.uint8),
                colors=None if colors is None else rows(colors).astype(np.uint8), landmark_offsets=lo[:L + 1].copy(), observations=obs[:no].copy(),
                constraints=cons)


def try_init(descriptors, counts, bearings, colors, center, options, pairs, n_pairs, model, inliers, n_inliers, found, cfg=None, tri=None):
    """The chain on the two-view outputs: init_reconstruction's oracle, then add_reconstruction when it accepts.  Returns dict(status,
    frames [3], init (the init oracle's dict), snapshot (or None))."""
    init = OINIT.init_reconstruction(bearings, center, options, pairs, n_pairs, model, inliers, n_inliers, found, cfg, tri)
    r = init["result"]
    status = {OINIT.ACCEPTED: CREATED, OINIT.NONE_BEARING_PAIRS: NONE_BEARING_PAIRS}.get(int(r["status"]), NONE)
    frames = [int(center), NO_FRAME, NO_FRAME]
    if int(r["status"]) != OINIT.NONE:
        frames[1:] = [int(options[r["first"]]), int(options[r["second"]])]
    snap = None
    if status == CREATED:
        snap = add_reconstruction(descriptors, counts, bearings, colors, *frames, r["first_pose"], r["second_pose"], init["combined"],
                                  init["first_matches"], init["second_matches"])
    return dict(status=status, frames=frames, init=init, snapshot=snap)
