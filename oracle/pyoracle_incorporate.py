"""ctypes binding of the CPU oracle of include/cvb200_incorporate.h (oracle/ref_incorporate.c in oracle/_build/libcvb_oracle_incorporate.so,
built by oracle/incorporate.mk): add_view with merge_landmarks and the replay of optimize_reconstruction's edits, restated on a slot map;
and incorporate_frame as the composition of the register, constraints and reconstruction oracles with those two edits.

TEST INFRASTRUCTURE ONLY, like oracle/pyoracle.py.  Snapshots are dicts with the keys of cv_b200.incorporate.SNAP_KEYS (host arrays)."""
import ctypes as C
import os
import subprocess

import numpy as np

from . import pyoracle_constraints as OC
from . import pyoracle_reconstruction as OREC
from . import pyoracle_register as OR

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "libcvb_oracle_incorporate.so")

NONE = 0xFFFFFFFF
MATCH_DTYPE = OR.MATCH_DTYPE
CONSTRAINT_DTYPE = OC.CONSTRAINT_DTYPE
COUNTS_DTYPE = np.dtype([("V", "<u4"), ("n_features", "<u4"), ("L", "<u4"), ("n_observations", "<u4"), ("C", "<u4"), ("merges", "<u4")])
VIEW_KEPT, VIEW_NO_EDGES = 0, 1
OBS_KEPT, OBS_SPLIT, OBS_DROPPED = 0, 1, 2

_L = None


def build(force=False):
    srcs = [os.path.join(_HERE, f) for f in ("ref_incorporate.c", "incorporate.mk")]
    if not force and os.path.exists(_LIB_PATH) and all(os.path.getmtime(_LIB_PATH) >= os.path.getmtime(s) for s in srcs):
        return _LIB_PATH
    subprocess.check_call(["make", "-s", "-C", _HERE, "-f", "incorporate.mk"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


def _lib():
    global _L
    if _L is None:
        build()
        L = C.CDLL(_LIB_PATH)
        vp, u32 = C.c_void_p, C.c_uint32
        L.ref_add_view.argtypes = [u32] + [vp] * 6 + [u32, vp, vp] + [vp] * 4 + [u32, vp, u32] + [vp] * 10
        L.ref_add_view.restype = C.c_int
        L.ref_apply_optimization.argtypes = [u32] + [vp] * 6 + [u32, vp, vp, vp, u32, vp, vp] + [vp] * 12
        L.ref_apply_optimization.restype = C.c_int
        _L = L
    return _L


def _ptr(a):
    return a.ctypes.data if a is not None and a.size else None


def _arrays(s):
    u = (lambda a: np.ascontiguousarray(a, np.uint32).reshape(-1))
    P = np.ascontiguousarray(s["poses"], np.float64).reshape(-1, 12)
    d = s.get("descriptors")
    col = s.get("colors")
    cons = s.get("constraints")
    return (P, u(s["view_offsets"]), u(s["view_landmarks"]), np.ascontiguousarray(s["bearings"], np.float64).reshape(-1, 3),
            None if d is None else np.ascontiguousarray(d, np.uint8).reshape(-1, 64),
            None if col is None else np.ascontiguousarray(col, np.uint8).reshape(-1, 3), u(s["landmark_offsets"]), u(s["observations"]),
            np.ascontiguousarray(cons if cons is not None else np.zeros(0, CONSTRAINT_DTYPE), CONSTRAINT_DTYPE).reshape(-1))


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


def add_view(s, pose, new_bearings, matches, new_descriptors=None, new_colors=None):
    """The snapshot after add_view (constraints unchanged), with landmark_map and merges; None where merge_landmarks' assert! fires."""
    P, vo, vl, bear, d, col, lo, ob, cons = _arrays(s)
    pose = np.ascontiguousarray(pose, np.float64).reshape(12)
    nb = np.ascontiguousarray(new_bearings, np.float64).reshape(-1, 3)
    nd = None if new_descriptors is None else np.ascontiguousarray(new_descriptors, np.uint8).reshape(-1, 64)
    nc = None if new_colors is None else np.ascontiguousarray(new_colors, np.uint8).reshape(-1, 3)
    m = np.ascontiguousarray(matches, MATCH_DTYPE).reshape(-1)
    V, Lm, nf, no, N = len(vo) - 1, len(lo) - 1, int(vo[-1]), int(lo[-1]), len(nb)
    o = _out(V + 1, nf + N, Lm + N, no + N, 0, d is not None, col is not None)
    lmap = np.zeros(max(Lm, 1), np.uint32)
    cnt = np.zeros(1, COUNTS_DTYPE)
    rc = _lib().ref_add_view(V, _ptr(P), _ptr(vo), _ptr(vl), _ptr(bear), _ptr(d), _ptr(col), Lm, _ptr(lo), _ptr(ob), pose.ctypes.data, _ptr(nb),
                             _ptr(nd), _ptr(nc), N, _ptr(m), len(m), o["poses"].ctypes.data, o["view_offsets"].ctypes.data,
                             o["view_landmarks"].ctypes.data, o["bearings"].ctypes.data, _ptr(o["descriptors"]), _ptr(o["colors"]),
                             o["landmark_offsets"].ctypes.data, o["observations"].ctypes.data, lmap.ctypes.data, cnt.ctypes.data)
    if rc:
        return None
    c = cnt[0].copy()
    c["C"] = len(cons)
    out = _trim(o, c)
    out["constraints"] = cons.copy()
    out.update(landmark_map=lmap[:Lm].copy(), merges=int(c["merges"]))
    return out


def apply_optimization(s, poses, view_state, obs_state):
    """The snapshot after optimize_reconstruction's edits, with view_map and landmark_map."""
    P, vo, vl, bear, d, col, lo, ob, cons = _arrays(s)
    P = np.ascontiguousarray(poses, np.float64).reshape(-1, 12)
    vs, os_ = np.ascontiguousarray(view_state, np.uint8), np.ascontiguousarray(obs_state, np.uint8)
    V, Lm, nf, no = len(vo) - 1, len(lo) - 1, int(vo[-1]), int(lo[-1])
    o = _out(V, nf, Lm + no, no, len(cons), d is not None, col is not None)
    vmap, lmap = np.zeros(max(V, 1), np.uint32), np.zeros(max(Lm, 1), np.uint32)
    cnt = np.zeros(1, COUNTS_DTYPE)
    assert _lib().ref_apply_optimization(V, _ptr(P), _ptr(vo), _ptr(vl), _ptr(bear), _ptr(d), _ptr(col), Lm, _ptr(lo), _ptr(ob), _ptr(cons),
                                         len(cons), _ptr(vs), _ptr(os_), o["poses"].ctypes.data, o["view_offsets"].ctypes.data,
                                         o["view_landmarks"].ctypes.data, o["bearings"].ctypes.data, _ptr(o["descriptors"]), _ptr(o["colors"]),
                                         o["landmark_offsets"].ctypes.data, o["observations"].ctypes.data, o["constraints"].ctypes.data,
                                         vmap.ctypes.data, lmap.ctypes.data, cnt.ctypes.data) == 0
    out = _trim(o, cnt[0])
    out.update(view_map=vmap[:V].copy(), landmark_map=lmap[:Lm].copy())
    return out


def remove_new_view(s):
    """remove_view of the last view, as apply_optimization's states"""
    V = len(s["view_offsets"]) - 1
    vs = np.zeros(V, np.uint8)
    vs[V - 1] = VIEW_NO_EDGES
    os_ = np.where(np.asarray(s["observations"]).reshape(-1, 2)[:, 0] == V - 1, OBS_DROPPED, OBS_KEPT).astype(np.uint8)
    return apply_optimization(s, s["poses"], vs, os_)


def _compose(first, second):
    first = np.asarray(first, np.uint32)
    out = np.full(len(first), NONE, np.uint32)
    ok = first != NONE
    out[ok] = np.asarray(second, np.uint32)[first[ok]]
    return out


def incorporate_frame(s, new_descriptors, new_bearings, view_matches, arrsac_cfg, rng, new_colors=None, register_cfg=None,
                      constraints_cfg=None, recon_cfg=None, tri=None):
    """The oracle chain: register_frame, add_view, generate_view_constraints of the new view with record_view_constraints' acceptance
    (remove_view when refused), optimize_reconstruction over the old constraints then the new ones, and its edits.  rng (an oracle Rng) is
    advanced like the reference's.  Returns dict(status, register, constraints, recon (the oracles' outputs, None where a stage did not
    run), snapshot or None, view_map, landmark_map, new_view)."""
    keys = ("poses", "view_offsets", "view_landmarks", "bearings", "descriptors", "landmark_offsets", "observations")
    V, Lm = len(s["view_offsets"]) - 1, len(s["landmark_offsets"]) - 1
    reg = OR.register_frame(*(s[k] for k in keys), new_descriptors, new_bearings, view_matches, arrsac_cfg, rng, cfg=register_cfg, tri=tri)
    out = dict(status=None, register=reg, constraints=None, recon=None, snapshot=None, view_map=np.full(V, NONE, np.uint32),
               landmark_map=np.full(Lm, NONE, np.uint32), new_view=None)
    if reg["status"] == "panic":
        out["status"] = "register_panic"
        return out
    if reg["status"] != "ok":
        out.update(status="not_registered", snapshot={k: (None if s.get(k) is None else np.array(s[k], copy=True)) for k in
                                                      keys + ("colors", "constraints")},
                   view_map=np.arange(V, dtype=np.uint32), landmark_map=np.arange(Lm, dtype=np.uint32))
        return out
    R, t = reg["pose"]
    a = add_view(s, np.concatenate([R.reshape(9), t]), new_bearings, reg["matches"], new_descriptors, new_colors)
    assert a is not None
    cons_in = np.ascontiguousarray(s.get("constraints") if s.get("constraints") is not None else np.zeros(0, CONSTRAINT_DTYPE),
                                   CONSTRAINT_DTYPE).reshape(-1)
    cr = OC.view_constraints(a["poses"], a["view_offsets"], a["view_landmarks"], a["bearings"], a["landmark_offsets"], a["observations"],
                             [V], cfg=constraints_cfg, tri=tri)
    out["constraints"] = cr
    if not cr["results"][0]["accepted"]:
        e = remove_new_view(a)
        out["status"] = "rejected"
    else:
        allc = np.concatenate([cons_in, np.asarray(cr["constraints"][0], CONSTRAINT_DTYPE).reshape(-1)])
        a["constraints"] = allc
        rr = OREC.optimize_reconstruction(a["poses"], a["view_offsets"], a["bearings"], a["landmark_offsets"], a["observations"], allc,
                                          cfg=recon_cfg, tri=tri)
        out["recon"] = rr
        st = int(rr["result"]["status"])
        if st != OREC_KEPT:
            out["status"] = {1: "removed_constraints", 2: "removed_filter", 3: "recon_panic"}[st]
            return out
        e = apply_optimization(a, rr["poses"], rr["view_state"], rr["obs_state"])
        out["status"] = "kept"
    nv = int(e["view_map"][V])
    vmap, lmap = e.pop("view_map"), e.pop("landmark_map")
    out.update(snapshot=e, view_map=vmap[:V].copy(), landmark_map=_compose(a["landmark_map"], lmap), new_view=None if nv == NONE else nv)
    return out


OREC_KEPT = 0
