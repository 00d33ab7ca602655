"""ctypes binding of the CPU oracle of include/cvb200_merge.h (oracle/ref_merge.c in oracle/_build/libcvb_oracle_merge.so, built by
oracle/merge.mk): incorporate_reconstruction's move restated on a slot map; incorporate_reconstruction as that move followed by the
constraints oracle called one view at a time, with remove_view between the calls (the reference's loop, not the device's speculation);
and try_merge_reconstructions + optimize_reconstruction as the composition of the register, incorporate, constraints and reconstruction
oracles.

TEST INFRASTRUCTURE ONLY, like oracle/pyoracle.py.  Snapshots are dicts with the keys of cv_b200.incorporate.SNAP_KEYS (host arrays)."""
import ctypes as C
import os
import subprocess

import numpy as np

from . import pyoracle_constraints as OC
from . import pyoracle_incorporate as OI
from . import pyoracle_reconstruction as OREC
from . import pyoracle_register as OR

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "libcvb_oracle_merge.so")

NONE = 0xFFFFFFFF
CONSTRAINT_DTYPE = OC.CONSTRAINT_DTYPE
COUNTS_DTYPE = OI.COUNTS_DTYPE
_L = None


def build(force=False):
    srcs = [os.path.join(_HERE, f) for f in ("ref_merge.c", "merge.mk")]
    if not force and os.path.exists(_LIB_PATH) and all(os.path.getmtime(_LIB_PATH) >= os.path.getmtime(s) for s in srcs):
        return _LIB_PATH
    subprocess.check_call(["make", "-s", "-C", _HERE, "-f", "merge.mk"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


def _lib():
    global _L
    if _L is None:
        build()
        L = C.CDLL(_LIB_PATH)
        vp, u32 = C.c_void_p, C.c_uint32
        L.ref_world_transform.argtypes = [vp, vp, vp]
        L.ref_move.argtypes = [u32] + [vp] * 6 + [u32, vp, vp, u32] + [vp] * 6 + [u32, u32, vp, vp] + [vp] * 11
        L.ref_move.restype = C.c_int
        _L = L
    return _L


def _ptr(a):
    return a.ctypes.data if a is not None and a.size else None


def world_transform(dest_pose, src_pose):
    """WorldToWorld::from_camera_poses(src, dest) = dest^-1 * src, as [12]"""
    d, s, o = (np.ascontiguousarray(dest_pose, np.float64).reshape(12), np.ascontiguousarray(src_pose, np.float64).reshape(12), np.zeros(12))
    _lib().ref_world_transform(d.ctypes.data, s.ctypes.data, o.ctypes.data)
    return o


def move(dest, src, wt, landmark_map, skip=NONE):
    """The move alone: the snapshot (dest's constraints kept), src_view_map, src_landmark_map (before any removal)."""
    P, vo, vl, bear, d, col, lo, ob, cons = OI._arrays(dest)
    Ps, vos, vls, bs, ds, cs, los, _, _ = OI._arrays(src)
    V, Lm, nf, no, VS, LS, nfs = len(vo) - 1, len(lo) - 1, int(vo[-1]), int(lo[-1]), len(vos) - 1, len(los) - 1, int(vos[-1])
    lm = np.ascontiguousarray(landmark_map, np.uint32).reshape(-1)
    w = np.ascontiguousarray(wt, np.float64).reshape(12)
    o = OI._out(V + VS, nf + nfs, Lm + nfs, no + nfs, 0, d is not None, col is not None)
    svm, slm = np.zeros(max(VS, 1), np.uint32), np.zeros(max(LS, 1), np.uint32)
    cnt = np.zeros(1, COUNTS_DTYPE)
    assert _lib().ref_move(V, _ptr(P), _ptr(vo), _ptr(vl), _ptr(bear), _ptr(d), _ptr(col), Lm, _ptr(lo), _ptr(ob), VS, _ptr(Ps), _ptr(vos),
                           _ptr(vls), _ptr(bs), _ptr(ds), _ptr(cs), LS, int(skip), w.ctypes.data, _ptr(lm), o["poses"].ctypes.data,
                           o["view_offsets"].ctypes.data, o["view_landmarks"].ctypes.data, o["bearings"].ctypes.data, _ptr(o["descriptors"]),
                           _ptr(o["colors"]), o["landmark_offsets"].ctypes.data, o["observations"].ctypes.data, svm.ctypes.data, slm.ctypes.data,
                           cnt.ctypes.data) == 0
    out = OI._trim(o, cnt[0])
    out["constraints"] = cons.copy()
    return out, svm[:VS].copy(), slm[:LS].copy()


def _remove_view(s, v):
    """remove_view(v) as apply_optimization's states"""
    V = len(s["view_offsets"]) - 1
    vs = np.zeros(V, np.uint8)
    vs[v] = OI.VIEW_NO_EDGES
    os_ = np.where(np.asarray(s["observations"]).reshape(-1, 2)[:, 0] == v, OI.OBS_DROPPED, OI.OBS_KEPT).astype(np.uint8)
    return OI.apply_optimization(s, s["poses"], vs, os_)


def incorporate_reconstruction(dest, src, wt, landmark_map, skip=NONE, constraints_cfg=None, tri=None):
    """The move, then record_view_constraints of each moved view in order against the snapshot as it stands, remove_view on refusal.
    Returns dict(snapshot, src_view_map, src_landmark_map, con_results [V_S] (OC.RESULT_DTYPE), refused, created)."""
    s, svm, slm = move(dest, src, wt, landmark_map, skip)
    VS, Ld = len(svm), len(dest["landmark_offsets"]) - 1
    created = len(s["landmark_offsets"]) - 1 - Ld
    res = np.zeros(VS, OC.RESULT_DTYPE)
    refused = 0
    for v in range(VS):
        if svm[v] == NONE:
            continue
        cr = OC.view_constraints(s["poses"], s["view_offsets"], s["view_landmarks"], s["bearings"], s["landmark_offsets"], s["observations"],
                                 [int(svm[v])], cfg=constraints_cfg, tri=tri)
        res[v] = cr["results"][0]
        if cr["results"][0]["accepted"]:
            s["constraints"] = np.concatenate([s["constraints"], np.asarray(cr["constraints"][0], CONSTRAINT_DTYPE).reshape(-1)])
            continue
        refused += 1
        e = _remove_view(s, int(svm[v]))
        vmap, lmap = e.pop("view_map"), e.pop("landmark_map")
        svm = OI._compose(svm, vmap)
        slm = OI._compose(slm, lmap)
        s = e
    return dict(snapshot=s, src_view_map=svm, src_landmark_map=slm, con_results=res, refused=refused, created=created)


def merge_reconstructions(dest, src, s_view, dest_view_matches, arrsac_cfg, rng, register_cfg=None, constraints_cfg=None, recon_cfg=None,
                          tri=None):
    """The oracle chain of try_merge_reconstructions followed by optimize_reconstruction.  Returns dict(status, register, constraints
    (the dest view's), move (incorporate_reconstruction's dict), recon, snapshot or None, dest_view_map, dest_landmark_map, src_view_map,
    src_landmark_map, dest_view)."""
    V, Lm = len(dest["view_offsets"]) - 1, len(dest["landmark_offsets"]) - 1
    VS, LS = len(src["view_offsets"]) - 1, len(src["landmark_offsets"]) - 1
    r0, r1 = int(src["view_offsets"][s_view]), int(src["view_offsets"][s_view + 1])
    nd, nb = np.asarray(src["descriptors"])[r0:r1], np.asarray(src["bearings"])[r0:r1]
    ncol = None if src.get("colors") is None else np.asarray(src["colors"])[r0:r1]
    keys = ("poses", "view_offsets", "view_landmarks", "bearings", "descriptors", "landmark_offsets", "observations")
    reg = OR.register_frame(*(dest[k] for k in keys), nd, nb, dest_view_matches, arrsac_cfg, rng, cfg=register_cfg, tri=tri)
    out = dict(status=None, register=reg, constraints=None, move=None, recon=None, snapshot=None, dest_view_map=np.full(V, NONE, np.uint32),
               dest_landmark_map=np.full(Lm, NONE, np.uint32), src_view_map=np.full(VS, NONE, np.uint32),
               src_landmark_map=np.full(LS, NONE, np.uint32), dest_view=None)
    if reg["status"] == "panic":
        out["status"] = "register_panic"
        return out
    if reg["status"] != "ok":
        out.update(status="not_registered", snapshot={k: (None if dest.get(k) is None else np.array(dest[k], copy=True)) for k in
                                                      keys + ("colors", "constraints")},
                   dest_view_map=np.arange(V, dtype=np.uint32), dest_landmark_map=np.arange(Lm, dtype=np.uint32))
        return out
    R, t = reg["pose"]
    dest_pose = np.concatenate([R.reshape(9), t])
    a = OI.add_view(dest, dest_pose, nb, reg["matches"], nd, ncol)
    cr = OC.view_constraints(a["poses"], a["view_offsets"], a["view_landmarks"], a["bearings"], a["landmark_offsets"], a["observations"], [V],
                             cfg=constraints_cfg, tri=tri)
    out["constraints"] = cr
    if not cr["results"][0]["accepted"]:
        e = _remove_view(a, V)
        vmap, lmap = e.pop("view_map"), e.pop("landmark_map")
        out.update(status="rejected", snapshot=e, dest_view_map=vmap[:V].copy(), dest_landmark_map=OI._compose(a["landmark_map"], lmap))
        return out
    a["constraints"] = np.concatenate([a["constraints"], np.asarray(cr["constraints"][0], CONSTRAINT_DTYPE).reshape(-1)])
    amap = a.pop("landmark_map")
    a.pop("merges")
    ltl = np.full(LS, NONE, np.uint32)
    svl = np.asarray(src["view_landmarks"])[r0:r1]
    for m in reg["matches"]:
        ltl[int(svl[int(m["feature"])])] = amap[int(m["landmark_a"])]
    wt = world_transform(dest_pose, np.asarray(src["poses"]).reshape(-1, 12)[s_view])
    mv = incorporate_reconstruction(a, src, wt, ltl, s_view, constraints_cfg, tri)
    out["move"] = mv
    f = mv["snapshot"]
    svm = mv["src_view_map"].copy()
    svm[s_view] = V
    rr = OREC.optimize_reconstruction(f["poses"], f["view_offsets"], f["bearings"], f["landmark_offsets"], f["observations"], f["constraints"],
                                      cfg=recon_cfg, tri=tri)
    out["recon"] = rr
    st = int(rr["result"]["status"])
    if st != 0:
        out["status"] = {1: "removed_constraints", 2: "removed_filter", 3: "recon_panic"}[st]
        return out
    e = OI.apply_optimization(f, rr["poses"], rr["view_state"], rr["obs_state"])
    vmap, lmap = e.pop("view_map"), e.pop("landmark_map")
    dv = int(vmap[V])
    out.update(status="merged", snapshot=e, dest_view_map=vmap[:V].copy(), dest_landmark_map=OI._compose(amap, lmap),
               src_view_map=OI._compose(svm, vmap), src_landmark_map=OI._compose(mv["src_landmark_map"], lmap),
               dest_view=None if dv == NONE else dv)
    return out
