"""Source and destination snapshots for the reconstruction-merging tests (include/cvb200_merge.h): one synthetic reconstruction of
tests/register_scenes.scene split into S (views 0 .. k, re-expressed in a world moved by a known isometry) and D (views k + 1 ..), with
s_view = k, the view both halves can see.  Built on tests/incorporate_scenes (colours, garbage constraints, sanity)."""
import numpy as np

from . import incorporate_scenes as IS
from . import register_scenes as RS

NONE = IS.NONE


def _rot(a, b, c):
    from .constraint_scenes import _rot_x, _rot_y
    return _rot_y(a) @ _rot_x(b) @ _rot_y(c)


def isometry(seed=0):
    """a world change (R, t): X' = R X + t"""
    rng = np.random.default_rng(seed)
    return _rot(*rng.uniform(-0.5, 0.5, 3)), rng.uniform(-2, 2, 3)


def subset(snap, views):
    """the snapshot of the given views (in that order) and the landmarks they observe, in index order; also the old -> new landmark map"""
    vo, vl, lo = np.asarray(snap["view_offsets"]), np.asarray(snap["view_landmarks"]), np.asarray(snap["landmark_offsets"])
    ob = np.asarray(snap["observations"]).reshape(-1, 2)
    vnew = {v: i for i, v in enumerate(views)}
    L = len(lo) - 1
    keep = [l for l in range(L) if any(int(v) in vnew for v in ob[lo[l]:lo[l + 1], 0])]
    lnew = np.full(L, NONE, np.uint32)
    lnew[keep] = np.arange(len(keep), dtype=np.uint32)
    rows = np.concatenate([np.arange(vo[v], vo[v + 1]) for v in views]).astype(np.int64)
    out = dict(poses=np.asarray(snap["poses"]).reshape(-1, 12)[list(views)].copy(),
               view_offsets=np.concatenate([[0], np.cumsum([vo[v + 1] - vo[v] for v in views])]).astype(np.uint32),
               view_landmarks=lnew[vl[rows]], bearings=np.asarray(snap["bearings"])[rows].copy(),
               descriptors=None if snap.get("descriptors") is None else np.asarray(snap["descriptors"])[rows].copy(),
               colors=None if snap.get("colors") is None else np.asarray(snap["colors"])[rows].copy())
    offs, obs = [0], []
    for l in keep:
        for v, f in ob[lo[l]:lo[l + 1]]:
            if int(v) in vnew:
                obs.append((vnew[int(v)], f))
        offs.append(len(obs))
    out.update(landmark_offsets=np.array(offs, np.uint32), observations=np.array(obs, np.uint32).reshape(-1, 2),
               constraints=np.zeros(0, IS.CONSTRAINT_DTYPE))
    return out, lnew


def moved_world(poses, iso):
    """WorldToCamera poses re-expressed in the world X' = R X + t: P' = P * iso^-1"""
    R, t = iso
    Ri, ti = R.T, -R.T @ t
    out = np.asarray(poses, np.float64).reshape(-1, 12).copy()
    for i, p in enumerate(out):
        Rp, tp = p[:9].reshape(3, 3), p[9:]
        out[i] = np.concatenate([(Rp @ Ri).reshape(9), Rp @ ti + tp])
    return out


def split(V=16, k=7, seed=0, per_view=1500, iso_seed=None, garbage=0, step=0.3, **kw):
    """dict(dest, src, s_view, iso, full, dest_lmap, src_lmap, dest_view_matches): views 0 .. k to S (moved world), k + 1 .. to D;
    garbage: random constraints given to S (never read)."""
    s = RS.scene(V=V, per_view=per_view, seed=seed, step=step, **kw)
    full = IS.snapshot(s, seed)
    full["descriptors"] = s["descriptors"]
    iso = isometry(seed if iso_seed is None else iso_seed)
    src, slmap = subset(full, list(range(k + 1)))
    src["poses"] = moved_world(src["poses"], iso)
    if garbage:
        src["constraints"] = IS.chain_constraints(k + 1, seed)[:garbage]
    dest, dlmap = subset(full, list(range(k + 1, V)))
    return dict(dest=dest, src=src, s_view=k, iso=iso, full=full, dest_lmap=dlmap, src_lmap=slmap,
                dest_view_matches=np.arange(V - k - 1, dtype=np.uint32))


def true_landmark_map(sc):
    """S landmark -> D landmark of the same original landmark (NONE when D does not observe it)"""
    out = np.full(len(sc["src"]["landmark_offsets"]) - 1, NONE, np.uint32)
    for o, n in enumerate(sc["src_lmap"]):
        if n != NONE and int(sc["dest_lmap"][o]) != NONE:
            out[int(n)] = sc["dest_lmap"][o]
    return out
