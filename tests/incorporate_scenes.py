"""Snapshots, matches and optimisation states for the frame-incorporation tests (include/cvb200_incorporate.h), built on
tests/register_scenes.scene (merge pairs, shared-view pairs and doubly claimed landmarks), plus cv-sfm's sanity_check invariant
(cv-sfm/src/lib.rs:3060-3094) checked both ways on a CSR snapshot."""
import numpy as np

from . import register_scenes as RS

NONE = 0xFFFFFFFF
MATCH_DTYPE = np.dtype([("feature", "<u4"), ("landmark_a", "<u4"), ("landmark_b", "<u4")])
CONSTRAINT_DTYPE = np.dtype([("views", "<u4", (3,)), ("landmarks", "<u4"), ("poses", [("r", "<f8", (9,)), ("t", "<f8", (3,))], (2,))])


def snapshot(s, colors_seed=None, constraints=None):
    """the incorporate snapshot of a register scene: its arrays, colours per feature, the given constraints"""
    nf = int(s["view_offsets"][-1])
    rng = np.random.default_rng(colors_seed if colors_seed is not None else 0)
    out = {k: s[k] for k in RS.SNAP_KEYS}
    out["colors"] = rng.integers(0, 256, (nf, 3), dtype=np.uint8)
    out["constraints"] = np.zeros(0, CONSTRAINT_DTYPE) if constraints is None else constraints
    return out


def chain_constraints(V, seed=0):
    """every window of three consecutive views as a constraint with random poses (the edits only move them)"""
    rng = np.random.default_rng(seed)
    c = np.zeros(max(V - 2, 0), CONSTRAINT_DTYPE)
    for i in range(len(c)):
        c[i]["views"] = (i, i + 1, i + 2)
        c[i]["landmarks"] = 30 + i
        c[i]["poses"]["r"] = rng.normal(size=(2, 9))
        c[i]["poses"]["t"] = rng.normal(size=(2, 3))
    return c


def landmark_views(s):
    lo, ob = s["landmark_offsets"], np.asarray(s["observations"]).reshape(-1, 2)
    return [set(ob[lo[l]:lo[l + 1], 0].tolist()) for l in range(len(lo) - 1)]


def random_matches(s, N, seed=0, n_match=None, merges=0):
    """register_frame-like matches of a new frame of N features: n_match features (ascending) matched to distinct landmarks, `merges`
    of them to two landmarks that share no view; no landmark in two matches"""
    rng = np.random.default_rng(seed)
    L = len(s["landmark_offsets"]) - 1
    n_match = N // 2 if n_match is None else n_match
    feats = np.sort(rng.choice(N, n_match, replace=False))
    lv = landmark_views(s)
    order = list(rng.permutation(L))
    used = set()
    out = np.zeros(n_match, MATCH_DTYPE)
    for i, f in enumerate(feats):
        a = order.pop()
        while a in used:
            a = order.pop()
        used.add(a)
        b = NONE
        if i < merges:
            for _ in range(200):
                c = int(order[int(rng.integers(len(order)))])
                if c not in used and not (lv[a] & lv[c]):
                    b = c
                    used.add(c)
                    order.remove(c)
                    break
        out[i] = (f, a, b)
    return out


def random_states(s, seed=0, removed=2, split=0.05):
    """optimize_reconstruction-like states: `removed` views removed (their observations DROPPED), a fraction of the others SPLIT, never
    every observation of a landmark"""
    rng = np.random.default_rng(seed)
    V = len(s["view_offsets"]) - 1
    lo, ob = s["landmark_offsets"], np.asarray(s["observations"]).reshape(-1, 2)
    vs = np.zeros(V, np.uint8)
    vs[rng.choice(V, removed, replace=False)] = rng.integers(1, 3, removed)
    os_ = np.where(vs[ob[:, 0]] != 0, 2, 0).astype(np.uint8)
    cand = (os_ == 0) & (rng.random(len(os_)) < split)
    os_[cand] = 1
    for l in range(len(lo) - 1):   # split_observation never splits the last observation
        seg = os_[lo[l]:lo[l + 1]]
        if len(seg) and (seg == 1).all():
            seg[-1] = 0
    return vs, os_


def sanity(s):
    """sanity_check both ways: every feature's landmark exists and lists (view, feature); every observation points back; no empty
    landmark; no landmark observes a view twice"""
    vo, vl, lo = np.asarray(s["view_offsets"]), np.asarray(s["view_landmarks"]), np.asarray(s["landmark_offsets"])
    ob = np.asarray(s["observations"]).reshape(-1, 2)
    V, L = len(vo) - 1, len(lo) - 1
    assert vo[0] == 0 and lo[0] == 0 and np.all(np.diff(vo.astype(np.int64)) >= 0) and np.all(np.diff(lo.astype(np.int64)) >= 1)
    assert vo[-1] == len(vl) and lo[-1] == len(ob)
    for l in range(L):
        views = ob[lo[l]:lo[l + 1], 0]
        assert len(set(views.tolist())) == len(views), l
        for v, f in ob[lo[l]:lo[l + 1]]:
            assert v < V and f < vo[v + 1] - vo[v] and vl[vo[v] + f] == l, (l, v, f)
    for v in range(V):
        for f in range(vo[v + 1] - vo[v]):
            l = int(vl[vo[v] + f])
            assert l < L and v in ob[lo[l]:lo[l + 1], 0], (v, f, l)
    assert len(ob) == len(vl)   # both ways: one observation per feature
    c = s.get("constraints")
    if c is not None and len(c):
        w = np.asarray(c["views"])
        assert (w < V).all() and (w[:, 0] < w[:, 1]).all() and (w[:, 1] < w[:, 2]).all()


def snap_equal(a, b, keys=("poses", "view_offsets", "view_landmarks", "bearings", "descriptors", "colors", "landmark_offsets", "observations",
                            "constraints")):
    for k in keys:
        x, y = a.get(k), b.get(k)
        assert (x is None) == (y is None), k
        if x is None:
            continue
        x, y = np.ascontiguousarray(x), np.ascontiguousarray(y)
        if k in ("view_offsets", "view_landmarks", "landmark_offsets", "observations"):
            x, y = x.astype(np.uint32), y.astype(np.uint32)
        assert x.shape == y.shape and x.tobytes() == y.tobytes(), k
