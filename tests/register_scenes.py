"""Synthetic reconstruction snapshots and new frames for the frame-registration tests (include/cvb200_register.h), built from seeds.

Every landmark has a random 512-bit descriptor; each of its features (in the views and in the new frame) flips a few bits of it, so a
feature's own landmark lies a few bits away and every other landmark about 256 bits away: the matching decisions have wide margins.
Bearings carry small noise (1e-5 rad by default), far inside the cosine thresholds, and the outliers of the new frame point at random
directions, far outside them, so that the decisions of the device and of the oracle agree even though their floating-point sums differ
in the last bits.  Arrays are in the layout of cvb_register_frame."""
import numpy as np

from .constraint_scenes import _rot_x, _rot_y


def _flip(rng, d, bits):
    d = d.copy()
    for b in rng.choice(512, bits, replace=False):
        d[b // 8] ^= np.uint8(1 << (b % 8))
    return d


def _bearing(R, t, p, rng, noise):
    x = R @ p + t
    b = x / np.linalg.norm(x)
    if noise:
        b = b + rng.normal(0, noise, 3)
        b /= np.linalg.norm(b)
    return b


def _pose(v, step):
    R = _rot_y(0.03 * v + 0.01 * np.sin(v)) @ _rot_x(0.01 * np.cos(0.7 * v))
    c = np.array([step * v, 0.05 * np.sin(0.5 * v), 0.05 * v * step])
    return R, -R @ c


def scene(V=8, per_view=2000, seed=0, noise=1e-5, outliers=0.0, merges=0, shared_merges=0, doubly=0, new_features=None, step=0.3,
          new_view=None, shuffle=True):
    """Returns dict(snapshot arrays, descriptors, new_descriptors, new_bearings, view_matches, true_pose (R, t), truth (landmark per
    new feature, -1 for an outlier)).  merges: points split into two landmarks over disjoint view sets (merge pairs); shared_merges:
    the same, but both landmarks also observed in one common view (the pair shares a view); doubly: new features duplicated, so two
    features claim one landmark; outliers: the fraction of new features whose bearing points at a random direction."""
    rng = np.random.default_rng(seed)
    poses = [_pose(v, step) for v in range(V)]
    span = step * V
    n_pts = int(per_view * 1.6)
    P = np.stack([rng.uniform(-4, span + 4, n_pts), rng.uniform(-3, 3, n_pts), rng.uniform(6, 14, n_pts)], 1)
    desc_pt = rng.integers(0, 256, (n_pts, 64), dtype=np.uint8)
    vis = []
    for v, (R, t) in enumerate(poses):
        x = P @ R.T + t
        ok = (x[:, 2] > 0) & (np.abs(x[:, 0] / x[:, 2]) < 0.9) & (np.abs(x[:, 1] / x[:, 2]) < 0.7)
        idx = np.where(ok)[0]
        if len(idx) > per_view:
            idx = np.sort(rng.choice(idx, per_view, replace=False))
        vis.append(idx)
    # landmark ids: one per point seen by at least one view; a merge point becomes two landmarks over disjoint halves of its views
    seen_by = [[] for _ in range(n_pts)]
    for v in range(V):
        for p in vis[v]:
            seen_by[p].append(v)
    cand = [p for p in range(n_pts) if len(seen_by[p]) >= 6]
    rng.shuffle(cand)
    split = {p: "merge" for p in cand[:merges]}
    split.update({p: "shared" for p in cand[merges:merges + shared_merges]})
    lm_of = {}          # (point, view) -> landmark
    L = 0
    lm_desc, lm_point = [], []
    extra = {}
    for p in range(n_pts):
        if not seen_by[p]:
            continue
        views = seen_by[p]
        if p in split:
            h = len(views) // 2
            for part, d in ((views[:h], desc_pt[p]), (views[h:], _flip(rng, desc_pt[p], 2))):
                for v in part:
                    lm_of[(p, v)] = L
                lm_desc.append(d); lm_point.append(p)
                L += 1
            if split[p] == "shared":      # the second landmark is also observed in the first one's first view
                extra.setdefault(views[0], []).append((p, L - 1))
        else:
            for v in views:
                lm_of[(p, v)] = L
            lm_desc.append(desc_pt[p]); lm_point.append(p)
            L += 1
    features, bearings, descs = [], [], []
    for v, (R, t) in enumerate(poses):
        items = [(p, lm_of[(p, v)]) for p in vis[v]]
        items += extra.get(v, [])
        order = rng.permutation(len(items)) if shuffle else np.arange(len(items))
        items = [items[i] for i in order]
        features.append([l for _, l in items])
        bearings.append(np.array([_bearing(R, t, P[p], rng, noise) for p, _ in items]).reshape(-1, 3))
        descs.append(np.array([_flip(rng, lm_desc[l], 3) for _, l in items], np.uint8).reshape(-1, 64))
    from .constraint_scenes import snapshot_from_lists
    poses_arr = np.array([np.concatenate([R.reshape(9), t]) for R, t in poses])
    snap = snapshot_from_lists(poses_arr, features, bearings)
    # the new frame: a pose beyond the trajectory's middle, its features the landmarks it sees
    nv = V / 2 + 0.35 if new_view is None else new_view
    Rn, tn = _pose(nv, step)
    x = P @ Rn.T + tn
    ok = (x[:, 2] > 0) & (np.abs(x[:, 0] / x[:, 2]) < 0.9) & (np.abs(x[:, 1] / x[:, 2]) < 0.7)
    pts = [p for p in np.where(ok)[0] if seen_by[p]]
    if new_features is not None and len(pts) > new_features:
        pts = list(rng.choice(pts, new_features, replace=False))
    pts = [int(p) for p in pts]
    pts += [pts[i] for i in rng.choice(len(pts), doubly, replace=False)] if doubly else []
    rng.shuffle(pts)
    nd, nb, truth = [], [], []
    n_out = int(round(outliers * len(pts)))
    out_set = set(rng.choice(len(pts), n_out, replace=False).tolist()) if n_out else set()
    for i, p in enumerate(pts):
        nd.append(_flip(rng, desc_pt[p], 3))
        if i in out_set:
            b = rng.normal(size=3); b[2] = abs(b[2]) + 0.5; b /= np.linalg.norm(b)
            nb.append(b); truth.append(-1)
        else:
            nb.append(_bearing(Rn, tn, P[p], rng, noise)); truth.append(p)
    out = dict(snap)
    out.update(descriptors=np.concatenate(descs), new_descriptors=np.array(nd, np.uint8).reshape(-1, 64),
               new_bearings=np.array(nb).reshape(-1, 3), view_matches=np.arange(V, dtype=np.uint32), true_pose=(Rn, tn),
               truth=np.array(truth), landmark_point=np.array(lm_point))
    return out


SNAP_KEYS = ("poses", "view_offsets", "view_landmarks", "bearings", "descriptors", "landmark_offsets", "observations")


def args(s):
    """the positional inputs of cv_b200.register_frame / oracle.pyoracle_register.register_frame up to view_matches"""
    return tuple(s[k] for k in SNAP_KEYS) + (s["new_descriptors"], s["new_bearings"], s["view_matches"])
