"""Synthetic reconstruction snapshots for the three-view constraint tests (include/cvb200_constraints.h): a camera trajectory, points seen
by the views whose frustum they fall in, shuffled feature order per view, single-observation landmarks, low-parallax points and outliers.
Arrays are in the layout of cvb_view_constraints."""
import numpy as np


def _rot_y(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])


def _rot_x(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[1, 0, 0], [0, c, -s], [0, s, c]])


def snapshot_from_lists(poses, features, bearings):
    """CSR arrays from per-view feature lists: features[v] = landmark index per feature, bearings[v] = [n, 3].  Observations of each
    landmark in ascending view order."""
    V = len(features)
    vo = np.zeros(V + 1, np.uint32)
    for v in range(V):
        vo[v + 1] = vo[v] + len(features[v])
    vl = np.concatenate([np.asarray(f, np.uint32) for f in features]) if vo[-1] else np.zeros(0, np.uint32)
    bear = np.concatenate([np.asarray(b, np.float64).reshape(-1, 3) for b in bearings]) if vo[-1] else np.zeros((0, 3))
    L = int(vl.max()) + 1 if len(vl) else 0
    obs = [[] for _ in range(L)]
    for v in range(V):
        for j, l in enumerate(features[v]):
            obs[l].append((v, j))
    lo = np.zeros(L + 1, np.uint32)
    for l in range(L):
        lo[l + 1] = lo[l] + len(obs[l])
    ob = np.array([o for ol in obs for o in ol], np.uint32).reshape(-1, 2)
    return dict(poses=np.ascontiguousarray(poses, np.float64).reshape(-1, 12), view_offsets=vo, view_landmarks=vl, bearings=bear,
                landmark_offsets=lo, observations=ob)


def scene(V, points=600, seed=0, noise=0.0, outliers=0.0, singles=20, far=30, fov_cos=0.75, step=0.25, exact=False):
    """A forward-moving camera over V views: returns (snapshot dict, true poses [V, 12], world points [L, 3])."""
    rng = np.random.default_rng(seed)
    poses = np.zeros((V, 12))
    for v in range(V):
        R = _rot_y(0.02 * v + 0.01 * np.sin(v)) @ _rot_x(0.01 * np.cos(0.7 * v))
        c = np.array([step * v, 0.05 * np.sin(0.5 * v), 0.1 * v * step])
        poses[v, :9] = R.reshape(9)
        poses[v, 9:] = -R @ c
    span = step * V
    P = np.stack([rng.uniform(-2, span + 2, points), rng.uniform(-2, 2, points), rng.uniform(3, 8, points) + 0.1 * step * V / 2], 1)
    if far:
        Pf = np.stack([rng.uniform(-50, 50, far), rng.uniform(-20, 20, far), rng.uniform(800, 1000, far)], 1)
        P = np.concatenate([P, Pf])
    feats, bears = [[] for _ in range(V)], [[] for _ in range(V)]
    L = 0
    for p in P:
        seen = []
        for v in range(V):
            R, t = poses[v, :9].reshape(3, 3), poses[v, 9:]
            x = R @ p + t
            b = x / np.linalg.norm(x)
            if b[2] > fov_cos:
                seen.append((v, b))
        if not seen:
            continue
        for v, b in seen:
            if not exact:
                if outliers and rng.random() < outliers:
                    b = b + rng.normal(0, 0.05, 3)
                elif noise:
                    b = b + rng.normal(0, noise, 3)
                b = b / np.linalg.norm(b)
            feats[v].append(L)
            bears[v].append(b)
        L += 1
    for v in range(V):   # single-observation landmarks
        for _ in range(singles):
            b = rng.normal(0, 0.2, 3) + np.array([0, 0, 1.0])
            feats[v].append(L)
            bears[v].append(b / np.linalg.norm(b))
            L += 1
    for v in range(V):   # shuffled feature order
        perm = rng.permutation(len(feats[v]))
        feats[v] = [feats[v][i] for i in perm]
        bears[v] = [bears[v][i] for i in perm]
    return snapshot_from_lists(poses, feats, bears), poses, P
