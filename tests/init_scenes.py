"""Synthetic inputs of cv-sfm's three-view initialisation (include/cvb200_init.h): a center frame and F option frames observing one set
of world points, each frame's features in its own order, per option an inlier match list (center feature, option feature) and the
two-view pose with a unit translation (what init_two_view returns: scale unknown)."""
import numpy as np

from tests.geom_util import rot_from_scaled_axis, unit


def init_scene(rng, F, n_points=600, cap=1024, noise=1e-5, outliers=0.05, seen=None, cluster=0):
    """seen[f]: the point indices option f matches (default: a random 80 %); the first `cluster` points lie in a tight cone (no robust
    bearing pairs among them).  Returns dict(bearings [F + 1, cap, 3], options [1 .. F], matches [F lists], poses [F (R, t unit)],
    true_t [F], points)."""
    X = np.stack([rng.uniform(-3, 3, n_points), rng.uniform(-2, 2, n_points), rng.uniform(4, 10, n_points)], 1)
    if cluster:
        X[:cluster] = np.array([0.5, 0.2, 6.0]) + rng.normal(0, 0.05, (cluster, 3))
    poses = []
    true_t = []
    for f in range(F):
        R = rot_from_scaled_axis(rng.uniform(-1, 1, 3) * 0.1)
        t = np.array([rng.uniform(-1.0, 1.0), rng.uniform(-0.3, 0.3), rng.uniform(-0.2, 0.2)])
        t *= rng.uniform(0.4, 1.2) / np.linalg.norm(t)
        poses.append((R, t / np.linalg.norm(t)))
        true_t.append(t)
    bear = np.zeros((F + 1, cap, 3))
    perms = [rng.permutation(n_points) for _ in range(F + 1)]
    inv = [np.argsort(p) for p in perms]        # feature index of point k in frame g: inv[g][k]
    for g in range(F + 1):
        Xg = X if g == 0 else X @ poses[g - 1][0].T + true_t[g - 1]
        b = unit(Xg)
        if noise:
            b = unit(b + rng.normal(0, noise, b.shape))
        bear[g, :n_points] = b[perms[g]]
    matches = []
    for f in range(F):
        pts = np.asarray(seen[f]) if seen is not None else np.sort(rng.choice(n_points, int(0.8 * n_points), replace=False))
        m = np.stack([inv[0][pts], inv[f + 1][pts]], 1)
        nout = int(outliers * len(m))
        if nout:
            rows = rng.choice(len(m), nout, replace=False)
            m[rows, 1] = rng.integers(0, n_points, nout)
            # keep one match per option feature (symmetric matching) by dropping duplicates
            _, first = np.unique(m[:, 1], return_index=True)
            m = m[np.sort(first)]
        matches.append(m)
    return dict(bearings=bear, options=list(range(1, F + 1)), matches=matches, poses=poses, true_t=true_t, points=X, inv=inv)
