"""Large synthetic reconstruction snapshots for the scale tests of the three-view constraints and the reconstruction optimisation
(tests/test_gpu_sfm_scale.py), built with numpy in time linear in the views.

The layout is tests/constraint_scenes.scene's (cvb_view_constraints): each landmark's observations in ascending view order, the feature
order of every view shuffled, and single-observation landmarks.  The camera moves sideways along x with a bounded wobble, so that a near
point is seen by a sliding window of consecutive views; only the views of that window are tested against the point.  Far points, when
asked for, are tested against every view and are seen by all of them, which makes every pair of views covisible.

The triangulators' cheirality test takes the world-frame bearing against the point's world position, not against the point seen from
the camera (the reference's behaviour), so a point far along x from the origin fails it.  The world origin is therefore put at the middle
of the path and far enough behind the cameras (trajectory's lift) that every point of the field of view passes it."""
import numpy as np

from oracle.pyoracle_reconstruction import CONSTRAINT_DTYPE


def _rodrigues(w):
    """[n, 3] rotation vectors -> [n, 3, 3] rotations"""
    a = np.linalg.norm(w, axis=1)
    k = np.divide(w, a[:, None], out=np.zeros_like(w), where=a[:, None] > 0)
    K = np.zeros((len(w), 3, 3))
    K[:, 0, 1], K[:, 0, 2], K[:, 1, 2] = -k[:, 2], k[:, 1], -k[:, 0]
    K = K - K.transpose(0, 2, 1)
    s, c = np.sin(a)[:, None, None], np.cos(a)[:, None, None]
    return np.eye(3) + s * K + (1 - c) * K @ K


def lift(V, step=0.25, width=16.0):
    """the cameras' height above the world origin along z: (p_z)^2 above |p_x| |c_x - p_x| <= (span / 2) (width / 2) for every point p
    seen from a centre c"""
    return 2.0 * np.sqrt(step * V * width) + 1.0


def trajectory(V, step=0.25):
    """[V, 12] WorldToCamera poses: centres step apart along x around x = 0 at z = lift(V, step), yaw within +-0.05 rad, pitch within
    +-0.01 rad"""
    v = np.arange(V, dtype=np.float64)
    yaw, pitch = 0.05 * np.sin(0.3 * v), 0.01 * np.cos(0.7 * v)
    cy, sy, cp, sp = np.cos(yaw), np.sin(yaw), np.cos(pitch), np.sin(pitch)
    Ry = np.zeros((V, 3, 3))
    Ry[:, 0, 0], Ry[:, 0, 2], Ry[:, 1, 1], Ry[:, 2, 0], Ry[:, 2, 2] = cy, sy, 1.0, -sy, cy
    Rx = np.zeros((V, 3, 3))
    Rx[:, 0, 0], Rx[:, 1, 1], Rx[:, 1, 2], Rx[:, 2, 1], Rx[:, 2, 2] = 1.0, cp, -sp, sp, cp
    R = Ry @ Rx
    c = np.stack([step * (v - (V - 1) / 2), 0.05 * np.sin(0.5 * v), lift(V, step) + 0.02 * np.sin(0.1 * v)], 1)
    return np.concatenate([R.reshape(V, 9), -np.einsum("vij,vj->vi", R, c)], 1)


def _observe(poses, P, views, fov_cos):
    """bearings [n, k, 3] of points P [n, 3] in views [n, k] (-1: none) and the mask of those inside the field of view"""
    ok = views >= 0
    vv = np.where(ok, views, 0)
    R, t = poses[vv, :9].reshape(*vv.shape, 3, 3), poses[vv, 9:]
    x = np.einsum("nkij,nj->nki", R, P) + t
    b = x / np.linalg.norm(x, axis=2, keepdims=True)
    return b, ok & (b[..., 2] > fov_cos)


def sliding_scene(V, per_view=150, seed=0, noise=0.0, outliers=0.0, singles=4, far=0, fov_cos=0.8, step=0.25, depth=(3.0, 8.0)):
    """A V-view snapshot: per_view near points in the strip of x each view sees (a fraction of them falls in its field of view), `far`
    points seen by every view, `singles` single-observation landmarks per view; bearing noise (standard deviation per component) and a fraction of outlier observations (noise 0.05).  Returns
    (snapshot dict with the true poses, true poses [V, 12])."""
    rng = np.random.default_rng(seed)
    poses = trajectory(V, step)
    tan = np.sqrt(1 - fov_cos ** 2) / fov_cos
    width = 2 * depth[1] * tan                      # the widest strip of x a view sees at the far depth
    n_near = int(round(per_view * V * step / width))
    half, z0 = step * (V - 1) / 2, lift(V, step)
    P = np.stack([rng.uniform(-half - width / 2, half + width / 2, n_near), rng.uniform(-2, 2, n_near), z0 + rng.uniform(*depth, n_near)], 1)
    H = int(np.ceil((depth[1] * tan + 0.5) / step)) + 2
    first = np.rint((P[:, 0] + half) / step).astype(np.int64) - H
    views = first[:, None] + np.arange(2 * H + 1)[None, :]
    views = np.where((views >= 0) & (views < V), views, -1)
    b_near, m_near = _observe(poses, P, views, fov_cos)
    pts_v, pts_b, pts_m = [views], [b_near], [m_near]
    if far:
        Pf = np.stack([rng.uniform(-half - 20, half + 20, far), rng.uniform(-10, 10, far), z0 + rng.uniform(800, 1000, far)], 1)
        vf = np.broadcast_to(np.arange(V), (far, V))
        b_far, m_far = _observe(poses, Pf, vf, fov_cos)
        assert m_far.all(), "far points must be seen by every view"
        pts_v, pts_b, pts_m = [views, vf], [b_near, b_far], [m_near, m_far]
    lm_v, lm_b, lm_id = [], [], []
    L = 0
    for vs, bs, ms in zip(pts_v, pts_b, pts_m):
        seen = ms.any(1)
        vs, bs, ms = vs[seen], bs[seen], ms[seen]
        ids = L + np.arange(len(vs))
        L += len(vs)
        r, k = np.nonzero(ms)                       # row-major: per landmark, views ascending
        lm_v.append(vs[r, k]); lm_b.append(bs[r, k]); lm_id.append(ids[r])
    sv = np.repeat(np.arange(V), singles)           # single-observation landmarks
    sb = rng.normal(0, 0.2, (len(sv), 3)) + np.array([0, 0, 1.0])
    lm_v.append(sv); lm_b.append(sb / np.linalg.norm(sb, axis=1, keepdims=True)); lm_id.append(L + np.arange(len(sv)))
    L += len(sv)
    ov, ob, ol = np.concatenate(lm_v), np.concatenate(lm_b), np.concatenate(lm_id)
    n = len(ov)
    if noise or outliers:
        out = rng.random(n) < outliers
        ob = ob + rng.normal(0, 1, (n, 3)) * np.where(out, 0.05, noise)[:, None]
        ob = ob / np.linalg.norm(ob, axis=1, keepdims=True)
    # view CSR: features of each view in random order
    order = np.lexsort((rng.random(n), ov))
    vo = np.zeros(V + 1, np.uint32)
    np.cumsum(np.bincount(ov, minlength=V), out=vo[1:])
    feat = np.empty(n, np.int64)
    feat[order] = np.arange(n) - vo[ov[order]]
    # landmark CSR: observations of each landmark in ascending view order
    lorder = np.lexsort((ov, ol))
    lo = np.zeros(L + 1, np.uint32)
    np.cumsum(np.bincount(ol, minlength=L), out=lo[1:])
    snap = dict(poses=poses.copy(), view_offsets=vo, view_landmarks=ol[order].astype(np.uint32), bearings=ob[order].copy(),
                landmark_offsets=lo, observations=np.stack([ov[lorder], feat[lorder]], 1).astype(np.uint32))
    return snap, poses


def _mul(A, B):
    """A * B of [n, 12] isometries"""
    Ra, Rb = A[:, :9].reshape(-1, 3, 3), B[:, :9].reshape(-1, 3, 3)
    return np.concatenate([(Ra @ Rb).reshape(-1, 9), np.einsum("nij,nj->ni", Ra, B[:, 9:]) + A[:, 9:]], 1)


def _inv(A):
    Rt = A[:, :9].reshape(-1, 3, 3).transpose(0, 2, 1)
    return np.concatenate([Rt.reshape(-1, 9), -np.einsum("nij,nj->ni", Rt, A[:, 9:])], 1)


def perturbed(poses, rot, trans, seed):
    """every pose times a random isometry (rotation and translation standard deviations per component)"""
    rng = np.random.default_rng(seed)
    n = len(poses)
    D = np.concatenate([_rodrigues(rng.normal(0, rot, (n, 3))).reshape(n, 9), rng.normal(0, trans, (n, 3))], 1)
    return _mul(D, poses)


def constraints(poses, per_view=8, window=6, noise_rot=0.0, noise_trans=0.0, seed=0):
    """tests/reconstruction_scenes.constraints_for without the Python loop: up to per_view triples (v, a, b) added by each view v, a and b
    drawn from the views within `window` of v, with the true relative poses P1 P0^-1 and P2 P0^-1 (views ascending) times a small random
    isometry.  A CONSTRAINT_DTYPE array in view order."""
    rng = np.random.default_rng(seed)
    V = len(poses)
    offs = np.array([d for d in range(-window, window + 1) if d])
    pa, pb = np.triu_indices(len(offs), 1)
    A = np.arange(V)[:, None] + offs[pa][None, :]
    B = np.arange(V)[:, None] + offs[pb][None, :]
    valid = (A >= 0) & (A < V) & (B >= 0) & (B < V)
    key = np.where(valid, rng.random(valid.shape), 2.0)
    pick = np.argsort(key, axis=1, kind="stable")[:, :per_view]
    rows = np.repeat(np.arange(V), pick.shape[1])
    keep = valid[rows, pick.reshape(-1)]
    w = np.sort(np.stack([rows, A[rows, pick.reshape(-1)], B[rows, pick.reshape(-1)]], 1)[keep], axis=1)
    out = np.zeros(len(w), CONSTRAINT_DTYPE)
    out["views"] = w
    out["landmarks"] = 32
    inv0 = _inv(poses[w[:, 0]])
    for k in range(2):
        rel = _mul(poses[w[:, k + 1]], inv0)
        if noise_rot or noise_trans:
            rel = perturbed(rel, noise_rot, noise_trans, seed * 2 + k + 1)
        out["poses"][:, k]["r"] = rel[:, :9]
        out["poses"][:, k]["t"] = rel[:, 9:]
    return out
