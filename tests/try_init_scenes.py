"""Inputs of cv-sfm's reconstruction creation (include/cvb200_try_init.h): frame stores in cvb_frame_features_batch_dev's layout and
match lists of the shape init_reconstruction returns (one-to-one per view, first_matches / second_matches without the common centers),
and an init scene whose features carry one descriptor per world point, so that symmetric matching finds the scene's correspondences."""
import numpy as np

from tests.init_scenes import init_scene


def random_lists(rng, nc, n1, n2, k, k1, k2):
    """combined [k, 3], first_matches [k1, 2], second_matches [k2, 2]: distinct centers per view, the common centers in neither list"""
    k = min(k, nc, n1, n2)
    centers = rng.permutation(nc)
    common, rest = centers[:k], centers[k:]
    k1, k2 = min(k1, len(rest), n1 - k), min(k2, len(rest), n2 - k)
    c1, c2 = rng.permutation(rest)[:k1], rng.permutation(rest)[:k2]
    f, s = rng.permutation(n1)[:k + k1], rng.permutation(n2)[:k + k2]
    comb = np.stack([common, f[:k], s[:k]], 1).astype(np.uint32).reshape(-1, 3)
    return comb, np.stack([c1, f[k:]], 1).astype(np.uint32).reshape(-1, 2), np.stack([c2, s[k:]], 1).astype(np.uint32).reshape(-1, 2)


def frame_store(rng, counts, cap, colors=True):
    """host frame store: random descriptors, unit bearings and colours in each frame's first counts[b] rows (the rest zero)"""
    frames = len(counts)
    d = np.zeros((frames, cap, 64), np.uint8)
    b = np.zeros((frames, cap, 3))
    c = np.zeros((frames, cap, 3), np.uint8)
    for g, n in enumerate(counts):
        d[g, :n] = rng.integers(0, 256, (n, 64))
        v = rng.normal(size=(n, 3))
        b[g, :n] = v / np.linalg.norm(v, axis=1, keepdims=True)
        c[g, :n] = rng.integers(0, 256, (n, 3))
    return dict(descriptors=d, counts=np.asarray(counts, np.int32), bearings=b, colors=c if colors else None)


def descriptor_scene(rng, F, n_points=600, cap=1024, noise=0.0, outliers=0.0, seen=None, cluster=0):
    """init_scene plus a frame store: every feature gets its world point's descriptor (so symmetric matching pairs exactly the features
    of one point) and a colour; option f sees its `seen[f]` points (default: a random 80 %), the center sees all."""
    sc = init_scene(rng, F, n_points=n_points, cap=cap, noise=noise, outliers=outliers, cluster=cluster)
    pd = rng.integers(0, 256, (n_points, 64), dtype=np.uint8)
    pc = rng.integers(0, 256, (n_points, 3), dtype=np.uint8)
    desc = np.zeros((F + 1, cap, 64), np.uint8)
    col = np.zeros((F + 1, cap, 3), np.uint8)
    counts = np.zeros(F + 1, np.int32)
    for g in range(F + 1):
        pts = np.argsort(sc["inv"][g])          # the point of feature j of frame g
        keep = np.ones(n_points, bool)
        if g and seen is not None:
            keep = np.isin(pts, seen[g - 1])
        desc[g, :n_points] = pd[pts]
        col[g, :n_points] = pc[pts]
        # an unseen point's feature gets a descriptor of its own, so it matches nothing
        desc[g, :n_points][~keep] = rng.integers(0, 256, ((~keep).sum(), 64), dtype=np.uint8)
        counts[g] = n_points
    sc.update(store=dict(descriptors=desc, counts=counts, bearings=sc["bearings"], colors=col))
    return sc
