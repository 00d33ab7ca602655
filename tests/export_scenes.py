"""Snapshots for the reconstruction export tests (include/cvb200_export.h): tests/constraint_scenes.py's scenes with feature colours, and
the edge cases the export and the normalisation must handle.  Arrays are in the layout of cvb_export_reconstruction."""
import numpy as np

from tests.constraint_scenes import scene, snapshot_from_lists


def colors_for(s, seed=0):
    """uint8 [n_features, 3] colours on the view CSR"""
    return np.random.default_rng(seed).integers(0, 256, (len(s["view_landmarks"]), 3), dtype=np.uint8)


def args(s):
    return (s["poses"], s["view_offsets"], s["view_landmarks"], s["bearings"], s["landmark_offsets"], s["observations"])


def _lists(s):
    vo, vl, b = s["view_offsets"], s["view_landmarks"], s["bearings"]
    return ([list(vl[vo[v]:vo[v + 1]]) for v in range(len(vo) - 1)], [b[vo[v]:vo[v + 1]] for v in range(len(vo) - 1)])


def with_empty_view(s, pose=None, singles=3):
    """s with one more view whose features are all single-observation landmarks, so that no value enters its mean distance"""
    feats, bears = _lists(s)
    L = len(s["landmark_offsets"]) - 1
    feats.append(list(range(L, L + singles)))
    bears.append(np.tile([0.0, 0.0, 1.0], (singles, 1)))
    poses = np.concatenate([s["poses"], (pose if pose is not None else s["poses"][-1])[None]])
    return snapshot_from_lists(poses, feats, bears)


def negate_landmark(s, l):
    """the bearings of landmark l negated, so that the triangulators' cheirality test fails"""
    s = {k: v.copy() for k, v in s.items()}
    lo, ob, vo = s["landmark_offsets"], s["observations"], s["view_offsets"]
    for o in range(lo[l], lo[l + 1]):
        s["bearings"][vo[ob[o, 0]] + ob[o, 1]] *= -1
    return s


def exact_scene(V, seed=5, points=120):
    """(snapshot with exact bearings and true poses, true world point of every landmark (NaN for the single-observation ones))"""
    s, true, P = scene(V, points=points, seed=seed, exact=True, singles=2, far=0)
    seen = []
    for p in P:
        x = (true[:, :9].reshape(-1, 3, 3) @ p) + true[:, 9:]
        if np.any(x[:, 2] / np.linalg.norm(x, axis=1) > 0.75):
            seen.append(p)
    L = len(s["landmark_offsets"]) - 1
    world = np.full((L, 3), np.nan)
    world[:len(seen)] = seen
    return s, world


def first_view_without_robust_landmark(V=5):
    """a snapshot whose view 0 observes only single-observation landmarks (its mean distance is NaN)"""
    s, _ = exact_scene(V)
    feats, bears = _lists(s)
    L = len(s["landmark_offsets"]) - 1
    feats = [list(range(L, L + 4))] + feats
    bears = [np.tile([0.0, 0.0, 1.0], (4, 1))] + bears
    return snapshot_from_lists(np.concatenate([s["poses"][:1], s["poses"]]), feats, bears)
