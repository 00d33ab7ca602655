"""Synthetic reconstructions with three-view constraints for the reconstruction optimisation tests (include/cvb200_reconstruction.h):
tests/constraint_scenes.py's camera trajectory and landmarks, constraints built from the true relative poses (plus noise) over nearby
view triples, and poses perturbed from the truth.  Arrays are in the layout of cvb_optimize_reconstruction."""
import numpy as np

from oracle.pyoracle_reconstruction import CONSTRAINT_DTYPE
from tests.constraint_scenes import scene


def _rot(w):
    a = np.linalg.norm(w)
    if a == 0:
        return np.eye(3)
    k = w / a
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(a) * K + (1 - np.cos(a)) * K @ K


def mul(A, B):
    """A * B of [12] isometries (rotation row-major, translation)"""
    Ra, Rb = A[:9].reshape(3, 3), B[:9].reshape(3, 3)
    return np.concatenate([(Ra @ Rb).reshape(9), Ra @ B[9:] + A[9:]])


def inv(A):
    R = A[:9].reshape(3, 3)
    return np.concatenate([R.T.reshape(9), -R.T @ A[9:]])


def perturb(P, rot, trans, rng):
    return mul(np.concatenate([_rot(rng.normal(0, rot, 3)).reshape(9), rng.normal(0, trans, 3)]), P)


def constraints_for(poses, per_view=8, window=6, noise_rot=0.0, noise_trans=0.0, seed=0):
    """Up to per_view constraints added by each view v: triples (v, a, b) of views within `window` of v, poses P1 P0^-1 and P2 P0^-1 of
    the true poses (views ascending) times a small random isometry.  Returns a CONSTRAINT_DTYPE array in view order."""
    rng = np.random.default_rng(seed)
    V = len(poses)
    out = []
    for v in range(V):
        near = [u for u in range(max(0, v - window), min(V, v + window + 1)) if u != v]
        pairs = [(a, b) for i, a in enumerate(near) for b in near[i + 1:]]
        rng.shuffle(pairs)
        for a, b in pairs[:per_view]:
            w = sorted([v, a, b])
            c = np.zeros(1, CONSTRAINT_DTYPE)
            c["views"] = w
            c["landmarks"] = 32
            for k in range(2):
                rel = mul(poses[w[k + 1]], inv(poses[w[0]]))
                if noise_rot or noise_trans:
                    rel = perturb(rel, noise_rot, noise_trans, rng)
                c["poses"][0, k]["r"] = rel[:9]
                c["poses"][0, k]["t"] = rel[9:]
            out.append(c)
    return np.concatenate(out) if out else np.zeros(0, CONSTRAINT_DTYPE)


def recon_scene(V, points=400, seed=0, noise=1e-4, per_view=8, window=6, noise_rot=1e-4, noise_trans=1e-4, pose_rot=2e-3, pose_trans=2e-3,
                singles=4, far=10):
    """(snapshot dict with perturbed poses, true poses [V, 12], constraints)"""
    rng = np.random.default_rng(seed + 1)
    s, true, _ = scene(V, points=points, seed=seed, noise=noise, singles=singles, far=far)
    s["poses"] = np.stack([perturb(p, pose_rot, pose_trans, rng) for p in true]) if (pose_rot or pose_trans) else true.copy()
    return s, true, constraints_for(true, per_view=per_view, window=window, noise_rot=noise_rot, noise_trans=noise_trans, seed=seed)


def args(s):
    return (s["poses"], s["view_offsets"], s["bearings"], s["landmark_offsets"], s["observations"])


def triples(poses, views, bad=(), inf_first=False):
    """Exact constraints over the given view triples (each sorted); those whose index is in `bad` get an infinite translation in their
    second pose (or first, with inf_first), as optimize_three_view's unguarded rescale can leave them."""
    out = np.zeros(len(views), CONSTRAINT_DTYPE)
    for i, w in enumerate(views):
        w = sorted(w)
        out[i]["views"] = w
        for k in range(2):
            rel = mul(poses[w[k + 1]], inv(poses[w[0]]))
            out[i]["poses"][k]["r"] = rel[:9]
            out[i]["poses"][k]["t"] = rel[9:]
        if i in bad:
            out[i]["poses"][0 if inf_first else 1]["t"][0] = np.inf
    return out


def small_scene(V, seed=5, **kw):
    """A V-view snapshot (exact bearings) and its true poses"""
    s, true, _ = scene(V, points=kw.pop("points", 120), seed=seed, exact=True, singles=2, far=0, **kw)
    return s, true


def py_pose_inverse(P):
    """pose_inverse in plain float arithmetic (bit for bit the C restatements)"""
    R = [P[3 * c + r] for r in range(3) for c in range(3)]
    nt = [-P[9], -P[10], -P[11]]
    return R + [R[3 * r] * nt[0] + R[3 * r + 1] * nt[1] + R[3 * r + 2] * nt[2] for r in range(3)]


def py_pose_mul(A, B):
    R = [A[3 * i] * B[c] + A[3 * i + 1] * B[3 + c] + A[3 * i + 2] * B[6 + c] for i in range(3) for c in range(3)]
    return R + [A[9 + i] + (A[3 * i] * B[9] + A[3 * i + 1] * B[10] + A[3 * i + 2] * B[11]) for i in range(3)]


def rot_log(m):
    """the header's scaled_axis restatement in numpy"""
    angle = np.arccos((m[0] + m[4] + m[8] - 1.0) / 2.0)
    a = np.array([m[7] - m[5], m[2] - m[6], m[3] - m[1]])
    n = np.linalg.norm(a)
    return a / n * angle if n > np.finfo(float).eps else np.zeros(3)


def view_delta_rotation_sum(poses, cons, v):
    """sum over view v's edges of the rotation part of se3(T_e P_other P_v^-1), rate 1 (the flattened edges of every constraint)"""
    order = {0: [(2, lambda f, s: inv(s)), (1, lambda f, s: inv(f))], 1: [(0, lambda f, s: f), (2, lambda f, s: inv(mul(s, inv(f))))],
             2: [(1, lambda f, s: mul(s, inv(f))), (0, lambda f, s: s)]}
    tot = np.zeros(3)
    for c in cons:
        w = [int(x) for x in c["views"]]
        if v not in w:
            continue
        f = np.concatenate([c["poses"][0]["r"], c["poses"][0]["t"]])
        s = np.concatenate([c["poses"][1]["r"], c["poses"][1]["t"]])
        for o, T in order[w.index(v)]:
            tot += rot_log(mul(mul(T(f, s), poses[w[o]]), inv(poses[v]))[:9])
    return tot


# Edge cases shared by the oracle's property tests and the device tests: name -> () -> (snapshot, constraints, cfg keywords)
def _no_edges():
    s, true = small_scene(4)
    s["poses"] = true
    return s, triples(true, [(0, 1, 2)]), dict(optimization_iterations=4, minimum_robust_landmarks=0)


def _two_updated():
    s, true = small_scene(5)
    return s, triples(true, [(0, 1, 2), (2, 3, 4)], bad={1}), dict(optimization_iterations=4, minimum_robust_landmarks=0)


def _panic(iterations, rounds=1):
    def build():
        s, true = small_scene(6)
        return s, triples(true, [(0, 1, 2), (2, 3, 4), (0, 1, 5)], bad={1}), dict(
            optimization_iterations=iterations, reconstruction_optimization_iterations=rounds, minimum_robust_landmarks=0)
    return build


def _exp_branch(side):
    def build():
        s, true = small_scene(3)
        rng = np.random.default_rng(9)
        s["poses"] = np.stack([perturb(p, 1e-3, 1e-3, rng) for p in true])
        cons = triples(true, [(0, 1, 2)])
        S = view_delta_rotation_sum(s["poses"], cons, 0)
        rate = np.sqrt(np.finfo(float).eps * (1.0 + side * 1e-6)) / np.linalg.norm(S)
        return s, cons, dict(optimization_iterations=1, graph_optimization_rate=rate, minimum_robust_landmarks=0)
    return build


def _empty(V, iterations):
    def build():
        s, true = small_scene(V)
        return s, np.zeros(0, CONSTRAINT_DTYPE), dict(optimization_iterations=iterations, minimum_robust_landmarks=0)
    return build


def _negated_landmark():
    """iterations 0; the bearings of the first landmark of 3+ observations negated, so that it no longer triangulates"""
    s, true = small_scene(5)
    s["poses"] = true
    lo, ob, vo = s["landmark_offsets"], s["observations"], s["view_offsets"]
    l = next(i for i in range(len(lo) - 1) if lo[i + 1] - lo[i] >= 3)
    for o in range(lo[l], lo[l + 1]):
        s["bearings"][vo[ob[o, 0]] + ob[o, 1]] *= -1
    s["negated"] = l
    return s, triples(true, [(0, 1, 2), (2, 3, 4)]), dict(optimization_iterations=0, minimum_robust_landmarks=0)


def _all_inconsistent():
    s, true = small_scene(5)
    s["poses"] = true
    return s, triples(true, [(0, 1, 2)]), dict(optimization_iterations=0, maximum_cosine_distance=-1.0, minimum_robust_landmarks=0)


def _fixed_point():
    s, true = small_scene(6)
    s["poses"] = true
    return s, triples(true, [(0, 1, 2), (1, 2, 3), (2, 3, 4), (3, 4, 5), (0, 2, 4), (1, 3, 5)]), dict(minimum_robust_landmarks=0)


def _converge():
    s, true, cons = recon_scene(12, points=200, noise=0.0, per_view=6, window=4, noise_rot=0.0, noise_trans=0.0)
    return s, cons, dict(minimum_robust_landmarks=0)


CASES = {"no_edges": _no_edges, "two_updated": _two_updated, "panic": _panic(4), "panic_on_last_step": _panic(1),
         "two_rounds": _panic(1, rounds=2), "exp_below": _exp_branch(-1), "exp_above": _exp_branch(1), "empty": _empty(4, 1),
         "empty_filter_only": _empty(4, 0), "two_views": _empty(2, 1), "two_views_filter_only": _empty(2, 0),
         "negated_landmark": _negated_landmark, "all_inconsistent": _all_inconsistent, "fixed_point": _fixed_point, "converge": _converge}
