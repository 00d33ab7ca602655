"""CPU-only: properties of the oracle of include/cvb200_constraints.h (oracle/ref_constraints.c) on synthetic reconstructions
(tests/constraint_scenes.py) and hand-built covisibility groups: the fixed point at exact geometry, the unique pass's short-circuit, each
threshold at and just below its limit, stable ties, the min(3, V) rule, the acceptance rule and the take limit."""
import numpy as np

from oracle.pyoracle_constraints import ConstraintsCfg, view_constraints
from tests.constraint_scenes import scene, snapshot_from_lists


def _poses(V):
    P = np.zeros((V, 12))
    for v in range(V):
        a = 0.05 * v
        R = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
        c = np.array([0.6 * v, 0.1 * (v % 2), 0.0])
        P[v, :9] = R.reshape(9)
        P[v, 9:] = -R @ c
    return P


def _groups(V, groups, seed=0):
    """A snapshot where group (views, n) holds n landmarks seen by exactly those views, at well spread depths and directions."""
    rng = np.random.default_rng(seed)
    P = _poses(V)
    feats, bears = [[] for _ in range(V)], [[] for _ in range(V)]
    L = 0
    for views, n in groups:
        for _ in range(n):
            x = np.array([rng.uniform(-3, 3 + 0.6 * V), rng.uniform(-2, 2), rng.uniform(6, 12)])
            for v in views:
                y = P[v, :9].reshape(3, 3) @ x + P[v, 9:]
                feats[v].append(L)
                bears[v].append(y / np.linalg.norm(y))
            L += 1
    return snapshot_from_lists(P, feats, bears), P


def _views(r, i=0):
    return [list(map(int, c)) for c in r["constraints"][i]["views"]]


def test_exact_geometry_is_a_fixed_point_with_the_scale_restored():
    s, P, _ = scene(10, points=300, seed=4, exact=True, singles=0, far=0)
    r = view_constraints(**s, queries=[0, 4, 9], cfg=ConstraintsCfg(constraint_patience=300))
    assert all(len(c) for c in r["constraints"])
    for cons in r["constraints"]:
        for c in cons:
            v0, v1, v2 = c["views"]
            R0, t0 = P[v0, :9].reshape(3, 3), P[v0, 9:]
            for k, v in enumerate((v1, v2)):
                R, t = P[v, :9].reshape(3, 3), P[v, 9:]
                Rr = R @ R0.T
                np.testing.assert_allclose(c["poses"][k]["r"].reshape(3, 3), Rr, atol=1e-12)
                np.testing.assert_allclose(c["poses"][k]["t"], t - Rr @ t0, atol=1e-12)


def test_unique_pass_short_circuits_any():
    # triples by count: A = (0,1,2) 40, B = (0,1,3) 35, C = (0,2,3) 30, D = (0,1,4) 28.  any() marks only the first new view: A marks
    # 0, B marks 1, C marks 2, D marks 4, so all four are unique (A, B, C, D).  Marking all three views would leave C not unique and
    # give A, B, D, C.
    s, _ = _groups(5, [((0, 1, 2), 40), ((0, 1, 3), 35), ((0, 2, 3), 30), ((0, 1, 4), 28)])
    r = view_constraints(**s, queries=[0], cfg=ConstraintsCfg(constraint_patience=0))
    assert r["stats"][0]["unique_triples"] == 4 and r["stats"][0]["triples"] == 4
    assert _views(r) == [[0, 1, 2], [0, 1, 3], [0, 2, 3], [0, 1, 4]]
    # the unique pass stops at the take limit: with two constraints, A and B
    r = view_constraints(**s, queries=[0], cfg=ConstraintsCfg(constraint_patience=0, optimization_maximum_three_view_constraints=2))
    assert r["stats"][0]["unique_triples"] == 2 and _views(r) == [[0, 1, 2], [0, 1, 3]]


def test_ties_keep_combination_order():
    s, _ = _groups(4, [((0, 2, 3), 30), ((0, 1, 3), 30), ((0, 1, 2), 30)])
    r = view_constraints(**s, queries=[0], cfg=ConstraintsCfg(constraint_patience=0))
    assert _views(r) == [[0, 1, 2], [0, 1, 3], [0, 2, 3]]


def test_covisibility_minimum_16_and_15():
    for n, triples in ((16, 1), (15, 0)):
        s, _ = _groups(3, [((0, 1, 2), n)])
        r = view_constraints(**s, queries=[0], cfg=ConstraintsCfg(constraint_patience=0, optimization_minimum_landmarks=1))
        st = r["stats"][0]
        assert st["robust_landmarks"] == n and st["coviews"] == 2 * triples and st["triples"] == triples


def test_optimisation_minimum_24_and_23():
    for n, ok in ((24, 1), (23, 0)):
        s, _ = _groups(3, [((0, 1, 2), n)])
        r = view_constraints(**s, queries=[0], cfg=ConstraintsCfg(constraint_patience=0))
        st = r["stats"][0]
        assert st["candidates"] == 1 and st["few_landmarks"] == 1 - ok and r["results"][0]["n_constraints"] == ok


def test_bearing_pairs_3_and_2():
    # 24 landmarks: 22 in a tight cluster (no pair of them is robust in all three views) and 2 or 3 far apart from everything
    P = _poses(3)

    def snap(spread):
        rng = np.random.default_rng(1)
        X = [np.array([0.6, 0.0, 10.0]) + rng.normal(0, 1e-3, 3) for _ in range(22)] + spread
        feats, bears = [[], [], []], [[], [], []]
        for i, x in enumerate(X):
            for v in range(3):
                y = P[v, :9].reshape(3, 3) @ x + P[v, 9:]
                feats[v].append(i)
                bears[v].append(y / np.linalg.norm(y))
        return snapshot_from_lists(P, feats, bears)
    far = [np.array([-6.0, 4.0, 8.0]), np.array([8.0, -4.0, 9.0])]
    cfg = ConstraintsCfg(constraint_patience=0, optimization_robust_covisibility_minimum_landmarks=16,
                         robust_observation_incidence_minimum_cosine_distance=0.0)
    # the cluster's 22 x 2 pairs with the far points are robust too, so count what the limit sees and put the limit there
    s = snap(far)
    o = s["observations"]
    B = np.stack([s["bearings"][s["view_offsets"][v] + np.arange(24)] for v in range(3)], 1)
    cnt = sum(all(1 - B[i, v] @ B[j, v] > 1e-2 for v in range(3)) for i in range(24) for j in range(i + 1, 24))
    assert cnt > 0 and len(o) == 72
    for need, ok in ((cnt, 1), (cnt + 1, 0)):
        cfg.robust_view_num_robust_bearing_pair = need
        r = view_constraints(**s, queries=[0], cfg=cfg)
        assert r["stats"][0]["few_bearing_pairs"] == 1 - ok and r["results"][0]["n_constraints"] == ok
    # and at cv-sfm's default of 3: the cluster alone has no robust pair, one far point gives 22, so the default limit passes with any
    cfg.robust_view_num_robust_bearing_pair = 3
    r = view_constraints(**snap([]), queries=[0], cfg=ConstraintsCfg(constraint_patience=0, optimization_minimum_landmarks=22,
                                                                        robust_observation_incidence_minimum_cosine_distance=0.0))
    assert r["stats"][0]["few_bearing_pairs"] == 1 and r["results"][0]["n_constraints"] == 0


def test_small_reconstructions_min_observations_and_acceptance():
    # V = 1: nothing to pair with; n = 0 and n + 1 < V fails, so the view is accepted
    s, _ = _groups(1, [((0,), 30)])
    r = view_constraints(**s, queries=[0], cfg=ConstraintsCfg(constraint_patience=0))
    assert r["results"][0]["n_constraints"] == 0 and r["results"][0]["accepted"] == 1
    # V = 2: min(3, 2) = 2 observations make a landmark robust; no triple, so n = 0 < 4 and 1 < 2: rejected
    s, _ = _groups(2, [((0, 1), 30)])
    r = view_constraints(**s, queries=[0, 1], cfg=ConstraintsCfg(constraint_patience=0))
    assert list(r["stats"]["robust_landmarks"]) == [30, 30] and list(r["results"]["accepted"]) == [0, 0]
    # V = 3: two observations are no longer enough; one triple: n = 1 < 4 and 2 < 3: rejected
    s, _ = _groups(3, [((0, 1), 30), ((0, 1, 2), 30)])
    r = view_constraints(**s, queries=[0], cfg=ConstraintsCfg(constraint_patience=0))
    assert r["stats"][0]["robust_landmarks"] == 30 and r["results"][0]["n_constraints"] == 1 and r["results"][0]["accepted"] == 0
    # with optimization_minimum_new_constraints = 1 the same view is accepted
    r = view_constraints(**s, queries=[0], cfg=ConstraintsCfg(constraint_patience=0, optimization_minimum_new_constraints=1))
    assert r["results"][0]["accepted"] == 1


def test_take_limit_and_padding_after_the_unique_triples():
    s, _, _ = scene(20, points=600, seed=3, noise=1e-4)
    r = view_constraints(**s, queries=[0, 10], cfg=ConstraintsCfg(constraint_patience=0))
    for i in range(2):
        st = r["stats"][i]
        assert st["triples"] > 64 and st["unique_triples"] < 64
        assert r["results"][i]["n_constraints"] == 64 and st["candidates"] >= 64
        assert r["results"][i]["accepted"] == 1
        # every triple holds the query and is distinct
        vs = [tuple(v) for v in r["constraints"][i]["views"]]
        q = [0, 10][i]
        assert len(set(vs)) == 64 and all(q in v and list(v) == sorted(v) for v in vs)
