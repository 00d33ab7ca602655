"""CPU-only: the oracle of include/cvb200_incorporate.h (oracle/ref_incorporate.c) -- add_view with merge_landmarks and the replay of
optimize_reconstruction's edits keep cv-sfm's sanity_check invariant both ways and pass the snapshot validators, and each edit does what
the reference's remove_view / split_observation / merge_landmarks do to the landmarks it touches."""
import numpy as np

from cv_b200.constraints import check_snapshot
from cv_b200.incorporate import check_incorporate
from oracle import pyoracle_incorporate as OI

from . import incorporate_scenes as IS
from . import register_scenes as RS


def _scene(V=6, seed=3, **kw):
    s = RS.scene(V=V, per_view=300, seed=seed, **kw)
    return IS.snapshot(s, seed, IS.chain_constraints(V, seed)), s


def _valid(s):
    IS.sanity(s)
    assert check_snapshot(s["view_offsets"], s["view_landmarks"], s["landmark_offsets"], s["observations"], []) == 0
    assert check_incorporate(s) == 0


def _pose(s):
    R, t = s["true_pose"]
    return np.concatenate([R.reshape(9), t])


def test_add_view_without_matches_appends_singletons():
    snap, s = _scene()
    N = 40
    a = OI.add_view(snap, _pose(s), s["new_bearings"][:N], np.zeros(0, OI.MATCH_DTYPE), s["new_descriptors"][:N], np.zeros((N, 3), np.uint8))
    _valid(a)
    L = len(snap["landmark_offsets"]) - 1
    assert len(a["landmark_offsets"]) - 1 == L + N and a["merges"] == 0
    assert np.array_equal(a["landmark_map"], np.arange(L))
    assert np.array_equal(a["view_landmarks"][-N:], L + np.arange(N))
    assert np.array_equal(a["observations"][-N:], np.stack([np.full(N, len(snap["view_offsets"]) - 1), np.arange(N)], 1))
    IS.snap_equal(dict(a, observations=a["observations"][:-N], landmark_offsets=a["landmark_offsets"][:-N], poses=a["poses"][:-1],
                       view_offsets=a["view_offsets"][:-1], view_landmarks=a["view_landmarks"][:-N], bearings=a["bearings"][:-N],
                       descriptors=a["descriptors"][:-N], colors=a["colors"][:-N]), snap)


def test_merge_removes_b_and_repoints_its_features():
    snap, s = _scene(merges=20)
    N = len(s["new_bearings"])
    m = IS.random_matches(snap, N, seed=1, n_match=N // 2, merges=10)
    k = int((m["landmark_b"] != IS.NONE).sum())
    assert k >= 5
    a = OI.add_view(snap, _pose(s), s["new_bearings"], m, s["new_descriptors"], np.zeros((N, 3), np.uint8))
    _valid(a)
    L = len(snap["landmark_offsets"]) - 1
    assert a["merges"] == k and len(a["landmark_offsets"]) - 1 == L - k + (N - len(m))
    lo, vl, vo = snap["landmark_offsets"], snap["view_landmarks"], snap["view_offsets"]
    for t in m[m["landmark_b"] != IS.NONE]:
        na = a["landmark_map"][t["landmark_a"]]
        assert a["landmark_map"][t["landmark_b"]] == na
        obs_a, obs_b = snap["observations"][lo[t["landmark_a"]]:lo[t["landmark_a"] + 1]], snap["observations"][lo[t["landmark_b"]]:lo[t["landmark_b"] + 1]]
        want = np.concatenate([obs_a, obs_b, [[len(vo) - 1, t["feature"]]]])
        assert np.array_equal(a["observations"][a["landmark_offsets"][na]:a["landmark_offsets"][na + 1]], want)
        for v, f in obs_b:
            assert a["view_landmarks"][vo[v] + f] == na and vl[vo[v] + f] == t["landmark_b"]


def test_add_view_refuses_a_pair_that_shares_a_view():
    snap, s = _scene()
    lo, ob = snap["landmark_offsets"], snap["observations"]
    v0 = ob[lo[0], 0]
    b = next(l for l in range(1, len(lo) - 1) if v0 in ob[lo[l]:lo[l + 1], 0])
    m = np.array([(0, 0, b)], OI.MATCH_DTYPE)
    assert OI.add_view(snap, _pose(s), s["new_bearings"], m) is None
    assert check_incorporate(snap, len(s["new_bearings"]), m) != 0


def test_rejection_keeps_the_merges_and_drops_only_the_new_singletons():
    snap, s = _scene(merges=20)
    N = len(s["new_bearings"])
    m = IS.random_matches(snap, N, seed=2, merges=8)
    a = OI.add_view(snap, _pose(s), s["new_bearings"], m, s["new_descriptors"], np.zeros((N, 3), np.uint8))
    r = OI.remove_new_view(a)
    _valid(r)
    V, L = len(snap["view_offsets"]) - 1, len(snap["landmark_offsets"]) - 1
    assert a["merges"] > 0 and len(r["view_offsets"]) - 1 == V and len(r["landmark_offsets"]) - 1 == L - a["merges"]
    # the old views' rows are the input's, with b's features naming a
    assert np.array_equal(r["bearings"], snap["bearings"]) and np.array_equal(r["colors"], snap["colors"])
    lmap = a["landmark_map"]
    assert np.array_equal(r["view_landmarks"], r["landmark_map"][lmap[snap["view_landmarks"]]])
    assert len(r["constraints"]) == len(snap["constraints"])


def test_apply_all_kept_is_the_identity():
    snap, s = _scene()
    V, no = len(snap["view_offsets"]) - 1, len(snap["observations"])
    r = OI.apply_optimization(snap, snap["poses"], np.zeros(V, np.uint8), np.zeros(no, np.uint8))
    IS.snap_equal(r, snap)
    assert np.array_equal(r["view_map"], np.arange(V)) and np.array_equal(r["landmark_map"], np.arange(len(snap["landmark_offsets"]) - 1))


def test_removing_a_view_drops_its_single_landmarks_and_constraints():
    # views 0..6 and a new view 7 of 20 singletons and 20 single matches; views 3 and 7 removed
    snap, s = _scene(V=7)
    N = 40
    m = IS.random_matches(snap, N, seed=6, n_match=20)
    a = OI.add_view(snap, _pose(s), s["new_bearings"][:N], m, s["new_descriptors"][:N], np.zeros((N, 3), np.uint8))
    c = np.concatenate([snap["constraints"], IS.chain_constraints(8, 1)[-1:]])
    a["constraints"] = c
    V, no = len(a["view_offsets"]) - 1, len(a["observations"])
    vs = np.zeros(V, np.uint8)
    vs[[3, 7]] = 1
    os_ = np.where(np.isin(a["observations"][:, 0], [3, 7]), 2, 0).astype(np.uint8)
    assert check_incorporate(a, view_state=vs, obs_state=os_) == 0
    r = OI.apply_optimization(a, a["poses"], vs, os_)
    _valid(r)
    lo = a["landmark_offsets"]
    gone = [l for l in range(len(lo) - 1) if set(a["observations"][lo[l]:lo[l + 1], 0].tolist()) <= {3, 7}]
    assert len(gone) >= 20 and all(r["landmark_map"][l] == IS.NONE for l in gone)
    assert len(r["landmark_offsets"]) - 1 == len(lo) - 1 - len(gone)
    assert np.array_equal(r["view_map"], [0, 1, 2, IS.NONE, 3, 4, 5, IS.NONE])
    # constraints (1,2,3), (2,3,4), (3,4,5) and (5,6,7) go; (0,1,2) and (4,5,6) stay, renumbered
    assert r["constraints"]["views"].tolist() == [[0, 1, 2], [3, 4, 5]]
    assert np.array_equal(r["poses"], np.delete(a["poses"], [3, 7], 0))


def test_a_split_observation_becomes_a_singleton():
    snap, s = _scene()
    V, no = len(snap["view_offsets"]) - 1, len(snap["observations"])
    lo = snap["landmark_offsets"]
    l = int(np.argmax(np.diff(lo) >= 3))
    os_ = np.zeros(no, np.uint8)
    os_[lo[l] + 1] = 1
    r = OI.apply_optimization(snap, snap["poses"], np.zeros(V, np.uint8), os_)
    _valid(r)
    L = len(lo) - 1
    assert len(r["landmark_offsets"]) - 1 == L + 1
    v, f = snap["observations"][lo[l] + 1]
    assert np.array_equal(r["observations"][r["landmark_offsets"][L]:], [[v, f]])
    assert r["view_landmarks"][snap["view_offsets"][v] + f] == L
    nl = r["landmark_map"][l]
    assert np.array_equal(r["observations"][r["landmark_offsets"][nl]:r["landmark_offsets"][nl + 1]],
                          np.delete(snap["observations"][lo[l]:lo[l + 1]], 1, 0))


def test_random_edits_keep_the_invariant():
    snap, s = _scene(V=8, seed=9, merges=20, shared_merges=5)
    N = len(s["new_bearings"])
    a = OI.add_view(snap, _pose(s), s["new_bearings"], IS.random_matches(snap, N, seed=4, merges=12), s["new_descriptors"],
                    np.zeros((N, 3), np.uint8))
    _valid(a)
    for seed in range(3):
        vs, os_ = IS.random_states(a, seed=seed, removed=2, split=0.1)
        assert check_incorporate(a, view_state=vs, obs_state=os_) == 0
        _valid(OI.apply_optimization(a, a["poses"], vs, os_))


def test_check_refuses_broken_preconditions():
    snap, s = _scene(merges=10)
    N = len(s["new_bearings"])
    m = IS.random_matches(snap, N, seed=5, merges=3)
    assert check_incorporate(snap, N, m) == 0
    L = len(snap["landmark_offsets"]) - 1
    bad = []
    x = m.copy(); x[[0, 1]] = x[[1, 0]]; bad.append(x)                                        # features not ascending
    x = m.copy(); x[-1]["feature"] = N; bad.append(x)                                          # feature >= N
    x = m.copy(); x[0]["landmark_a"] = L; bad.append(x)                                        # a >= L
    x = m.copy(); x[0]["landmark_b"] = x[0]["landmark_a"]; bad.append(x)                       # a == b
    x = m.copy(); x[1]["landmark_a"] = x[0]["landmark_a"]; bad.append(x)                       # a landmark in two matches
    x = m.copy(); x[5]["landmark_a"] = m[0]["landmark_b"]; bad.append(x)                       # ... as a and as b
    for x in bad:
        assert check_incorporate(snap, N, x) != 0
    V, no = len(snap["view_offsets"]) - 1, len(snap["observations"])
    vs, os_ = np.zeros(V, np.uint8), np.zeros(no, np.uint8)
    assert check_incorporate(snap, view_state=vs, obs_state=os_) == 0
    assert check_incorporate(snap, view_state=vs[:-1], obs_state=os_) != 0                      # wrong lengths
    assert check_incorporate(snap, view_state=vs, obs_state=os_[:-1]) != 0
    assert check_incorporate(snap, view_state=np.full(V, 3, np.uint8), obs_state=np.full(no, 2, np.uint8)) != 0   # out of range
    assert check_incorporate(snap, view_state=vs, obs_state=np.full(no, 3, np.uint8)) != 0
    o2 = os_.copy(); o2[0] = 2
    assert check_incorporate(snap, view_state=vs, obs_state=o2) != 0                            # DROPPED in a kept view
    v2 = vs.copy(); v2[0] = 1
    assert check_incorporate(snap, view_state=v2, obs_state=os_) != 0                           # kept observation of a removed view
    lo = snap["landmark_offsets"]
    o3 = os_.copy(); o3[lo[0]:lo[1]] = 1
    assert check_incorporate(snap, view_state=vs, obs_state=o3) != 0                            # every observation SPLIT
    c = snap["constraints"].copy(); c[0]["views"] = (0, 0, 1)
    assert check_incorporate(dict(snap, constraints=c)) != 0                                    # bad constraints
    c = snap["constraints"].copy(); c[0]["views"] = (0, 1, V)
    assert check_incorporate(dict(snap, constraints=c)) != 0
