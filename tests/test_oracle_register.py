"""CPU: properties of the frame-registration oracle (oracle/ref_register.c), the reference the device is held to in
tests/test_gpu_register.py."""
import numpy as np
import pytest

from oracle import pyoracle as O
from oracle import pyoracle_register as OR

from . import register_scenes as RS


def _run(s, seed=5, **kw):
    return OR.register_frame(*RS.args(s), O.arrsac_cfg(1e-5), O.rng_xoshiro(seed), cfg=OR.RegisterCfg(**kw))


def test_own_view_recovers_its_pose_and_landmarks():
    s = RS.scene(V=6, per_view=700, seed=1, noise=0.0)
    v = 3
    vo = s["view_offsets"]
    s["new_descriptors"] = s["descriptors"][vo[v]:vo[v + 1]]
    s["new_bearings"] = s["bearings"][vo[v]:vo[v + 1]]
    r = _run(s)
    assert r["status"] == "ok"
    P = s["poses"][v]
    assert np.abs(r["pose"][0] - P[:9].reshape(3, 3)).max() < 1e-9 and np.abs(r["pose"][1] - P[9:]).max() < 1e-9
    m = r["matches"]
    assert len(m) > 0 and np.all(m["landmark_b"] == OR.NONE)
    assert np.array_equal(m["landmark_a"], s["view_landmarks"][vo[v] + m["feature"]])


def test_frame_from_a_known_pose_is_registered():
    s = RS.scene(V=6, per_view=700, seed=2, noise=0.0)
    r = _run(s)
    R, t = s["true_pose"]
    assert r["status"] == "ok"
    assert np.abs(r["pose"][0] - R).max() < 1e-8 and np.abs(r["pose"][1] - t).max() < 1e-8
    assert all(s["landmark_point"][m["landmark_a"]] == s["truth"][m["feature"]] for m in r["matches"])


@pytest.mark.parametrize("status,kw,scene_kw", [
    ("few_robust_landmarks", dict(single_view_minimum_landmarks=100000), dict()),
    ("few_matches", dict(single_view_minimum_robust_landmarks=100000), dict()),
    ("filter_half", dict(maximum_cosine_distance=1e-14, maximum_sine_distance=1e-14), dict(noise=1e-3)),
    ("final_half", dict(single_view_filter_loop_iterations=1, maximum_cosine_distance=1e-14, maximum_sine_distance=1e-14), dict(noise=1e-3)),
    ("final_robust_half", dict(single_view_filter_loop_iterations=0, maximum_cosine_distance=1e-14, maximum_sine_distance=1e-14),
     dict(noise=1e-3)),
    ("no_consensus", dict(), dict(outliers=1.0)),
])
def test_each_status_is_reached(status, kw, scene_kw):
    s = RS.scene(V=6, per_view=500, seed=41, **scene_kw)
    r = _run(s, **kw)
    assert r["status"] == status
    assert r["pose"] is None and len(r["matches"]) == 0


def test_panic_without_three_candidate_landmarks():
    s = RS.scene(V=6, per_view=500, seed=42)
    s["view_matches"] = np.array([], np.uint32)
    rng = O.rng_xoshiro(5)
    before = list(rng.s)
    r = OR.register_frame(*RS.args(s), O.arrsac_cfg(1e-5), rng)
    assert r["status"] == "panic" and list(rng.s) == before


def test_subsets_accumulate_the_match_list():
    s = RS.scene(V=6, per_view=800, seed=31, outliers=0.2)
    r = _run(s, single_view_initial_features=40)
    assert r["status"] == "ok" and r["stats"]["subsets"] >= 2
    # the last subset's list holds every feature matched so far: the accumulated count of a one-subset run over the same range
    end = min(40 << (int(r["stats"]["subsets"]) - 1), len(s["new_descriptors"]))
    one = _run(s, single_view_initial_features=end)
    assert one["stats"]["subsets"] == 1 and one["stats"]["matches"] == r["stats"]["matches"]


def test_matching_stage_equals_landmark_matches_ref():
    # no outliers and no noise: every claim-filtered match is consistent under the registered pose, so the final list is the whole
    # matching stage's list, merge-pair orientation included
    s = RS.scene(V=8, per_view=300, seed=7, merges=8, shared_merges=4, doubly=6, noise=0.0)
    vo, vl, lo, ob = s["view_offsets"], s["view_landmarks"], s["landmark_offsets"], s["observations"]
    views = [(s["descriptors"][vo[v]:vo[v + 1]], vl[vo[v]:vo[v + 1]]) for v in range(len(vo) - 1)]
    lv = {l: ob[lo[l]:lo[l + 1], 0].tolist() for l in range(len(lo) - 1)}
    oc = {l: int(lo[l + 1] - lo[l]) for l in range(len(lo) - 1)}
    want = O.landmark_matches_ref(s["new_descriptors"], views, 24, lv, oc)
    r = _run(s)
    assert r["stats"]["claimed"] == len(want)
    assert any(len(ls) == 2 for ls, _ in want)
    tuples = sorted((f, ls[0], ls[1] if len(ls) > 1 else OR.NONE) for ls, f in want)
    assert r["status"] == "ok"
    assert [(int(m["feature"]), int(m["landmark_a"]), int(m["landmark_b"])) for m in r["matches"]] == tuples


def test_inliers_index_the_robust_matches():
    s = RS.scene(V=6, per_view=700, seed=3, outliers=0.2)
    r = _run(s)
    inl = r["inliers"]
    assert r["status"] == "ok" and len(inl) == r["stats"]["inliers"] and r["result"]["n_inliers"] == len(inl)
    assert len(set(inl.tolist())) == len(inl) and inl.max() < r["stats"]["matches_3d"]


def test_empty_first_subset_is_refused():
    s = RS.scene(V=6, per_view=300, seed=4)
    with pytest.raises(AssertionError):
        _run(s, single_view_initial_features=0)
