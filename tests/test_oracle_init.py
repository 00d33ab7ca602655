"""CPU-only: properties of the oracle of include/cvb200_init.h (oracle/ref_init.c), cv-sfm's three-view initialisation over the two-view
options (cv-sfm/src/lib.rs:986-1303), on synthetic scenes with noise and outliers."""
import numpy as np
import pytest

from oracle import pyoracle_init as OI
from oracle import pyoracle_tri as OT
from tests.init_scenes import init_scene

FAST = dict(three_view_patience=200)


def _run(sc, F=None, found=None, n_inl=None, **cfg):
    F = len(sc["options"]) if F is None else F
    pairs, npairs, model, inl, ninl, fnd = OI.options_from_matches(F, sc["bearings"].shape[1], sc["matches"][:F], sc["poses"][:F], found)
    if n_inl is not None:
        ninl = np.asarray(n_inl, np.uint32)
    return OI.init_reconstruction(sc["bearings"], 0, sc["options"][:F], pairs, npairs, model, inl, ninl, fnd, OI.InitCfg(**cfg))


def test_clean_scene_is_accepted_at_pair_zero_with_the_true_scale():
    sc = init_scene(np.random.default_rng(1), 3, noise=0.0, outliers=0.0)
    r = _run(sc, **FAST)
    res = r["result"]
    assert res["status"] == OI.ACCEPTED and res["pair"] == 0 and (res["first"], res["second"]) == (0, 1)
    t1, t2 = sc["true_t"][0], sc["true_t"][1]
    want = np.linalg.norm(t2) / np.linalg.norm(t1)
    assert abs(r["stats"][0]["median_scale"] - want) < 1e-6 * want
    assert np.allclose(res["second_pose"]["t"], t2 / np.linalg.norm(t1), atol=1e-6)
    # every true triple is in combined
    m0, m1 = sc["matches"][0], sc["matches"][1]
    common = set(m0[:, 0]) & set(m1[:, 0])
    assert len(r["combined"]) == len(common)
    assert set(r["combined"][:, 0]) == common
    assert all(s["outcome"] == OI.PAIR_NOT_EVALUATED for s in r["stats"][1:])


def test_first_pair_without_robust_bearing_pairs_makes_the_call_none():
    rng = np.random.default_rng(2)
    n = 600
    spread = np.arange(100, n)
    a, b = spread[:250], spread[250:]
    # options 0 and 1 share only the tight cluster (points 0..99); option 2 sees everything, so pair (0, 2) would be accepted
    sc = init_scene(rng, 3, n_points=n, noise=0.0, outliers=0.0, cluster=100,
                    seen=[np.r_[np.arange(100), a], np.r_[np.arange(100), b], np.arange(n)])
    r = _run(sc, **FAST)
    assert r["result"]["status"] == OI.NONE_BEARING_PAIRS and r["result"]["pair"] == 0
    assert r["stats"][0]["outcome"] == OI.PAIR_BEARING_PAIRS and r["stats"][0]["bearing_pairs"] < 3
    assert r["stats"][1]["outcome"] == OI.PAIR_NOT_EVALUATED
    # without the first pair the next one is accepted
    r2 = _run(sc, found=[1, 0, 1], **FAST)
    assert r2["result"]["status"] == OI.ACCEPTED and (r2["result"]["first"], r2["result"]["second"]) == (0, 2)


@pytest.mark.parametrize("shared,outcome", [(10, OI.PAIR_FEW_SCALES), (24, OI.PAIR_FEW_MATCHES)])
def test_small_overlaps_pass_on_to_the_next_pair(shared, outcome):
    rng = np.random.default_rng(3)
    n = 800
    a = np.arange(shared, 400)
    b = np.arange(400, n)
    sc = init_scene(rng, 3, n_points=n, noise=0.0, outliers=0.0, seen=[np.r_[np.arange(shared), a], np.r_[np.arange(shared), b], np.arange(n)])
    r = _run(sc, **FAST)
    assert r["stats"][0]["outcome"] == outcome
    assert r["result"]["status"] == OI.ACCEPTED and r["result"]["pair"] == 1


def test_at_most_half_robust_passes_on():
    sc = init_scene(np.random.default_rng(4), 3, noise=2e-3, outliers=0.0)
    seen = None
    for max_cos in (1e-7, 3e-7, 1e-6, 3e-6):
        r = _run(sc, maximum_cosine_distance=max_cos, three_view_patience=0)
        if r["stats"][0]["outcome"] == OI.PAIR_HALF_MATCHES:
            seen = r
            break
    assert seen is not None
    assert seen["stats"][1]["outcome"] != OI.PAIR_NOT_EVALUATED


def test_options_not_taking_part_are_skipped_without_shifting_the_pairs():
    sc = init_scene(np.random.default_rng(5), 4, noise=1e-5)
    counts = [len(m) for m in sc["matches"]]
    r = _run(sc, found=[1, 0, 1, 1], **FAST)
    assert r["result"]["n_pairs"] == 3 and (r["result"]["first"], r["result"]["second"]) == (0, 2)
    r = _run(sc, n_inl=[counts[0], 100, counts[2], counts[3]], **FAST)      # option 1 below the two-view minimum
    assert r["result"]["n_pairs"] == 3 and (r["result"]["first"], r["result"]["second"]) == (0, 2)
    st = r["stats"]
    assert (st[0]["first"], st[0]["second"]) == (0, 2)


def test_one_or_no_option_is_none():
    sc = init_scene(np.random.default_rng(6), 2)
    for F in (0, 1):
        r = _run(sc, F=F)
        assert r["result"]["status"] == OI.NONE and r["result"]["n_pairs"] == 0 and len(r["stats"]) == 0
    r = _run(sc, found=[1, 0])
    assert r["result"]["status"] == OI.NONE and r["result"]["n_pairs"] == 0


def test_first_and_second_lists_exclude_center_features_of_the_other_option():
    sc = init_scene(np.random.default_rng(7), 2, noise=1e-5)
    r = _run(sc, **FAST)
    assert r["result"]["status"] == OI.ACCEPTED
    c0, c1 = set(sc["matches"][0][:, 0]), set(sc["matches"][1][:, 0])
    assert len(r["first_matches"]) > 0 and len(r["second_matches"]) > 0
    assert not set(r["first_matches"][:, 0]) & c1 and not set(r["second_matches"][:, 0]) & c0
    assert set(map(tuple, r["first_matches"])) <= set(map(tuple, sc["matches"][0]))


@pytest.mark.parametrize("method", [OT.SINE_L1, OT.MEAN_MEAN])
def test_other_observation_triangulators_accept_a_clean_scene(method):
    sc = init_scene(np.random.default_rng(8), 2, noise=0.0, outliers=0.0)
    F = 2
    pairs, npairs, model, inl, ninl, fnd = OI.options_from_matches(F, sc["bearings"].shape[1], sc["matches"], sc["poses"])
    r = OI.init_reconstruction(sc["bearings"], 0, sc["options"], pairs, npairs, model, inl, ninl, fnd, OI.InitCfg(**FAST),
                               OT.triangulator(method))
    assert r["result"]["status"] == OI.ACCEPTED
