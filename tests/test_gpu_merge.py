"""GPU: cv_b200.incorporate_reconstruction / merge_reconstructions (include/cvb200_merge.h) against the oracle of oracle/pyoracle_merge.py,
whose constraint loop calls the constraints oracle one view at a time with remove_view between the calls.  The move only copies rows and
moves integers, and its poses use the same unfused FP64 formulas as the oracle, so the standalone incorporate_reconstruction is held bit
for bit.  The merge starts from register_frame's pose, which agrees with the oracle's to rounding (include/cvb200_register.h), and the
world transform carries that difference to every moved view: without optimisation steps the poses are held to 1e-12, after
optimize_reconstruction's steps over 16 to 64 views to 5e-8 (1.9e-8 was the largest difference seen); everything else -- statuses,
states, counts, the four maps, every other array of the snapshot -- must be equal."""
import numpy as np
import pytest
import torch

import cv_b200
from cv_b200._lib import CvbError
from cv_b200.incorporate import snapshot_to_device, snapshot_to_host
from cv_b200.merge import incorporate_reconstruction_dev, merge_reconstructions_dev
from oracle import pyoracle as O
from oracle import pyoracle_constraints as OC
from oracle import pyoracle_merge as OM
from oracle import pyoracle_reconstruction as OREC
from oracle import pyoracle_register as OR
from oracle.pyoracle_tri import LINEAR_EIGEN, MEAN_MEAN, SINE_L1, triangulator as o_tri

from . import incorporate_scenes as IS
from . import merge_scenes as MS

pytestmark = pytest.mark.gpu

TRIS = {LINEAR_EIGEN: cv_b200.LinearEigenTriangulator, SINE_L1: cv_b200.SineL1Triangulator, MEAN_MEAN: cv_b200.MeanMeanTriangulator}
NONPOSE = ("view_offsets", "view_landmarks", "bearings", "descriptors", "colors", "landmark_offsets", "observations")
NONE = MS.NONE


@pytest.fixture(scope="module")
def ctx():
    return cv_b200.Context(0)


def _wt(sc):
    R, t = sc["iso"]
    return np.concatenate([R.T.reshape(9), -R.T @ t])


def _scene(n, seed=3, **kw):
    return MS.split(V=2 * n, k=n - 1, seed=seed, per_view=800 if n <= 8 else 500, step=0.3 if n <= 8 else 0.1, **kw)


def _cons_equal(g, w, tol):
    assert len(g) == len(w)
    assert np.array_equal(g["views"], w["views"]) and np.array_equal(g["landmarks"], w["landmarks"])
    for x in ("r", "t"):
        d = np.abs(g["poses"][x] - w["poses"][x]).max(initial=0)
        assert d <= tol, d


# views 0, 1, 2, 4, 7 refused, 3, 5, 6 accepted; view 4's removal changes view 6's constraints and overturns view 7's speculative
# acceptance, and drops constraints of views 3 and 5 (tests/test_oracle_merge.py checks these facts on the oracle)
REFUSING = dict(optimization_robust_covisibility_minimum_landmarks=380, optimization_minimum_new_constraints=10)


@pytest.mark.parametrize("n,con", [
    (8, REFUSING),
    (8, {}),
    (8, dict(optimization_maximum_three_view_constraints=2, optimization_minimum_new_constraints=3)),
    (8, dict(optimization_robust_covisibility_minimum_landmarks=120, optimization_minimum_new_constraints=6)),
    (32, {}),
    (32, dict(optimization_maximum_three_view_constraints=3, optimization_minimum_new_constraints=4)),
])
def test_incorporate_reconstruction_equals_the_oracle(ctx, n, con):
    sc = _scene(n, garbage=3)
    lm = MS.true_landmark_map(sc)
    got = cv_b200.incorporate_reconstruction(ctx, sc["dest"], sc["src"], _wt(sc), lm, constraint_settings=cv_b200.ConstraintSettings(**con))
    want = OM.incorporate_reconstruction(sc["dest"], sc["src"], _wt(sc), lm, constraints_cfg=OC.ConstraintsCfg(**con))
    IS.snap_equal(got["snapshot"], want["snapshot"], keys=NONPOSE + ("poses",))
    IS.sanity(got["snapshot"])
    assert np.array_equal(got["src_view_map"], want["src_view_map"]) and np.array_equal(got["src_landmark_map"], want["src_landmark_map"])
    assert got["con_results"].tobytes() == want["con_results"].tobytes()
    r = got["result"]
    assert int(r["refused_views"]) == want["refused"] and int(r["created_landmarks"]) == want["created"]
    last_refused = int(want["src_view_map"][n - 1] == NONE)   # a refusal of the last moved view needs no rerun
    assert int(r["constraint_calls"]) == want["refused"] + 1 - last_refused
    print(f"n={n} con={con}: refused {want['refused']} of {n}, constraint calls {int(r['constraint_calls'])}")


def test_speculation_reruns_after_a_refusal(ctx):
    sc = _scene(8)
    got = cv_b200.incorporate_reconstruction(ctx, sc["dest"], sc["src"], _wt(sc), MS.true_landmark_map(sc),
                                             constraint_settings=cv_b200.ConstraintSettings(**REFUSING))
    acc = [bool(r["accepted"]) for r in got["con_results"]]
    assert acc == [False, False, False, True, False, True, True, False]
    assert int(got["result"]["refused_views"]) == 5 and int(got["result"]["constraint_calls"]) == 5   # the last view's refusal ends it
    recorded = sum(int(r["n_constraints"]) for r in got["con_results"] if r["accepted"])
    assert len(got["snapshot"]["constraints"]) < recorded


def test_merge_with_refused_moved_views_equals_the_oracle_chain(ctx):
    sc = _scene(8)
    got, want = _merge_both(ctx, sc, con=dict(optimization_robust_covisibility_minimum_landmarks=375, optimization_minimum_new_constraints=12))
    assert want["status"] == "merged" and want["move"]["refused"] > 1
    _assert_merge(got, want)
    assert int(got["result"]["move"]["constraint_calls"]) > 1


def _merge_both(ctx, sc, method=LINEAR_EIGEN, reg=None, con=None, rec=None, seed=5):
    reg, con, rec = dict(reg or {}), dict(con or {}), dict(rec or {})
    ars = cv_b200.Arrsac(1e-5, cv_b200.Xoshiro256PlusPlus(seed), ctx)
    got = cv_b200.merge_reconstructions(ctx, sc["dest"], sc["src"], sc["s_view"], sc["dest_view_matches"], ars,
                                        register_settings=cv_b200.RegisterSettings(**reg), constraint_settings=cv_b200.ConstraintSettings(**con),
                                        reconstruction_settings=cv_b200.ReconstructionSettings(**rec), triangulator=TRIS[method]())
    orng = O.rng_xoshiro(seed)
    want = OM.merge_reconstructions(sc["dest"], sc["src"], sc["s_view"], sc["dest_view_matches"], O.arrsac_cfg(1e-5), orng,
                                    register_cfg=OR.RegisterCfg(**reg), constraints_cfg=OC.ConstraintsCfg(**con), recon_cfg=OREC.ReconCfg(**rec),
                                    tri=o_tri(method))
    assert list(ars.rng.state.s) == list(orng.s)
    return got, want


def _assert_merge(got, want, tol=5e-8):
    assert got["status"] == want["status"], (got["status"], want["status"])
    r = got["result"]
    assert OR.STATUS_NAMES[int(r["reg"]["status"])] == want["register"]["status"]
    if want["constraints"] is not None:
        wc = want["constraints"]["results"][0]
        assert int(r["con"]["n_constraints"]) == int(wc["n_constraints"]) and int(r["con"]["accepted"]) == int(wc["accepted"])
    if want["move"] is not None:
        assert got["con_results"].tobytes() == want["move"]["con_results"].tobytes()
        assert int(r["move"]["refused_views"]) == want["move"]["refused"]
    if want["recon"] is not None:
        for k in ("status", "round", "step", "views_removed", "robust_before", "robust_after", "observations_split"):
            assert int(r["recon"][k]) == int(want["recon"]["result"][k]), k
    for k in ("dest_view_map", "dest_landmark_map", "src_view_map", "src_landmark_map"):
        assert np.array_equal(got[k], want[k]), k
    assert got["dest_view"] == want["dest_view"]
    if want["snapshot"] is None:
        assert got["snapshot"] is None
        return
    g, w = got["snapshot"], want["snapshot"]
    IS.snap_equal(g, w, keys=NONPOSE)
    IS.sanity(g)
    d = np.abs(g["poses"] - w["poses"]).max()
    assert d <= tol, d
    _cons_equal(g["constraints"], w["constraints"], tol)


@pytest.mark.parametrize("n,method", [(8, LINEAR_EIGEN), (8, SINE_L1), (8, MEAN_MEAN), (32, LINEAR_EIGEN)])
def test_merge_equals_the_oracle_chain(ctx, n, method):
    sc = _scene(n, seed=4, garbage=3, outliers=0.1, merges=20, shared_merges=5)
    got, want = _merge_both(ctx, sc, method)
    assert want["status"] == "merged"
    _assert_merge(got, want)


def test_merge_bit_for_bit_without_steps(ctx):
    sc = _scene(8, seed=4)
    got, want = _merge_both(ctx, sc, con=dict(constraint_patience=0), rec=dict(optimization_iterations=0))
    assert want["status"] == "merged"
    # the registered pose is held to the oracle's only to rounding (include/cvb200_register.h); when it is equal, so is every pose
    R, t = want["register"]["pose"]
    reg_equal = (got["result"]["reg"]["pose"]["r"].tobytes() == R.reshape(9).tobytes() and
                 got["result"]["reg"]["pose"]["t"].tobytes() == t.tobytes())
    print("registered pose bit for bit:", reg_equal)
    _assert_merge(got, want, tol=0 if reg_equal else 1e-12)


@pytest.mark.parametrize("status,kw", [
    ("not_registered", dict(reg=dict(single_view_minimum_landmarks=100000))),
    ("rejected", dict(con=dict(optimization_minimum_new_constraints=1000, optimization_robust_covisibility_minimum_landmarks=10 ** 6))),
    ("removed_filter", dict(rec=dict(minimum_robust_landmarks=10 ** 7))),
])
def test_merge_statuses_equal_the_oracle(ctx, status, kw):
    sc = _scene(8, seed=4, merges=20)
    got, want = _merge_both(ctx, sc, **kw)
    assert want["status"] == status
    _assert_merge(got, want, tol=0 if status == "not_registered" else 1e-12 if status == "rejected" else 5e-8)


def test_dev_forms_equal_the_host_forms_and_repeat(ctx):
    sc = _scene(8, seed=4)
    dd, sd = snapshot_to_device(sc["dest"]), snapshot_to_device(sc["src"])
    lm = MS.true_landmark_map(sc)
    h = cv_b200.incorporate_reconstruction(ctx, sc["dest"], sc["src"], _wt(sc), lm)
    for _ in range(2):
        d = incorporate_reconstruction_dev(ctx, dd, sd, torch.from_numpy(_wt(sc)).cuda(), torch.from_numpy(lm.view(np.int32)).cuda())
        IS.snap_equal(snapshot_to_host(d["snapshot"]), h["snapshot"])
        assert np.array_equal(d["src_landmark_map"].cpu().numpy().view(np.uint32), h["src_landmark_map"])
    hm = []
    for dev in (False, True, True):
        ars = cv_b200.Arrsac(1e-5, cv_b200.Xoshiro256PlusPlus(5), ctx)
        if dev:
            r = merge_reconstructions_dev(ctx, dd, sd, sc["s_view"], sc["dest_view_matches"], ars)
            r = dict(r, snapshot=snapshot_to_host(r["snapshot"]), src_view_map=r["src_view_map"].cpu().numpy().view(np.uint32))
        else:
            r = cv_b200.merge_reconstructions(ctx, sc["dest"], sc["src"], sc["s_view"], sc["dest_view_matches"], ars)
        hm.append(r)
    assert hm[0]["status"] == "merged"
    for r in hm[1:]:
        assert r["status"] == hm[0]["status"]
        IS.snap_equal(r["snapshot"], hm[0]["snapshot"])
        assert np.array_equal(r["src_view_map"], hm[0]["src_view_map"])


def test_bad_arguments(ctx):
    sc = _scene(8, seed=4)
    lm = MS.true_landmark_map(sc)
    with pytest.raises(CvbError):
        cv_b200.incorporate_reconstruction(ctx, sc["dest"], sc["src"], _wt(sc), lm, skip_view=8)
    dup = np.full_like(lm, NONE); dup[:2] = 0
    with pytest.raises(CvbError):
        cv_b200.incorporate_reconstruction(ctx, sc["dest"], sc["src"], _wt(sc), dup)
    ars = cv_b200.Arrsac(1e-5, cv_b200.Xoshiro256PlusPlus(5), ctx)
    with pytest.raises(CvbError):
        cv_b200.merge_reconstructions(ctx, sc["dest"], sc["src"], 8, sc["dest_view_matches"], ars)
    with pytest.raises(CvbError):
        cv_b200.merge_reconstructions(ctx, sc["dest"], sc["src"], sc["s_view"], sc["dest_view_matches"], ars,
                                      triangulator=cv_b200.RelativeDltTriangulator())
