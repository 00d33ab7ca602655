"""GPU: cv_b200.register_frame (include/cvb200_register.h) against the loop-for-loop C oracle (oracle/ref_register.c).

The scenes (tests/register_scenes.py) have margin on purpose: inlier bearings carry 1e-5 rad of noise, far inside the consensus and
consistency thresholds, outliers point at random directions, far outside them, and descriptors put a feature's own landmark a few bits
away and every other landmark about 256 bits away.  Lambda Twist's rotation uses CUDA's sin / cos and the optimiser's sums run in another
order, so the pose is held to 1e-8, not bit for bit; with that margin every decision -- status, each count, the inlier set, the final
match list and the generator's state -- must be equal."""
import ctypes as C

import numpy as np
import pytest
import torch

import cv_b200
from oracle import pyoracle as O
from oracle import pyoracle_register as OR
from oracle.pyoracle_tri import LINEAR_EIGEN, MEAN_MEAN, SINE_L1, triangulator as o_tri

from . import register_scenes as RS

pytestmark = pytest.mark.gpu

TRIS = {LINEAR_EIGEN: cv_b200.LinearEigenTriangulator, SINE_L1: cv_b200.SineL1Triangulator, MEAN_MEAN: cv_b200.MeanMeanTriangulator}
STAT_KEYS = ("subsets", "matches", "claimed", "matches_3d", "inliers", "final_robust", "final_matches", "iterations",
             "final_stage_matches")


@pytest.fixture(scope="module")
def ctx():
    return cv_b200.Context(0)


def _run_both(ctx, s, seed=5, method=LINEAR_EIGEN, **kw):
    dev_cfg = cv_b200.RegisterSettings(**kw)
    ars = cv_b200.Arrsac(1e-5, cv_b200.Xoshiro256PlusPlus(seed), ctx)
    got = cv_b200.register_frame(ctx, *RS.args(s), ars, settings=dev_cfg, triangulator=TRIS[method](), stats=True)
    orng = O.rng_xoshiro(seed)
    want = OR.register_frame(*RS.args(s), O.arrsac_cfg(1e-5), orng, cfg=OR.RegisterCfg(**kw), tri=o_tri(method))
    return got, want, ars, orng


def _assert_equal(got, want, ars, orng):
    status, pose, matches, st, inliers = got
    assert status == want["status"], (status, want["status"], st, want["stats"])
    for k in STAT_KEYS:
        assert int(st[k]) == int(want["stats"][k]), (k, st, want["stats"])
    assert np.array_equal(st["filter_matches"], want["stats"]["filter_matches"])
    assert np.array_equal(matches, want["matches"])
    assert np.array_equal(inliers, want["inliers"])      # the consensus' inlier set, in its order
    assert list(ars.rng.state.s) == list(orng.s)
    if status == "ok":
        assert np.abs(pose[0] - want["pose"][0]).max() < 1e-8 and np.abs(pose[1] - want["pose"][1]).max() < 1e-8


SCENES = {
    "8v": dict(V=8, per_view=2000, seed=11),
    "8v_outliers": dict(V=8, per_view=2500, seed=12, outliers=0.25),
    "32v": dict(V=32, per_view=2000, seed=13, outliers=0.1, step=0.12),
    "merges_doubly": dict(V=10, per_view=2000, seed=14, merges=40, shared_merges=15, doubly=25, outliers=0.1),
}


@pytest.mark.parametrize("name", sorted(SCENES))
def test_device_equals_oracle(ctx, name):
    s = RS.scene(**SCENES[name])
    got, want, ars, orng = _run_both(ctx, s)
    assert want["status"] == "ok"
    _assert_equal(got, want, ars, orng)
    if name == "merges_doubly":
        assert (got[2]["landmark_b"] != RS_NONE).any()
        assert want["stats"]["claimed"] < want["stats"]["matches"]


RS_NONE = 0xFFFFFFFF


@pytest.mark.parametrize("method", [SINE_L1, MEAN_MEAN])
def test_device_equals_oracle_other_triangulators(ctx, method):
    s = RS.scene(V=8, per_view=1500, seed=21, outliers=0.15, merges=10)
    _assert_equal(*_run_both(ctx, s, method=method))


def test_multi_subset_accumulates(ctx):
    # a first subset of 40 features cannot reach 32 robust landmarks once 20 % are outliers; the doubled range succeeds
    s = RS.scene(V=8, per_view=1500, seed=31, outliers=0.2)
    got, want, ars, orng = _run_both(ctx, s, single_view_initial_features=40)
    assert want["stats"]["subsets"] >= 2 and want["status"] == "ok"
    _assert_equal(got, want, ars, orng)


@pytest.mark.parametrize("status,kw,scene_kw", [
    ("few_robust_landmarks", dict(single_view_minimum_landmarks=100000), dict()),
    ("few_matches", dict(single_view_minimum_robust_landmarks=100000), dict()),
    ("filter_half", dict(maximum_cosine_distance=1e-14, maximum_sine_distance=1e-14), dict(noise=1e-3)),
    # one filter iteration leaves nothing consistent under the tightened thresholds: the final stage's check fails
    ("final_half", dict(single_view_filter_loop_iterations=1, maximum_cosine_distance=1e-14, maximum_sine_distance=1e-14), dict(noise=1e-3)),
    # no filter iteration: the inliers pass the final check, and none of them is consistent after the final optimisation
    ("final_robust_half", dict(single_view_filter_loop_iterations=0, maximum_cosine_distance=1e-14, maximum_sine_distance=1e-14),
     dict(noise=1e-3)),
    ("no_consensus", dict(), dict(outliers=1.0)),
])
def test_failure_statuses(ctx, status, kw, scene_kw):
    s = RS.scene(V=6, per_view=800, seed=41, **scene_kw)
    got, want, ars, orng = _run_both(ctx, s, **kw)
    assert want["status"] == status, (want["status"], want["stats"])
    _assert_equal(got, want, ars, orng)


def test_panic(ctx):
    s = RS.scene(V=6, per_view=800, seed=42)
    s["view_matches"] = np.array([], np.uint32)
    got, want, ars, orng = _run_both(ctx, s)
    assert want["status"] == "panic" and got[0] == "panic"
    _assert_equal(got, want, ars, orng)


def test_matching_stage_equals_landmark_matches(ctx):
    # a scene without outliers or noise: every claim-filtered match is consistent under the registered pose, so the final list is the
    # matching stage's whole list -- tuples and merge-pair orientation included -- and its length the claimed count.  Its order (the
    # stable sort) is what the consensus sees: test_device_equals_oracle holds the inlier indices into it to the oracle's.
    s = RS.scene(V=6, per_view=800, seed=43, merges=15, doubly=10, noise=0.0)
    vo, vl, lo, ob = s["view_offsets"], s["view_landmarks"], s["landmark_offsets"], s["observations"]
    views = [(s["descriptors"][vo[v]:vo[v + 1]], vl[vo[v]:vo[v + 1]]) for v in range(len(vo) - 1)]
    lv = {l: set(ob[lo[l]:lo[l + 1], 0].tolist()) for l in range(len(lo) - 1)}
    oc = {l: int(lo[l + 1] - lo[l]) for l in range(len(lo) - 1)}
    want = cv_b200.landmark_matches(s["new_descriptors"], views, 24, lv, oc, ctx=ctx)
    ars = cv_b200.Arrsac(1e-5, cv_b200.Xoshiro256PlusPlus(1), ctx)
    status, pose, matches, st, _ = cv_b200.register_frame(ctx, *RS.args(s), ars, stats=True)
    assert status == "ok" and int(st["claimed"]) == len(want)
    assert any(len(ls) == 2 for ls, _ in want)
    tuples = sorted((f, ls[0], ls[1] if len(ls) > 1 else RS_NONE) for ls, f in want)
    assert [(int(m["feature"]), int(m["landmark_a"]), int(m["landmark_b"])) for m in matches] == tuples


def test_dev_form_equals_host_form_and_repeats(ctx):
    s = RS.scene(V=8, per_view=1500, seed=51, outliers=0.1, merges=10)
    ars = cv_b200.Arrsac(1e-5, cv_b200.Xoshiro256PlusPlus(3), ctx)
    host = cv_b200.register_frame(ctx, *RS.args(s), ars, stats=True)
    again = cv_b200.register_frame(ctx, *RS.args(s), cv_b200.Arrsac(1e-5, cv_b200.Xoshiro256PlusPlus(3), ctx), stats=True)
    assert host[0] == again[0] == "ok" and np.array_equal(host[2], again[2]) and host[3].tobytes() == again[3].tobytes()
    assert np.array_equal(host[4], again[4])
    assert np.array_equal(host[1][0], again[1][0]) and np.array_equal(host[1][1], again[1][1])
    dev = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dt)).cuda()
    P = dev(s["poses"], np.float64)
    vo, vl, bear, desc = dev(s["view_offsets"], np.int32), dev(s["view_landmarks"], np.int32), dev(s["bearings"], np.float64), \
        dev(s["descriptors"], np.uint8)
    lo, ob = dev(s["landmark_offsets"], np.int32), dev(s["observations"], np.int32)
    nd, nb = dev(s["new_descriptors"], np.uint8), dev(s["new_bearings"], np.float64)
    N = len(s["new_descriptors"])
    res = torch.zeros(112, dtype=torch.uint8, device="cuda")
    out = torch.zeros(N * 12, dtype=torch.uint8, device="cuda")
    st = torch.zeros(112, dtype=torch.uint8, device="cuda")
    inl = torch.zeros(N, dtype=torch.int32, device="cuda")
    vm = np.ascontiguousarray(s["view_matches"], np.uint32)
    torch.cuda.synchronize()     # the copies above run on torch's stream, the call on the context's
    ars2 = cv_b200.Arrsac(1e-5, cv_b200.Xoshiro256PlusPlus(3), ctx)
    cfg, tri = cv_b200.RegisterSettings(), cv_b200.LinearEigenTriangulator()     # alive for the whole call
    L = cv_b200._lib.load_register_library()
    ctx.check(L.cvb_register_frame_dev(ctx.handle, C.addressof(cfg), C.addressof(tri.cfg),
                                       C.addressof(ars2.cfg), C.addressof(ars2.rng.state), len(s["view_offsets"]) - 1, P.data_ptr(),
                                       vo.data_ptr(), vl.data_ptr(), bear.data_ptr(), desc.data_ptr(), int(s["view_offsets"][-1]),
                                       len(s["landmark_offsets"]) - 1, lo.data_ptr(), ob.data_ptr(), int(s["landmark_offsets"][-1]),
                                       nd.data_ptr(), nb.data_ptr(), N, vm.ctypes.data, len(vm), res.data_ptr(), out.data_ptr(),
                                       inl.data_ptr(), st.data_ptr()))
    r = np.frombuffer(res.cpu().numpy().tobytes(), cv_b200.register.RESULT_DTYPE)[0]
    m = np.frombuffer(out.cpu().numpy().tobytes(), cv_b200.register.MATCH_DTYPE)[:int(r["n_matches"])]
    assert r["status"] == 0 and np.array_equal(m, host[2]) and st.cpu().numpy().tobytes() == host[3].tobytes()
    assert np.array_equal(inl.cpu().numpy()[:int(r["n_inliers"])].view(np.uint32), host[4])
    assert list(ars2.rng.state.s) == list(ars.rng.state.s)
    assert np.array_equal(r["pose"]["r"].reshape(3, 3), host[1][0]) and np.array_equal(r["pose"]["t"], host[1][1])


def test_registered_pose_is_the_true_pose(ctx):
    s = RS.scene(V=8, per_view=2000, seed=61, noise=0.0)
    status, pose, matches = cv_b200.register_frame(ctx, *RS.args(s), cv_b200.Arrsac(1e-5, cv_b200.Xoshiro256PlusPlus(2), ctx))
    R, t = s["true_pose"]
    assert status == "ok" and np.abs(pose[0] - R).max() < 1e-6 and np.abs(pose[1] - t).max() < 1e-5
    lp = s["landmark_point"]
    assert all(lp[m["landmark_a"]] == s["truth"][m["feature"]] for m in matches)


def _add_view(s, pose, matches, new_bearings):
    """add_view (cv-sfm/src/lib.rs:430-480) on the numpy CSR, for matches of single landmarks: the new view's feature j joins its matched
    landmark, every other feature starts a landmark of its own.  Returns the new snapshot (the new view is the last)."""
    from .constraint_scenes import snapshot_from_lists
    vo, vl = s["view_offsets"], s["view_landmarks"]
    V, L = len(vo) - 1, len(s["landmark_offsets"]) - 1
    feats = [list(vl[vo[v]:vo[v + 1]]) for v in range(V)]
    bears = [s["bearings"][vo[v]:vo[v + 1]] for v in range(V)]
    matched = {int(m["feature"]): int(m["landmark_a"]) for m in matches}
    assert np.all(matches["landmark_b"] == RS_NONE)
    new = []
    for j in range(len(new_bearings)):
        if j in matched:
            new.append(matched[j])
        else:
            new.append(L)
            L += 1
    poses = np.concatenate([s["poses"], np.concatenate([pose[0].reshape(9), pose[1]])[None]])
    return snapshot_from_lists(poses, feats + [new], bears + [new_bearings])


def test_registration_plugs_into_constraints_and_optimisation(ctx):
    # register a frame, add it as a view on the numpy CSR, generate its three-view constraints (accepted), then optimise (kept)
    s = RS.scene(V=8, per_view=1500, seed=71, outliers=0.1)
    status, pose, matches = cv_b200.register_frame(ctx, *RS.args(s), cv_b200.Arrsac(1e-5, cv_b200.Xoshiro256PlusPlus(4), ctx))
    assert status == "ok"
    snap = _add_view(s, pose, matches, s["new_bearings"])
    keys = ("poses", "view_offsets", "view_landmarks", "bearings", "landmark_offsets", "observations")
    V = len(snap["view_offsets"]) - 1
    cons = cv_b200.generate_view_constraints(ctx, *(snap[k] for k in keys), [V - 1])
    assert cons["results"][0]["accepted"] and cons["results"][0]["n_constraints"] > 0
    out = cv_b200.optimize_reconstruction(ctx, *(snap[k] for k in keys), cons["constraints"][0])
    from cv_b200.reconstruction import KEPT
    assert out["result"]["status"] == KEPT
