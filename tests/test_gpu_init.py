"""GPU: cv-sfm's three-view initialisation on the device (include/cvb200_init.h) against its oracle (oracle/ref_init.c) -- bit for bit
when the optimiser runs no iterations, to the optimiser's rounding otherwise -- across waves, chained from frames, and its argument
errors."""
import ctypes as C

import numpy as np
import pytest
import torch

import cv_b200
from cv_b200._lib import CVB_EINVAL, CVB_EUNSUPPORTED, default_context, load_init_library
from cv_b200.pair import INIT_PAIR_STATS_DTYPE, INIT_RESULT_DTYPE, InitSettings, init_reconstruction_dev
from oracle import pyoracle_init as OI
from oracle import pyoracle_tri as OT
from tests.init_scenes import init_scene
from tests.synth import synth_frame, warp_frame

pytestmark = pytest.mark.gpu

TRIS = {OT.LINEAR_EIGEN: cv_b200.LinearEigenTriangulator, OT.SINE_L1: cv_b200.SineL1Triangulator, OT.MEAN_MEAN: cv_b200.MeanMeanTriangulator}


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _device_inputs(sc, found=None):
    F = len(sc["options"])
    cap = sc["bearings"].shape[1]
    arrs = OI.options_from_matches(F, cap, sc["matches"], sc["poses"], found)
    names = ("pairs", "n_pairs", "model", "inliers", "n_inliers", "found")
    dev = {k: torch.from_numpy(np.ascontiguousarray(a).view(np.int32) if a.dtype != np.float64 else np.ascontiguousarray(a)).cuda()
           for k, a in zip(names, arrs)}
    return arrs, dev


def _both(sc, cfg_kw, method=OT.LINEAR_EIGEN, found=None):
    arrs, dev = _device_inputs(sc, found)
    ctx = default_context(0)
    got = init_reconstruction_dev(ctx, torch.from_numpy(sc["bearings"]).cuda(), 0, sc["options"], dev, InitSettings(**cfg_kw),
                                  TRIS[method](), stats=True)
    want = OI.init_reconstruction(sc["bearings"], 0, sc["options"], *arrs, OI.InitCfg(**cfg_kw), OT.triangulator(method))
    return got, want


def _assert_exact(got, want):
    assert got["result"].tobytes() == want["result"].tobytes(), (got["result"], want["result"])
    assert got["stats"].tobytes() == want["stats"].tobytes(), (got["stats"], want["stats"])
    for k in ("combined", "first_matches", "second_matches"):
        assert np.array_equal(got[k], want[k].astype(np.int64)), k


@pytest.mark.parametrize("method", [OT.LINEAR_EIGEN, OT.SINE_L1, OT.MEAN_MEAN])
@pytest.mark.parametrize("seed", [0, 1])
def test_bit_for_bit_without_optimiser_iterations(method, seed):
    sc = init_scene(np.random.default_rng(100 + seed), 4, noise=1e-4 * (seed + 1), outliers=0.1 + 0.1 * seed)
    got, want = _both(sc, dict(three_view_patience=0), method)
    assert want["result"]["status"] == OI.ACCEPTED or seed
    _assert_exact(got, want)


@pytest.mark.parametrize("patience", [200, 1 << 16])
def test_optimised_decision_and_lists_match_the_oracle(patience):
    # low noise keeps every triple far from the 1e-5 cosine threshold, so the optimiser's last-bit differences decide nothing
    sc = init_scene(np.random.default_rng(7), 3, noise=1e-7, outliers=0.05)
    got, want = _both(sc, dict(three_view_patience=patience))
    g, w = got["result"], want["result"]
    assert (g["status"], g["pair"], g["first"], g["second"]) == (w["status"], w["pair"], w["first"], w["second"]) and w["status"] == OI.ACCEPTED
    assert np.array_equal(got["stats"]["outcome"], want["stats"]["outcome"])
    for k in ("combined", "first_matches", "second_matches"):
        assert np.array_equal(got[k], want[k].astype(np.int64)), k
    for p in ("first_pose", "second_pose"):
        assert np.allclose(g[p]["r"], w[p]["r"], atol=1e-8) and np.allclose(g[p]["t"], w[p]["t"], atol=1e-8)


def _pair_index(F, i, j):
    return sum(F - 1 - k for k in range(i)) + (j - i - 1)


def _pair_of(F, p):
    for i in range(F):
        for j in range(i + 1, F):
            if _pair_index(F, i, j) == p:
                return i, j


def _wave_scene(F, accept=None, block=40, shared=200):
    """option f sees its own `block` points; the options of pair `accept` also share `shared` points"""
    rng = np.random.default_rng(F + 31 * (accept[0] if accept else 0) + (accept[1] if accept else 0))
    n = F * block + shared
    seen = [list(range(f * block, (f + 1) * block)) for f in range(F)]
    if accept is not None:
        for f in accept:
            seen[f] += list(range(F * block, n))
    cap = 1 << int(np.ceil(np.log2(n)))
    return init_scene(rng, F, n_points=n, cap=cap, noise=0.0, outliers=0.0, seen=[np.array(s) for s in seen])


WAVE_CFG = dict(two_view_minimum_robust_matches=32, three_view_patience=50)


@pytest.mark.parametrize("where", ["first", "W-1", "W", "last"])
def test_decisive_pair_in_any_wave(where):
    F, W = 64, _sms()
    P = F * (F - 1) // 2
    p = {"first": 0, "W-1": W - 1, "W": W, "last": P - 1}[where]
    sc = _wave_scene(F, accept=_pair_of(F, p))
    got, want = _both(sc, WAVE_CFG)
    assert want["result"]["status"] == OI.ACCEPTED and want["result"]["pair"] == p
    _assert_exact_or_close(got, want)
    # pairs after the decisive one are not evaluated
    assert np.all(got["stats"]["outcome"][p + 1:] == OI.PAIR_NOT_EVALUATED)
    assert np.all(got["stats"]["outcome"][:p] == OI.PAIR_FEW_SCALES)


def _assert_exact_or_close(got, want):
    g, w = got["result"], want["result"]
    assert (g["status"], g["pair"], g["first"], g["second"], g["n_pairs"]) == (w["status"], w["pair"], w["first"], w["second"], w["n_pairs"])
    assert np.array_equal(got["stats"]["outcome"], want["stats"]["outcome"])
    for k in ("combined", "first_matches", "second_matches"):
        assert np.array_equal(got[k], want[k].astype(np.int64)), k
    for p in ("first_pose", "second_pose"):
        assert np.allclose(g[p]["r"], w[p]["r"], atol=1e-8) and np.allclose(g[p]["t"], w[p]["t"], atol=1e-8)


def test_no_decisive_pair_and_a_bearing_pair_abort():
    F = 64
    sc = _wave_scene(F)
    got, want = _both(sc, WAVE_CFG)
    assert want["result"]["status"] == OI.NONE and want["result"]["n_pairs"] == F * (F - 1) // 2
    _assert_exact(got, want)
    # a tight cluster shared by pair 5 in front of an accepted pair 200
    rng = np.random.default_rng(3)
    n = 6 * 40 + 400
    seen = [list(range(f * 40, (f + 1) * 40)) for f in range(6)]
    for f in _pair_of(6, 3):
        seen[f] += list(range(240, 440))
    for f in _pair_of(6, 10):
        seen[f] += list(range(440, 640))
    sc = init_scene(rng, 6, n_points=n, cap=1024, noise=0.0, outliers=0.0, seen=[np.array(s) for s in seen])
    # the cluster: points 240..439 into a tight cone, bearings of every frame recomputed
    X = sc["points"].copy()
    X[240:440] = np.array([0.5, 0.2, 6.0]) + rng.normal(0, 0.03, (200, 3))
    for g in range(7):
        Xg = X if g == 0 else X @ sc["poses"][g - 1][0].T + sc["true_t"][g - 1]
        b = Xg / np.linalg.norm(Xg, axis=1, keepdims=True)
        sc["bearings"][g, :n] = b[np.argsort(sc["inv"][g])]
    got, want = _both(sc, WAVE_CFG)
    assert want["result"]["status"] == OI.NONE_BEARING_PAIRS and want["result"]["pair"] == 3
    _assert_exact_or_close(got, want)


@pytest.mark.parametrize("F", [0, 1, 2])
def test_few_options(F):
    sc = init_scene(np.random.default_rng(9), max(F, 1), noise=1e-5)
    sc = dict(sc, options=sc["options"][:F], matches=sc["matches"][:F], poses=sc["poses"][:F])
    if F == 0:
        ctx = default_context(0)
        got = init_reconstruction_dev(ctx, torch.from_numpy(sc["bearings"]).cuda(), 0, [], None, InitSettings(three_view_patience=0), stats=True)
        assert got["result"]["status"] == OI.NONE and got["result"]["n_pairs"] == 0
        return
    got, want = _both(sc, dict(three_view_patience=0))
    _assert_exact(got, want)
    assert (want["result"]["status"] == OI.ACCEPTED) == (F == 2)


def test_chained_from_frames_equals_the_oracle_and_the_wrapper():
    base = synth_frame(11, h=360, w=640, nblobs=1200)
    frames = np.stack([base] + [warp_frame(base, 100 + i, shift=(1.5 * i, -0.7 * i)) for i in range(1, 5)])
    camera = cv_b200.CameraIntrinsics(focals=(600.0, 600.0), principal_point=(320.0, 180.0))
    cap = 4096
    ak = cv_b200.Akaze(maximum_features=cap)
    feats = cv_b200.frame_features(ak, frames, (np.clip(frames, 0, 1) * 255).astype(np.uint8), camera)
    Fr = len(frames)
    desc = np.zeros((Fr, cap, 64), np.uint8); bear = np.zeros((Fr, cap, 3)); n = np.zeros(Fr, np.int32)
    for f, d in enumerate(feats):
        k = len(d["keypoints"])
        desc[f, :k] = d["descriptors"]; bear[f, :k] = d["bearings"]; n[f] = k
    features = dict(descriptors=torch.from_numpy(desc).cuda(), counts=torch.from_numpy(n).cuda(), bearings=torch.from_numpy(bear).cuda())
    ctx = default_context(0)
    ars = cv_b200.Arrsac(1e-6, cv_b200.Xoshiro256PlusPlus(0), ctx=ctx)
    options = [1, 2, 3, 4]
    settings = dict(three_view_patience=0, two_view_minimum_robust_matches=64)
    _, _, opts, two = cv_b200.pair._two_view_options_dev(features, 0, options, ars, [cv_b200.Xoshiro256PlusPlus(s) for s in (1, 2, 3, 4)], 24)
    got = init_reconstruction_dev(ctx, features["bearings"], 0, opts, two, InitSettings(**settings), stats=True)
    h = {k: v.cpu().numpy() for k, v in two.items()}
    want = OI.init_reconstruction(bear, 0, options, h["pairs"].view(np.uint32), h["n_pairs"].view(np.uint32), h["model"],
                                  h["inliers"].view(np.uint32), h["n_inliers"].view(np.uint32), h["found"], OI.InitCfg(**settings))
    _assert_exact(got, want)
    wrap = cv_b200.init_reconstruction(features, 0, options, ars, [cv_b200.Xoshiro256PlusPlus(s) for s in (1, 2, 3, 4)],
                                       settings=InitSettings(**settings))
    w = want["result"]
    if w["status"] != OI.ACCEPTED:
        assert wrap is None
    else:
        assert wrap["first"] == options[w["first"]] and wrap["second"] == options[w["second"]]
        assert np.array_equal(wrap["combined"], want["combined"].astype(np.int64))
        assert np.array_equal(wrap["first_matches"], want["first_matches"].astype(np.int64))
        assert wrap["first_pose"][1].tobytes() == np.array(w["first_pose"]["t"]).tobytes()


def test_errors_and_repeats():
    sc = init_scene(np.random.default_rng(11), 3, noise=1e-5)
    arrs, dev = _device_inputs(sc)
    ctx = default_context(0)
    IL = load_init_library()
    bear = torch.from_numpy(sc["bearings"]).cuda()
    frames, cap = bear.shape[0], bear.shape[1]
    outs = [torch.zeros(n, dtype=torch.int32, device="cuda") for n in (64, cap * 3, cap * 2, cap * 2, 3 * 16)]
    cfg = InitSettings(three_view_patience=100)
    tri = cv_b200.LinearEigenTriangulator()

    def call(cfg_p=C.addressof(cfg), tri_cfg=tri.cfg, options=(1, 2, 3), F=None, center=0, cap_=cap, bear_p=bear.data_ptr()):
        opts = np.array(options, np.uint32)
        F = len(opts) if F is None else F
        return IL.cvb_init_reconstruction_dev(ctx.handle, cfg_p, C.addressof(tri_cfg), bear_p, frames, cap_, center,
                                              opts.ctypes.data, F, dev["pairs"].data_ptr(), dev["n_pairs"].data_ptr(),
                                              dev["model"].data_ptr(), dev["inliers"].data_ptr(), dev["n_inliers"].data_ptr(),
                                              dev["found"].data_ptr(), *[o.data_ptr() for o in outs])
    torch.cuda.synchronize()
    assert call(cfg_p=None) == CVB_EINVAL
    assert call(bear_p=None) == CVB_EINVAL
    assert call(cap_=0) == CVB_EINVAL
    assert call(center=frames) == CVB_EINVAL
    assert call(options=(1, 2, frames)) == CVB_EINVAL
    assert call(options=[1] * 65) == CVB_EUNSUPPORTED
    for m in (cv_b200.RelativeDltTriangulator(), cv_b200.AngularL1Triangulator(), cv_b200.AngularLInfinityTriangulator()):
        assert call(tri_cfg=m.cfg) == CVB_EUNSUPPORTED
    def written():
        r = np.frombuffer(outs[0].cpu().numpy().tobytes()[:INIT_RESULT_DTYPE.itemsize], INIT_RESULT_DTYPE)[0]
        return (r.tobytes(), outs[1][:3 * int(r["n_combined"])].cpu().numpy().tobytes(),
                outs[2][:2 * int(r["n_first_matches"])].cpu().numpy().tobytes(),
                outs[3][:2 * int(r["n_second_matches"])].cpu().numpy().tobytes(),
                outs[4].cpu().numpy().tobytes()[:3 * INIT_PAIR_STATS_DTYPE.itemsize])
    ctx.check(call())
    torch.cuda.synchronize()
    first = written()
    assert np.frombuffer(first[0], INIT_RESULT_DTYPE)[0]["status"] == OI.ACCEPTED
    for o in outs:
        o.fill_(7)
    ctx.check(call())
    torch.cuda.synchronize()
    assert written() == first
