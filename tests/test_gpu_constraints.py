"""GPU: include/cvb200_constraints.h against the CPU oracle (oracle/ref_constraints.c) and the warp-per-problem optimiser against
cvb_three_view_optimize_l2 (adaptive), bit for bit where the arithmetic is the same."""
import ctypes as C

import numpy as np
import pytest

import cv_b200
from cv_b200._lib import CVB_EINVAL, CVB_EUNSUPPORTED
from cv_b200.constraints import ConstraintSettings, generate_view_constraints, three_view_adaptive_optimize_l2_dev
from oracle.pyoracle_constraints import ConstraintsCfg, view_constraints
from oracle.pyoracle_tri import LINEAR_EIGEN, MEAN_MEAN, SINE_L1, triangulator

from tests.constraint_scenes import scene, snapshot_from_lists

pytestmark = pytest.mark.gpu
TRIS = {LINEAR_EIGEN: cv_b200.LinearEigenTriangulator, SINE_L1: cv_b200.SineL1Triangulator, MEAN_MEAN: cv_b200.MeanMeanTriangulator}


@pytest.fixture(scope="module")
def ctx():
    return cv_b200.Context(0)


def _cfgs(**kw):
    return ConstraintSettings(**kw), ConstraintsCfg(**kw)


def _run(ctx, s, queries, method=LINEAR_EIGEN, **kw):
    dc, oc = _cfgs(**kw)
    d = generate_view_constraints(ctx, **s, queries=queries, settings=dc, triangulator=TRIS[method](), stats=True)
    o = view_constraints(**s, queries=queries, cfg=oc, tri=triangulator(method))
    return d, o


def _same(d, o, poses_exact=True, tol=1e-8):
    assert d["results"].tobytes() == o["results"].tobytes()
    st_d, st_o = d["stats"].copy(), o["stats"].copy()
    assert st_d.tobytes() == st_o.tobytes()
    for cd, co in zip(d["constraints"], o["constraints"]):
        assert np.array_equal(cd["views"], co["views"]) and np.array_equal(cd["landmarks"], co["landmarks"])
        if poses_exact:
            assert cd.tobytes() == co.tobytes()
        else:
            for f in ("r", "t"):
                np.testing.assert_allclose(cd["poses"][f], co["poses"][f], rtol=0, atol=tol)


# ------------------------------------------------------------------------------------------------ the warp optimiser
def _opt_problems(ns, seed=3):
    rng = np.random.default_rng(seed)
    obs, off, poses = [], [0], []
    for n in ns:
        s, P, X = scene(3, points=max(n, 1) * 2, seed=seed + n, noise=1e-3, singles=0, far=0, fov_cos=0.3)
        pts = rng.normal(0, 1, (n, 3)) + np.array([0, 0, 6.0])
        rows = []
        for p in pts:
            r = []
            for v in range(3):
                R, t = P[v, :9].reshape(3, 3), P[v, 9:]
                x = R @ p + t + rng.normal(0, 1e-3, 3)
                r.append(x / np.linalg.norm(x))
            rows.append(np.concatenate(r))
        obs += rows
        off.append(off[-1] + n)
        R0, t0 = P[0, :9].reshape(3, 3), P[0, 9:]
        for v in (1, 2):
            R, t = P[v, :9].reshape(3, 3), P[v, 9:]
            Rr = R @ R0.T
            poses.append(np.concatenate([Rr.reshape(9), t - Rr @ t0 + rng.normal(0, 1e-2, 3)]))
    return np.asarray(poses), np.asarray(obs, np.float64).reshape(-1, 9), np.asarray(off, np.uint32)


@pytest.mark.parametrize("iterations", [0, 1, 4096])
def test_warp_optimiser_equals_three_view_optimize_l2_adaptive(ctx, iterations):
    import torch
    from cv_b200.optimize import _lib as opt_lib
    ns = [0, 1, 31, 32, 33, 64, 65, 512]
    poses, obs, off = _opt_problems(ns)
    B = len(ns)
    _, L = opt_lib(ctx)
    want = np.zeros(2 * B * 12)
    wupd = np.zeros(B, np.uint32)
    p = np.ascontiguousarray(poses)
    ctx.check(L.cvb_three_view_optimize_l2(ctx.handle, p.ctypes.data, B, 1, 0.0, iterations, obs.ctypes.data, off.ctypes.data,
                                           want.ctypes.data, wupd.ctypes.data))
    dev = torch.device("cuda", 0)
    got, upd = three_view_adaptive_optimize_l2_dev(ctx, torch.from_numpy(p).to(dev), torch.from_numpy(obs).to(dev),
                                                   torch.from_numpy(off.astype(np.int32)).to(dev), iterations)
    assert got.cpu().numpy().tobytes() == want.tobytes()
    assert np.array_equal(upd.cpu().numpy().astype(np.uint32), wupd)


def test_warp_optimiser_rejects_more_than_512_landmarks(ctx):
    import torch
    poses, obs, off = _opt_problems([513])
    dev = torch.device("cuda", 0)
    with pytest.raises(cv_b200.CvbError) as e:
        three_view_adaptive_optimize_l2_dev(ctx, torch.from_numpy(poses).to(dev), torch.from_numpy(obs).to(dev),
                                            torch.from_numpy(off.astype(np.int32)).to(dev), 1)
    assert e.value.code == CVB_EUNSUPPORTED


# ------------------------------------------------------------------------------------------------ the whole call
@pytest.mark.parametrize("method", [LINEAR_EIGEN, SINE_L1, MEAN_MEAN])
def test_every_view_equals_oracle_at_patience_0(ctx, method):
    s, _, _ = scene(64, points=900, seed=11, noise=2e-4, outliers=0.02, fov_cos=0.8)
    d, o = _run(ctx, s, np.arange(64), method, constraint_patience=0)
    assert sum(len(c) for c in d["constraints"]) > 64 * 8
    _same(d, o)


def test_default_patience_matches_oracle(ctx):
    """At cv-sfm's patience (4 096) views, order, counts, statistics and acceptance are the oracle's.  With exact bearings the true
    relative poses are a fixed point of the adaptive step and the poses agree within 1e-8.  With noisy bearings the adaptive step does
    not settle, and the oracle's landmark-order sums and the device's tree sums drift apart over the iterations (DESIGN section 4l), so
    only the rest is compared there."""
    s, _, _ = scene(12, points=400, seed=5, exact=True, singles=0, far=0)
    d, o = _run(ctx, s, [0, 5, 11])
    assert all(len(c) for c in d["constraints"])
    _same(d, o, poses_exact=False)
    s, _, _ = scene(12, points=400, seed=5, noise=2e-4, outliers=0.02)
    d, o = _run(ctx, s, [0, 11])
    assert all(len(c) for c in d["constraints"])
    _same(d, o, poses_exact=False, tol=np.inf)


def test_many_queries_equal_single_queries(ctx):
    s, _, _ = scene(20, points=500, seed=8, noise=2e-4)
    dc, _ = _cfgs(constraint_patience=50)
    qs = [3, 0, 19, 3, 7]
    d = generate_view_constraints(ctx, **s, queries=qs, settings=dc, stats=True)
    for i, q in enumerate(qs):
        one = generate_view_constraints(ctx, **s, queries=[q], settings=dc, stats=True)
        assert one["results"].tobytes() == d["results"][i:i + 1].tobytes()
        assert one["stats"].tobytes() == d["stats"][i:i + 1].tobytes()
        assert one["constraints"][0].tobytes() == d["constraints"][i].tobytes()
    again = generate_view_constraints(ctx, **s, queries=qs, settings=dc, stats=True)     # repeated call on the same buffers
    assert again["results"].tobytes() == d["results"].tobytes()
    assert all(a.tobytes() == b.tobytes() for a, b in zip(again["constraints"], d["constraints"]))


def test_query_without_robust_landmarks_and_small_reconstructions(ctx):
    s, _, _ = scene(6, points=300, seed=9)
    # a seventh view whose features are all single-observation landmarks
    L = len(s["landmark_offsets"]) - 1
    feats = [list(s["view_landmarks"][s["view_offsets"][v]:s["view_offsets"][v + 1]]) for v in range(6)] + [list(range(L, L + 40))]
    bears = [s["bearings"][s["view_offsets"][v]:s["view_offsets"][v + 1]] for v in range(6)] + [np.tile([0, 0, 1.0], (40, 1))]
    s7 = snapshot_from_lists(np.concatenate([s["poses"], s["poses"][:1]]), feats, bears)
    d, o = _run(ctx, s7, [6, 0, 6], constraint_patience=0)
    _same(d, o)
    assert d["stats"][0]["robust_landmarks"] == 0 and d["results"][0]["n_constraints"] == 0 and d["results"][0]["accepted"] == 0
    for V in (1, 2, 3):
        sv, _, _ = scene(V, points=200, seed=V)
        d, o = _run(ctx, sv, list(range(V)) * 2, constraint_patience=10)
        _same(d, o, poses_exact=False)


def test_argument_errors(ctx):
    s, _, _ = scene(4, points=100, seed=1)
    with pytest.raises(cv_b200.CvbError) as e:
        generate_view_constraints(ctx, **s, queries=[0], triangulator=cv_b200.RelativeDltTriangulator())
    assert e.value.code == CVB_EUNSUPPORTED
    with pytest.raises(cv_b200.CvbError) as e:
        generate_view_constraints(ctx, **s, queries=[0], settings=ConstraintSettings(optimization_maximum_landmarks=513))
    assert e.value.code == CVB_EUNSUPPORTED
    with pytest.raises(cv_b200.CvbError) as e:
        generate_view_constraints(ctx, **s, queries=[4])
    assert e.value.code == CVB_EINVAL
    L = cv_b200._lib.load_constraints_library()
    dc = ConstraintSettings()
    tri = cv_b200.LinearEigenTriangulator()
    q = np.zeros(1, np.uint32)
    assert L.cvb_view_constraints_dev(ctx.handle, C.addressof(dc), C.addressof(tri.cfg), 4, None, None, None, None, 0, 0, None, None, 0,
                                      q.ctypes.data, 1, None, None, None) == CVB_EINVAL
    assert L.cvb_view_constraints(None, C.addressof(dc), C.addressof(tri.cfg), 0, None, None, None, None, 0, None, None, None, 0, None, None,
                                  None) == CVB_EINVAL
