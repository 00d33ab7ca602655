"""GPU: cv-sfm's reconstruction optimisation on the device (include/cvb200_reconstruction.h) against its CPU oracle
(oracle/ref_reconstruction.c): bit for bit when no step runs, for the three triangulators; after 1, 16 and 1 024 steps on noisy scenes of 32
and 128 views, identical statuses, states and counts with poses within 1e-8 (the device's FP64 sin, cos and acos are not glibc's); every
edge case of tests/reconstruction_scenes.py; regenerate_reconstruction against the same chain run through the host; repeated calls; and
argument errors."""
import ctypes as C

import numpy as np
import pytest

import cv_b200
from cv_b200._lib import CVB_EINVAL, CVB_EUNSUPPORTED
from cv_b200.constraints import generate_view_constraints
from cv_b200.reconstruction import ReconstructionSettings, optimize_reconstruction, regenerate_reconstruction
from oracle.pyoracle_reconstruction import ReconCfg
from oracle.pyoracle_reconstruction import optimize_reconstruction as ref_optimize
from oracle.pyoracle_tri import LINEAR_EIGEN, MEAN_MEAN, SINE_L1, triangulator
from tests.reconstruction_scenes import CASES, args, recon_scene

pytestmark = pytest.mark.gpu

TRI = {LINEAR_EIGEN: "LinearEigenTriangulator", SINE_L1: "SineL1Triangulator", MEAN_MEAN: "MeanMeanTriangulator"}


@pytest.fixture(scope="module")
def ctx():
    return cv_b200.Context()


def _run(ctx, s, cons, method=LINEAR_EIGEN, **kw):
    d = optimize_reconstruction(ctx, s["poses"], s["view_offsets"], s["view_landmarks"], s["bearings"], s["landmark_offsets"],
                                s["observations"], cons, settings=ReconstructionSettings(**kw), triangulator=getattr(cv_b200, TRI[method])())
    o = ref_optimize(*args(s), cons, cfg=ReconCfg(**kw), tri=triangulator(method))
    return d, o


def _same(d, o, tol=1e-8, small_slack=0):
    """small_slack: where the updates shrink through |delta|^2 = f64::EPSILON (exact constraints), the device's and glibc's acos can put a
    view update on either side of it; that count may then differ by this much, and every other output must still agree"""
    fields = [f for f in d["result"].dtype.names if f != "small_angle_updates"]
    assert all(d["result"][f] == o["result"][f] for f in fields), (d["result"], o["result"])
    assert abs(int(d["result"]["small_angle_updates"]) - int(o["result"]["small_angle_updates"])) <= small_slack, (d["result"], o["result"])
    assert np.array_equal(d["view_state"], o["view_state"])
    assert np.array_equal(d["obs_state"], o["obs_state"])
    if tol == 0:
        assert d["poses"].tobytes() == o["poses"].tobytes()
    else:
        fin = np.isfinite(o["poses"])
        assert np.array_equal(fin, np.isfinite(d["poses"]))
        assert np.abs(d["poses"][fin] - o["poses"][fin]).max(initial=0.0) <= tol


@pytest.mark.parametrize("method", [LINEAR_EIGEN, SINE_L1, MEAN_MEAN])
def test_filter_alone_equals_oracle_bit_for_bit(ctx, method):
    s, _, cons = recon_scene(32, seed=2)
    d, o = _run(ctx, s, cons, method, optimization_iterations=0)
    assert o["result"]["observations_split"] > 0 and o["result"]["robust_after"] > 0
    _same(d, o, tol=0)


@pytest.mark.parametrize("V", [32, 128])
@pytest.mark.parametrize("steps", [1, 16, 1024])
def test_steps_match_oracle(ctx, V, steps):
    s, _, cons = recon_scene(V, seed=V + steps)
    d, o = _run(ctx, s, cons, optimization_iterations=steps)
    assert o["result"]["status"] == 0
    _same(d, o)


@pytest.mark.parametrize("name", sorted(CASES))
def test_edge_cases_match_oracle(ctx, name):
    """With exact constraints ("converge", "fixed_point") the updates shrink to rounding level, where the device's acos and glibc's part:
    the small-angle count may differ by 2 and, after 1 024 steps from perturbed poses, the poses by up to 1e-7 (2.9e-8 measured)."""
    s, cons, kw = CASES[name]()
    d, o = _run(ctx, s, cons, **kw)
    exact = name in ("converge", "fixed_point")
    _same(d, o, tol=0 if kw.get("optimization_iterations", 1) == 0 else (1e-7 if exact else 1e-8), small_slack=2 if exact else 0)


def test_regenerate_reconstruction_equals_host_chain(ctx):
    s, _, _ = recon_scene(24, seed=4, per_view=0)
    cset = cv_b200.ConstraintSettings(constraint_patience=64)
    rset = ReconstructionSettings(optimization_iterations=64, minimum_robust_landmarks=8)
    g = regenerate_reconstruction(ctx, s["poses"], s["view_offsets"], s["view_landmarks"], s["bearings"], s["landmark_offsets"],
                                  s["observations"], settings=rset, constraint_settings=cset)
    V = len(s["view_offsets"]) - 1
    c = generate_view_constraints(ctx, s["poses"], s["view_offsets"], s["view_landmarks"], s["bearings"], s["landmark_offsets"],
                                  s["observations"], np.arange(V), settings=cset)
    cons = np.concatenate([c["constraints"][q] for q in range(V) if c["results"][q]["accepted"]])
    assert g["n_constraints"] == len(cons) > 0
    h = optimize_reconstruction(ctx, s["poses"], s["view_offsets"], s["view_landmarks"], s["bearings"], s["landmark_offsets"],
                                s["observations"], cons, settings=rset)
    for k in ("result", "poses", "view_state", "obs_state"):
        assert g[k].tobytes() == h[k].tobytes(), k


def test_repeated_calls_are_identical(ctx):
    s, _, cons = recon_scene(32, seed=6)
    a = optimize_reconstruction(ctx, s["poses"], s["view_offsets"], s["view_landmarks"], s["bearings"], s["landmark_offsets"],
                                s["observations"], cons)
    for _ in range(2):
        b = optimize_reconstruction(ctx, s["poses"], s["view_offsets"], s["view_landmarks"], s["bearings"], s["landmark_offsets"],
                                    s["observations"], cons)
        for k in ("result", "poses", "view_state", "obs_state"):
            assert a[k].tobytes() == b[k].tobytes(), k


def test_argument_errors(ctx):
    s, _, cons = recon_scene(8, seed=7, per_view=2, window=3)
    L = cv_b200._lib.load_reconstruction_library()
    call = (lambda **kw: optimize_reconstruction(ctx, s["poses"], s["view_offsets"], s["view_landmarks"], s["bearings"],
                                                 s["landmark_offsets"], s["observations"], kw.pop("cons", cons), **kw))
    with pytest.raises(cv_b200.CvbError) as e:
        call(triangulator=cv_b200.RelativeDltTriangulator())
    assert e.value.code == CVB_EUNSUPPORTED
    bad = cons.copy()
    bad[0]["views"][2] = 8
    with pytest.raises(cv_b200.CvbError) as e:
        call(cons=bad)
    assert e.value.code == CVB_EINVAL
    bad = cons.copy()
    bad[0]["views"][1] = bad[0]["views"][0]
    with pytest.raises(cv_b200.CvbError) as e:
        call(cons=bad)
    assert e.value.code == CVB_EINVAL
    # the device entry: NULL outputs, V = 0, view_offsets[V] != n_features
    cfg, tri = ReconstructionSettings(), cv_b200.LinearEigenTriangulator()
    assert L.cvb_optimize_reconstruction_dev(ctx.handle, C.addressof(cfg), C.addressof(tri.cfg), 8, None, None, None, None, 0, 0, None,
                                             None, 0, None, 0, None, None, None, None) == CVB_EINVAL
    import torch
    dev = torch.device("cuda", ctx.device)
    P = torch.from_numpy(s["poses"]).to(dev)
    vo = torch.from_numpy(s["view_offsets"].astype(np.int32)).to(dev)
    out = torch.zeros(8 * 12 + 16, dtype=torch.float64, device=dev)
    assert L.cvb_optimize_reconstruction_dev(ctx.handle, C.addressof(cfg), C.addressof(tri.cfg), 0, P.data_ptr(), vo.data_ptr(), None, None,
                                             0, 0, vo.data_ptr(), None, 0, None, 0, out.data_ptr(), out.data_ptr(), out.data_ptr(),
                                             None) == CVB_EINVAL
    n_features = int(s["view_offsets"][-1])
    torch.cuda.synchronize(dev)
    assert L.cvb_optimize_reconstruction_dev(ctx.handle, C.addressof(cfg), C.addressof(tri.cfg), 8, P.data_ptr(), vo.data_ptr(), vo.data_ptr(),
                                             P.data_ptr(), n_features + 1, 0, vo.data_ptr(), None, 0, None, 0, out.data_ptr(), out.data_ptr(),
                                             out.data_ptr(), None) == CVB_EINVAL
