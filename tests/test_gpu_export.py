"""GPU: cv-sfm's reconstruction export on the device (include/cvb200_export.h) against its oracle (oracle/ref_export.c), bit for bit.
Every operation involved is an IEEE add, multiply, divide or square root, or a triangulator that is already bit-exact, so the points,
states, colours, cameras, mean distances, normalised poses and constraints must have the oracle's bytes, and the PLY text written from the
device's outputs the oracle's characters."""
import ctypes as C
import os

import numpy as np
import pytest

import cv_b200
from cv_b200._lib import CVB_EINVAL, CVB_EUNSUPPORTED, CvbError, load_export_library
from cv_b200.export import (CAMERA_DTYPE, NORMALIZE_RESULT_DTYPE, ExportSettings, export_reconstruction, normalize_reconstruction,
                            robust_landmarks, write_ply)
from cv_b200.triangulation import LinearEigenTriangulator, MeanMeanTriangulator, RelativeDltTriangulator, SineL1Triangulator
from oracle import pyoracle_export as X
from oracle.pyoracle_reconstruction import CONSTRAINT_DTYPE
from oracle.pyoracle_tri import triangulator as otri
from tests.export_scenes import args, colors_for, exact_scene, first_view_without_robust_landmark, with_empty_view
from tests.reconstruction_scenes import recon_scene

pytestmark = pytest.mark.gpu
TRIS = {0: LinearEigenTriangulator, 1: SineL1Triangulator, 2: MeanMeanTriangulator}


@pytest.fixture(scope="module")
def ctx():
    return cv_b200.Context(0)


def _same(dev, ora):
    for k in ora:
        a, b = np.ascontiguousarray(dev[k]), np.ascontiguousarray(ora[k])
        assert a.shape == b.shape and a.tobytes() == b.tobytes(), k


def _check_all(ctx, s, cons, method=0, first_view=0, settings=None, tmp=None):
    settings = settings if settings is not None else ExportSettings()
    cfg = X.ExportCfg(robust_observation_incidence_minimum_cosine_distance=settings.robust_observation_incidence_minimum_cosine_distance,
                      robust_minimum_observations=settings.robust_minimum_observations)
    tri, ot = TRIS[method](), otri(method)
    col = colors_for(s)
    _same(robust_landmarks(ctx, *args(s), settings=settings, triangulator=tri), X.robust_landmarks(*args(s), cfg=cfg, tri=ot))
    d = export_reconstruction(ctx, *args(s), col, settings=settings, triangulator=tri)
    o = X.export_reconstruction(*args(s), col, cfg=cfg, tri=ot)
    _same(d, o)
    n_d = normalize_reconstruction(ctx, *args(s), cons, first_view=first_view, settings=settings, triangulator=tri)
    n_o = X.normalize_reconstruction(*args(s), cons, first_view=first_view, cfg=cfg, tri=ot)
    assert np.asarray(n_d["result"]).tobytes() == np.asarray(n_o["result"]).tobytes()
    _same(n_d, {"poses": n_o["poses"], "constraints": n_o["constraints"]})
    if tmp is not None:
        write_ply(os.path.join(tmp, "dev.ply"), d["points"], d["colors"], d["cameras"])
        write_ply(os.path.join(tmp, "ora.ply"), o["points"], o["colors"], o["cameras"])
        assert open(os.path.join(tmp, "dev.ply"), "rb").read() == open(os.path.join(tmp, "ora.ply"), "rb").read()
    return d, n_d


@pytest.mark.parametrize("V", [32, 128])
@pytest.mark.parametrize("method", [0, 1, 2])
def test_device_equals_oracle_bit_for_bit(ctx, V, method, tmp_path):
    s, _, cons = recon_scene(V)
    d, n = _check_all(ctx, s, cons, method, first_view=V // 3, tmp=str(tmp_path))
    assert len(d["points"]) > 0 and n["result"]["normalized"] == 1
    # the Python writer's path argument writes the same file
    p = str(tmp_path / "via_path.ply")
    export_reconstruction(ctx, *args(s), colors_for(s), path=p, triangulator=TRIS[method]())
    assert open(p, "rb").read() == open(str(tmp_path / "dev.ply"), "rb").read()


def _no_landmarks(V):
    s, _ = exact_scene(V)
    return dict(poses=s["poses"], view_offsets=np.zeros(V + 1, np.uint32), view_landmarks=np.zeros(0, np.uint32),
                bearings=np.zeros((0, 3)), landmark_offsets=np.zeros(1, np.uint32), observations=np.zeros((0, 2), np.uint32))


@pytest.mark.parametrize("case", ["no_landmarks", "one_view", "no_constraints", "empty_view", "first_view_not_robust", "first_view_last",
                                  "min_obs_2", "min_obs_above_V"])
def test_edge_cases_equal_the_oracle(ctx, case, tmp_path):
    s, _, cons = recon_scene(12, points=200)
    first, settings = 0, None
    if case == "no_landmarks":
        s = _no_landmarks(4)
        cons = cons[:0]
    elif case == "one_view":
        s, _ = exact_scene(1)
        cons = cons[:0]
    elif case == "no_constraints":
        cons = cons[:0]
    elif case == "empty_view":
        s = with_empty_view(s)
        first = 12
    elif case == "first_view_not_robust":
        s = first_view_without_robust_landmark()
        cons = cons[:0]
    elif case == "first_view_last":
        first = 11
    elif case == "min_obs_2":
        settings = ExportSettings(robust_minimum_observations=2)
    elif case == "min_obs_above_V":
        settings = ExportSettings(robust_minimum_observations=100)
    d, n = _check_all(ctx, s, cons, 0, first_view=first, settings=settings, tmp=str(tmp_path))
    if case in ("no_landmarks", "empty_view", "first_view_not_robust"):
        assert n["result"]["normalized"] == 0 and np.isnan(n["result"]["mean_distance"])
        assert n["poses"].tobytes() == np.ascontiguousarray(s["poses"]).tobytes()
    if case == "one_view":
        assert len(d["points"]) == 0   # one observation per landmark is never robust


def test_scale_above_one_resident_grid(ctx):
    """512 views and more than 1.1 M observations, with more landmarks than one H100 holds threads resident (2 048 x 132)."""
    from tests.scale_scenes import sliding_scene
    s, _ = sliding_scene(512, per_view=2700, seed=3, noise=1e-4, singles=560)
    L, n_obs = len(s["landmark_offsets"]) - 1, len(s["observations"])
    assert L > 2048 * 132 and n_obs > 1_100_000, (L, n_obs)
    col = colors_for(s)
    d = export_reconstruction(ctx, *args(s), col)
    _same(d, X.export_reconstruction(*args(s), col))
    _same(robust_landmarks(ctx, *args(s)), X.robust_landmarks(*args(s)))
    n_d = normalize_reconstruction(ctx, *args(s), np.zeros(0, CONSTRAINT_DTYPE), first_view=200)
    n_o = X.normalize_reconstruction(*args(s), np.zeros(0, CONSTRAINT_DTYPE), first_view=200)
    assert np.asarray(n_d["result"]).tobytes() == np.asarray(n_o["result"]).tobytes() and n_d["poses"].tobytes() == n_o["poses"].tobytes()


def _dev_calls(ctx, s, cons, col, first_view, tri):
    """the three _dev entry points on torch device tensors; returns host copies in the host forms' layout"""
    import torch
    dev = torch.device("cuda", ctx.device)
    t = (lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dt).reshape(-1).copy()).to(dev))
    P, vo, vl = t(s["poses"], np.float64), t(s["view_offsets"], np.uint32), t(s["view_landmarks"], np.uint32)
    bear, lo, ob = t(s["bearings"], np.float64), t(s["landmark_offsets"], np.uint32), t(s["observations"], np.uint32)
    colt = t(col, np.uint8)
    consb = t(np.ascontiguousarray(cons, CONSTRAINT_DTYPE).view(np.uint8), np.uint8)
    V, Lm, nf, no = len(s["view_offsets"]) - 1, len(s["landmark_offsets"]) - 1, len(s["view_landmarks"]), len(s["observations"])
    ptr = (lambda x: x.data_ptr() if x.numel() else None)
    lib, st = load_export_library(), ExportSettings()
    pts4 = torch.zeros(max(Lm, 1) * 4, dtype=torch.float64, device=dev)
    state = torch.zeros(max(Lm, 1), dtype=torch.uint8, device=dev)
    torch.cuda.synchronize(dev)
    ctx.check(lib.cvb_robust_landmarks_dev(ctx.handle, C.addressof(st), C.addressof(tri.cfg), V, ptr(P), ptr(vo), ptr(vl), ptr(bear), nf, Lm,
                                           ptr(lo), ptr(ob), no, pts4.data_ptr(), state.data_ptr()))
    pout = torch.zeros(max(V, 1) * 12, dtype=torch.float64, device=dev)
    cout = torch.zeros(max(len(cons), 1) * CONSTRAINT_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    res = torch.zeros(NORMALIZE_RESULT_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    ctx.check(lib.cvb_normalize_reconstruction_dev(ctx.handle, C.addressof(st), C.addressof(tri.cfg), V, ptr(P), ptr(vo), ptr(vl), ptr(bear),
                                                   nf, Lm, ptr(lo), ptr(ob), no, ptr(consb), len(cons), first_view, pout.data_ptr(),
                                                   cout.data_ptr(), res.data_ptr()))
    # the export runs on the normalised poses without leaving the device
    pts = torch.zeros(max(Lm, 1) * 3, dtype=torch.float64, device=dev)
    pcol = torch.zeros(max(Lm, 1) * 3, dtype=torch.uint8, device=dev)
    npt = torch.zeros(1, dtype=torch.int32, device=dev)
    cams = torch.zeros(max(V, 1) * CAMERA_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    mean = torch.zeros(max(V, 1), dtype=torch.float64, device=dev)
    ctx.check(lib.cvb_export_reconstruction_dev(ctx.handle, C.addressof(st), C.addressof(tri.cfg), V, pout.data_ptr(), ptr(vo), ptr(vl),
                                                ptr(bear), ptr(colt), nf, Lm, ptr(lo), ptr(ob), no, pts.data_ptr(), pcol.data_ptr(),
                                                npt.data_ptr(), cams.data_ptr(), mean.data_ptr()))
    n = int(npt.item())
    return (dict(points=pts4.cpu().numpy().reshape(-1, 4)[:Lm], state=state.cpu().numpy()[:Lm]),
            dict(result=res.cpu().numpy().view(NORMALIZE_RESULT_DTYPE)[0], poses=pout.cpu().numpy().reshape(-1, 12)[:V],
                 constraints=cout.cpu().numpy().view(CONSTRAINT_DTYPE)[:len(cons)]),
            dict(points=pts.cpu().numpy().reshape(-1, 3)[:n], colors=pcol.cpu().numpy().reshape(-1, 3)[:n],
                 cameras=cams.cpu().numpy().view(CAMERA_DTYPE)[:V], mean_distance=mean.cpu().numpy()[:V]))


@pytest.mark.parametrize("method", [0, 1])
def test_dev_forms_equal_host_forms_and_chain_on_device(ctx, method):
    s, _, cons = recon_scene(32)
    col = colors_for(s)
    tri = TRIS[method]()
    r_d, n_d, e_d = _dev_calls(ctx, s, cons, col, 7, tri)
    _same(r_d, robust_landmarks(ctx, *args(s), triangulator=tri))
    n_h = normalize_reconstruction(ctx, *args(s), cons, first_view=7, triangulator=tri)
    assert np.asarray(n_d["result"]).tobytes() == np.asarray(n_h["result"]).tobytes()
    _same(n_d, {"poses": n_h["poses"], "constraints": n_h["constraints"]})
    s2 = dict(s, poses=n_h["poses"])
    _same(e_d, export_reconstruction(ctx, *args(s2), col, triangulator=tri))


def test_chain_on_regenerate_reconstruction_outputs(ctx):
    """normalize then export on the poses regenerate_reconstruction leaves (constraints, pose graph and filter all on the device) equal
    the host chain through the oracles"""
    s, _, _ = recon_scene(32)
    out = cv_b200.regenerate_reconstruction(ctx, *(s[k] for k in ("poses", "view_offsets", "view_landmarks", "bearings", "landmark_offsets",
                                                                   "observations")))
    s2 = dict(s, poses=out["poses"])
    col = colors_for(s)
    cons = np.zeros(0, CONSTRAINT_DTYPE)
    _, n_d, e_d = _dev_calls(ctx, s2, cons, col, 0, LinearEigenTriangulator())
    n_o = X.normalize_reconstruction(*args(s2), cons, first_view=0)
    _same(n_d, {"poses": n_o["poses"]})
    _same(e_d, X.export_reconstruction(*args(dict(s2, poses=n_o["poses"])), col))


def test_repeated_calls_are_identical(ctx):
    s, _, cons = recon_scene(32)
    col = colors_for(s)
    a = [export_reconstruction(ctx, *args(s), col, triangulator=SineL1Triangulator()) for _ in range(3)]
    b = [normalize_reconstruction(ctx, *args(s), cons, first_view=3) for _ in range(3)]
    for x in a[1:]:
        _same(x, a[0])
    for x in b[1:]:
        assert np.asarray(x["result"]).tobytes() == np.asarray(b[0]["result"]).tobytes()
        _same(x, {"poses": b[0]["poses"], "constraints": b[0]["constraints"]})


def test_argument_errors(ctx):
    s, _, cons = recon_scene(8, points=100)
    col = colors_for(s)
    for tri in (RelativeDltTriangulator(),):
        with pytest.raises(CvbError) as e:
            export_reconstruction(ctx, *args(s), col, triangulator=tri)
        assert e.value.code == CVB_EUNSUPPORTED
    from cv_b200.triangulation import AngularL1Triangulator, AngularLInfinityTriangulator
    for tri in (AngularL1Triangulator(), AngularLInfinityTriangulator()):
        for f in (lambda t: robust_landmarks(ctx, *args(s), triangulator=t), lambda t: normalize_reconstruction(ctx, *args(s), cons, triangulator=t)):
            with pytest.raises(CvbError) as e:
                f(tri)
            assert e.value.code == CVB_EUNSUPPORTED
    for first in (8, 1 << 20):
        with pytest.raises(CvbError) as e:
            normalize_reconstruction(ctx, *args(s), cons, first_view=first)
        assert e.value.code == CVB_EINVAL
    lib, st, tri = load_export_library(), ExportSettings(), LinearEigenTriangulator()
    # V = 0 and NULL device arguments
    assert lib.cvb_robust_landmarks_dev(ctx.handle, C.addressof(st), C.addressof(tri.cfg), 0, 1, 1, None, None, 0, 0, 1, None, 0, None,
                                        None) == CVB_EINVAL
    assert lib.cvb_export_reconstruction_dev(ctx.handle, None, C.addressof(tri.cfg), 1, 1, 1, None, None, None, 0, 0, 1, None, 0, None, None,
                                             1, 1, None) == CVB_EINVAL
    assert lib.cvb_normalize_reconstruction_dev(ctx.handle, C.addressof(st), C.addressof(tri.cfg), 2, 1, 1, None, None, 0, 0, 1, None, 0,
                                                None, 0, 2, 1, None, 1) == CVB_EINVAL
    assert lib.cvb_normalize_reconstruction_dev(ctx.handle, C.addressof(st), C.addressof(tri.cfg), 2, None, 1, None, None, 0, 0, 1, None, 0,
                                                None, 0, 0, 1, None, 1) == CVB_EINVAL
