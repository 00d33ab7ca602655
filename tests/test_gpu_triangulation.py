"""GPU parity for cv-geom's triangulators (include/cvb200_tri.h): every method equals the CPU oracle (oracle/ref_triangulation.c)
bit for bit on seeded batches of more than 10k items that include degenerate and failing cases.  Both sides use only +, -, x, / and
sqrt in f64 without contraction (the library is built with -fmad=false, the oracle with -ffp-contract=off)."""
import ctypes as C

import numpy as np
import pytest

import cv_b200
from cv_b200.geom import POSE_DTYPE
from oracle import pyoracle_tri as T
from tests.geom_util import rot_from_scaled_axis, three_view_scene, unit

pytestmark = pytest.mark.gpu

OBS_CLASSES = [cv_b200.LinearEigenTriangulator, cv_b200.SineL1Triangulator, cv_b200.MeanMeanTriangulator]
REL_CLASSES = OBS_CLASSES + [cv_b200.RelativeDltTriangulator, cv_b200.AngularL1Triangulator, cv_b200.AngularLInfinityTriangulator]


def _oracle_cfg(tri):
    c = tri.cfg
    return T.triangulator(c.method, c.epsilon, c.max_iterations, c.optimization_rate)


def _pose_arr(Rs, ts):
    p = np.zeros(len(Rs), POSE_DTYPE)
    p["r"] = np.asarray(Rs).reshape(-1, 9); p["t"] = ts
    return p


def observation_batch(rng, L=12000):
    """L landmarks of 0..8 observations; every tenth kind is a degenerate one"""
    Rs, ts, bs, off = [], [], [], [0]
    d_par = unit(rng.normal(size=3))
    for l in range(L):
        kind = l % 10
        X = rng.uniform([-3, -3, 2], [3, 3, 12])
        n = int(rng.integers(0, 2)) if kind == 0 else int(rng.integers(2, 9))
        for k in range(n):
            R = rot_from_scaled_axis(rng.normal(0, 0.2, 3))
            t = np.zeros(3) if kind == 1 else rng.normal(0, 1.0, 3)    # kind 1: zero baseline (every centre at the origin: w = 0)
            b = unit(R @ X + t + rng.normal(0, 1e-3, 3))
            if kind == 2 and k == n - 1:
                b = -b                                                  # behind one camera
            if kind == 3:
                b = R @ d_par                                           # parallel bearings
            if kind == 4 and k == 0:
                b = np.full(3, np.nan)                                  # NaN-producing
            if kind == 5 and k == 0:
                b = np.zeros(3)
            Rs.append(R); ts.append(t); bs.append(b)
        off.append(len(bs))
    return _pose_arr(Rs, ts), np.array(bs, np.float64).reshape(-1, 3), np.array(off, np.uint32)


def relative_batch(rng, n=12000):
    Rs, ts, As, Bs = [], [], [], []
    for i in range(n):
        kind = i % 8
        X = rng.uniform([-3, -3, 2], [3, 3, 12])
        R = rot_from_scaled_axis(rng.normal(0, 0.2, 3))
        t = np.zeros(3) if kind == 1 else rng.normal(0, 1.0, 3)
        a = unit(X + rng.normal(0, 1e-3, 3)); b = unit(R @ X + t + rng.normal(0, 1e-3, 3))
        if kind == 2:
            b = -b
        if kind == 3:
            b = R @ a                                                   # parallel bearings
        if kind == 4:
            b = np.full(3, np.nan)
        if kind == 5:
            a = unit(rng.normal(size=3))                                # unrelated rays, often behind
        Rs.append(R); ts.append(t); As.append(a); Bs.append(b)
    return _pose_arr(Rs, ts), np.array(As), np.array(Bs)


@pytest.fixture(scope="module")
def obs_data():
    return observation_batch(np.random.default_rng(82))


@pytest.fixture(scope="module")
def rel_data():
    return relative_batch(np.random.default_rng(322))


@pytest.mark.parametrize("cls", OBS_CLASSES + [lambda: cv_b200.SineL1Triangulator(1e-9, 50, 0.5), lambda: cv_b200.LinearEigenTriangulator(1e-8, 5)])
def test_observations_bit_equal_to_oracle(cls, obs_data):
    poses, bearings, off = obs_data
    tri = cls()
    got, ok = tri.triangulate_batch(poses, bearings, off)
    want, wok, _ = T.triangulate_observations_batch(_oracle_cfg(tri), poses, bearings, off)
    assert np.array_equal(ok, wok) and got.tobytes() == want.tobytes()
    assert 0.2 < ok.mean() < 0.95, ok.mean()          # both outcomes well represented
    assert not ok[np.diff(off.astype(np.int64)) < 2].any()


@pytest.mark.parametrize("shared", [True, False])
@pytest.mark.parametrize("cls", REL_CLASSES)
def test_relative_bit_equal_to_oracle(cls, shared, rel_data):
    poses, a, b = rel_data
    if shared:
        poses = poses[:1]
    tri = cls()
    got, ok = tri.triangulate_relative_batch(poses, a, b)
    want, wok = T.triangulate_relative_batch(_oracle_cfg(tri), poses, a, b)
    assert np.array_equal(ok, wok) and got.tobytes() == want.tobytes()
    assert ok.any() and not ok.all()
    assert not got[~ok].any()


def test_observations_entry_point_equals_linear_eigen_entry_point(obs_data):
    poses, bearings, off = obs_data
    got, ok = cv_b200.LinearEigenTriangulator().triangulate_batch(poses, bearings, off)
    ctx = cv_b200._lib.default_context(0)
    L = ctx.lib
    L.cvb_triangulate_linear_eigen.argtypes = [C.c_void_p] * 4 + [C.c_uint32, C.c_void_p, C.c_void_p]
    nl = len(off) - 1
    out = np.zeros((nl, 4)); ok2 = np.zeros(nl, np.uint8)
    ctx.check(L.cvb_triangulate_linear_eigen(ctx.handle, poses.ctypes.data, bearings.ctypes.data, off.ctypes.data, nl, out.ctypes.data,
                                             ok2.ctypes.data))
    assert np.array_equal(ok, ok2.astype(bool)) and got.tobytes() == out.tobytes()


def _from_homogeneous(p):
    p = -p if np.signbit(p[3]) else p
    return p / np.sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2])


@pytest.mark.parametrize("cls", OBS_CLASSES)
def test_relative_form_is_the_blanket_impl(cls, rel_data):
    poses, a, b = rel_data
    n = 3000
    tri = cls()
    got, ok = tri.triangulate_relative_batch(poses[:n], a[:n], b[:n])
    ident = _pose_arr([np.eye(3)] * n, np.zeros((n, 3)))
    obs_poses = np.empty(2 * n, POSE_DTYPE); obs_poses[0::2] = ident; obs_poses[1::2] = poses[:n]
    obs_b = np.empty((2 * n, 3)); obs_b[0::2] = a[:n]; obs_b[1::2] = b[:n]
    w, wok = tri.triangulate_batch(obs_poses, obs_b, np.arange(0, 2 * n + 1, 2, dtype=np.uint32))
    assert np.array_equal(ok, wok)
    want = np.array([_from_homogeneous(p) if k else np.zeros(4) for p, k in zip(w, wok)])
    assert got.tobytes() == want.tobytes()


@pytest.mark.parametrize("cls,tol", [(cv_b200.LinearEigenTriangulator, 1e-6), (cv_b200.SineL1Triangulator, 1e-6), (cv_b200.MeanMeanTriangulator, 1e-2),
                                     (cv_b200.RelativeDltTriangulator, 1e-6), (cv_b200.AngularL1Triangulator, 1e-6),
                                     (cv_b200.AngularLInfinityTriangulator, 1e-6)])
def test_doc_tests_on_the_device(cls, tol):
    """cv-geom/src/triangulation.rs:26-38,150-162,371-388,452-468,538-554"""
    R, t = rot_from_scaled_axis(np.array([0.1, 0.1, 0.1])), np.array([0.1, 0.1, 0.1])
    point = np.array([0.3, 0.1, 2.0])
    got = cls().triangulate_relative((R, t), unit(point), unit(R @ point + t))
    assert got is not None and np.linalg.norm(got[:3] / got[3] - point) < tol


def test_losses_and_robustness_with_a_triangulator(obs_data):
    poses, bearings, off = obs_data
    L = 3000
    p, b, o = poses[:off[L]], bearings[:off[L]], off[:L + 1]
    base = cv_b200.observation_losses(p, b, o)
    assert base.tobytes() == cv_b200.observation_losses(p, b, o, triangulator=cv_b200.LinearEigenTriangulator()).tobytes()
    cnt = np.diff(o.astype(np.int64))
    three = np.repeat(cnt >= 3, cnt)
    for tri in (cv_b200.SineL1Triangulator(), cv_b200.MeanMeanTriangulator()):
        got = cv_b200.observation_losses(p, b, o, triangulator=tri)
        want = T.observation_losses(_oracle_cfg(tri), p, b, o)
        assert got[three].tobytes() == want[three].tobytes()                 # the triangulated landmarks: bit for bit
        assert np.allclose(got[~three], want[~three], rtol=1e-9, atol=1e-14)  # two views go through asin / cos
        assert (got[three] < 2.0).sum() > 1000
    rng = np.random.default_rng(1332)
    tposes, obs = three_view_scene(rng, 4000, noise=1.5e-3)
    obs = np.array(obs).reshape(-1, 9)
    obs[::97, 0:3] = -obs[::97, 0:3]
    args = (tposes[0], tposes[1], obs, 1e-5, 1e-3)
    base = cv_b200.tri_landmarks_robust(*args)
    assert np.array_equal(base, cv_b200.tri_landmarks_robust(*args, triangulator=cv_b200.LinearEigenTriangulator()))
    for tri in (cv_b200.SineL1Triangulator(), cv_b200.MeanMeanTriangulator()):
        got = cv_b200.tri_landmarks_robust(*args, triangulator=tri)
        assert np.array_equal(got, T.tri_landmarks_robust(_oracle_cfg(tri), *args))
        assert 0 < got.sum() < len(got)


def test_relative_only_methods_are_rejected_by_the_observations_entry_points(obs_data):
    poses, bearings, off = obs_data
    for tri in (cv_b200.RelativeDltTriangulator(), cv_b200.AngularL1Triangulator()):
        with pytest.raises(cv_b200.CvbError) as e:
            cv_b200.observation_losses(poses[:off[10]], bearings[:off[10]], off[:11], triangulator=tri)
        assert e.value.code == cv_b200._lib.CVB_EINVAL
    with pytest.raises(ValueError):
        cv_b200.AngularL1Triangulator().triangulate_relative_batch(poses[:3], bearings[:5], bearings[:5])
