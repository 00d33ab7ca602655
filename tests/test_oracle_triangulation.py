"""CPU-only: the oracle of cv-geom's triangulators (oracle/ref_triangulation.c) against the reference's own checks and against
independent numpy transcriptions.

  cv-geom/src/triangulation.rs:26-38,150-162,371-388,452-468,538-554   doc-tests: (0.3, 0.1, 2.0) recovered to 1e-6 (MeanMean 1e-2)
  cv-geom/src/triangulation.rs:651-680                                  RelativeDlt = the SVD null vector, 100 random cases
"""
import numpy as np
import pytest

from oracle import pyoracle as O
from oracle import pyoracle_tri as T


def rot(v):
    """Rotation3::new / from_scaled_axis (Rodrigues)"""
    v = np.asarray(v, np.float64)
    th = np.linalg.norm(v)
    if th == 0.0:
        return np.eye(3)
    k = v / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K


def from_homogeneous(p):
    p = np.asarray(p, np.float64)
    if np.signbit(p[3]):
        p = -p
    return p / np.linalg.norm(p[:3])


def doc_scene():
    R, t = rot([0.1, 0.1, 0.1]), np.array([0.1, 0.1, 0.1])
    point = np.array([0.3, 0.1, 2.0])
    a = point / np.linalg.norm(point)
    q = R @ point + t
    return (R, t), point, a, q / np.linalg.norm(q)


@pytest.mark.parametrize("method,tol", [(T.LINEAR_EIGEN, 1e-6), (T.SINE_L1, 1e-6), (T.MEAN_MEAN, 1e-2), (T.RELATIVE_DLT, 1e-6),
                                        (T.ANGULAR_L1, 1e-6), (T.ANGULAR_LINF, 1e-6)])
def test_doc_tests(method, tol):
    pose, point, a, b = doc_scene()
    got = T.triangulate_relative(T.triangulator(method), pose, a, b)
    assert got is not None and got[3] > 0
    assert np.linalg.norm(got[:3] / got[3] - point) < tol


def test_defaults_follow_the_default_impls_not_the_doc_comments():
    s = T.triangulator(T.SINE_L1)
    assert (s.epsilon, s.max_iterations, s.optimization_rate) == (1e-12, 1000, 1.0)
    d = T.triangulator(T.RELATIVE_DLT)
    assert (d.epsilon, d.max_iterations) == (1e-12, 1000)


def _design(R, t, a, b):
    P = np.hstack([R, t[:, None]])
    return np.array([[-a[2], 0.0, a[0], 0.0], [0.0, -a[2], a[1], 0.0], b[0] * P[2] - b[2] * P[0], b[1] * P[2] - b[2] * P[1]])


def test_relative_dlt_is_the_svd_null_vector():
    """triangulation.rs:651-680: 100 random (pose, homogeneous point) cases; the point equals the right singular vector of the smallest
    singular value of the design matrix (numpy's SVD) to 1e-9, and None exactly where that vector fails the cheirality test"""
    rng = np.random.default_rng(651)
    tri = T.triangulator(T.RELATIVE_DLT)
    checked = 0
    for _ in range(100):
        R, t = rot(rng.random(3)), rng.random(3)
        X = from_homogeneous(rng.random(4))
        a = X[:3]
        q = R @ X[:3] + t * X[3]
        b = q / np.linalg.norm(q)
        want = from_homogeneous(np.linalg.svd(_design(R, t, a, b))[2][3])
        front = not np.signbit(want[:3] @ a) and not np.signbit(want[:3] @ (R.T @ b))
        got = T.triangulate_relative(tri, (R, t), a, b)
        assert (got is not None) == front
        if got is not None:
            assert np.abs(got - want).max() < 1e-9, (got, want)
            assert np.abs(got - X).max() < 1e-6
            checked += 1
    assert checked > 50


# ---- independent numpy transcriptions (same operation order as the reference's nalgebra code)
def np_mean_mean(poses, bearings):
    n = len(poses)
    cs = [R.T @ -t for R, t in poses]
    wbs = [R.T @ b for (R, _), b in zip(poses, bearings)]
    with np.errstate(all="ignore"):
        total = float(n)
        ac = (np.sum(cs, axis=0) if n else np.zeros(3)) / total
        sb = np.sum(wbs, axis=0) if n else np.zeros(3)
        ab = sb / np.linalg.norm(sb)
        s = 0.0
        for c, wb in zip(cs, wbs):
            q = np.cross(ab, wb)
            s += (q * (1.0 / (q @ q))) @ np.cross(wb, ac - c)
        w = 1.0 / (s / total)
        p = from_homogeneous(np.append(ab + ac * w, w))
    if not np.isfinite(p).all() or any(np.signbit(wb @ p[:3]) for wb in wbs):
        return None
    return p


def np_angular(linf, R, t, a_in, b_in):
    with np.errstate(all="ignore"):
        a, b, tt = R.T @ b_in, np.asarray(a_in, np.float64), R.T @ -t
        nt = tt / np.linalg.norm(tt)
        if not linf:
            ca, cb = np.cross(a, nt), np.cross(b, nt)
            if np.linalg.norm(ca) < np.linalg.norm(cb):
                nb = cb / np.linalg.norm(cb)
                v = a - (a @ nb) * nb
                a = v / np.linalg.norm(v)
            else:
                na = ca / np.linalg.norm(ca)
                v = b - (b @ na) * na
                b = v / np.linalg.norm(v)
        else:
            na, nb = np.cross(a + b, nt), np.cross(a - b, nt)
            n = na / np.sqrt(na @ na) if na @ na > nb @ nb else nb / np.sqrt(nb @ nb)
            va, vb = a - (a @ n) * n, b - (b @ n) * n
            a, b = va / np.linalg.norm(va), vb / np.linalg.norm(vb)
        z = np.cross(b, a)
        p = from_homogeneous(np.append(b, (z @ z) / (z @ np.cross(tt, a))))
    if not np.isfinite(p).all() or np.signbit(p[:3] @ a) or np.signbit(p[:3] @ b):
        return None
    return p


def _random_views(rng, n):
    X = rng.uniform([-2, -2, 4], [2, 2, 8])
    poses, bearings = [], []
    for _ in range(n):
        R, t = rot(rng.normal(0, 0.1, 3)), rng.normal(0, 0.5, 3)
        q = R @ X + t
        b = q / np.linalg.norm(q) + rng.normal(0, 1e-3, 3)
        poses.append((R, t)); bearings.append(b / np.linalg.norm(b))
    return poses, np.array(bearings).reshape(-1, 3)


def _close(got, want, tol=1e-12):
    assert (got is None) == (want is None), (got, want)
    if got is not None:
        assert np.abs(got - want).max() < tol, (got, want)


def test_mean_mean_matches_numpy():
    rng = np.random.default_rng(389)
    tri = T.triangulator(T.MEAN_MEAN)
    some = 0
    for n in [2, 3, 5, 8] * 25:
        poses, bearings = _random_views(rng, n)
        out, ok, _ = T.triangulate_observations_batch(tri, poses, bearings, [0, n])
        want = np_mean_mean(poses, bearings)
        _close(out[0] if ok[0] else None, want)
        some += want is not None
    assert some > 50


@pytest.mark.parametrize("linf", [False, True])
def test_angular_matches_numpy(linf):
    rng = np.random.default_rng(469 + linf)
    tri = T.triangulator(T.ANGULAR_LINF if linf else T.ANGULAR_L1)
    some = 0
    for _ in range(200):
        poses, bearings = _random_views(rng, 2)
        (R0, t0), (R1, t1) = poses
        Rr, tr = R1 @ R0.T, t1 - R1 @ R0.T @ t0     # CameraToCamera from view 0 to view 1
        a, b = bearings
        want = np_angular(linf, Rr, tr, a, b)
        _close(T.triangulate_relative(tri, (Rr, tr), a, b), want)
        some += want is not None
    assert some > 100


def test_degenerate_inputs_are_none():
    """MeanMean with 0 or 1 observations, and MeanMean / AngularL1 / AngularL-infinity on a zero baseline, parallel bearings or a NaN
    bearing, return None (MeanMean divides by zero and its finiteness filter catches it)"""
    pose, _, a, b = doc_scene()
    I = (np.eye(3), np.zeros(3))
    for m in (T.LINEAR_EIGEN, T.SINE_L1, T.MEAN_MEAN):
        out, ok, _ = T.triangulate_observations_batch(T.triangulator(m), [pose], [b], [0, 0, 1])   # zero and one observation
        assert not ok.any() and not out.any()
    nan = np.full(3, np.nan)
    for m in (T.MEAN_MEAN, T.ANGULAR_L1, T.ANGULAR_LINF):
        tri = T.triangulator(m)
        assert T.triangulate_relative(tri, I, a, a) is None                     # zero baseline, one ray
        assert T.triangulate_relative(tri, I, a, b) is None                     # zero baseline
        assert T.triangulate_relative(tri, (np.eye(3), np.array([1.0, 0, 0])), a, a) is None   # parallel bearings
        assert T.triangulate_relative(tri, pose, a, nan) is None


def test_linear_eigen_default_and_filters_equal_the_existing_oracle():
    """ref_triangulation.c restates LinearEigen with its settings and cv-sfm's two filters with a triangulator argument; with
    LinearEigen's Default they are bit for bit ref_geom.c's ref_triangulate_linear_eigen and ref_optimize.c's filters"""
    rng = np.random.default_rng(130)
    tri = T.triangulator(T.LINEAR_EIGEN)
    some = 0
    for n in [0, 1, 2, 3, 4, 6, 8] * 30:
        poses, bearings = _random_views(rng, n) if n else ([], np.zeros((0, 3)))
        if n and rng.random() < 0.2:
            bearings[-1] = -bearings[-1]
        out, ok, _ = T.triangulate_observations_batch(tri, poses, bearings, [0, n])
        want = O.triangulate_linear_eigen(poses, bearings) if n else None
        assert bool(ok[0]) == (want is not None)
        if want is not None:
            assert out[0].tobytes() == want.tobytes()
            some += 1
        if n:
            assert T.observation_losses(tri, poses, bearings, [0, n]).tobytes() == O.observation_losses(poses, bearings).tobytes()
    assert some > 50
    for _ in range(200):
        poses, bearings = _random_views(rng, 3)
        (R0, t0), (R1, t1), (R2, t2) = poses
        first, second = (R1 @ R0.T, t1 - R1 @ R0.T @ t0), (R2 @ R0.T, t2 - R2 @ R0.T @ t0)
        for mc, inc in ((1e-5, 1e-6), (1e-6, 1e-3)):
            want = O.is_tri_landmark_robust(first, second, bearings[0], bearings[1], bearings[2], mc, inc)
            assert T.tri_landmarks_robust(tri, first, second, bearings.reshape(1, 9), mc, inc)[0] == want
