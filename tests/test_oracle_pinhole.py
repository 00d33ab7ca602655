"""CPU-only: the oracle of include/cvb200_pinhole.h (oracle/ref_pinhole.c).  Its essential routines from ref_geom.c are already pinned by
tests/test_oracle_geom.py (random.rs, essential.rs:93-113 and 197-216); this file covers what is new:

  cv-pinhole/src/lib.rs:291-313, 344-364   pose_reprojection_error / average_pose_reprojection_error doc-tests (< 1e-6, LinearEigen)
  cv-pinhole/src/essential.rs:168-183      the possible_rotations doc-test
  the reprojection error equals a numpy transcription of lib.rs:314-372 over the oracle's own triangulated points, every triangulator
  EssentialMatrix::recondition equals a numpy-SVD restatement (recondition does not depend on the SVD's sign conventions)"""
import numpy as np
import pytest

from oracle import pyoracle_pinhole as O
from oracle import pyoracle_tri as T
from tests.geom_util import rot_angle, skew, unit
from tests.pinhole_cases import DOC_POSE, essential_batch, reprojection_batch

METHODS = [T.LINEAR_EIGEN, T.SINE_L1, T.MEAN_MEAN, T.RELATIVE_DLT, T.ANGULAR_L1, T.ANGULAR_LINF]


def test_reprojection_doc_tests():
    pa = np.array([0.4, -0.25, 5.0]); R, t = np.eye(3), np.array([0.1, 0.2, -0.5])
    a, b = unit(pa)[None], unit(R @ pa + t)[None]
    err, avg, ok = O.pose_reprojection_error_batch(T.triangulator(T.LINEAR_EIGEN), [(R, t)], a, b)
    assert ok[0] and avg[0] < 1e-6
    assert np.linalg.norm(err[0].reshape(2, 2), axis=1).sum() * 0.5 == avg[0]


def _numpy_reprojection(poses, a, b, xyzw):
    """lib.rs:314-341 transcribed on the triangulated CameraPoints xyzw"""
    with np.errstate(divide="ignore", invalid="ignore"):
        an, bn = a[:, :2] / a[:, 2:3], b[:, :2] / b[:, 2:3]
        R = poses["r"].reshape(-1, 3, 3); t = poses["t"]
        q = np.einsum("nij,nj->ni", R, xyzw[:, :3]) + t * xyzw[:, 3:4]
        q = q / np.linalg.norm(q, axis=1, keepdims=True)               # w >= 0 already: from_homogeneous only normalises
        ea = an - xyzw[:, :2] / xyzw[:, 2:3]; eb = bn - q[:, :2] / q[:, 2:3]
    ok = ~np.signbit(xyzw[:, 2]) & ~np.signbit(q[:, 2])
    return np.concatenate([ea, eb], 1), ok


@pytest.mark.parametrize("method", METHODS)
def test_reprojection_equals_numpy_transcription(method):
    Rs, ts, a, b = reprojection_batch(np.random.default_rng(3), 3000)
    poses = np.zeros(len(Rs), T.POSE_DTYPE); poses["r"] = Rs.reshape(-1, 9); poses["t"] = ts
    tri = T.triangulator(method)
    err, avg, ok = O.pose_reprojection_error_batch(tri, poses, a, b)
    xyzw, tok = T.triangulate_relative_batch(tri, poses, a, b)
    want, wok = _numpy_reprojection(poses, a, b, xyzw)
    assert np.isnan(err[~ok]).all() and np.isnan(avg[~ok]).all()
    assert not (ok & ~tok).any()
    # non-degenerate rows (the kinds without a zero, NaN, parallel or behind-the-camera bearing): where the sign tests cannot flip on
    # rounding, ok and the errors agree with the transcription
    normal = np.isin(np.arange(len(ok)) % 10, [0, 9])
    assert np.array_equal(ok[normal], (tok & wok)[normal])
    fin = ok & normal
    assert fin.sum() > 0.9 * normal.sum()
    with np.errstate(divide="ignore", invalid="ignore"):
        rep = np.concatenate([a[:, :2] / a[:, 2:3], b[:, :2] / b[:, 2:3]], 1) - want      # the reprojected coordinates
    assert (np.abs(err[fin] - want[fin]) <= 1e-12 * np.maximum(1.0, np.abs(rep[fin]))).all()
    e = err[ok]
    assert np.array_equal(avg[ok], ((0.0 + np.sqrt(e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1])) + np.sqrt(e[:, 2] * e[:, 2] + e[:, 3] * e[:, 3])) * 0.5,
                          equal_nan=True)
    if method == T.LINEAR_EIGEN:
        assert np.median(avg[fin]) < 1e-2


def test_reprojection_sign_tests():
    """a bearing whose z is +0.0 passes the reference's is_sign_positive test and reaches the error as an infinity; -0.0 does not"""
    R, t = np.eye(3), np.array([1.0, 0.0, 0.0])
    X = np.array([0.3, -0.2, 4.0])
    a, b = unit(X), unit(X + t)
    tri = T.triangulator(T.LINEAR_EIGEN)
    a0 = a.copy(); a0[2] = 0.0
    a1 = a.copy(); a1[2] = -0.0
    err, avg, ok = O.pose_reprojection_error_batch(tri, [(R, t)], np.array([a, a0, a1]), np.array([b, b, b]))
    assert ok[0] and avg[0] < 1e-9
    for k in (1, 2):   # a's own z only enters a_norm: the point itself may still be triangulated in front
        assert not ok[k] or (np.isinf(err[k, 0]) and np.signbit(err[k, 0]) != (k == 1) or np.isnan(err[k, 0]))


def test_possible_rotations_doc_test():
    # essential.rs:168-183
    R, t = DOC_POSE
    ra, rb, tt, ok = O.essential_decompose_batch(skew(t) @ R, 1e-6, 50)
    assert ok[0]
    assert any(rot_angle(r, R) < 1e-4 for r in (ra[0], rb[0]))


def _numpy_recondition(E):
    U, s, Vt = np.linalg.svd(E)
    m = (s[0] + s[1]) / 2.0
    return U @ np.diag([m, m, 0.0]) @ Vt


def test_recondition_equals_numpy_svd():
    Es = essential_batch(np.random.default_rng(5), 2048)
    keep = np.isin(np.arange(len(Es)) % 8, [0, 1, 4, 6, 7])             # well-separated s0, s1 (E of a pose, noisy or scaled)
    out, ok = O.essential_recondition_batch(Es, 1e-12, 1000)
    assert ok[keep].all()
    for E, R in zip(Es[keep], out[keep]):
        assert np.abs(R - _numpy_recondition(E)).max() <= 1e-12 * np.linalg.norm(E, 2)
    assert not ok[2::8].any() and not ok[3::8].any()                    # exactly rank one, zero: no decomposition (documented)
    assert np.isnan(out[~ok]).all()
    _, ok0 = O.essential_recondition_batch(Es[:16], 1e-12, 0)            # no sweep: no result
    assert not ok0.any()


def test_recondition_is_an_essential_matrix_and_a_fixed_point():
    R, t = DOC_POSE
    E = skew(t) @ R + np.random.default_rng(9).normal(0, 1e-2, (3, 3))
    (Er,), ok = O.essential_recondition_batch(E, 1e-12, 1000)
    s = np.linalg.svd(Er, compute_uv=False)
    assert ok[0] and abs(s[0] - s[1]) < 1e-12 * s[0] and s[2] < 1e-12 * s[0]
    (Er2,), _ = O.essential_recondition_batch(Er, 1e-12, 1000)
    assert np.abs(Er2 - Er).max() < 1e-12 * np.abs(Er).max()
