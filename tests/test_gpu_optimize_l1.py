"""GPU parity of cv-optimize's L1 (Weiszfeld) optimizers (include/cvb200_opt.h) with the CPU oracle (oracle/ref_optimize_l1.c).
The device adds the per-iteration sums in its own fixed order and its sin / cos are not glibc's, so results agree to rounding, not bit for
bit: every problem is compared with the oracle in the device's summation order and in the reference's landmark order, with the
tolerances measured on the CPU for these batches (tests/opt_l1_cases.py)."""
import numpy as np
import pytest

import cv_b200
from oracle import pyoracle_opt as P
from tests import opt_l1_cases as K

pytestmark = pytest.mark.gpu


def _diff(p, q):
    return max(np.abs(p[0] - q[0]).max(), np.abs(p[1] - q[1]).max())


@pytest.mark.parametrize("eps", K.EPSILONS)
def test_single_view_l1_batch_matches_oracle(eps):
    poses, B, W, off = K.single_view_batch()
    assert (W[:, 3] == 0).sum() > 50                      # points at infinity are in the batch
    for iters in K.ITERATIONS:
        got, upd = cv_b200.single_view_simple_optimize_l1_batch(poses, eps, K.RATE, iters, B, W, off)
        for k in range(len(poses)):
            s = slice(off[k], off[k + 1])
            for order in (P.DEVICE_ORDER, P.LANDMARK_ORDER):
                Rw, tw, uw = P.single_view_optimize_l1(poses[k], eps, K.RATE, iters, B[s], W[s], order)
                assert abs(int(upd[k]) - uw) <= K.UPDATE_DRIFT, (k, iters, order, upd[k], uw)
                assert _diff(got[k], (Rw, tw)) < K.POSE_TOL, (k, iters, order, _diff(got[k], (Rw, tw)))
        assert upd[K.SINGLE_SIZES.index(0)] == 0
        empty = K.SINGLE_SIZES.index(0)
        assert got[empty][0].tobytes() == np.asarray(poses[empty][0]).tobytes()
    # the single-problem surface equals the batch
    k = 0
    s = slice(off[k], off[k + 1])
    batch, _ = cv_b200.single_view_simple_optimize_l1_batch(poses, eps, K.RATE, 150, B, W, off)
    one = cv_b200.single_view_simple_optimize_l1(poses[k], eps, K.RATE, 150, (B[s], W[s]))
    assert one[0].tobytes() == batch[k][0].tobytes() and one[1].tobytes() == batch[k][1].tobytes()
    assert cv_b200.single_view_simple_optimize_l1(poses[0], eps, K.RATE, 10, (np.zeros((0, 3)), np.zeros((0, 4)))) is poses[0]


@pytest.mark.parametrize("eps", K.EPSILONS)
def test_three_view_l1_batch_matches_oracle(eps):
    starts, obs, off = K.three_view_batch()
    obs_all = np.concatenate(obs)
    for iters in K.ITERATIONS:
        got, upd = cv_b200.three_view_simple_optimize_l1_batch(starts, eps, K.RATE, iters, obs_all, off)
        for k in range(len(starts)):
            for order in (P.DEVICE_ORDER, P.LANDMARK_ORDER):
                want, uw = P.three_view_optimize_l1(starts[k], eps, K.RATE, iters, obs[k], order)
                assert abs(int(upd[k]) - uw) <= K.UPDATE_DRIFT, (k, iters, order, upd[k], uw)
                for v in range(2):
                    assert _diff(got[k][v], want[v]) < K.POSE_TOL, (k, v, iters, order)
        empty = K.THREE_SIZES.index(0)
        assert upd[empty] == 0
        assert all(got[empty][v][j].tobytes() == np.asarray(starts[empty][v][j]).tobytes() for v in range(2) for j in range(2))
    batch, _ = cv_b200.three_view_simple_optimize_l1_batch(starts, eps, K.RATE, 150, obs_all, off)
    one = cv_b200.three_view_simple_optimize_l1(starts[0], eps, K.RATE, 150, obs[0])
    assert all(one[v][j].tobytes() == batch[0][v][j].tobytes() for v in range(2) for j in range(2))


def test_l1_entry_points_reject_bad_arguments():
    from cv_b200._lib import CVB_EINVAL
    poses, B, W, off = K.single_view_batch()
    bad = np.array([0, 2, 1, 3], np.uint32)                 # decreasing offsets
    with pytest.raises(cv_b200.CvbError) as e:
        cv_b200.single_view_simple_optimize_l1_batch(poses[:3], 1e-12, 0.1, 10, B[:3], W[:3], bad)
    assert e.value.code == CVB_EINVAL
    starts, obs, _ = K.three_view_batch()
    with pytest.raises(cv_b200.CvbError) as e:
        cv_b200.three_view_simple_optimize_l1_batch(starts[:3], 1e-12, 0.1, 10, obs[2], np.array([0, 2, 1, 3], np.uint32))
    assert e.value.code == CVB_EINVAL
    # B == 0 is a no-op
    out, upd = cv_b200.single_view_simple_optimize_l1_batch([], 1e-12, 0.1, 10, np.zeros((0, 3)), np.zeros((0, 4)), [0])
    assert out == [] and len(upd) == 0
