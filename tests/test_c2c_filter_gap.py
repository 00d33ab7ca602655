"""CPU: the filter's certificate for a small spectral gap (cv_b200/csrc/c2c_filter.cuh: the ladder of upper shifts below s_hi).

Predicates of good hypotheses on low-parallax data have a small second eigenvalue l2 of the design matrix; with one upper shift
s_hi the filter left them all to the exact evaluation.  Checked: the filter still never contradicts the oracle's exact
`residual < threshold`, and on the bench pair's good poses it leaves almost nothing undecided."""
import os

import numpy as np

from oracle import pyoracle as O
from tests.geom_util import rot_from_scaled_axis, unit
from tests.test_c2c_filter import HERE, _check, _poses, filt  # noqa: F401  (filt: the host build of the filter, a module fixture)


def _run(filt, poses, a, b, thr):
    P = np.ascontiguousarray([np.concatenate([R.reshape(9), t]) for R, t in poses], np.float64)
    out = np.zeros((len(P), len(a)), np.int8)
    filt.c2c_filter_batch(P.ctypes.data, len(P), a.ctypes.data, b.ctypes.data, len(a), thr, out.ctypes.data)
    return out


def test_bench_pair_good_poses_are_decided(filt):
    # 60 eight-point hypotheses on the bench pair, the 20 with the most inliers: the block loop's candidates look like these
    z = np.load(os.path.join(HERE, "golden", "bench_pair0.npz"))
    a, b = np.ascontiguousarray(z["ba"]), np.ascontiguousarray(z["bb"])
    poses = _poses(a, b, np.random.default_rng(1), 60)
    out = _run(filt, poses, a, b, 1e-7)
    best = np.argsort(-(out != 0).sum(1), kind="stable")[:20]
    good = [poses[i] for i in best]
    ob = out[best]
    n = len(a) // 32 * 32
    assert (ob == -1).mean() <= 1e-3                                          # undecided predicates
    assert (ob[:, :n].reshape(len(best), -1, 32) == -1).any(2).mean() <= 0.02     # 32-datum units with an undecided lane
    exact = np.array([[O.residual_c2c(R, t, a[i], b[i]) < 1e-7 for i in range(len(a))] for R, t in good])
    d = ob >= 0
    assert np.array_equal(ob[d] == 1, exact[d])


def test_low_parallax_scenes_agree_with_exact_predicate(filt):
    # far points (depth 20-150 for a unit baseline): l2 down to ~1e-5, below s_hi at every threshold tried
    rng = np.random.default_rng(5)
    for thr, noise in [(1e-7, 3e-5), (1e-8, 1e-5), (1e-6, 1e-4), (1e-9, 0.0)]:
        n = 400
        R = rot_from_scaled_axis(rng.uniform(-1, 1, 3) * 0.1)
        t = unit(rng.uniform(-1, 1, 3))
        X = np.stack([rng.uniform(-20, 20, n), rng.uniform(-20, 20, n), rng.uniform(20, 150, n)], 1)
        a, b = unit(X), unit(X @ R.T + t)
        if noise:
            a = unit(a + rng.normal(0, noise, a.shape)); b = unit(b + rng.normal(0, noise, b.shape))
        a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
        dec, _ = _check(filt, _poses(a, b, rng, 6) + [(R, t)], a, b, thr)
        assert dec > 0.95, (thr, dec)
