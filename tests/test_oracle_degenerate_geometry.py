"""CPU: the degenerate scenes of tests/degenerate_scenes.py have the degeneracy they claim, and the geometry oracle handles them.

The GPU tests (tests/test_gpu_degenerate_geometry.py) hold the device to the oracle on these scenes bit for bit; that is only
worth something if the scenes really reach the branches where the solvers make choices: near-tied smallest eigenvalues of the
eight-point design, the 40-pose cap of a five-point sample, P3P's failing inv3 and w == 0 landmarks, non-finite rows."""
import time

import numpy as np
import pytest

from oracle import pyoracle as O
from tests import degenerate_scenes as S
from tests.geom_util import two_view_scene

ORACLE_SECONDS = 60.0          # per ARRSAC call; measured 0.1-1.3 s on these sizes


def _null_dim(a, b, rel=1e-12):
    s = np.linalg.svd(S.design_matrix(a, b), compute_uv=False)
    return int((s < rel * s[0]).sum()), s


def _samples(rng, n, k, count):
    return np.stack([rng.choice(n, k, replace=False) for _ in range(count)])


def _timed_arrsac(cfg, kind, a, b, seed=0):
    rng = O.rng_xoshiro(seed)
    t0 = time.perf_counter()
    out = O.arrsac(cfg, kind, a, b, rng)
    assert time.perf_counter() - t0 < ORACLE_SECONDS
    return out


@pytest.mark.parametrize("scene", ["planar", "rotation_only"])
def test_design_null_space_is_three_dimensional(scene):
    a, b = getattr(S, scene)(1, 300, outlier_frac=0.0)
    dim, s = _null_dim(a, b)
    assert dim == 3 and s[-4] > 1e-6 * s[0], s / s[0]
    # every 8-sample of it has near-tied smallest eigenvalues of AtA: the eight-point's choice among them is decided by the last bits
    rng = np.random.default_rng(2)
    for idx in _samples(rng, 300, 8, 20):
        w = np.linalg.eigvalsh(S.design_matrix(a[idx], b[idx]).T @ S.design_matrix(a[idx], b[idx]))
        assert abs(w[2]) < 1e-14 * w[-1] and w[3] > 1e-9 * w[-1], w / w[-1]      # three eigenvalues at the rounding floor


def test_general_and_small_baseline_designs():
    _, _, a, b, _ = two_view_scene(np.random.default_rng(3), 300)
    assert _null_dim(a, b)[0] == 1
    a, b = S.small_baseline(4, 300, outlier_frac=0.0)
    dim, s = _null_dim(a, b, rel=1e-6)
    assert dim >= 2 and s[-1] < 1e-15 * s[0]       # t = 1e-5: numerically close to rotation only


def test_repeated_and_duplicated_rows():
    a, b, src = S.repeated(5, 400)
    assert len(a) == 400 and 2.0 <= 400 / len(np.unique(src)) <= 3.0
    assert np.array_equal(a, a[np.unique(src, return_index=True)[1]][np.searchsorted(np.unique(src), src)])
    bear, world = S.pnp_duplicated(6, 400)
    assert len(np.unique(world, axis=0)) < 400 // 2 + 20


def test_five_point_reaches_the_forty_pose_cap_on_a_planar_scene():
    a, b = S.planar(1, 400, noise=1e-4)
    counts = [len(O.five_point(a[s], b[s])) for s in S.five_point_cap_samples()]
    assert max(counts) == 40 and all(c % 4 == 0 for c in counts)
    a, b = S.rotation_only(9, 400)
    counts = [len(O.five_point(a[s], b[s])) for s in _samples(np.random.default_rng(10), 400, 5, 200)]
    assert np.mean(np.array(counts) == 0) > 0.5


def test_p3p_on_degenerate_world_points():
    bear, world = S.pnp_collinear(11, 200, 40)
    for s in _samples(np.random.default_rng(12), 40, 3, 100):
        assert O.p3p(bear[s], world[s]) == []                     # collinear: inv3 fails
    bear, world = S.pnp_planar(13, 300)
    counts = {len(O.p3p(bear[s], world[s])) for s in _samples(np.random.default_rng(14), 300, 3, 600)}
    assert counts == {0, 1, 2, 3, 4}
    bear, world, k = S.pnp_at_infinity(15, 300)
    zero = k[:len(k) // 2]
    for s in _samples(np.random.default_rng(16), len(zero), 2, 30):
        assert O.p3p(bear[[zero[s[0]], zero[s[1]], 0]], world[[zero[s[0]], zero[s[1]], 0]]) == []    # w = 0 -> Projective::point() None


def test_oracle_arrsac_terminates_on_every_degenerate_scene():
    scenes2 = dict(planar=S.planar(20, 400), planar_noisy=S.planar(21, 400, noise=1e-4), rotation=S.rotation_only(22, 400),
                   small_baseline=S.small_baseline(23, 400), repeated=S.repeated(24, 400)[:2])
    for name, (a, b) in scenes2.items():
        _timed_arrsac(O.arrsac_cfg(1e-6, initialization_hypotheses=512, max_candidate_hypotheses=128), 0, a, b)
    scenes3 = dict(planar=S.pnp_planar(25, 400), collinear=S.pnp_collinear(26, 400, 60), infinity=S.pnp_at_infinity(27, 400)[:2],
                   duplicated=S.pnp_duplicated(28, 400))
    for name, (bear, world) in scenes3.items():
        out = _timed_arrsac(O.arrsac_cfg(1e-5, initialization_hypotheses=512, max_candidate_hypotheses=128), 1, bear, world)
        assert out is not None, name


def test_oracle_arrsac_on_poisoned_rows():
    a, b, rows = S.two_view_poisoned(30, 400)
    assert not np.isfinite(a[rows[:12]]).all() and (a[rows[:12]] == 0).all(axis=1).any()
    out = _timed_arrsac(O.arrsac_cfg(1e-6, initialization_hypotheses=1024, max_candidate_hypotheses=128), 0, a, b)
    assert out is not None and not np.isin(rows, out[2]).any() and len(out[2]) > 200
    bear, world, rows = S.pnp_poisoned(31, 400)
    out = _timed_arrsac(O.arrsac_cfg(1e-5, initialization_hypotheses=512, max_candidate_hypotheses=128), 1, bear, world)
    assert out is not None and len(out[2]) > 200
    # WorldToCamera::residual is 1 - bearing . q (cv-core/src/pose.rs:194-202): an infinite bearing component makes it -inf when
    # its q component is positive, and -inf < threshold.  Every other poisoned row gives NaN or a residual >= 0.5.
    res = np.array([O.residual_w2c(out[0], out[1], bear[r], world[r]) for r in rows])
    taken = np.isin(rows, out[2])
    assert np.array_equal(taken, res == -np.inf) and np.isinf(bear[rows[taken]]).any(axis=1).all()


def test_endless_loop_case_returns_every_landmark():
    bear, world = S.endless_loop()
    out = _timed_arrsac(O.arrsac_cfg(0.01), 1, bear, world)
    assert out is not None and out[2].tolist() == list(range(9))


@pytest.mark.parametrize("kind,K", [(0, 8), (2, 5), (1, 3)])
def test_fewer_data_than_the_sample_size(kind, K):
    rng = np.random.default_rng(40 + K)
    if kind == 1:
        from tests.geom_util import pnp_scene
        _, _, a, b, _ = pnp_scene(rng, K + 1)
    else:
        _, _, a, b, _ = two_view_scene(rng, K + 1)
    r = O.rng_xoshiro(0)
    s0 = [int(x) for x in r.s]
    assert O.arrsac(O.arrsac_cfg(1e-6), kind, a[:K - 1], b[:K - 1], r) is None
    assert [int(x) for x in r.s] == s0                           # no draw consumed
    assert O.arrsac(O.arrsac_cfg(1e-6), kind, a[:0], b[:0], r) is None
    out = O.arrsac(O.arrsac_cfg(1e-6), kind, a[:K], b[:K], r)
    if kind == 0:
        assert out is not None and out[2].tolist() == list(range(8))
