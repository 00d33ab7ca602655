"""GPU: the block loop's queued exact evaluation (k_ars_resolve_block) under every way the driver runs the loop.

The vslam-sandbox two-view configuration, Arrsac(1e-7).initialization_hypotheses(8192).max_candidate_hypotheses(1024) + EightPoint,
on the bench's frame pair and on a low-parallax scene (far points: small second eigenvalue of the design matrix, where the
filter leaves the most predicates undecided).  Each run mode gets a fresh context and three calls with a continuing generator
(eager, capture + launch, replay); every call's inlier set, pose and generator state must equal the oracle's, and the
block scoring must have queued predicates."""
import os
import re

import numpy as np
import pytest

import cv_b200
from oracle import pyoracle as O
from tests.common import GOLDEN
from tests.geom_util import rot_from_scaled_axis, unit

pytestmark = pytest.mark.gpu

THR = 1e-7
CFG = dict(initialization_hypotheses=8192, max_candidate_hypotheses=1024)
MODES = {"eager": {"CVB_ARS_NO_GRAPH": "1"}, "while": {"CVB_ARS_WHILE": "1"}, "unrolled": {"CVB_ARS_WHILE": "0"}}


def _bench_pair():
    z = np.load(os.path.join(GOLDEN, "bench_pair0.npz"))
    return z["ba"], z["bb"]


def _low_parallax_scene(n=2500, outlier_frac=0.25, noise=3e-5):
    rng = np.random.default_rng(1234)
    R = rot_from_scaled_axis(rng.uniform(-1, 1, 3) * 0.1)
    t = unit(rng.uniform(-1, 1, 3))
    P = np.stack([rng.uniform(-20, 20, n), rng.uniform(-20, 20, n), rng.uniform(20, 150, n)], 1)
    a, b = unit(P), unit(P @ R.T + t)
    a = unit(a + rng.normal(0, noise, a.shape)); b = unit(b + rng.normal(0, noise, b.shape))
    bad = rng.choice(n, int(n * outlier_frac), replace=False)
    b[bad] = b[rng.permutation(bad)]
    return np.ascontiguousarray(a), np.ascontiguousarray(b)


SCENES = {"bench_pair": _bench_pair, "low_parallax": _low_parallax_scene}
_want = {}


def _oracle(scene, a, b):
    if scene not in _want:
        orng = O.rng_xoshiro(0)
        calls = []
        for _ in range(3):
            w = O.arrsac(O.arrsac_cfg(THR, **CFG), 0, a, b, orng)
            calls.append((w, [int(x) for x in orng.s]))
        _want[scene] = calls
    return _want[scene]


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("scene", list(SCENES))
def test_block_queue_equals_oracle(scene, mode, monkeypatch, capfd):
    a, b = SCENES[scene]()
    want = _oracle(scene, a, b)
    assert want[0][0] is not None and len(want[0][0][2]) > len(a) // 2
    for k, v in MODES[mode].items():
        monkeypatch.setenv(k, v)
    monkeypatch.setenv("CVB_ARS_DEBUG", "1")
    capfd.readouterr()
    ctx = cv_b200.Context(0)
    try:
        ars = cv_b200.Arrsac(THR, cv_b200.Xoshiro256PlusPlus(0), ctx=ctx).initialization_hypotheses(8192).max_candidate_hypotheses(1024)
        for call, (w, state) in enumerate(want):
            got = ars.model_inliers(cv_b200.EightPoint(), a, b)
            assert (got is None) == (w is None), call
            if got is not None:
                assert np.array_equal(got[2], w[2]), call
                assert np.allclose(got[0], w[0], rtol=1e-6, atol=1e-12) and np.allclose(got[1], w[1], rtol=1e-6, atol=1e-12), call
            assert [int(x) for x in ars.rng.state.s] == state, call
    finally:
        ctx.close()
    err = capfd.readouterr().err
    queued = [int(x) for x in re.findall(r"undecided predicates queued: initial \d+ block (\d+)", err)]
    assert len(queued) == 3 and all(q > 0 for q in queued), err
