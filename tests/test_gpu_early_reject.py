"""GPU: early rejection in the block loop's scoring (k_ars_score phase 1) changes no result.

A new hypothesis whose certain outliers in [0, acc_hi) reach acc_hi - worst can no longer join the candidates, and the scoring
writes its remaining mask words as 0 instead of scoring them; when worst >= acc_hi no new hypothesis can join, and the block's
samples are drawn but not estimated.  Every scene runs three calls on one generator with early rejection
on (the default) and forced off (CVB_ARS_EARLY_REJECT=0); model, inlier set and the committed generator state must be the same,
and equal to the oracle's.  The CVB_ARS_DEBUG line shows that the interesting cases were reached: units skipped at all, a block
scored under worst == 0 (nothing can be skipped before every word below acc_hi is decided), a bar below one mask word, and blocks
with the bar at 0 (the median candidate holds every datum so far: nothing is estimated)."""
import os
import re

import numpy as np
import pytest

import cv_b200
import tests.degenerate_scenes as S
from oracle import pyoracle as O
from tests.common import GOLDEN
from tests.geom_util import two_view_scene

pytestmark = pytest.mark.gpu

VSLAM = dict(initialization_hypotheses=8192, max_candidate_hypotheses=1024)
SMALL = dict(initialization_hypotheses=512, max_candidate_hypotheses=128)
# every initial model passes the likelihood-ratio test: 16 samples give <= 64 candidates of which only the one right decomposition
# per sample has inliers, so the median candidate after the first halving has none (worst == 0)
ALL_PASS = dict(initialization_hypotheses=16, max_candidate_hypotheses=64, likelihood_ratio_threshold=float("inf"))


def _bench_pair():
    z = np.load(os.path.join(GOLDEN, "bench_pair0.npz"))
    return z["ba"], z["bb"]


SCENES = {   # name: (bearings, threshold, configuration, what the debug counters must show with early rejection on)
    "bench_pair": (_bench_pair, 1e-7, VSLAM, "bar0"),
    "planar": (lambda: S.planar(120, 600, noise=3e-5), 1e-7, VSLAM, "skip"),
    "rotation_only": (lambda: S.rotation_only(103, 400), 1e-6, SMALL, None),
    "small_baseline": (lambda: S.small_baseline(104, 400), 1e-6, SMALL, None),
    "repeated": (lambda: S.repeated(105, 400)[:2], 1e-6, SMALL, None),
    "worst_zero": (lambda: two_view_scene(np.random.default_rng(7), 1000, noise=1e-5)[2:4], 1e-6, ALL_PASS, "worst0"),
    "bar_below_word": (lambda: two_view_scene(np.random.default_rng(8), 600, outlier_frac=0.02)[2:4], 1e-6, SMALL, "lt32"),
    "bar_zero": (lambda: two_view_scene(np.random.default_rng(9), 400, outlier_frac=0.25, noise=1e-4)[2:4], 2.5, SMALL, "none_estimated"),
}
DEBUG = re.compile(r"block units: kept (\d+) new (\d+) skipped (\d+) \| blocks worst0 (\d+) bar<32 (\d+) not estimated (\d+)")


def _run(a, b, thr, cfg, early, monkeypatch, capfd):
    monkeypatch.setenv("CVB_ARS_DEBUG", "1")
    if early:
        monkeypatch.delenv("CVB_ARS_EARLY_REJECT", raising=False)
    else:
        monkeypatch.setenv("CVB_ARS_EARLY_REJECT", "0")
    capfd.readouterr()
    ctx = cv_b200.Context(0)
    out = []
    try:
        ars = cv_b200.Arrsac(thr, cv_b200.Xoshiro256PlusPlus(0), ctx=ctx)
        for k, v in cfg.items():
            if k == "likelihood_ratio_threshold":
                ars.cfg.likelihood_ratio_threshold = v
            else:
                getattr(ars, k)(v)
        for _ in range(3):      # eager, capture + launch, replay
            got = ars.model_inliers(cv_b200.EightPoint(), a, b)
            out.append((got, [int(x) for x in ars.rng.state.s]))
    finally:
        ctx.close()
    stats = [tuple(int(x) for x in m) for m in DEBUG.findall(capfd.readouterr().err)]
    assert len(stats) == 3, stats
    return out, stats


@pytest.mark.parametrize("scene", list(SCENES))
def test_early_rejection_changes_no_result(scene, monkeypatch, capfd):
    make, thr, cfg, expect = SCENES[scene]
    a, b = make()
    on, st_on = _run(a, b, thr, cfg, True, monkeypatch, capfd)
    off, st_off = _run(a, b, thr, cfg, False, monkeypatch, capfd)
    orng = O.rng_xoshiro(0)
    for call in range(3):
        w = O.arrsac(O.arrsac_cfg(thr, **cfg), 0, a, b, orng)
        for got, state in (on[call], off[call]):
            assert (got is None) == (w is None), call
            if got is not None:
                assert np.array_equal(got[2], w[2]), call
                assert got[0].tobytes() == on[call][0][0].tobytes() and got[1].tobytes() == on[call][0][1].tobytes(), call
                assert np.allclose(got[0], w[0], rtol=1e-6, atol=1e-12) and np.allclose(got[1], w[1], rtol=1e-6, atol=1e-12), call
            assert state == [int(x) for x in orng.s], call
    assert on[0][0] is not None
    # the same blocks are scored either way; forced off, nothing is skipped
    assert [s[:2] + s[3:] for s in st_on] == [s[:2] + s[3:] for s in st_off], (st_on, st_off)
    assert all(s[2] == 0 for s in st_off), st_off
    kept, new, skipped, w0, lt32, bar0 = st_on[0]
    assert skipped <= new, st_on
    if expect == "skip":
        assert skipped > 0, st_on
    elif expect == "bar0":
        assert bar0 > 0, st_on
    elif expect == "worst0":
        assert w0 > 0, st_on
    elif expect == "lt32":
        assert lt32 > 0 and skipped > 0, st_on
    elif expect == "none_estimated":     # every datum is an inlier of every model: every block's bar is 0
        assert bar0 > 0 and new == 0, st_on
