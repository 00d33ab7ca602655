"""GPU: the minimal solvers and the ARRSAC driver against the CPU oracle on degenerate geometry (tests/degenerate_scenes.py).

On well-conditioned data a one-ulp difference between device and oracle cannot change a result; here it can.  Planar and
rotation-only scenes make the eight-point's smallest eigenvalues tie to the rounding floor, planar five-point samples reach the
40-pose cap, collinear and w == 0 landmarks make P3P fail, repeated matches and poisoned rows (NaN, +-inf, zero vectors, z = 0,
z < 0) flow through the exact-predicate filter into the exact path, and device-side counts fall below the sample size.

  (a) EightPoint / NisterStewenius (both row modes) / LambdaTwist .estimate_batch == O.eight_point / O.five_point / O.p3p per
      sample: equal counts, equal NaN positions, eight- and five-point bit for bit, P3P to 1e-8 (its final rotation uses CUDA's
      sin / cos, not glibc's).
  (b) Arrsac.model_inliers under each run mode (eager, WHILE node, unrolled graph), fresh context, three calls on one generator:
      found, inlier set, generator state and (two-view) pose bits equal the oracle's, and the inlier set is
      { i : oracle residual of the returned model < threshold }.
  (c) cvb_arrsac_eight_point_dev / cvb_arrsac_p3p_dev with device counts 0, 1, K - 1, K, n below a 4096-row buffer whose rows past the
      count are copies of true inliers (or NaN) == the host entry on the counted rows; outputs past the count keep their sentinel.
  (d) cvb_two_view_pair_dev on synthetic keypoints and descriptors with fewer than 8 symmetric matches: the pairs equal the host
      restatement of symmetric matching, no model is found and the generator is where the oracle leaves it."""
import ctypes as C

import numpy as np
import pytest

import cv_b200
from cv_b200._lib import KP_DTYPE
from oracle import pyoracle as O
from tests import degenerate_scenes as S
from tests.geom_util import pnp_scene, two_view_scene
from tests.synth import random_descriptors

pytestmark = pytest.mark.gpu

MODES = {"eager": {"CVB_ARS_NO_GRAPH": "1"}, "while": {"CVB_ARS_WHILE": "1"}, "unrolled": {"CVB_ARS_WHILE": "0"}}
ROW0 = {"eight": None, "five": 5, "five_corrected": 6, "p3p": None}
KIND = {"eight": 0, "five": 2, "five_corrected": 2, "p3p": 1}
MIN_SAMPLES = {"eight": 8, "five": 5, "five_corrected": 5, "p3p": 3}
THR = {"eight": 1e-6, "five": 1e-6, "five_corrected": 1e-6, "p3p": 1e-5}
CFG = {"eight": dict(initialization_hypotheses=512, max_candidate_hypotheses=128),
       "five": dict(initialization_hypotheses=256, max_candidate_hypotheses=64),
       "five_corrected": dict(initialization_hypotheses=256, max_candidate_hypotheses=64),
       "p3p": dict(initialization_hypotheses=512, max_candidate_hypotheses=128)}

TWO_VIEW = {
    "general": lambda: two_view_scene(np.random.default_rng(100), 400, outlier_frac=0.25, noise=1e-4)[2:4],   # the control
    "planar": lambda: S.planar(101, 400),
    "planar_noisy": lambda: S.planar(1, 400, noise=1e-4),
    "rotation_only": lambda: S.rotation_only(103, 400),
    "baseline_1e-5": lambda: S.small_baseline(104, 400),
    "repeated": lambda: S.repeated(105, 400)[:2],
    "poisoned": lambda: S.two_view_poisoned(106, 400)[:2],
}
PNP = {
    "planar": lambda: S.pnp_planar(13, 400),
    "collinear": lambda: S.pnp_collinear(112, 400, 60),
    "infinity": lambda: S.pnp_at_infinity(113, 400)[:2],
    "duplicated": lambda: S.pnp_duplicated(114, 400),
    "poisoned": lambda: S.pnp_poisoned(115, 400)[:2],
    "endless_loop": S.endless_loop,
}


def _estimator(name):
    if name == "eight":
        return cv_b200.EightPoint()
    if name == "p3p":
        return cv_b200.LambdaTwist()
    return cv_b200.NisterStewenius(corrected=name == "five_corrected")


def _bits_equal(x, y):
    """equal NaN positions, every other value bit for bit"""
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    nx, ny = np.isnan(x), np.isnan(y)
    return x.shape == y.shape and np.array_equal(nx, ny) and np.array_equal(x[~nx].view(np.uint64), y[~ny].view(np.uint64))


def _close(x, y, tol=1e-8):
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    nx, ny = np.isnan(x), np.isnan(y)
    return x.shape == y.shape and np.array_equal(nx, ny) and np.allclose(x[~nx], y[~ny], rtol=tol, atol=tol)


def _flat(poses):
    return np.array([np.concatenate([np.asarray(R).reshape(9), np.asarray(t)]) for R, t in poses]).reshape(-1, 12)


class _Row0:
    """O.five_point / O.arrsac(kind 2) read a process-wide eigenvector row; restore the reference's after use"""

    def __init__(self, row0):
        self.row0 = row0

    def __enter__(self):
        if self.row0 is not None:
            O.five_point_set_row0(self.row0)

    def __exit__(self, *exc):
        O.five_point_set_row0(5)


# ---- (a) minimal solvers per sample ----------------------------------------------------------------------------------------
def _samples(rng, n, K, special=()):
    """300 random samples, 24 built from repeated rows, and any rows of `special` (poisoned, collinear, w = 0) forced into 60 more"""
    s = [rng.choice(n, K, replace=False) for _ in range(300)]
    for j in range(24):
        r = rng.choice(n, 1 + j % (K - 1), replace=False)
        s.append(np.resize(r, K))
    special = np.asarray(special)
    if len(special):
        for _ in range(60):
            x = rng.choice(n, K, replace=False)
            x[rng.integers(0, K)] = special[rng.integers(0, len(special))]
            s.append(x)
    return np.array(s, np.uint32)


@pytest.mark.parametrize("solver", ["eight", "five", "five_corrected"])
@pytest.mark.parametrize("scene", list(TWO_VIEW))
def test_two_view_solvers_equal_oracle_bit_for_bit(scene, solver):
    a, b = TWO_VIEW[scene]()
    K = MIN_SAMPLES[solver]
    special = S.two_view_poisoned(106, 400)[2] if scene == "poisoned" else ()
    samples = _samples(np.random.default_rng(10 * list(TWO_VIEW).index(scene) + len(solver)), len(a), K, special)
    if scene == "planar_noisy" and solver != "eight":
        samples = np.concatenate([samples, S.five_point_cap_samples()])
    poses, cnt = _estimator(solver).estimate_batch(a, b, samples)
    oracle = O.eight_point if solver == "eight" else O.five_point
    counts = []
    with _Row0(ROW0[solver]):
        for h, s in enumerate(samples):
            want = _flat(oracle(a[s], b[s]))
            assert cnt[h] == len(want), (h, s)
            got = np.concatenate([poses[h, :cnt[h]]["r"], poses[h, :cnt[h]]["t"]], 1)
            assert _bits_equal(got, want), (h, s)
            counts.append(len(want))
    if scene == "planar_noisy" and solver == "five":
        assert max(counts) == 40                                   # the ModelIter cap is reached


@pytest.mark.parametrize("scene", list(PNP))
def test_p3p_equals_oracle(scene):
    bear, world = PNP[scene]()
    rng = np.random.default_rng(7)
    if scene == "endless_loop":
        import itertools
        samples = np.array(list(itertools.permutations(range(9), 3)), np.uint32)
    else:
        special = {"collinear": np.arange(60), "infinity": S.pnp_at_infinity(113, 400)[2],
                   "poisoned": S.pnp_poisoned(115, 400)[2]}.get(scene, ())
        samples = _samples(rng, len(bear), 3, special)
        if scene == "collinear":
            samples = np.concatenate([samples, np.array([rng.choice(60, 3, replace=False) for _ in range(100)], np.uint32)])
    poses, cnt = cv_b200.LambdaTwist().estimate_batch(bear, world, samples)
    counts = []
    for h, s in enumerate(samples):
        want = _flat(O.p3p(bear[s], world[s]))
        assert cnt[h] == len(want), (h, s)
        got = np.concatenate([poses[h, :cnt[h]]["r"], poses[h, :cnt[h]]["t"]], 1)
        assert _close(got, want), (h, s)
        counts.append(len(want))
    if scene == "collinear":
        assert not any(counts[-100:])                               # inv3 fails on every all-collinear sample
    if scene == "planar":
        assert set(counts) == {0, 1, 2, 3, 4}


# ---- (b) consensus through the host entry, every run mode ------------------------------------------------------------------
_want = {}


def _oracle_calls(key, solver, a, b, thr, cfg, seed, calls=3):
    if key not in _want:
        orng = O.rng_xoshiro(seed)
        out = []
        with _Row0(ROW0[solver]):
            for _ in range(calls):
                w = O.arrsac(O.arrsac_cfg(thr, **cfg), KIND[solver], a, b, orng)
                out.append((w, [int(x) for x in orng.s]))
        _want[key] = out
    return _want[key]


def _predicate_set(solver, R, t, a, b, thr):
    res = O.residual_w2c if solver == "p3p" else O.residual_c2c
    return np.array([i for i in range(len(a)) if res(R, t, a[i], b[i]) < thr], np.uint32)


def _check_modes(key, solver, a, b, thr, cfg, monkeypatch, seed=0):
    want = _oracle_calls(key, solver, a, b, thr, cfg, seed)
    for mode in MODES:
        for k in ("CVB_ARS_NO_GRAPH", "CVB_ARS_WHILE"):
            monkeypatch.delenv(k, raising=False)
        for k, v in MODES[mode].items():
            monkeypatch.setenv(k, v)
        ctx = cv_b200.Context(0)
        try:
            ars = cv_b200.Arrsac(thr, cv_b200.Xoshiro256PlusPlus(seed), ctx=ctx)
            for k, v in cfg.items():
                getattr(ars, k)(v)
            for call, (w, state) in enumerate(want):
                got = ars.model_inliers(_estimator(solver), a, b)
                where = (mode, call)
                assert (got is None) == (w is None), where
                if got is not None:
                    assert np.array_equal(got[2], w[2]), where
                    if solver == "p3p":
                        assert _close(got[0], w[0]) and _close(got[1], w[1]), where
                    else:
                        assert _bits_equal(got[0], w[0]) and _bits_equal(got[1], w[1]), where
                    if mode == "eager":                         # the same results in the other modes
                        assert np.array_equal(got[2], _predicate_set(solver, got[0], got[1], a, b, thr)), where
                assert [int(x) for x in ars.rng.state.s] == state, where
        finally:
            ctx.close()
    return want


@pytest.mark.parametrize("solver", ["eight", "five", "five_corrected"])
@pytest.mark.parametrize("scene", list(TWO_VIEW))
def test_two_view_consensus_equals_oracle_in_every_mode(scene, solver, monkeypatch):
    a, b = TWO_VIEW[scene]()
    want = _check_modes((scene, solver), solver, a, b, THR[solver], CFG[solver], monkeypatch)
    if scene == "poisoned":
        rows = S.two_view_poisoned(106, 400)[2]
        assert all(w is None or not np.isin(rows, w[2]).any() for w, _ in want)


@pytest.mark.parametrize("scene", list(PNP))
def test_p3p_consensus_equals_oracle_in_every_mode(scene, monkeypatch):
    bear, world = PNP[scene]()
    thr, cfg = (0.01, {}) if scene == "endless_loop" else (THR["p3p"], CFG["p3p"])
    want = _check_modes(("pnp", scene), "p3p", bear, world, thr, cfg, monkeypatch)
    assert want[0][0] is not None
    if scene == "endless_loop":
        assert want[0][0][2].tolist() == list(range(9))             # lambda-twist/tests/consensus.rs:68-134


def test_vslam_sandbox_configuration_on_a_planar_scene(monkeypatch):
    # vslam-sandbox/src/main.rs:112-117: Arrsac(1e-7).initialization_hypotheses(8192).max_candidate_hypotheses(1024) + EightPoint
    a, b = S.planar(120, 600, noise=3e-5)
    cfg = dict(initialization_hypotheses=8192, max_candidate_hypotheses=1024)
    want = _check_modes(("vslam_planar", "eight"), "eight", a, b, 1e-7, cfg, monkeypatch)
    assert want[0][0] is not None


@pytest.mark.parametrize("thr", [0.0, 1e-12, 2.5])
def test_threshold_edges_equal_oracle(thr, monkeypatch):
    _, _, a, b, _ = two_view_scene(np.random.default_rng(130), 300, outlier_frac=0.3, noise=1e-4)
    want = _check_modes(("thr", thr), "eight", a, b, thr, CFG["eight"], monkeypatch)
    if thr == 2.5:
        assert all(w is not None and len(w[2]) == 300 for w, _ in want)     # a residual is at most 2


@pytest.mark.parametrize("delta", [-1, 0, 1])
@pytest.mark.parametrize("solver", ["eight", "five", "five_corrected", "p3p"])
def test_data_count_around_the_sample_size(solver, delta, monkeypatch):
    n = MIN_SAMPLES[solver] + delta
    rng = np.random.default_rng(140 + n)
    if solver == "p3p":
        _, _, a, b, _ = pnp_scene(rng, n)
    else:
        _, _, a, b, _ = two_view_scene(rng, n)
    want = _check_modes(("count", solver, n), solver, a, b, 0.1 if solver == "p3p" else 1e-6, {}, monkeypatch)
    assert (want[0][0] is None) == (delta < 0)


# ---- (c) device-count entries --------------------------------------------------------------------------------------------
NMAX = 4096
SENT_U32 = 0xFFFFFFF9
SENT_F64 = -1234.5


def _dev_entry(kind_name, a, b, n_dev, fill_rows, thr, cfg, seed):
    import torch
    from cv_b200.pair import bind
    ctx = cv_b200.Context(0)
    try:
        bind(ctx.lib)
        cv_b200.geom._lib(ctx)
        dev = torch.device("cuda", 0)
        A = np.full((NMAX, 3), np.nan); B = np.full((NMAX, b.shape[1]), np.nan)
        A[:n_dev] = a[:n_dev]; B[:n_dev] = b[:n_dev]
        if fill_rows is not None:
            src = np.resize(fill_rows, NMAX - n_dev)
            A[n_dev:] = a[src]; B[n_dev:] = b[src]
        ta, tb = torch.from_numpy(A.reshape(-1)).to(dev), torch.from_numpy(B.reshape(-1)).to(dev)
        tn = torch.tensor([n_dev], dtype=torch.int32, device=dev)
        model = torch.full((12,), SENT_F64, dtype=torch.float64, device=dev)
        inl = torch.from_numpy(np.full(NMAX, SENT_U32, np.uint32).view(np.int32)).to(dev)
        cnt = torch.from_numpy(np.array([SENT_U32, 7], np.uint32).view(np.int32)).to(dev)      # n_inliers, found
        ars = cv_b200.Arrsac(thr, cv_b200.Xoshiro256PlusPlus(seed), ctx)
        for k, v in cfg.items():
            getattr(ars, k)(v)
        torch.cuda.synchronize()
        fn = ctx.lib.cvb_arrsac_eight_point_dev if kind_name == "eight" else ctx.lib.cvb_arrsac_p3p_dev
        ctx.check(fn(ctx.handle, C.addressof(ars.cfg), ta.data_ptr(), tb.data_ptr(), tn.data_ptr(), NMAX, C.addressof(ars.rng.state),
                     model.data_ptr(), inl.data_ptr(), NMAX, cnt.data_ptr(), cnt.data_ptr() + 4))
        ctx.check(ctx.lib.cvb_arrsac_commit_rng(ctx.handle, C.addressof(ars.rng.state), None))
        c = cnt.cpu().numpy().view(np.uint32)
        return dict(model=model.cpu().numpy(), inl=inl.cpu().numpy().view(np.uint32), n_inliers=int(c[0]), found=int(c[1]),
                    state=[int(x) for x in ars.rng.state.s])
    finally:
        ctx.close()


@pytest.mark.parametrize("fill", ["inlier_copies", "nan"])
@pytest.mark.parametrize("solver", ["eight", "p3p"])
def test_device_count_entries_equal_host_entry(solver, fill):
    rng = np.random.default_rng(150)
    if solver == "eight":
        _, _, a, b, good = two_view_scene(rng, 400, outlier_frac=0.25, noise=1e-4)
    else:
        _, _, a, b, good = pnp_scene(rng, 400, outlier_frac=0.25, noise=1e-4)
    K, thr, cfg = MIN_SAMPLES[solver], THR[solver], CFG[solver]
    fill_rows = np.flatnonzero(good) if fill == "inlier_copies" else None
    for n_dev in (0, 1, K - 1, K, len(a)):
        got = _dev_entry(solver, a, b, n_dev, fill_rows, thr, cfg, 9)
        ars = cv_b200.Arrsac(thr, cv_b200.Xoshiro256PlusPlus(9))
        for k, v in cfg.items():
            getattr(ars, k)(v)
        want = ars.model_inliers(_estimator(solver), a[:n_dev], b[:n_dev])
        assert got["state"] == [int(x) for x in ars.rng.state.s], n_dev
        assert got["found"] == (want is not None), n_dev
        if want is None:
            assert got["n_inliers"] == 0 and (got["model"] == SENT_F64).all() and (got["inl"] == SENT_U32).all(), n_dev
            continue
        m = got["n_inliers"]
        assert np.array_equal(got["inl"][:m], want[2]) and (got["inl"][m:] == SENT_U32).all(), n_dev
        assert _bits_equal(got["model"][:9], want[0].reshape(9)) and _bits_equal(got["model"][9:], want[1]), n_dev
    assert got["found"] and got["n_inliers"] > 250                    # n_dev = n: the scene's consensus


# ---- (d) the fused pair below the sample size ----------------------------------------------------------------------------
def _symmetric_pairs(da, db, better_by=24):
    """cv-sfm's symmetric_matching (cv-sfm/src/lib.rs:3097-3133) restated on the oracle's 2-NN: a pair needs a best match better
    than the second by better_by in both directions and the two best matches pointing at each other"""
    if len(da) < 2 or len(db) < 2:
        return np.zeros((0, 2), np.int64)
    fi, fd = O.hamming_knn(da, db, 2)
    ri, rd = O.hamming_knn(db, da, 2)
    return np.array([(i, int(fi[i, 0])) for i in range(len(da))
                     if fd[i, 0] + better_by <= fd[i, 1] and rd[fi[i, 0], 0] + better_by <= rd[fi[i, 0], 1] and ri[fi[i, 0], 0] == i],
                    np.int64).reshape(-1, 2)


@pytest.mark.parametrize("n_b", [0, 1, 2, 5, 8])
@pytest.mark.parametrize("n_a", [0, 1, 2, 5, 8])
def test_fused_pair_with_fewer_than_eight_matches(n_a, n_b):
    import torch
    from cv_b200.pair import Intrinsics, bind
    cap = 64
    rng = np.random.default_rng(160 + 10 * n_a + n_b)
    da, db = random_descriptors(cap, 170 + n_a), random_descriptors(cap, 180 + n_b)
    m = min(n_a, n_b, 7)
    for j, i in enumerate(rng.permutation(n_a)[:m]):                # m true matches, 4 bits apart
        db[j] = da[i]
        for bit in rng.choice(486, 4, replace=False):
            db[j, bit // 8] ^= np.uint8(1 << (bit % 8))
    hi = max(n_a, n_b)
    db[hi:] = da[hi:]                                                # rows past both counts match each other exactly
    kp = np.zeros((2, cap), KP_DTYPE)
    kp["x"] = rng.uniform(0, 1920, (2, cap)); kp["y"] = rng.uniform(0, 1080, (2, cap))
    want_pairs = _symmetric_pairs(da[:n_a], db[:n_b])
    assert len(want_pairs) < 8
    dev = torch.device("cuda", 0)
    ctx = cv_b200.Context(0)
    try:
        bind(ctx.lib)
        cv_b200.geom._lib(ctx)
        tkp = torch.from_numpy(kp.view(np.uint8).reshape(-1)).to(dev)
        tdesc = torch.from_numpy(np.stack([da, db]).reshape(-1)).to(dev)
        tn = torch.tensor([n_a, n_b], dtype=torch.int32, device=dev)
        pairs = torch.from_numpy(np.full(2 * cap, SENT_U32, np.uint32).view(np.int32)).to(dev)
        cnt = torch.from_numpy(np.array([SENT_U32, SENT_U32, 7], np.uint32).view(np.int32)).to(dev)   # n_pairs, n_inliers, found
        model = torch.full((12,), SENT_F64, dtype=torch.float64, device=dev)
        inl = torch.from_numpy(np.full(cap, SENT_U32, np.uint32).view(np.int32)).to(dev)
        intr = Intrinsics(1000.0, 1000.0, 960.0, 540.0, 0.0)
        ars = cv_b200.Arrsac(1e-7, cv_b200.Xoshiro256PlusPlus(4), ctx).initialization_hypotheses(8192).max_candidate_hypotheses(1024)
        torch.cuda.synchronize()
        ctx.check(ctx.lib.cvb_two_view_pair_dev(ctx.handle, tkp.data_ptr(), tdesc.data_ptr(), tn.data_ptr(),
                                                tkp.data_ptr() + cap * KP_DTYPE.itemsize, tdesc.data_ptr() + cap * 64, tn.data_ptr() + 4,
                                                cap, 24, C.byref(intr), C.addressof(ars.cfg), C.addressof(ars.rng.state), pairs.data_ptr(),
                                                cap, cnt.data_ptr(), model.data_ptr(), inl.data_ptr(), cnt.data_ptr() + 4, cnt.data_ptr() + 8))
        ctx.check(ctx.lib.cvb_arrsac_commit_rng(ctx.handle, C.addressof(ars.rng.state), None))
        c = cnt.cpu().numpy().view(np.uint32)
        got_pairs = pairs.cpu().numpy().view(np.uint32).reshape(cap, 2)
        assert c[0] == len(want_pairs)
        assert np.array_equal(got_pairs[:c[0]].astype(np.int64), want_pairs)
        assert c[2] == 0 and c[1] == 0
        assert (model.cpu().numpy() == SENT_F64).all() and (inl.cpu().numpy().view(np.uint32) == SENT_U32).all()
        ba = np.array([O.calibrate(1000.0, 1000.0, 960.0, 540.0, 0.0, float(kp[0, i]["x"]), float(kp[0, i]["y"])) for i, _ in want_pairs])
        bb = np.array([O.calibrate(1000.0, 1000.0, 960.0, 540.0, 0.0, float(kp[1, j]["x"]), float(kp[1, j]["y"])) for _, j in want_pairs])
        orng = O.rng_xoshiro(4)
        assert O.arrsac(O.arrsac_cfg(1e-7, initialization_hypotheses=8192, max_candidate_hypotheses=1024), 0, ba.reshape(-1, 3),
                        bb.reshape(-1, 3), orng) is None
        assert [int(x) for x in ars.rng.state.s] == [int(x) for x in orng.s]
    finally:
        ctx.close()
