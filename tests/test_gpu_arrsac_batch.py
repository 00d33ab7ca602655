"""GPU: batched device ARRSAC (include/cvb200_batch.h).  Every problem of a batch must equal the oracle's ref_arrsac and the single
call on the same rows with the same generator: pose, inlier set, found and the generator state after the commit -- for every
estimator (eight-point, five-point with both eigenvector rows, P3P) and every way the driver runs the block loop (eager, WHILE node,
unrolled graph).  Mixed batches put problems of 0, K - 1, K and K + 1 data, a problem without consensus and device counts below n_max
next to a 5 000-match problem, under every run mode; B = 1 must be the single entry launch for launch; graph replay must repeat the
result; a commit of the wrong kind is refused.  The fused cvb_two_view_options_dev must equal F separate cvb_two_view_pair_k1_dev calls
on KITTI golden frames and synthetic frames."""
import ctypes as C

import numpy as np
import pytest
import torch

import cv_b200
from cv_b200._lib import ARRSAC_BATCH_MAX, CVB_EINVAL, CVB_EUNSUPPORTED, default_context, load_batch_library
from cv_b200.geom import Pose, Rng
from oracle import pyoracle as O
from tests.common import kitti_frame
from tests.geom_util import pnp_scene, two_view_scene, unit
from tests.synth import synth_frame, warp_frame

pytestmark = pytest.mark.gpu

MODES = {"eager": {"CVB_ARS_NO_GRAPH": "1"}, "while": {"CVB_ARS_WHILE": "1"}, "unrolled": {"CVB_ARS_WHILE": "0"}}
# estimator, oracle kind, eigenvector row, threshold, configuration, problem sizes
KINDS = {
    "eight": (lambda: cv_b200.EightPoint(), 0, 5, 1e-6, {}, (60, 300, 900, 2000)),
    "five_ref": (lambda: cv_b200.NisterStewenius(corrected=False), 2, 5, 1e-6,
                 dict(initialization_hypotheses=64, max_candidate_hypotheses=32, estimations_per_block=16), (40, 250, 600)),
    "five_corr": (lambda: cv_b200.NisterStewenius(corrected=True), 2, 6, 1e-6,
                  dict(initialization_hypotheses=64, max_candidate_hypotheses=32, estimations_per_block=16), (40, 250, 600)),
    "p3p": (lambda: cv_b200.LambdaTwist(), 1, 5, 1e-5, {}, (50, 400, 1500)),
}


def _problems(kind, sizes, seed):
    rng = np.random.default_rng(seed)
    out = []
    for i, n in enumerate(sizes):
        if kind == 1:
            _, _, a, b, _ = pnp_scene(rng, n, outlier_frac=0.1 + 0.1 * (i % 3), noise=1e-4)
        else:
            _, _, a, b, _ = two_view_scene(rng, n, outlier_frac=0.1 + 0.15 * (i % 3), noise=1e-4)
        out.append((a, b))
    return out


def _arrsac(thr, cfg, seed, ctx):
    ars = cv_b200.Arrsac(thr, cv_b200.Xoshiro256PlusPlus(seed), ctx=ctx)
    for k, v in cfg.items():
        getattr(ars, k)(v)
    return ars


def _state(r):
    return [int(x) for x in r.s]


def _same(got, want, exact=True):
    assert (got is None) == (want is None)
    if got is None:
        return
    assert np.array_equal(got[2], want[2])
    if exact:
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    else:
        assert np.allclose(got[0], want[0], atol=1e-9) and np.allclose(got[1], want[1], atol=1e-9)


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("name", list(KINDS))
def test_batch_equals_single_calls_and_oracle(name, mode, monkeypatch):
    est_f, okind, row0, thr, cfg, sizes = KINDS[name]
    for k, v in MODES[mode].items():
        monkeypatch.setenv(k, v)
    probs = _problems(okind, sizes, 10 + okind)
    B = len(probs)
    seeds = [100 + i for i in range(B)]
    ctx = cv_b200.Context(0)
    try:
        ars = _arrsac(thr, cfg, 0, ctx)
        rngs = [cv_b200.Xoshiro256PlusPlus(s, ctx=ctx) for s in seeds]
        singles = [_arrsac(thr, cfg, s, ctx) for s in seeds]
        orngs = [O.rng_xoshiro(s) for s in seeds]
        O.five_point_set_row0(row0)
        try:
            for call in range(2):             # eager, then captured (graph modes)
                got = ars.model_inliers_batch(est_f(), probs, rngs)
                assert len(got) == B
                for i, (a, b) in enumerate(probs):
                    one = singles[i].model_inliers(est_f(), a, b)
                    want = O.arrsac(O.arrsac_cfg(thr, **cfg), okind, a, b, orngs[i])
                    _same(got[i], one, exact=True)
                    _same(got[i], want, exact=False)
                    assert _state(rngs[i].state) == _state(singles[i].rng.state) == _state(orngs[i]), (call, i)
                assert any(g is not None for g in got)
        finally:
            O.five_point_set_row0(5)
    finally:
        ctx.close()


def _dev_batch(ctx, cfg, kind, row0, probs, n_max, counts, rng_states, cap, bufs=None):
    """cvb_arrsac_batch_dev on torch device buffers (problem b at rows b * n_max); returns (per-problem results, stats, rng states).
    bufs: a dict that keeps the device buffers between calls (the same pointers every call)."""
    BL = load_batch_library()
    B = len(probs)
    bc = 4 if kind == 1 else 3
    bufs = {} if bufs is None else bufs
    if not bufs:
        a = np.zeros((B * n_max, 3)); b = np.zeros((B * n_max, bc))
        for i, (pa, pb) in enumerate(probs):
            a[i * n_max:i * n_max + len(pa)] = pa; b[i * n_max:i * n_max + len(pb)] = pb
        bufs.update(ad=torch.from_numpy(a).cuda(), bd=torch.from_numpy(b).cuda(),
                    nd=torch.tensor(counts, dtype=torch.int32).cuda() if counts is not None else None,
                    model=torch.zeros(B * 12, dtype=torch.float64, device="cuda"), inl=torch.zeros(B * cap, dtype=torch.int32, device="cuda"),
                    ninl=torch.zeros(B, dtype=torch.int32, device="cuda"), found=torch.zeros(B, dtype=torch.int32, device="cuda"))
    ad, bd, nd, model, inl, ninl, found = (bufs[k] for k in ("ad", "bd", "nd", "model", "inl", "ninl", "found"))
    for t in (model, inl, ninl, found):
        t.zero_()
    states = (Rng * B)(*rng_states)
    torch.cuda.synchronize()
    ctx.check(BL.cvb_arrsac_batch_dev(ctx.handle, C.addressof(cfg), kind, row0, ad.data_ptr(), bd.data_ptr(),
                                      nd.data_ptr() if nd is not None else None, n_max, B, C.addressof(states), model.data_ptr(),
                                      inl.data_ptr(), cap, ninl.data_ptr(), found.data_ptr()))
    stats = np.zeros(16 * B, np.uint32)
    ctx.check(BL.cvb_arrsac_commit_rng_batch(ctx.handle, C.addressof(states), B, stats.ctypes.data))
    model, inl, ninl, found = model.cpu().numpy(), inl.cpu().numpy().view(np.uint32), ninl.cpu().numpy(), found.cpu().numpy()
    out = []
    for i in range(B):
        if not found[i]:
            out.append(None)
            continue
        out.append((model[i * 12:i * 12 + 9].reshape(3, 3).copy(), model[i * 12 + 9:i * 12 + 12].copy(), inl[i * cap:i * cap + ninl[i]].copy()))
    return out, stats.reshape(B, 16), [_state(states[i]) for i in range(B)]


def _seed_states(seeds):
    out = []
    for s in seeds:
        r = cv_b200.Xoshiro256PlusPlus(s)
        out.append(r.state)
    return out


@pytest.mark.parametrize("mode", list(MODES))
def test_mixed_batch_with_device_counts_equals_oracle(mode, monkeypatch):
    rng = np.random.default_rng(77)
    _, _, a_big, b_big, _ = two_view_scene(rng, 5000, outlier_frac=0.3, noise=1e-4)
    _, _, a_mid, b_mid, _ = two_view_scene(rng, 700, outlier_frac=0.2, noise=1e-4)
    noise_a, noise_b = unit(rng.normal(size=(600, 3))), unit(rng.normal(size=(600, 3)))     # no consensus
    rows = [(a_big[:0], b_big[:0]), (a_mid[:7], b_mid[:7]), (a_mid[:8], b_mid[:8]), (a_mid[:9], b_mid[:9]), (a_big, b_big),
            (noise_a, noise_b), (a_mid, b_mid)]
    n_max = 5120
    counts = [len(x[0]) for x in rows]
    # device counts below n_max; the rows beyond each count hold the big problem's data and must not be read
    probs = [(np.concatenate([pa, a_big[:n_max - len(pa)]]), np.concatenate([pb, b_big[:n_max - len(pb)]])) for pa, pb in rows]
    seeds = [31 + i for i in range(len(rows))]
    for k, v in MODES[mode].items():
        monkeypatch.setenv(k, v)
    ctx = cv_b200.Context(0)
    try:
        ars = cv_b200.Arrsac(1e-6, cv_b200.Xoshiro256PlusPlus(0), ctx=ctx)
        # three runs on the same buffers (graph modes: eager, capture, replay); problems that finish before the block loop retire
        # next to ones that run many blocks, and the WHILE node must still end exactly when the last one does
        bufs = {}
        runs = [_dev_batch(ctx, ars.cfg, 0, 5, probs, n_max, counts, _seed_states(seeds), n_max, bufs) for _ in range(3)]
    finally:
        ctx.close()
    got, stats, states = runs[0]
    for g2, s2, st2 in runs[1:]:
        for i in range(len(rows)):
            _same(g2[i], got[i], exact=True)
        assert st2 == states and np.array_equal(s2[:, :8], stats[:, :8])
    for i, (a, b) in enumerate(rows):
        orng = O.rng_xoshiro(seeds[i])
        want = O.arrsac(O.arrsac_cfg(1e-6), 0, a, b, orng)
        _same(got[i], want, exact=False)
        assert states[i] == _state(orng), i
        assert stats[i][0] == counts[i]
    assert got[0] is None and got[1] is None and got[4] is not None and got[6] is not None
    # the problems leave the block loop on very different iterations: before it (below the initialisation data) and after several blocks
    assert stats[2][4] == 0 and stats[3][4] == 0 and stats[4][4] >= 5


def test_batch_of_one_is_the_single_entry_launch_for_launch():
    rng = np.random.default_rng(5)
    _, _, a, b, _ = two_view_scene(rng, 1500, outlier_frac=0.3, noise=1e-4)
    n = len(a)
    L, BL = cv_b200.load_library(), load_batch_library()
    L.cvb_arrsac_eight_point_dev.argtypes = [C.c_void_p] * 5 + [C.c_uint32] + [C.c_void_p] * 3 + [C.c_uint32] + [C.c_void_p] * 2
    L.cvb_arrsac_commit_rng.argtypes = [C.c_void_p] * 3
    res = []
    for batched in (False, True):
        ctx = cv_b200.Context(0)
        try:
            ars = cv_b200.Arrsac(1e-6, cv_b200.Xoshiro256PlusPlus(0), ctx=ctx)
            ad, bd = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
            nd = torch.tensor([n], dtype=torch.int32).cuda()
            md = torch.zeros(12, dtype=torch.float64, device="cuda"); inl = torch.zeros(n, dtype=torch.int32, device="cuda")
            ninl = torch.zeros(1, dtype=torch.int32, device="cuda"); found = torch.zeros(1, dtype=torch.int32, device="cuda")
            runs = []
            for call in range(3):                     # the same buffers every time: eager, capture, replay
                st = (Rng * 1)(*_seed_states([9]))
                torch.cuda.synchronize()
                l0 = ctx.launch_count()
                if batched:
                    ctx.check(BL.cvb_arrsac_batch_dev(ctx.handle, C.addressof(ars.cfg), 0, 5, ad.data_ptr(), bd.data_ptr(), nd.data_ptr(), n, 1,
                                                      C.addressof(st), md.data_ptr(), inl.data_ptr(), n, ninl.data_ptr(), found.data_ptr()))
                    ctx.check(BL.cvb_arrsac_commit_rng_batch(ctx.handle, C.addressof(st), 1, None))
                else:
                    ctx.check(L.cvb_arrsac_eight_point_dev(ctx.handle, C.addressof(ars.cfg), ad.data_ptr(), bd.data_ptr(), nd.data_ptr(), n,
                                                           C.addressof(st), md.data_ptr(), inl.data_ptr(), n, ninl.data_ptr(), found.data_ptr()))
                    ctx.check(L.cvb_arrsac_commit_rng(ctx.handle, C.addressof(st), None))
                launches = ctx.launch_count() - l0
                m = md.cpu().numpy()
                got = (m[:9].reshape(3, 3), m[9:].copy(), inl.cpu().numpy().view(np.uint32)[:int(ninl.cpu()[0])].copy()) if int(found.cpu()[0]) else None
                runs.append((got, _state(st[0]), launches))
            res.append(runs)
        finally:
            ctx.close()
    orng = O.rng_xoshiro(9)
    want = O.arrsac(O.arrsac_cfg(1e-6), 0, a, b, orng)
    for (g1, s1, l1), (g2, s2, l2) in zip(*res):
        _same(g1, g2, exact=True)
        _same(g1, want, exact=False)
        assert s1 == s2 == _state(orng) and l1 == l2


def test_graph_replay_repeats_the_batch():
    probs = _problems(0, (120, 800, 2500), 3)
    n_max = 2500
    counts = [len(p[0]) for p in probs]
    probs = [(np.concatenate([a, np.zeros((n_max - len(a), 3))]), np.concatenate([b, np.zeros((n_max - len(b), 3))])) for a, b in probs]
    ctx = cv_b200.Context(0)
    try:
        ars = cv_b200.Arrsac(1e-6, cv_b200.Xoshiro256PlusPlus(0), ctx=ctx)
        BL = load_batch_library()
        B = len(probs)
        ad = torch.from_numpy(np.concatenate([p[0] for p in probs])).cuda(); bd = torch.from_numpy(np.concatenate([p[1] for p in probs])).cuda()
        nd = torch.tensor(counts, dtype=torch.int32).cuda()
        model = torch.zeros(B * 12, dtype=torch.float64, device="cuda"); inl = torch.zeros(B * n_max, dtype=torch.int32, device="cuda")
        ninl = torch.zeros(B, dtype=torch.int32, device="cuda"); found = torch.zeros(B, dtype=torch.int32, device="cuda")
        outs = []
        for call in range(3):                         # the same pointers every time: eager, capture, replay
            states = (Rng * B)(*_seed_states([5, 6, 7]))
            model.zero_(); inl.zero_(); ninl.zero_(); found.zero_()
            torch.cuda.synchronize()
            ctx.check(BL.cvb_arrsac_batch_dev(ctx.handle, C.addressof(ars.cfg), 0, 5, ad.data_ptr(), bd.data_ptr(), nd.data_ptr(), n_max, B,
                                              C.addressof(states), model.data_ptr(), inl.data_ptr(), n_max, ninl.data_ptr(), found.data_ptr()))
            ctx.check(BL.cvb_arrsac_commit_rng_batch(ctx.handle, C.addressof(states), B, None))
            outs.append((model.cpu().numpy().tobytes(), inl.cpu().numpy().tobytes(), ninl.cpu().numpy().tobytes(),
                         found.cpu().numpy().tobytes(), [_state(states[i]) for i in range(B)]))
        assert outs[0] == outs[1] == outs[2]
        assert all(np.frombuffer(outs[0][3], np.int32))
    finally:
        ctx.close()


def test_batch_at_the_maximum_and_limits():
    rng = np.random.default_rng(8)
    probs = []
    for i in range(ARRSAC_BATCH_MAX):
        _, _, a, b, _ = two_view_scene(rng, 64 + 8 * i, outlier_frac=0.2, noise=1e-4)
        probs.append((a, b))
    seeds = list(range(200, 200 + ARRSAC_BATCH_MAX))
    ctx = cv_b200.Context(0)
    try:
        ars = cv_b200.Arrsac(1e-6, cv_b200.Xoshiro256PlusPlus(0), ctx=ctx)
        rngs = [cv_b200.Xoshiro256PlusPlus(s, ctx=ctx) for s in seeds]
        got = ars.model_inliers_batch(cv_b200.EightPoint(), probs, rngs)
        for i, (a, b) in enumerate(probs):
            orng = O.rng_xoshiro(seeds[i])
            _same(got[i], O.arrsac(O.arrsac_cfg(1e-6), 0, a, b, orng), exact=False)
            assert _state(rngs[i].state) == _state(orng)
        assert ars.model_inliers_batch(cv_b200.EightPoint(), [], []) == []
        BL = load_batch_library()
        states = (Rng * (ARRSAC_BATCH_MAX + 1))()
        x = torch.zeros(8, dtype=torch.float64, device="cuda")
        rc = BL.cvb_arrsac_batch_dev(ctx.handle, C.addressof(ars.cfg), 0, 5, x.data_ptr(), x.data_ptr(), None, 1, ARRSAC_BATCH_MAX + 1,
                                     C.addressof(states), x.data_ptr(), None, 1, x.data_ptr(), x.data_ptr())
        assert rc == CVB_EUNSUPPORTED
        assert BL.cvb_arrsac_batch_dev(ctx.handle, C.addressof(ars.cfg), 0, 5, x.data_ptr(), x.data_ptr(), None, 1, 0,
                                       C.addressof(states), x.data_ptr(), None, 1, x.data_ptr(), x.data_ptr()) == 0
        assert BL.cvb_arrsac_batch_dev(ctx.handle, C.addressof(ars.cfg), 0, 5, None, x.data_ptr(), None, 1, 2,
                                       C.addressof(states), x.data_ptr(), None, 1, x.data_ptr(), x.data_ptr()) == CVB_EINVAL
        assert BL.cvb_arrsac_batch_dev(ctx.handle, C.addressof(ars.cfg), 3, 5, x.data_ptr(), x.data_ptr(), None, 1, 2,
                                       C.addressof(states), x.data_ptr(), None, 1, x.data_ptr(), x.data_ptr()) == CVB_EINVAL
    finally:
        ctx.close()


def test_commit_of_the_wrong_kind_is_refused():
    rng = np.random.default_rng(4)
    _, _, a, b, _ = two_view_scene(rng, 400, outlier_frac=0.2, noise=1e-4)
    ctx = cv_b200.Context(0)
    try:
        ars = cv_b200.Arrsac(1e-6, cv_b200.Xoshiro256PlusPlus(0), ctx=ctx)
        L, BL = cv_b200.load_library(), load_batch_library()
        L.cvb_arrsac_eight_point_dev.argtypes = [C.c_void_p] * 5 + [C.c_uint32] + [C.c_void_p] * 3 + [C.c_uint32] + [C.c_void_p] * 2
        L.cvb_arrsac_commit_rng.argtypes = [C.c_void_p] * 3
        ad, bd = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
        md = torch.zeros(24, dtype=torch.float64, device="cuda"); w = torch.zeros(8, dtype=torch.int32, device="cuda")
        nd = torch.tensor([400], dtype=torch.int32).cuda()
        states = (Rng * 2)(*_seed_states([1, 2]))
        before = [_state(states[i]) for i in range(2)]
        torch.cuda.synchronize()
        # a batch run, committed as a single run: refused, nothing moves; the batch commit then succeeds
        ctx.check(BL.cvb_arrsac_batch_dev(ctx.handle, C.addressof(ars.cfg), 0, 5, ad.data_ptr(), bd.data_ptr(), None, 200, 2,
                                          C.addressof(states), md.data_ptr(), None, 0, w.data_ptr(), w.data_ptr() + 16))
        assert L.cvb_arrsac_commit_rng(ctx.handle, C.addressof(states), None) == CVB_EINVAL
        assert [_state(states[i]) for i in range(2)] == before
        assert BL.cvb_arrsac_commit_rng_batch(ctx.handle, C.addressof(states), 3, None) == CVB_EINVAL        # another size
        ctx.check(BL.cvb_arrsac_commit_rng_batch(ctx.handle, C.addressof(states), 2, None))
        assert [_state(states[i]) for i in range(2)] != before
        # a single run, committed as a batch: refused; the single commit then succeeds
        st = _seed_states([3])[0]
        ctx.check(L.cvb_arrsac_eight_point_dev(ctx.handle, C.addressof(ars.cfg), ad.data_ptr(), bd.data_ptr(), nd.data_ptr(), 400,
                                               C.addressof(st), md.data_ptr(), None, 0, w.data_ptr(), w.data_ptr() + 16))
        one = (Rng * 1)(st)
        assert BL.cvb_arrsac_commit_rng_batch(ctx.handle, C.addressof(one), 1, None) == CVB_EINVAL
        assert _state(one[0]) == _state(st)
        ctx.check(L.cvb_arrsac_commit_rng(ctx.handle, C.addressof(st), None))
    finally:
        ctx.close()


def _frames_features(frames, camera, cap):
    """kp, desc, counts and K1 bearings of the frames on the device, as cvb_frame_features_batch(_dev) lays them out (frame b at b * cap)"""
    ak = cv_b200.Akaze(maximum_features=cap)
    feats = cv_b200.frame_features(ak, frames, (np.clip(frames, 0, 1) * 255).astype(np.uint8), camera)
    F = len(frames)
    kp = np.zeros((F, cap), cv_b200.KP_DTYPE); desc = np.zeros((F, cap, 64), np.uint8); bear = np.zeros((F, cap, 3)); n = np.zeros(F, np.int32)
    for f, d in enumerate(feats):
        k = len(d["keypoints"])
        kp[f, :k] = d["keypoints"]; desc[f, :k] = d["descriptors"]; bear[f, :k] = d["bearings"]; n[f] = k
    return (torch.from_numpy(kp.view(np.uint8)).cuda(), torch.from_numpy(desc).cuda(), torch.from_numpy(n).cuda(),
            torch.from_numpy(bear).cuda())


@pytest.mark.parametrize("source", ["kitti", "synthetic"])
def test_two_view_options_equals_separate_pair_calls(source):
    if source == "kitti":
        f0, f1 = kitti_frame("0000000000"), kitti_frame("0000000014")
        frames = np.stack([f0, f1, warp_frame(f0, 7, shift=(2.0, 1.0)), warp_frame(f1, 8, shift=(-3.0, 0.5)), f0[:, ::-1].copy()])
        camera = cv_b200.CameraIntrinsicsK1Distortion(cv_b200.CameraIntrinsics(focals=(984.2439, 980.8141), principal_point=(690.0, 233.1966)),
                                                     -0.3728755)
    else:
        base = synth_frame(11, h=360, w=640, nblobs=1200)
        frames = np.stack([base] + [warp_frame(base, 100 + i, shift=(1.5 * i, -0.7 * i)) for i in range(1, 5)] + [synth_frame(12, h=360, w=640, nblobs=1200)])
        camera = cv_b200.CameraIntrinsics(focals=(600.0, 600.0), principal_point=(320.0, 180.0))
    cap = 4096
    kp, desc, n, bear = _frames_features(frames, camera, cap)
    center, options = 0, list(range(1, len(frames)))
    F = len(options)
    ctx = default_context(0)
    ars = cv_b200.Arrsac(1e-6, cv_b200.Xoshiro256PlusPlus(0), ctx=ctx)
    L, BL = cv_b200.load_library(), load_batch_library()
    cv_b200.pair.bind(L)
    K = cv_b200.IntrinsicsK1.from_camera(camera)
    seeds = [40 + f for f in range(F)]
    # the fused call
    pairs = torch.zeros((F, cap, 2), dtype=torch.int32, device="cuda"); npairs = torch.zeros(F, dtype=torch.int32, device="cuda")
    model = torch.zeros((F, 12), dtype=torch.float64, device="cuda"); inl = torch.zeros((F, cap), dtype=torch.int32, device="cuda")
    ninl = torch.zeros(F, dtype=torch.int32, device="cuda"); found = torch.zeros(F, dtype=torch.int32, device="cuda")
    opts = np.array(options, np.uint32)
    states = (Rng * F)(*_seed_states(seeds))
    torch.cuda.synchronize()
    ctx.check(BL.cvb_two_view_options_dev(ctx.handle, desc.data_ptr(), n.data_ptr(), bear.data_ptr(), len(frames), cap, center, opts.ctypes.data, F,
                                          24, C.addressof(ars.cfg), C.addressof(states), pairs.data_ptr(), npairs.data_ptr(), model.data_ptr(),
                                          inl.data_ptr(), ninl.data_ptr(), found.data_ptr()))
    ctx.check(BL.cvb_arrsac_commit_rng_batch(ctx.handle, C.addressof(states), F, None))
    # F separate pair calls, the same camera and generators
    kpb = kp.view(-1)
    kp_size = cv_b200.KP_DTYPE.itemsize
    any_found = 0
    for f, o in enumerate(options):
        p1 = torch.zeros((cap, 2), dtype=torch.int32, device="cuda"); np1 = torch.zeros(1, dtype=torch.int32, device="cuda")
        m1 = torch.zeros(12, dtype=torch.float64, device="cuda"); i1 = torch.zeros(cap, dtype=torch.int32, device="cuda")
        ni1 = torch.zeros(1, dtype=torch.int32, device="cuda"); fd1 = torch.zeros(1, dtype=torch.int32, device="cuda")
        st = _seed_states([seeds[f]])[0]
        torch.cuda.synchronize()
        ctx.check(L.cvb_two_view_pair_k1_dev(ctx.handle, kpb.data_ptr(), desc.data_ptr(), n.data_ptr(), kpb.data_ptr() + o * cap * kp_size,
                                             desc.data_ptr() + o * cap * 64, n.data_ptr() + 4 * o, cap, 24, C.byref(K), C.addressof(ars.cfg),
                                             C.addressof(st), p1.data_ptr(), cap, np1.data_ptr(), m1.data_ptr(), i1.data_ptr(), ni1.data_ptr(),
                                             fd1.data_ptr()))
        L.cvb_arrsac_commit_rng.argtypes = [C.c_void_p] * 3
        ctx.check(L.cvb_arrsac_commit_rng(ctx.handle, C.addressof(st), None))
        k = int(np1.cpu()[0])
        assert int(npairs[f].cpu()) == k and torch.equal(pairs[f, :k].cpu(), p1[:k].cpu()), f
        assert int(found[f].cpu()) == int(fd1.cpu()[0]), f
        if int(fd1.cpu()[0]):
            any_found += 1
            c = int(ni1.cpu()[0])
            assert int(ninl[f].cpu()) == c and torch.equal(inl[f, :c].cpu(), i1[:c].cpu()), f
            assert model[f].cpu().numpy().tobytes() == m1.cpu().numpy().tobytes(), f
        assert _state(states[f]) == _state(st), f
    assert any_found >= 2
    # the Python wrapper: the same results, two_view_minimum_robust_matches applied on the host
    rngs = [cv_b200.Xoshiro256PlusPlus(s) for s in seeds]
    res = cv_b200.init_two_view_options(dict(descriptors=desc, counts=n, bearings=bear), center, options, ars, rngs, minimum_robust_matches=0)
    res_min = cv_b200.init_two_view_options(dict(descriptors=desc, counts=n, bearings=bear), center, options, ars,
                                            [cv_b200.Xoshiro256PlusPlus(s) for s in seeds])
    pairs_h, inl_h, ninl_h, found_h = pairs.cpu().numpy(), inl.cpu().numpy(), ninl.cpu().numpy(), found.cpu().numpy()
    for f in range(F):
        assert _state(rngs[f].state) == _state(states[f])
        if not found_h[f]:
            assert res[f] is None and res_min[f] is None
            continue
        want = pairs_h[f][inl_h[f, :ninl_h[f]]]
        assert np.array_equal(res[f][2], want.astype(np.int64))
        assert (res_min[f] is None) == (ninl_h[f] < 256)
