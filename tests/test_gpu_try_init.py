"""GPU: cv-sfm's reconstruction creation on the device (include/cvb200_try_init.h) -- add_reconstruction bit for bit against its oracle
(oracle/ref_try_init.c), try_init against the oracle chain (the init oracle, then ref_try_init) and against the composition of the public
calls, its statuses, the snapshot's geometry on a noise-free scene, its use by incorporate_frame and export, and argument errors."""
import ctypes as C

import numpy as np
import pytest
import torch

import cv_b200
from cv_b200._lib import CVB_EINVAL, CVB_EUNSUPPORTED, default_context, load_init_library, load_try_init_library
from cv_b200.incorporate import check_incorporate, incorporate_frame_dev, snapshot_to_device, snapshot_to_host
from cv_b200.pair import INIT_RESULT_DTYPE, InitSettings
from cv_b200.reconstruction import check_reconstruction
from cv_b200.try_init import RESULT_DTYPE, add_reconstruction, add_reconstruction_dev, try_init, try_init_dev
from oracle import pyoracle_init as OI
from oracle import pyoracle_try_init as OT
from tests.synth import synth_frame, warp_frame
from tests.try_init_scenes import descriptor_scene, frame_store, random_lists

pytestmark = pytest.mark.gpu

KEYS = ("poses", "view_offsets", "view_landmarks", "bearings", "descriptors", "colors", "landmark_offsets", "observations", "constraints")
SETTINGS = dict(three_view_patience=0, two_view_minimum_robust_matches=64)


@pytest.fixture(scope="module")
def ctx():
    return default_context(0)


def _equal(got, want, keys=KEYS):
    for k in keys:
        g, w = got[k], want[k]
        if g is None or w is None:
            assert g is None and w is None, k
            continue
        assert np.ascontiguousarray(g).tobytes() == np.ascontiguousarray(w).tobytes(), k


def _dev_store(st):
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return dict(descriptors=t(st["descriptors"]), counts=t(np.asarray(st["counts"], np.int32)), bearings=t(st["bearings"]),
                colors=t(st["colors"]))


def _init_record(comb, fm, sm, fp, sp):
    ir = np.zeros(1, INIT_RESULT_DTYPE)
    ir["status"] = OI.ACCEPTED
    ir["n_combined"], ir["n_first_matches"], ir["n_second_matches"] = len(comb), len(fm), len(sm)
    ir["first_pose"]["r"], ir["first_pose"]["t"] = fp[:9], fp[9:]
    ir["second_pose"]["r"], ir["second_pose"]["t"] = sp[:9], sp[9:]
    return ir


def _padded(a, cap, k):
    p = np.zeros((cap, k), np.uint32)
    p[:len(a)] = a
    return torch.from_numpy(p.view(np.int32)).cuda()


# ---- 1. add_reconstruction against the oracle -----------------------------------------------------------------------------------------
CASES = {"random": ((1001, 777, 333), (200, 150, 120)), "empty_lists": ((517, 300, 299), (0, 0, 0)), "zero_first": ((700, 0, 455), (0, 0, 100)),
         "zero_second": ((259, 901, 0), (0, 120, 0)), "full": ((1024, 1024, 1024), (500, 300, 200))}


@pytest.mark.parametrize("cap", [1024, 8192])
@pytest.mark.parametrize("colors", [True, False])
@pytest.mark.parametrize("case", list(CASES))
def test_add_reconstruction_equals_the_oracle(ctx, cap, colors, case):
    rng = np.random.default_rng(cap + len(case) + colors)
    n, ks = CASES[case]
    n = tuple(x * cap // 1024 - (x * cap // 1024 > 0 and case != "full") * 3 for x in n)   # counts that are not block multiples
    comb, fm, sm = random_lists(rng, *n, *[k * cap // 1024 for k in ks])
    st = frame_store(rng, [n[1], 5, n[0], n[2]], cap, colors)
    fp, sp = rng.normal(size=12), rng.normal(size=12)
    want = OT.add_reconstruction(st["descriptors"], st["counts"], st["bearings"], st["colors"], 2, 0, 3, fp, sp, comb, fm, sm)
    ir = torch.from_numpy(_init_record(comb, fm, sm, fp, sp).view(np.uint8)).cuda()
    sd, cnt = add_reconstruction_dev(ctx, _dev_store(st), 2, 0, 3, ir, _padded(comb, cap, 3), _padded(fm, cap, 2), _padded(sm, cap, 2))
    _equal(snapshot_to_host(sd), want)
    assert (cnt["V"], cnt["n_features"], cnt["C"], cnt["merges"]) == (3, sum(n), 1, 0) and cnt["n_observations"] == sum(n)
    host, hcnt = add_reconstruction(ctx, st, 2, 0, 3, fp, sp, comb, fm, sm)
    _equal(host, want)
    assert hcnt.tobytes() == cnt.tobytes()


# ---- 2. / 3. try_init against the oracle chain and the composition of the public calls ------------------------------------------------
def _akaze_store():
    base = synth_frame(11, h=360, w=640, nblobs=1200)
    frames = np.stack([base] + [warp_frame(base, 100 + i, shift=(1.5 * i, -0.7 * i)) for i in range(1, 5)])
    camera = cv_b200.CameraIntrinsics(focals=(600.0, 600.0), principal_point=(320.0, 180.0))
    cap = 4096
    feats = cv_b200.frame_features(cv_b200.Akaze(maximum_features=cap), frames, (np.clip(frames, 0, 1) * 255).astype(np.uint8), camera)
    Fr = len(frames)
    st = dict(descriptors=np.zeros((Fr, cap, 64), np.uint8), bearings=np.zeros((Fr, cap, 3)), colors=np.zeros((Fr, cap, 3), np.uint8),
              counts=np.zeros(Fr, np.int32))
    for f, d in enumerate(feats):
        k = len(d["keypoints"])
        st["descriptors"][f, :k], st["bearings"][f, :k], st["colors"][f, :k], st["counts"][f] = d["descriptors"], d["bearings"], d["colors"], k
    return st


def _rngs(seeds=(1, 2, 3, 4)):
    return [cv_b200.Xoshiro256PlusPlus(s) for s in seeds]


def _composition(ctx, store, center, options, settings, seeds):
    """two_view_options_dev + commit, cvb_init_reconstruction_dev into device tensors, add_reconstruction_dev; and the oracle chain on
    the downloaded two-view outputs"""
    ars = cv_b200.Arrsac(1e-6, cv_b200.Xoshiro256PlusPlus(0), ctx=ctx)
    rngs = _rngs(seeds)
    ds = _dev_store(store)
    frames, cap, opts, two = cv_b200.pair._two_view_options_dev(ds, center, options, ars, rngs, 24)
    res = torch.zeros(INIT_RESULT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    lists = [torch.zeros((cap, k), dtype=torch.int32, device="cuda") for k in (3, 2, 2)]
    tri = cv_b200.LinearEigenTriangulator()
    torch.cuda.synchronize()
    ctx.check(load_init_library().cvb_init_reconstruction_dev(
        ctx.handle, C.addressof(settings), C.addressof(tri.cfg), ds["bearings"].data_ptr(), frames, cap, center, opts.ctypes.data, len(opts),
        *[two[k].data_ptr() for k in ("pairs", "n_pairs", "model", "inliers", "n_inliers", "found")], res.data_ptr(),
        *[x.data_ptr() for x in lists], None))
    torch.cuda.synchronize()
    r = np.frombuffer(res.cpu().numpy().tobytes(), INIT_RESULT_DTYPE)[0]
    sd = None
    if r["status"] == OI.ACCEPTED:
        sd, _ = add_reconstruction_dev(ctx, ds, center, options[r["first"]], options[r["second"]], res, *lists)
    h = {k: v.cpu().numpy() for k, v in two.items()}
    want = OT.try_init(store["descriptors"], store["counts"], store["bearings"], store["colors"], center, options, h["pairs"].view(np.uint32),
                       h["n_pairs"].view(np.uint32), h["model"], h["inliers"].view(np.uint32), h["n_inliers"].view(np.uint32), h["found"],
                       OI.InitCfg(**{k: getattr(settings, k) for k, *_ in settings._fields_}))
    return r, sd, rngs, want


def _run(ctx, store, center, options, settings, seeds=(1, 2, 3, 4)):
    ars = cv_b200.Arrsac(1e-6, cv_b200.Xoshiro256PlusPlus(0), ctx=ctx)
    rngs = _rngs(seeds)
    got = try_init_dev(_dev_store(store), center, options, ars, rngs, settings=settings)
    return got, rngs


def _same_rngs(a, b):
    assert [bytes(x.state) for x in a] == [bytes(x.state) for x in b]


def _scene_store(seed=5, noise=0.0):
    return descriptor_scene(np.random.default_rng(seed), 4, n_points=700, cap=1024, noise=noise)


@pytest.mark.parametrize("source", ["akaze", "scene"])
def test_try_init_equals_the_oracle_chain_and_the_composition(ctx, source):
    store = _akaze_store() if source == "akaze" else _scene_store()["store"]
    options = [1, 2, 3, 4] if source == "akaze" else [1, 2, 3]
    settings = InitSettings(**SETTINGS)
    got, rngs = _run(ctx, store, 0, options, settings, seeds=(1, 2, 3, 4)[:len(options)])
    r, sd, crngs, want = _composition(ctx, store, 0, options, settings, (1, 2, 3, 4)[:len(options)])
    _same_rngs(rngs, crngs)
    assert got["result"]["init"].tobytes() == r.tobytes() == want["init"]["result"].tobytes()
    assert got["result"]["status"] == want["status"] and list(got["result"]["frames"]) == want["frames"]
    if source == "scene":
        assert want["status"] == OT.CREATED
    if want["status"] == OT.CREATED:
        _equal(snapshot_to_host(got["snapshot"]), want["snapshot"])
        _equal(snapshot_to_host(sd), want["snapshot"])
        assert got["frames"] == want["frames"]
    else:
        assert got["snapshot"] is None and sd is None and got["result"]["counts"].tobytes() == bytes(24)


def test_optimised_init_matches_the_oracle_chain_but_the_poses(ctx):
    sc = _scene_store(seed=7, noise=1e-7)
    settings = InitSettings(three_view_patience=200, two_view_minimum_robust_matches=64)
    got, rngs = _run(ctx, sc["store"], 0, [1, 2, 3], settings, seeds=(1, 2, 3))
    _, _, crngs, want = _composition(ctx, sc["store"], 0, [1, 2, 3], settings, (1, 2, 3))
    _same_rngs(rngs, crngs)
    assert want["status"] == OT.CREATED and got["result"]["status"] == OT.CREATED and got["frames"] == want["frames"]
    g = snapshot_to_host(got["snapshot"])
    _equal(g, want["snapshot"], keys=[k for k in KEYS if k not in ("poses", "constraints")])
    assert np.abs(g["poses"] - want["snapshot"]["poses"]).max() < 1e-8
    gc, wc = g["constraints"][0], want["snapshot"]["constraints"][0]
    assert list(gc["views"]) == [0, 1, 2] and np.abs(gc["poses"]["t"] - wc["poses"]["t"]).max() < 1e-8


# ---- 4. statuses --------------------------------------------------------------------------------------------------------------------
def _assert_none(ctx, store, options, settings, status):
    got, rngs = _run(ctx, store, 0, options, settings, seeds=tuple(range(1, len(options) + 1)))
    r, sd, crngs, want = _composition(ctx, store, 0, options, settings, tuple(range(1, len(options) + 1)))
    assert got["status"] == status and want["status"] == {"none": OT.NONE, "none_bearing_pairs": OT.NONE_BEARING_PAIRS}[status]
    assert got["result"]["status"] == want["status"] and got["snapshot"] is None and sd is None
    assert got["result"]["counts"].tobytes() == bytes(24) and got["result"]["init"].tobytes() == r.tobytes()
    _same_rngs(rngs, crngs)
    if options:
        assert [bytes(x.state) for x in rngs] != [bytes(x.state) for x in _rngs(tuple(range(1, len(options) + 1)))]   # advanced
    return got


def test_statuses_without_a_snapshot(ctx):
    st = _scene_store()["store"]
    cfg = InitSettings(**SETTINGS)
    assert _assert_none(ctx, st, [1], cfg, "none")["frames"][1] is None        # fewer than two options
    # every option sees a block of its own: no pair has common matches
    n = 900
    sc = descriptor_scene(np.random.default_rng(9), 3, n_points=n, cap=1024, seen=[np.arange(f * 300, (f + 1) * 300) for f in range(3)])
    _assert_none(ctx, sc["store"], [1, 2, 3], InitSettings(three_view_patience=0, two_view_minimum_robust_matches=32), "none")
    # options 1 and 2 share only a tight cluster: the bearing-pair abort
    sc = descriptor_scene(np.random.default_rng(3), 3, n_points=n, cap=1024, cluster=200,
                          seen=[np.r_[0:200, 200:400], np.r_[0:200, 400:600], np.r_[600:800]])
    got = _assert_none(ctx, sc["store"], [1, 2, 3], InitSettings(three_view_patience=50, two_view_minimum_robust_matches=32),
                       "none_bearing_pairs")
    assert got["frames"] == [0, 1, 2]


# ---- 5. the snapshot's geometry on a noise-free scene ---------------------------------------------------------------------------------
def test_noise_free_snapshot_joins_one_point_per_landmark(ctx):
    sc = _scene_store(seed=11)
    got, _ = _run(ctx, sc["store"], 0, [1, 2, 3], InitSettings(**SETTINGS), seeds=(1, 2, 3))
    assert got["status"] == "created"
    s = snapshot_to_host(got["snapshot"])
    fr = got["frames"]
    pts = [np.argsort(sc["inv"][f]) for f in fr]                  # the world point of each feature of views 0, 1, 2
    vo, lo, ob = s["view_offsets"], s["landmark_offsets"], s["observations"]
    shared = [0, 0]
    for l in range(len(lo) - 1):
        o = ob[lo[l]:lo[l + 1]]
        assert list(o[:, 0]) == sorted(o[:, 0]) and len(set(o[:, 0])) == len(o)
        if len(o) > 1:
            assert len({int(pts[v][f]) for v, f in o}) == 1
            for v in o[1:, 0]:
                shared[v - 1] += 1
        for v, f in o:
            assert s["view_landmarks"][vo[v] + f] == l
    N = [int(vo[i + 1] - vo[i]) for i in range(3)]
    ir = got["result"]["init"]
    assert len(lo) - 1 == sum(N) - shared[0] - shared[1]
    assert shared == [ir["n_first_matches"] + ir["n_combined"], ir["n_second_matches"] + ir["n_combined"]]
    c = s["constraints"][0]
    assert c["poses"][0].tobytes() == ir["first_pose"].tobytes() and c["poses"][1].tobytes() == ir["second_pose"].tobytes()
    assert s["poses"][1].tobytes() == np.concatenate([ir["first_pose"]["r"], ir["first_pose"]["t"]]).tobytes()
    assert check_incorporate(s) == 0
    assert check_reconstruction(s["view_offsets"], s["view_landmarks"], s["landmark_offsets"], s["observations"], s["constraints"]) == 0


# ---- 6. downstream: incorporate_frame and export ---------------------------------------------------------------------------------------
def test_incorporate_a_fourth_frame_and_export(ctx):
    sc = _scene_store(seed=13)
    st = sc["store"]
    got, _ = _run(ctx, st, 0, [1, 2, 3], InitSettings(**SETTINGS), seeds=(1, 2, 3))
    assert got["status"] == "created"
    frames = got["frames"]
    new = next(f for f in (1, 2, 3, 4) if f not in frames)
    n = int(st["counts"][new])
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    ir = got["result"]["init"]
    oracle_sd = snapshot_to_device(OT.add_reconstruction(st["descriptors"], st["counts"], st["bearings"], st["colors"], *frames, ir["first_pose"],
                                                         ir["second_pose"], *_lists_of(ctx, st, frames)))
    outs = []
    for sd in (got["snapshot"], oracle_sd):
        ars = cv_b200.Arrsac(1e-5, cv_b200.Xoshiro256PlusPlus(21), ctx)
        outs.append(incorporate_frame_dev(ctx, sd, dev(st["descriptors"][new, :n]), dev(st["bearings"][new, :n]), np.arange(3, dtype=np.uint32),
                                          ars, new_colors=dev(st["colors"][new, :n])))
    a, b = outs
    assert a["status"] == b["status"] == "kept"
    _equal(snapshot_to_host(a["snapshot"]), snapshot_to_host(b["snapshot"]))
    h = snapshot_to_host(a["snapshot"])
    ex = cv_b200.export_reconstruction(ctx, h["poses"], h["view_offsets"], h["view_landmarks"], h["bearings"], h["landmark_offsets"],
                                       h["observations"], h["colors"])
    assert len(ex["points"]) > 100 and len(ex["cameras"]) == 4


def _lists_of(ctx, st, frames):
    """the init's lists, recomputed by the oracle chain from the same two-view outputs"""
    _, _, _, want = _composition(ctx, st, 0, [1, 2, 3], InitSettings(**SETTINGS), (1, 2, 3))
    assert want["frames"] == frames
    return want["init"]["combined"], want["init"]["first_matches"], want["init"]["second_matches"]


# ---- 7. host forms, repeats, argument errors ---------------------------------------------------------------------------------------------
def test_dev_equals_host_repeats_and_errors(ctx):
    st = _scene_store(seed=17)["store"]
    cfg = InitSettings(**SETTINGS)
    got, r1 = _run(ctx, st, 0, [1, 2, 3], cfg, seeds=(1, 2, 3))
    ars = cv_b200.Arrsac(1e-6, cv_b200.Xoshiro256PlusPlus(0), ctx=ctx)
    hr = _rngs((1, 2, 3))
    host = try_init(st, 0, [1, 2, 3], ars, hr, settings=cfg)
    _same_rngs(r1, hr)
    assert host["result"].tobytes() == got["result"].tobytes() and host["status"] == "created"
    _equal(host["snapshot"], snapshot_to_host(got["snapshot"]))
    again, _ = _run(ctx, st, 0, [1, 2, 3], cfg, seeds=(1, 2, 3))
    assert again["result"].tobytes() == got["result"].tobytes()
    _equal(snapshot_to_host(again["snapshot"]), snapshot_to_host(got["snapshot"]))
    # argument errors of the C entries
    L = load_try_init_library()
    ds = _dev_store(st)
    frames, cap = ds["descriptors"].shape[0], ds["descriptors"].shape[1]
    outs = [torch.zeros(n, dtype=torch.uint8, device="cuda") for n in (3 * 96, 16, 12 * cap, 72 * cap, 192 * cap, 9 * cap, 12 * cap + 4,
                                                                        24 * cap, 208, RESULT_DTYPE.itemsize)]
    tri = cv_b200.LinearEigenTriangulator()
    states = (cv_b200.geom.Rng * 65)()

    def call(options=(1, 2, 3), center=0, tri_cfg=tri.cfg, desc=ds["descriptors"].data_ptr(), res=outs[-1].data_ptr()):
        opts = np.array(options, np.uint32)
        return L.cvb_try_init_dev(ctx.handle, C.addressof(cfg), C.addressof(tri_cfg), C.addressof(ars.cfg), C.addressof(states), 24, desc,
                                  ds["counts"].data_ptr(), ds["bearings"].data_ptr(), None, frames, cap, center, opts.ctypes.data, len(opts),
                                  *[o.data_ptr() for o in outs[:5]], None, *[o.data_ptr() for o in outs[6:-1]], res)
    assert call(desc=None) == CVB_EINVAL and call(res=None) == CVB_EINVAL
    assert call(center=frames) == CVB_EINVAL and call(options=(1, 2, frames)) == CVB_EINVAL
    assert call(options=[1] * 65) == CVB_EUNSUPPORTED
    for m in (cv_b200.RelativeDltTriangulator(), cv_b200.AngularL1Triangulator(), cv_b200.AngularLInfinityTriangulator()):
        assert call(tri_cfg=m.cfg) == CVB_EUNSUPPORTED
    ir = torch.zeros(INIT_RESULT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    lst = torch.zeros(3 * cap, dtype=torch.int32, device="cuda")

    def add(f=(0, 1, 2), desc=ds["descriptors"].data_ptr(), ir_p=ir.data_ptr()):
        return L.cvb_add_reconstruction_dev(ctx.handle, desc, ds["counts"].data_ptr(), ds["bearings"].data_ptr(), None, frames, cap, *f, ir_p,
                                            lst.data_ptr(), lst.data_ptr(), lst.data_ptr(), *[o.data_ptr() for o in outs[:5]], None,
                                            *[o.data_ptr() for o in outs[6:-1]], outs[-1].data_ptr())
    assert add(desc=None) == CVB_EINVAL and add(ir_p=None) == CVB_EINVAL
    assert add(f=(0, 1, frames)) == CVB_EINVAL and add(f=(0, 1, 1)) == CVB_EINVAL and add(f=(2, 1, 2)) == CVB_EINVAL
    assert add() == 0
    col = torch.zeros(9 * cap, dtype=torch.uint8, device="cuda")
    assert L.cvb_add_reconstruction_dev(ctx.handle, ds["descriptors"].data_ptr(), ds["counts"].data_ptr(), ds["bearings"].data_ptr(), None, frames,
                                        cap, 0, 1, 2, ir.data_ptr(), lst.data_ptr(), lst.data_ptr(), lst.data_ptr(),
                                        *[o.data_ptr() for o in outs[:5]], col.data_ptr(), *[o.data_ptr() for o in outs[6:-1]],
                                        outs[-1].data_ptr()) == CVB_EINVAL    # colours out without colours in
