"""AKAZE's keypoint stages past their first plan, bit for bit against the CPU oracle (the bar of tests/test_gpu_akaze.py: every plane,
the candidates / extrema / refined / sorted stages, keypoints and descriptors).

  - a dense 1080p frame: duplicate suppression falls back from k_suppress_smem's ring to k_suppress_par, and the chunk loops of
    k_filter_upper, k_rank_count and k_rank_scatter and the grid-stride loop of k_refine_orient wrap;
  - tiled frames with bit-identical responses, cut by maximum_features inside a run of equal responses, on both suppression paths;
  - batches mixing frames that fall back with frames that keep the ring, in both orders;
  - frames that need more candidates or cached keypoints than the default capacities: the host calls grow the workspace and run again,
    the _dev call reports flag 1 or 2 with clamped counts and leaves the context usable.

Each test proves from the oracle's counts that its path is reached (tests/test_akaze_scenes.py restates the limits)."""
import ctypes as C
import functools

import numpy as np
import pytest

import cv_b200
from cv_b200 import DynamicImage
from cv_b200._lib import KP_DTYPE
from oracle import pyoracle as O
from tests import akaze_scenes as S
from tests.synth import synth_frame
from tests.test_akaze_scenes import SUP_CAPS, capc, capk, chunk_span, pair

pytestmark = pytest.mark.gpu

CAP = 1 << 16   # output slots per frame (the tests' frames have up to 47 263 keypoints)
STAGES = ("candidates", "extrema", "refined", "sorted")


def _bits_equal(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


_ORACLE = {}


def _oracle(key, cfg, planes=False):
    """(keypoints, descriptors, {stage: keypoints}, contrast factor, planes) of the oracle on the frame named `key` (see _frame).  Only
    the small results are kept between tests; the planes (~260 MB for a 1080p frame) are returned to the caller that asks for them."""
    k = (key, tuple(sorted(cfg.items())))
    if k in _ORACLE and not planes:
        return _ORACLE[k] + (None,)
    o = O.Akaze(**cfg)
    kps, desc = o.extract(_frame(key))
    _ORACLE[k] = (kps, desc, {s: o.stage(s) for s in STAGES}, o.contrast_factor())
    pl = None
    if planes:
        pl = [{n: o.plane(i, n) for n in ("Lsmooth", "Lflow", "Lt", "Lx", "Ly", "Ldet") if i or n != "Lflow"}
              for i in range(o.num_evolutions())]
    return _ORACLE[k] + (pl,)


@functools.lru_cache(maxsize=None)
def _frame(key):
    if key == "ring":      # 1920x1080 at 1e-4 with 3 161 candidates in two adjacent classes: the ring path
        return np.float32(0.3) * synth_frame(1)
    if key == "tied3":     # the tied frame at 1e-4: 105 905 candidates, 47 263 keypoints with 127 distinct responses, fallback
        return np.float32(3) * S.tied()[0]
    if key == "vga_fit":   # 640x480 at 1e-4 within the default capacities
        return np.float32(0.3) * synth_frame(2, h=480, w=640, nblobs=1500)
    return getattr(S, key)()[0]


def _check(ak, key, cfg, frame=0, planes=True, got=None):
    """the last extract of `ak` on `frame` equals the oracle on frame `key`; returns the oracle's result"""
    okp, odesc, ostages, kc, oplanes = _oracle(key, cfg, planes)
    if planes:
        assert ak.debug_contrast(frame) == kc
        for i, d in enumerate(oplanes):
            for name, want in d.items():
                assert _bits_equal(ak.debug_plane(i, name, frame), want), (key, i, name)
    for st in STAGES:
        g = ak.debug_stage(st, frame)
        assert len(g) == len(ostages[st]) and g.tobytes() == ostages[st].tobytes(), (key, st, len(g), len(ostages[st]))
    if got is not None:
        assert got[0].tobytes() == okp.tobytes() and np.array_equal(got[1], odesc), key
    return okp, odesc, ostages


def _extract(ak, imgs):
    kps, descs = ak.extract_batch(np.stack(imgs))
    return list(zip(kps, descs))


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


DENSE = dict(detector_threshold=1e-4, maximum_features=-1)


def test_dense_frame_falls_back_wraps_and_replays():
    img = _frame("dense")
    ak = cv_b200.Akaze(ctx=cv_b200.Context(0), max_keypoints=CAP, **DENSE)
    got = _extract(ak, [img])[0]
    _, _, ost = _check(ak, "dense", DENSE, got=got)
    assert pair(ost["candidates"]) > SUP_CAPS                            # k_suppress_par
    n = len(ost["extrema"])                                             # <= the cache the chunk loops run over
    assert n > chunk_span(img.size) and n > _sms() * 2 * (256 // 32)    # chunk loops and k_refine_orient's grid wrap
    again = _extract(ak, [img])[0]
    assert again[0].tobytes() == got[0].tobytes() and np.array_equal(again[1], got[1])
    # the frame fits the default capacities: the device-resident call raises no flag
    _dev_extract(ak.ctx, ak.config, img, 0)


def _check_oracle_only(key, cfg):
    return _oracle(key, cfg)[:3]


def _cut_inside_run(sorted_kps):
    """maximum_features that cuts the longest run of equal responses in the middle, and the run's value"""
    r = sorted_kps["response"]
    starts = np.flatnonzero(np.r_[True, r[1:] != r[:-1]])
    lens = np.diff(np.r_[starts, len(r)])
    k = int(np.argmax(lens))
    assert lens[k] >= 4
    return int(starts[k] + lens[k] // 2), r[starts[k]]


@pytest.mark.parametrize("name,fallback", [("tied", True), ("tied_small", False)])
def test_tied_frame_cut_inside_a_run_of_equal_responses(name, fallback):
    img, cfg = getattr(S, name)()
    _, _, ost = _check_oracle_only(name, cfg)
    assert (pair(ost["candidates"]) > SUP_CAPS) == fallback
    assert len(np.unique(ost["sorted"]["response"])) < 40
    m, v = _cut_inside_run(ost["sorted"])
    cut = dict(cfg, maximum_features=m)
    ak = cv_b200.Akaze(ctx=cv_b200.Context(0), max_keypoints=CAP, **cut)
    kps, desc = _extract(ak, [img])[0]
    okp, _, cst = _check(ak, name, cut, got=(kps, desc))
    assert len(cst["sorted"]) == m
    # both sides of the cut hold the cut value: the last kept keypoint and the first one cut off
    assert cst["sorted"]["response"][-1] == v and ost["sorted"]["response"][m] == v
    # the kept ones of the run are its first ones in the reference's order
    assert cst["sorted"].tobytes() == ost["sorted"][:m].tobytes()


@pytest.mark.parametrize("order", [("dense", "ring"), ("ring", "dense"), ("ring", "dense", "tied3"), ("tied3", "ring", "dense")])
def test_batches_mix_fallback_and_ring_frames(order):
    for key in set(order):
        fb = pair(_check_oracle_only(key, DENSE)[2]["candidates"]) > SUP_CAPS
        assert fb == (key != "ring"), key
    ak = cv_b200.Akaze(ctx=cv_b200.Context(0), max_keypoints=CAP, **DENSE)
    got = _extract(ak, [_frame(k) for k in order])
    for b, key in enumerate(order):
        _check(ak, key, DENSE, frame=b, planes=False, got=got[b])
    for b, key in enumerate(order):
        single = _extract(ak, [_frame(key)])[0]
        assert single[0].tobytes() == got[b][0].tobytes() and np.array_equal(single[1], got[b][1]), key


def test_find_image_keypoints_on_the_dense_frame():
    ak = cv_b200.Akaze(ctx=cv_b200.Context(0), max_keypoints=CAP, **DENSE)
    ss = ak.create_scale_space(_frame("dense"))
    found = ak.find_image_keypoints(ss)[0]
    assert found.tobytes() == _check_oracle_only("dense", DENSE)[2]["refined"].tobytes()
    assert ak.find_image_keypoints(ss)[0].tobytes() == found.tobytes()


@pytest.mark.parametrize("name", sorted(S.CAPACITY))
def test_capacity_frames_extract_on_a_fresh_context(name):
    img, cfg = S.CAPACITY[name]()
    ak = cv_b200.Akaze(ctx=cv_b200.Context(0), max_keypoints=CAP, **cfg)
    got = _extract(ak, [img])[0]
    _, _, ost = _check(ak, name, cfg, got=got)
    assert len(ost["extrema"]) > capk(img.size)
    # the staged find grows the workspace of a scale space without replacing its planes
    ak2 = cv_b200.Akaze(ctx=cv_b200.Context(0), max_keypoints=CAP, **cfg)
    ss = ak2.create_scale_space(img)
    assert ak2.find_image_keypoints(ss)[0].tobytes() == ost["refined"].tobytes()
    kd, dd = ak2.extract_descriptors(ss, ost["sorted"])
    assert len(kd[0]) == len(got[0]) and np.array_equal(dd[0], got[1])


def test_capacity_frame_through_the_dynamic_format_batch():
    img, cfg = S.noise_vga()
    px = (img * np.float32(65535)).astype(np.uint16)
    gray = px.astype(np.float32) / np.float32(65535)
    o = O.Akaze(**cfg)
    okp, odesc = o.extract(gray)
    assert len(o.stage("extrema")) > capk(img.size)
    ak = cv_b200.Akaze(ctx=cv_b200.Context(0), max_keypoints=CAP, **cfg)
    kps, descs = ak.extract_batch([DynamicImage("luma16", px), DynamicImage("luma16", px[::-1].copy())])
    assert kps[0].tobytes() == okp.tobytes() and np.array_equal(descs[0], odesc)
    k1, d1 = ak.extract_from_gray_float_image(np.ascontiguousarray(gray[::-1]))
    assert kps[1].tobytes() == k1.tobytes() and np.array_equal(descs[1], d1)


def test_capacity_frame_through_frame_features():
    """cvb_frame_features_batch (cv-sfm's kps_descriptors) grows the extractor's capacities and runs again, like the extract calls"""
    from oracle import pyoracle_sfm as OS
    img, cfg = S.noise_vga()
    rgb = (np.random.default_rng(7).random((1,) + img.shape + (3,)) * 255).astype(np.uint8)
    K = (500.0, 510.0, 320.0, 240.0, 0.0, -0.1)
    cam = cv_b200.CameraIntrinsicsK1Distortion(cv_b200.CameraIntrinsics(K[:2], K[2:4], K[4]), K[5])
    ak = cv_b200.Akaze(ctx=cv_b200.Context(0), max_keypoints=CAP, **cfg)
    g = cv_b200.frame_features(ak, img[None], rgb, cam)[0]
    okp, odesc, obear, _, ocol = OS.kps_descriptors(O.Akaze(**cfg), img, rgb[0], K)
    assert len(okp) > capk(img.size)
    assert g["keypoints"].tobytes() == okp.tobytes() and np.array_equal(g["descriptors"], odesc)
    assert np.array_equal(g["bearings"].view(np.uint64), obear.view(np.uint64)) and np.array_equal(g["colors"], ocol)


def test_capacity_growth_in_a_mixed_batch():
    cfg = dict(detector_threshold=1e-4, maximum_features=-1)
    ak = cv_b200.Akaze(ctx=cv_b200.Context(0), max_keypoints=CAP, **cfg)
    got = _extract(ak, [_frame("vga_fit"), _frame("noise_vga")])
    _check(ak, "vga_fit", cfg, frame=0, planes=False, got=got[0])
    _check(ak, "noise_vga", cfg, frame=1, planes=False, got=got[1])


def _dev_extract(ctx, config, img, want_flag):
    """cvb_akaze_extract_batch_dev on one frame; asserts the overflow flag and returns (n, keypoints) read back"""
    import torch
    dev = torch.device("cuda", 0)
    t = torch.from_numpy(np.ascontiguousarray(img)[None]).to(dev)
    kp = torch.zeros(CAP * KP_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    d = torch.zeros(CAP * 64, dtype=torch.uint8, device=dev)
    n = torch.zeros(1, dtype=torch.int32, device=dev)
    cfg = config.to_c()
    ctx.check(ctx.lib.cvb_akaze_extract_batch_dev(ctx.handle, C.byref(cfg), t.data_ptr(), 1, img.shape[1], img.shape[0], kp.data_ptr(),
                                                  d.data_ptr(), CAP, n.data_ptr()))
    flag = C.c_uint32()
    ctx.check(ctx.lib.cvb_akaze_dev_overflow(ctx.handle, C.byref(flag)))
    assert flag.value in (want_flag if isinstance(want_flag, tuple) else (want_flag,)), flag.value
    cnt = int(n.cpu()[0])
    return cnt, np.frombuffer(kp.cpu().numpy().tobytes(), KP_DTYPE)[:cnt], d.cpu().numpy().reshape(CAP, 64)[:cnt]


def test_dev_call_flags_the_overflow_and_leaves_the_context_usable():
    img, cfg = S.noise_vga()
    P = img.size
    okp, odesc, ost = _check_oracle_only("noise_vga", cfg)
    ak = cv_b200.Akaze(ctx=cv_b200.Context(0), max_keypoints=CAP, **cfg)
    n, _, _ = _dev_extract(ak.ctx, ak.config, img, 2)            # more cached keypoints than capk: flag 2, counts clamped
    assert len(ost["candidates"]) <= capc(P) and len(ak.debug_stage("candidates")) == len(ost["candidates"])
    assert len(ak.debug_stage("extrema")) <= capk(P) and n <= capk(P) < len(okp)
    # the next call on the context, a frame that fits, is exact and raises no flag
    n2, k2, d2 = _dev_extract(ak.ctx, ak.config, _frame("vga_fit"), 0)
    fkp, fdesc, _ = _check_oracle_only("vga_fit", cfg)
    assert n2 == len(fkp) and k2.tobytes() == fkp.tobytes() and np.array_equal(d2, fdesc)
    # the host call grows the workspace; the _dev call then fits too
    got = _extract(ak, [img])[0]
    assert got[0].tobytes() == okp.tobytes() and np.array_equal(got[1], odesc)
    n3, k3, d3 = _dev_extract(ak.ctx, ak.config, img, 0)
    assert n3 == len(okp) and k3.tobytes() == okp.tobytes() and np.array_equal(d3, odesc)
    # a candidate overflow (the lattice): flag 1 or 2, the candidates clamped to capc
    lat, lcfg = S.lattice()
    ak2 = cv_b200.Akaze(ctx=cv_b200.Context(0), max_keypoints=CAP, **lcfg)
    n4, _, _ = _dev_extract(ak2.ctx, ak2.config, lat, (1, 2))   # 2 when the clamped candidates still overflow the cache
    assert len(ak2.debug_stage("candidates")) == capc(P) and n4 <= capk(P)
