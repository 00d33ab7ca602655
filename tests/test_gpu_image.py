"""GPU: the extractor's input on the device (include/cvb200_image.h, libcvb200_image.so).

  * k_from_dynamic equals the oracle (GrayFloatImage::from_dynamic, to_rgb8) bit for bit for all eight formats: batches, row widths
    whose bytes are not a multiple of 16, 1 x 1 frames, unaligned sources and the exhaustive 8- and 16-bit value sweeps;
  * the KITTI frames as Luma8 at Akaze::sparse() give the reference's 399 / 343 descriptors, the same bytes as the f32 path; 16-bit and
    RGB(A) copies of them give the same output; a synthetic colour frame equals the f32 entry on the oracle-converted plane;
  * frame_features from one 8-bit image equals cvb_frame_features_batch on the oracle's (gray, rgb8) pair; the two-view entry on the
    KITTI pair as Luma8 reproduces tutorial chapter 5 with the f32 entry's generator state;
  * mixed and repeated calls in one context give the bytes of fresh contexts; unsupported formats are refused."""
import ctypes as C

import numpy as np
import pytest

import cv_b200
from cv_b200 import CameraIntrinsics, CameraIntrinsicsK1Distortion, DynamicImage
from cv_b200._lib import CVB_EINVAL, CVB_EUNSUPPORTED, KP_DTYPE
from cv_b200.image import FORMATS
from cv_b200.image import lib as image_lib
from oracle import pyoracle_image as OI
from tests.common import GOLDEN, kitti_frame
from tests.synth import synth_frame

pytestmark = pytest.mark.gpu

TUTORIAL = (9.842439e+02, 9.808141e+02, 6.900000e+02, 2.331966e+02, 0.0, -3.728755e-01)  # tutorial chapter 5 main.rs:36-42


def _cam(fx, fy, cx, cy, skew, k1):
    return CameraIntrinsicsK1Distortion(CameraIntrinsics((fx, fy), (cx, cy), skew), k1)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _kitti8(name):
    return np.load(f"{GOLDEN}/kitti_{name}.npz")["image"]


def _random_pixels(kind, shape, seed):
    _, ch, dt = FORMATS[kind]
    rng = np.random.default_rng(seed)
    full = shape if ch == 1 else shape + (ch,)
    return rng.integers(0, np.iinfo(dt).max + 1, full, dtype=dt)


def _device_convert(kind, pixels, rgb=False, offset=0):
    """cvb_gray_float_from_dynamic_dev on pixels [B, H, W(, C)] uploaded to the device (offset: bytes the source starts behind a 16-byte
    boundary); returns (gray [B, H, W], rgb8 [B, H, W, 3] or None)."""
    import torch
    code = FORMATS[kind][0]
    B, H, W = pixels.shape[:3]
    raw = np.ascontiguousarray(pixels).view(np.uint8).reshape(-1)
    dev = torch.device("cuda", 0)
    buf = torch.zeros(raw.size + 16, dtype=torch.uint8, device=dev)
    buf[offset:offset + raw.size] = torch.from_numpy(raw.copy()).to(dev)
    gray = torch.full((B * H * W,), float("nan"), dtype=torch.float32, device=dev)
    col = torch.zeros(B * H * W * 3, dtype=torch.uint8, device=dev) if rgb else None
    torch.cuda.synchronize()
    ctx = cv_b200.Context(0)
    L = image_lib()
    ctx.check(L.cvb_gray_float_from_dynamic_dev(ctx.handle, code, buf.data_ptr() + offset, B, W, H, gray.data_ptr(),
                                                col.data_ptr() if rgb else None))
    ctx.sync()
    ctx.close()
    return gray.cpu().numpy().reshape(B, H, W), (col.cpu().numpy().reshape(B, H, W, 3) if rgb else None)


def _oracle(kind, pixels):
    code = FORMATS[kind][0]
    gray = OI.from_dynamic(code, pixels)
    return gray, (OI.to_rgb8(code, pixels) if code <= 3 else None)


@pytest.mark.parametrize("kind", list(FORMATS))
def test_kernel_equals_oracle_bit_for_bit(kind):
    rgb = FORMATS[kind][0] <= 3
    for seed, (B, H, W), offset in ((1, (3, 7, 13), 0), (2, (1, 1, 1), 0), (3, (2, 33, 50), 0), (4, (1, 17, 101), 0),
                                    (5, (4, 9, 31), 1), (6, (1, 64, 64), 0), (7, (2, 5, 7), 3)):
        px = _random_pixels(kind, (B, H, W), seed)
        g, c = _device_convert(kind, px, rgb, offset)
        wg, wc = _oracle(kind, px)
        assert np.array_equal(_bits(g), _bits(wg)), (kind, B, H, W, offset)
        if rgb:
            assert np.array_equal(c, wc), (kind, B, H, W, offset)


@pytest.mark.parametrize("kind", list(FORMATS))
def test_exhaustive_value_sweep(kind):
    """every value of the channel width: in the luma (luma formats) or in all of R = G = B and, one channel at a time, in R, G and B"""
    _, ch, dt = FORMATS[kind]
    v = np.arange(np.iinfo(dt).max + 1, dtype=np.uint32).astype(dt)
    n = v.size
    if ch <= 2:
        px = np.stack([v, v[::-1]], -1) if ch == 2 else v
        px = px.reshape((1, n // 256, 256) + px.shape[1:])
    else:
        z = np.zeros_like(v)
        rows = [np.stack([v, v, v], -1), np.stack([v, z, z], -1), np.stack([z, v, z], -1), np.stack([z, z, v], -1)]
        if ch == 4:
            rows = [np.concatenate([r, v[::-1, None]], -1) for r in rows]
        px = np.stack(rows).reshape(4, n // 256, 256, ch)
    g, c = _device_convert(kind, px, FORMATS[kind][0] <= 3)
    wg, wc = _oracle(kind, px)
    assert np.array_equal(_bits(g), _bits(wg))
    if c is not None:
        assert np.array_equal(c, wc)
    if ch >= 3:     # a gray pixel is its own luma
        assert np.array_equal(_bits(g[0].reshape(-1)), _bits(v.astype(np.float32) / np.float32(np.iinfo(dt).max)))


def test_kitti_luma8_sparse_equals_the_f32_path_and_the_reference_counts():
    ak = cv_b200.Akaze.sparse()
    for name, count in (("0000000000", 399), ("0000000014", 343)):      # akaze/tests/estimate_pose.rs:41-42
        kps, d = ak.extract(DynamicImage.luma8(_kitti8(name)))
        fk, fd = ak.extract_from_gray_float_image(kitti_frame(name))
        assert len(d) == count and kps.tobytes() == fk.tobytes() and np.array_equal(d, fd)
    # the 16-bit case of test_gpu_akaze's from_dynamic test through the device conversion
    im16 = _kitti8("0000000000").astype(np.uint16) * np.uint16(257) + np.uint16(3)
    k16, d16 = ak.extract(DynamicImage.luma16(im16))
    hk, hd = ak.extract(im16)
    assert len(d16) > 0 and k16.tobytes() == hk.tobytes() and np.array_equal(d16, hd)


def test_kitti_replicated_into_rgb8_and_rgba8_equals_luma8():
    ak = cv_b200.Akaze.sparse()
    a, b = _kitti8("0000000000"), _kitti8("0000000014")
    want = ak.extract_batch([DynamicImage.luma8(a), DynamicImage.luma8(b)])
    alpha = np.random.default_rng(0).integers(0, 256, a.shape, dtype=np.uint8)
    for frames in ([DynamicImage.rgb8(np.repeat(x[..., None], 3, -1)) for x in (a, b)],
                   [DynamicImage.rgba8(np.stack([x, x, x, alpha], -1)) for x in (a, b)],
                   [DynamicImage.luma_a8(np.stack([x, alpha], -1)) for x in (a, b)]):
        got = ak.extract_batch(frames)
        for f in range(2):
            assert got[0][f].tobytes() == want[0][f].tobytes() and np.array_equal(got[1][f], want[1][f])
    assert [len(d) for d in want[1]] == [399, 343]


@pytest.mark.parametrize("kind", ["rgb8", "rgba8", "rgb16", "rgba16", "luma_a16"])
def test_synthetic_colour_frame_equals_the_f32_entry_on_the_oracle_plane(kind):
    _, ch, dt = FORMATS[kind]
    mx = np.iinfo(dt).max
    t = synth_frame(21, h=301, w=415, nblobs=600)
    rng = np.random.default_rng(22)
    chans = [np.round(t * mx), rng.integers(0, mx + 1, t.shape), np.round((1 - t) * mx), rng.integers(0, mx + 1, t.shape)]
    px = np.stack([c.astype(dt) for c in chans[:ch]], -1)
    ak = cv_b200.Akaze(0.001)
    kps, d = ak.extract(DynamicImage(kind, px))
    fk, fd = ak.extract_from_gray_float_image(OI.from_dynamic(FORMATS[kind][0], px))
    assert len(d) > 50 and kps.tobytes() == fk.tobytes() and np.array_equal(d, fd)


@pytest.mark.parametrize("kind", ["luma8", "rgb8", "rgba8"])
def test_frame_features_from_one_image_equals_the_pair_entry(kind):
    _, ch, _ = FORMATS[kind]
    t = synth_frame(31, h=540, w=960, nblobs=2500)
    rng = np.random.default_rng(32)
    chans = [np.round(t * 255), rng.integers(0, 256, t.shape), np.round((1 - t) * 255), rng.integers(0, 256, t.shape)]
    px = np.stack([c.astype(np.uint8) for c in chans[:ch]], -1) if ch > 1 else chans[0].astype(np.uint8)
    px2 = np.roll(px, 7, axis=1)
    cam = _cam(*TUTORIAL)
    ak = cv_b200.Akaze(maximum_features=3000)
    got = cv_b200.frame_features(ak, [DynamicImage(kind, px), DynamicImage(kind, px2)], cam)
    code = FORMATS[kind][0]
    gray = np.stack([OI.from_dynamic(code, p) for p in (px, px2)])
    rgb = np.stack([OI.to_rgb8(code, p) for p in (px, px2)])
    want = cv_b200.frame_features(ak, gray, rgb, cam)
    for f in range(2):
        assert len(got[f]["keypoints"]) > 500
        for key in ("keypoints", "descriptors", "bearings", "responses", "colors"):
            assert got[f][key].tobytes() == want[f][key].tobytes(), (f, key)


def test_two_view_luma8_reproduces_tutorial_chapter5():
    a, b = _kitti8("0000000000"), _kitti8("0000000014")
    cam = _cam(*TUTORIAL)
    ars = cv_b200.Arrsac(1e-7, cv_b200.Xoshiro256PlusPlus(0))
    got = cv_b200.two_view_frames(cv_b200.Akaze(), [DynamicImage.luma8(a), DynamicImage.luma8(b)], cam, ars, better_by=25)
    ars_f = cv_b200.Arrsac(1e-7, cv_b200.Xoshiro256PlusPlus(0))
    want = cv_b200.two_view_frames(cv_b200.Akaze(), np.stack([kitti_frame("0000000000"), kitti_frame("0000000014")]), cam, ars_f,
                                   better_by=25)
    assert len(got["matches"]) == 127 and len(got["inliers"]) == 81
    assert np.array_equal(got["matches"], want["matches"]) and np.array_equal(got["inliers"], want["inliers"])
    for f in range(2):
        assert got["keypoints"][f].tobytes() == want["keypoints"][f].tobytes()
    assert np.array_equal(got["pose"][0], want["pose"][0]) and np.array_equal(got["pose"][1], want["pose"][1])
    assert [int(x) for x in ars.rng.state.s] == [int(x) for x in ars_f.rng.state.s]


def _fingerprint(kps, descs):
    return [k.tobytes() + d.tobytes() for k, d in zip(kps, descs)]


def test_mixed_and_repeated_calls_in_one_context_equal_fresh_contexts():
    a8, b8 = _kitti8("0000000000"), _kitti8("0000000014")
    rgb = np.stack([b8, a8, b8], -1)
    calls = [("f32", np.stack([kitti_frame("0000000000")])), ("dyn", [DynamicImage.luma8(a8)]), ("dyn", [DynamicImage.rgb8(rgb)]),
             ("f32", np.stack([kitti_frame("0000000014"), kitti_frame("0000000000")])), ("dyn", [DynamicImage.luma8(b8)] * 2),
             ("dyn", [DynamicImage.luma8(a8)])]
    fresh = []
    for _, x in calls:
        ctx = cv_b200.Context(0)
        fresh.append(_fingerprint(*cv_b200.Akaze.sparse(ctx=ctx).extract_batch(x)))
        ctx.close()
    ctx = cv_b200.Context(0)
    ak = cv_b200.Akaze.sparse(ctx=ctx)
    for _ in range(2):
        for (_, x), want in zip(calls, fresh):
            assert _fingerprint(*ak.extract_batch(x)) == want
    # a repeated call on the same buffers replays the cached graph: the same launches and the same bytes
    frames = [DynamicImage.luma8(a8)]
    ak.extract_batch(frames)
    l0 = ctx.launch_count()
    first = _fingerprint(*ak.extract_batch(frames))
    l1 = ctx.launch_count()
    second = _fingerprint(*ak.extract_batch(frames))
    assert ctx.launch_count() - l1 == l1 - l0 and first == second == fresh[1]
    ctx.close()


def test_device_entry_equals_the_host_entry():
    import torch
    a8 = _kitti8("0000000000")
    dev = torch.device("cuda", 0)
    px = torch.from_numpy(np.stack([a8, a8[::-1].copy()])).to(dev)
    cap = 4096
    kp = torch.zeros((2, cap, KP_DTYPE.itemsize), dtype=torch.uint8, device=dev)
    desc = torch.zeros((2, cap, 64), dtype=torch.uint8, device=dev)
    n = torch.zeros(2, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    ctx = cv_b200.Context(0)
    ak = cv_b200.Akaze.sparse(ctx=ctx)
    cfg = ak.config.to_c()
    L = image_lib()
    H, W = a8.shape
    for _ in range(2):
        ctx.check(L.cvb_akaze_extract_dynamic_batch_dev(ctx.handle, C.byref(cfg), 0, px.data_ptr(), 2, W, H, kp.data_ptr(), desc.data_ptr(),
                                                        cap, n.data_ptr()))
        ctx.sync()
        want = ak.extract_batch([DynamicImage.luma8(a8), DynamicImage.luma8(a8[::-1].copy())])
        nn = n.cpu().numpy()
        for f in range(2):
            assert nn[f] == len(want[1][f])
            assert kp[f, :nn[f]].cpu().numpy().tobytes() == want[0][f].tobytes()
            assert np.array_equal(desc[f, :nn[f]].cpu().numpy(), want[1][f])
    ctx.close()


def test_unsupported_formats_and_bad_arguments():
    ctx = cv_b200.Context(0)
    L = image_lib()
    cfg = cv_b200.Akaze().config.to_c()
    px = np.zeros(64 * 64 * 16, np.uint8)
    kp = np.zeros(16, KP_DTYPE)
    desc = np.zeros((16, 64), np.uint8)
    n = np.zeros(1, np.uint32)
    for fmt, want in ((8, CVB_EUNSUPPORTED), (9, CVB_EUNSUPPORTED), (10, CVB_EINVAL), (0xFFFFFFFF, CVB_EINVAL)):
        assert L.cvb_akaze_extract_dynamic_batch(ctx.handle, C.byref(cfg), fmt, px.ctypes.data, 1, 64, 64, kp.ctypes.data, desc.ctypes.data,
                                                 16, n.ctypes.data) == want
    assert L.cvb_akaze_extract_dynamic_batch(ctx.handle, C.byref(cfg), 0, px.ctypes.data, 0, 64, 64, kp.ctypes.data, desc.ctypes.data,
                                             16, n.ctypes.data) == CVB_EINVAL
    assert L.cvb_akaze_extract_dynamic_batch(None, C.byref(cfg), 0, px.ctypes.data, 1, 64, 64, kp.ctypes.data, desc.ctypes.data,
                                             16, n.ctypes.data) == CVB_EINVAL
    cam = _cam(*TUTORIAL)
    for kind in ("luma16", "luma_a16", "rgb16", "rgba16"):
        _, ch, dt = FORMATS[kind]
        with pytest.raises(cv_b200.CvbError) as e:
            cv_b200.frame_features(cv_b200.Akaze(ctx=ctx), DynamicImage(kind, np.zeros((64, 64) if ch == 1 else (64, 64, ch), dt)), cam)
        assert e.value.code == CVB_EUNSUPPORTED
    # an output capacity too small is CVB_ECAP, as for the f32 entry
    ak = cv_b200.Akaze.sparse(ctx=ctx, max_keypoints=16)
    with pytest.raises(cv_b200.CvbError) as e:
        ak.extract(DynamicImage.luma8(_kitti8("0000000000")))
    with pytest.raises(cv_b200.CvbError) as e2:
        ak.extract_from_gray_float_image(kitti_frame("0000000000"))
    assert e.value.code == e2.value.code and "capacity" in str(e.value)
    ctx.close()
