"""GPU: akaze::image on the device (include/cvb200_filter.h, libcvb200_filter.so).

  * every filter and its _dev form equals the oracle (oracle/ref_filter.c, tail taps included) bit for bit: kernel sizes 1 .. 1023,
    1 x 1, 1 x N, N x 1 and odd planes, kernels longer than the plane, KITTI, batches of different planes, asymmetric and negative
    taps, -0.0 pixels and taps, and NaN / +-inf under real and tail taps (NaN outputs compared as NaN: payloads are not specified);
  * gaussian_blur for sigma 0.5 .. 40, half_size on odd dimensions;
  * gaussian_blur(KITTI, 1.6) is the extractor's evolution-0 Lt; the reference's image.rs:414-432 test (KITTI, gaussian_kernel(3, 7),
    within 1e-4 of a float64 replicate-border correlation);
  * filter calls interleaved with extractor calls in one context give the bytes of fresh contexts;
  * argument errors: even and too long kernels, sigma <= 0 or NaN, empty planes, overlapping buffers, a null context."""
import ctypes as C

import numpy as np
import pytest

import cv_b200
from cv_b200 import filter as F
from cv_b200._lib import CVB_EINVAL, CVB_EUNSUPPORTED
from oracle import pyoracle_filter as OF
from tests.common import kitti_frame

pytestmark = pytest.mark.gpu

SIZES = [1, 3, 5, 7, 9, 11, 33, 35, 71, 73, 255, 1023]
SHAPES = [(1, 1), (1, 37), (37, 1), (13, 29), (3, 19, 23)]   # [H, W] or [B, H, W]
SIGMAS = [0.5, 1.0, 1.6, 3.0, 8.0, 10.0, 40.0]


@pytest.fixture(scope="module")
def ctx():
    c = cv_b200.Context()
    yield c
    c.close()


def _same(got, want):
    """bit-equal, every NaN equal to every NaN"""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    assert got.shape == want.shape, (got.shape, want.shape)
    gn, wn = np.isnan(got), np.isnan(want)
    assert np.array_equal(gn, wn), f"NaN at {np.argwhere(gn != wn)[:5].tolist()}"
    gb, wb = got.view(np.uint32)[~gn], want.view(np.uint32)[~wn]
    bad = np.flatnonzero(gb != wb)
    assert bad.size == 0, f"{bad.size} of {gb.size} differ, first {got[~gn][bad[:3]]} vs {want[~wn][bad[:3]]}"


def _taps(ks, seed):
    """asymmetric, signed, with a -0.0 tap"""
    k = np.random.default_rng(seed).standard_normal(ks).astype(np.float32)
    k[ks // 3] = -0.0
    return k


def _planes(shape, seed):
    """signed pixels with -0.0 and +0.0 among them"""
    a = np.random.default_rng(seed).standard_normal(shape).astype(np.float32)
    flat = a.reshape(-1)
    flat[::5] = -0.0
    flat[2::7] = 0.0
    return a


def _dev(fn, img, *args, out_hw=None):
    """the _dev entry point on device copies of img ([H, W] or [B, H, W]); returns the result on the host"""
    import torch
    a = np.ascontiguousarray(img, np.float32).reshape((-1,) + img.shape[-2:])
    B, H, W = a.shape
    oh, ow = out_hw if out_hw else (H, W)
    dev = torch.device("cuda", 0)
    src = torch.from_numpy(a).to(dev)
    dst = torch.full((B, oh, ow), float("nan"), dtype=torch.float32, device=dev)
    torch.cuda.synchronize()
    ctx = cv_b200.Context()
    ctx.check(getattr(F.lib(), fn)(ctx.handle, src.data_ptr(), B, W, H, *args, dst.data_ptr()))
    ctx.sync()
    out = dst.cpu().numpy().reshape(img.shape[:-2] + (oh, ow))
    ctx.close()
    return out


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("ks", SIZES)
def test_filters_equal_the_oracle(ctx, ks, shape):
    img = _planes(shape, ks)
    k = _taps(ks, 1000 + ks)
    vk = _taps(2 * (ks % 7) + 1, 2000 + ks)
    want_h, want_v = OF.horizontal_filter(img, k), OF.vertical_filter(img, k)
    want_s = OF.separable_filter(img, k, vk)
    _same(F.horizontal_filter(img, k, ctx=ctx), want_h)
    _same(F.vertical_filter(img, k, ctx=ctx), want_v)
    _same(F.separable_filter(img, k, vk, ctx=ctx), want_s)
    _same(_dev("cvb_horizontal_filter_dev", img, k.ctypes.data, ks), want_h)
    _same(_dev("cvb_vertical_filter_dev", img, k.ctypes.data, ks), want_v)
    _same(_dev("cvb_separable_filter_dev", img, k.ctypes.data, ks, vk.ctypes.data, len(vk)), want_s)


@pytest.mark.parametrize("ks", [7, 71])
def test_kitti_and_a_batch_of_different_planes(ctx, ks):
    k0, k1 = kitti_frame("0000000000"), kitti_frame("0000000014")
    for k in (F.gaussian_kernel(10.0 if ks == 71 else 1.0, ks), _taps(ks, ks)):
        _same(F.horizontal_filter(k0, k, ctx=ctx), OF.horizontal_filter(k0, k))
        _same(F.vertical_filter(k0, k, ctx=ctx), OF.vertical_filter(k0, k))
        batch = np.stack([k0, k1, k0[::-1].copy()])
        want = OF.separable_filter(batch, k, k[::-1].copy())
        _same(F.separable_filter(batch, k, k[::-1].copy(), ctx=ctx), want)
        _same(_dev("cvb_separable_filter_dev", batch, k.ctypes.data, ks, k[::-1].copy().ctypes.data, ks), want)


@pytest.mark.parametrize("ks", [3, 5, 7, 9, 11, 13, 71, 73])
def test_nan_and_inf_under_real_and_tail_taps(ctx, ks):
    """a NaN at q: output q - half - 1 sees it only through a tail tap (when ks is not a multiple of 4, which odd sizes never are);
    -inf first, +inf last and a NaN column / row in a batch plane"""
    n, q, half = 96, 60, ks // 2
    img = _planes((3, n, n), 7 * ks)
    img[0, :, q] = np.nan
    img[0, q, :] = np.nan
    img[1, :, 0] = -np.inf
    img[1, :, -1] = np.inf
    img[2, -1, :] = np.inf
    img[2, 0, :] = -np.inf
    k = _taps(ks, ks)
    want_h, want_v = OF.horizontal_filter(img, k), OF.vertical_filter(img, k)
    if q - half - 1 >= 0:
        assert np.isnan(want_h[0, 5, q - half - 1])   # the oracle does evaluate the tail taps
    _same(F.horizontal_filter(img, k, ctx=ctx), want_h)
    _same(F.vertical_filter(img, k, ctx=ctx), want_v)
    _same(F.separable_filter(img, k, k, ctx=ctx), OF.separable_filter(img, k, k))
    _same(_dev("cvb_horizontal_filter_dev", img, k.ctypes.data, ks), want_h)
    _same(_dev("cvb_vertical_filter_dev", img, k.ctypes.data, ks), want_v)


@pytest.mark.parametrize("r", SIGMAS)
def test_gaussian_blur_equals_the_oracle(ctx, r):
    k0 = kitti_frame("0000000000")
    imgs = [k0, _planes((2, 33, 47), 3), _planes((5, 3), 4)]
    for img in imgs:
        want = OF.gaussian_blur(img, r)
        _same(F.gaussian_blur(img, r, ctx=ctx), want)
        _same(_dev("cvb_gaussian_blur_dev", img, C.c_float(r)), want)


@pytest.mark.parametrize("shape", [(1, 1), (1, 9), (9, 1), (2, 2), (3, 3), (7, 5), (2, 31, 17), (513, 1391)],
                         ids=lambda s: "x".join(map(str, s)))
def test_half_size_equals_the_oracle(ctx, shape):
    img = _planes(shape, sum(shape))
    want = OF.half_size(img)
    _same(F.half_size(img, ctx=ctx), want)
    oh, ow = shape[-2] // 2, shape[-1] // 2
    if oh and ow:
        _same(_dev("cvb_half_size_dev", img, out_hw=(oh, ow)), want)
    k0 = kitti_frame("0000000000")[:511, :1391]
    _same(F.half_size(k0, ctx=ctx), OF.half_size(k0))


def test_gaussian_blur_is_the_extractors_first_evolution():
    k0 = kitti_frame("0000000000")
    ak = cv_b200.Akaze.sparse(ctx=cv_b200.Context())
    ak.extract_from_gray_float_image(k0)
    _same(F.gaussian_blur(k0, 1.6), ak.debug_plane(0, "Lt"))


def test_reference_filter_tests_on_kitti(ctx):
    """image.rs:414-432: horizontal / vertical_filter(KITTI, gaussian_kernel(3.0, 7)) within 1e-4 of a plain correlation"""
    img = kitti_frame("0000000000")
    k = F.gaussian_kernel(3.0, 7)
    want = np.array([0.10628852, 0.14032133, 0.16577007, 0.17524014, 0.16577007, 0.14032133, 0.10628852], np.float32)
    assert np.abs(k - want).max() < 1e-4
    p = np.pad(img.astype(np.float64), 3, mode="edge")
    H, W = img.shape
    hor = sum(k[j] * p[3:3 + H, j:j + W] for j in range(7))
    ver = sum(k[j] * p[j:j + H, 3:3 + W] for j in range(7))
    assert np.abs(F.horizontal_filter(img, k, ctx=ctx) - hor).max() < 1e-4
    assert np.abs(F.vertical_filter(img, k, ctx=ctx) - ver).max() < 1e-4


def test_interleaved_with_the_extractor_in_one_context():
    k0, k1 = kitti_frame("0000000000"), kitti_frame("0000000014")
    k = _taps(71, 5)

    def fresh_extract(img):
        return cv_b200.Akaze.sparse(ctx=cv_b200.Context()).extract_from_gray_float_image(img)

    want_e0, want_e1 = fresh_extract(k0), fresh_extract(k1)
    want_b = F.gaussian_blur(k1, 3.0, ctx=cv_b200.Context())
    want_s = F.separable_filter(np.stack([k0, k1]), k, k, ctx=cv_b200.Context())
    want_half = F.half_size(k1, ctx=cv_b200.Context())
    c = cv_b200.Context()
    ak = cv_b200.Akaze.sparse(ctx=c)
    for _ in range(2):
        e0 = ak.extract_from_gray_float_image(k0)
        b = F.gaussian_blur(k1, 3.0, ctx=c)
        s = F.separable_filter(np.stack([k0, k1]), k, k, ctx=c)
        e1 = ak.extract_from_gray_float_image(k1)
        half = F.half_size(k1, ctx=c)
        for got, want in ((e0, want_e0), (e1, want_e1)):
            assert got[0].tobytes() == want[0].tobytes() and np.array_equal(got[1], want[1])
        for got, want in ((b, want_b), (s, want_s), (half, want_half)):
            assert got.tobytes() == want.tobytes()


def test_argument_errors(ctx):
    import torch
    L = F.lib()
    img = _planes((8, 9), 0)
    k3 = _taps(3, 0)
    out = np.empty_like(img)

    def code(call):
        with pytest.raises(cv_b200.CvbError) as e:
            call()
        return e.value.code

    assert code(lambda: F.horizontal_filter(img, _taps(4, 0), ctx=ctx)) == CVB_EINVAL
    assert code(lambda: F.vertical_filter(img, np.zeros(0, np.float32), ctx=ctx)) == CVB_EINVAL
    assert code(lambda: F.separable_filter(img, k3, _taps(2, 0), ctx=ctx)) == CVB_EINVAL
    assert code(lambda: F.vertical_filter(img, _taps(1025, 0), ctx=ctx)) == CVB_EUNSUPPORTED
    assert code(lambda: F.gaussian_kernel(1.0, 4)) == CVB_EINVAL
    for r in (0.0, -1.0, float("nan")):
        assert code(lambda: F.gaussian_blur(img, r, ctx=ctx)) == CVB_EINVAL
    assert code(lambda: F.gaussian_blur(img, 256.0, ctx=ctx)) == CVB_EUNSUPPORTED
    assert F.gaussian_blur(img, 255.5, ctx=ctx).shape == img.shape   # 1023 taps
    with pytest.raises(TypeError):
        F.horizontal_filter(img.astype(np.float64), k3, ctx=ctx)
    with pytest.raises(ValueError):
        F.half_size(np.zeros((2, 2, 2, 2), np.float32), ctx=ctx)
    h = ctx.handle
    p, o, kp = img.ctypes.data, out.ctypes.data, k3.ctypes.data
    for b, w, hh in ((0, 9, 8), (1, 0, 8), (1, 9, 0)):
        assert L.cvb_horizontal_filter(h, p, b, w, hh, kp, 3, o) == CVB_EINVAL
        assert L.cvb_gaussian_blur(h, p, b, w, hh, C.c_float(1.0), o) == CVB_EINVAL
        assert L.cvb_half_size(h, p, b, w, hh, o) == CVB_EINVAL
    assert L.cvb_horizontal_filter(None, p, 1, 9, 8, kp, 3, o) == CVB_EINVAL
    assert L.cvb_separable_filter_dev(None, p, 1, 9, 8, kp, 3, kp, 3, o) == CVB_EINVAL
    assert L.cvb_half_size_dev(None, p, 1, 9, 8, o) == CVB_EINVAL
    assert L.cvb_horizontal_filter(h, p, 1, 9, 8, None, 3, o) == CVB_EINVAL
    assert L.cvb_vertical_filter(h, p, 1, 9, 8, kp, 3, None) == CVB_EINVAL
    # overlapping buffers, host and device
    assert L.cvb_vertical_filter(h, p, 1, 9, 8, kp, 3, p + 4) == CVB_EINVAL
    assert L.cvb_separable_filter(h, p, 1, 9, 8, kp, 3, kp, 3, p) == CVB_EINVAL
    assert L.cvb_half_size(h, p, 1, 9, 8, p + 4 * 70) == CVB_EINVAL
    buf = torch.zeros(4 * 72, dtype=torch.float32, device="cuda:0")
    d = buf.data_ptr()
    torch.cuda.synchronize()
    assert L.cvb_horizontal_filter_dev(h, d, 1, 9, 8, kp, 3, d + 4 * 71) == CVB_EINVAL
    assert L.cvb_gaussian_blur_dev(h, d, 1, 9, 8, C.c_float(1.0), d) == CVB_EINVAL
    assert L.cvb_half_size_dev(h, d, 1, 9, 8, d + 4 * 71) == CVB_EINVAL
    assert L.cvb_horizontal_filter_dev(h, d, 1, 9, 8, kp, 3, d + 4 * 72) == 0   # adjacent, not overlapping
    ctx.sync()
    # a 1-pixel dimension: half_size is empty, nothing written
    assert F.half_size(np.ones((1, 7), np.float32), ctx=ctx).shape == (0, 3)
    assert L.cvb_half_size_dev(h, d, 1, 1, 7, d + 4 * 72) == 0
