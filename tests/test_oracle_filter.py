"""CPU-only: the oracle of include/cvb200_filter.h (oracle/ref_filter.c) is the reference's filter loops (akaze/src/image.rs:202-331).

The reference is transcribed here literally in numpy float32: the zero-padded f32x4 kernel (kernel.chunks(4)), the scratch line
[half x first][line][half x last][3 x 0.0] with kernel_simd_size = 4 * (ks + 3) / 4, windows(kernel_simd_size), chunks_exact(4) zipped with
the kernel's chunks, lane folds acc = (pixel * k) + acc from +0, and reduce_add = (l0 + l2) + (l1 + l3).  The oracle equals it bit for
bit (every NaN equal to every NaN) for kernel sizes 1 .. 13 and 71, on planes narrower and shorter than the kernel, with NaN and +-inf
under real taps and under the zero-weighted tail taps; on finite data it equals the extractor's oracle (oracle/ref_akaze.c), which skips
those taps."""
import numpy as np
import pytest

from oracle import pyoracle as O
from oracle import pyoracle_filter as OF

SIZES = list(range(1, 14, 2)) + [71]


def _ref_line(line, kernel):
    """horizontal_filter's loop for one row (image.rs:214-249), in f32"""
    line = np.asarray(line, np.float32)
    kernel = np.asarray(kernel, np.float32)
    ks = len(kernel)
    half = ks // 2
    chunks = [np.array([kernel[i + u] if i + u < ks else 0.0 for u in range(4)], np.float32) for i in range(0, ks, 4)]
    simd_size = 4 * (ks + 3) // 4                     # operator precedence as written: ks + 3
    extra = simd_size - ks
    width = len(line)
    scratch = np.zeros(width + 2 * half + extra, np.float32)
    scratch[0:half] = line[0]
    scratch[half:half + width] = line
    scratch[half + width:2 * half + width] = line[width - 1]
    scratch[2 * half + width:] = 0.0
    out = np.empty(width, np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        for x in range(len(scratch) - simd_size + 1):  # windows(simd_size)
            window = scratch[x:x + simd_size]
            acc = np.zeros(4, np.float32)
            for c, kc in zip(range(len(window) // 4), chunks):   # chunks_exact(4).zip(kernel_simd)
                acc = window[4 * c:4 * c + 4] * kc + acc           # a.mul_add(b, acc) without FMA: two roundings
            out[x] = (acc[0] + acc[2]) + (acc[1] + acc[3])
    return out


def ref_horizontal(img, kernel):
    return np.stack([_ref_line(row, kernel) for row in img])


def ref_vertical(img, kernel):
    return np.stack([_ref_line(col, kernel) for col in img.T]).T


def _same(got, want):
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    assert got.shape == want.shape
    gn, wn = np.isnan(got), np.isnan(want)
    assert np.array_equal(gn, wn), np.argwhere(gn != wn)[:5].tolist()
    assert np.array_equal(got.view(np.uint32)[~gn], want.view(np.uint32)[~wn])


def _taps(ks, seed):
    k = np.random.default_rng(seed).standard_normal(ks).astype(np.float32)
    k[ks // 2] = -0.0 if ks > 1 else k[0]
    return k


@pytest.mark.parametrize("shape", [(1, 1), (1, 5), (6, 1), (4, 3), (9, 17), (31, 24)], ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("ks", SIZES)
def test_oracle_equals_the_reference_loop(ks, shape):
    rng = np.random.default_rng(ks * 100 + shape[0])
    img = rng.standard_normal(shape).astype(np.float32)
    img.reshape(-1)[::4] = -0.0
    k = _taps(ks, ks)
    _same(OF.horizontal_filter(img, k), ref_horizontal(img, k))
    _same(OF.vertical_filter(img, k), ref_vertical(img, k))
    # finite data: the tail taps are a no-op, the extractor's oracle (which skips them) agrees
    _same(OF.horizontal_filter(img, k), O.horizontal_filter(img, k))
    _same(OF.vertical_filter(img, k), O.vertical_filter(img, k))


@pytest.mark.parametrize("ks", SIZES)
def test_non_finite_pixels_under_real_and_tail_taps(ks):
    half, n = ks // 2, 40
    rng = np.random.default_rng(ks)
    img = rng.standard_normal((n, n)).astype(np.float32)
    q = 25
    img[3, q] = np.nan            # row 3: a NaN mid-row
    img[5, -1] = np.inf           # row 5: +inf at the end, replicated into the right border and the tail
    img[7, 0] = -np.inf           # row 7: -inf at the start
    img[q, 9] = np.nan            # column 9: a NaN mid-column
    img[-1, 11] = -np.inf         # column 11: -inf at the bottom
    k = _taps(ks, 7 * ks)
    got_h, got_v = OF.horizontal_filter(img, k), OF.vertical_filter(img, k)
    _same(got_h, ref_horizontal(img, k))
    _same(got_v, ref_vertical(img, k))
    tail = 4 * ((ks + 3) // 4) - ks
    x = q - half - 1              # the NaN lies only under tap ks of output x, a tail tap
    if tail and x >= 0:
        assert np.isnan(got_h[3, x]) and not np.isnan(O.horizontal_filter(img, k)[3, x])
        assert np.isnan(got_v[x, 9]) and not np.isnan(O.vertical_filter(img, k)[x, 9])
    # +inf at the last pixel: every output whose window reaches past the row's end (the replicated border or the tail) is non-finite
    assert not np.isfinite(got_h[5, n - 1 - half:]).any()


def test_kernels_longer_than_the_plane_and_batches():
    rng = np.random.default_rng(3)
    k = _taps(71, 71)
    img = rng.standard_normal((3, 5, 7)).astype(np.float32)
    got = OF.separable_filter(img, k, k[::-1].copy())
    for b in range(3):
        _same(got[b], ref_vertical(ref_horizontal(img[b], k), k[::-1].copy()))
    _same(OF.half_size(img)[1], O.half_size(img[1]))


def test_gaussian_blur_size_is_the_references():
    """image.rs:385-386: 2 * ceil(2 r) + 1 in f32"""
    assert [OF.blur_size(r) for r in (0.5, 1.0, 1.6, 3.0, 8.0, 10.0, 40.0, 255.5)] == [3, 5, 9, 13, 33, 41, 161, 1023]
