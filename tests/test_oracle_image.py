"""CPU-only: the oracle of include/cvb200_image.h (oracle/ref_image.c) -- GrayFloatImage::from_dynamic (akaze/src/image.rs:45-109) of
the eight integer DynamicImage variants and DynamicImage::to_rgb8() of the 8-bit ones.

  * Luma8 / Luma16 equal numpy's v.astype(f32) / f32(255 or 65535) bit for bit, over every 8- and 16-bit value;
  * RGB(A)8 / RGB(A)16 equal a numpy integer transcription of image 0.24's rgb_to_luma (restated, parity unpinned) then the division;
  * a gray RGB pixel gives exactly the luma's value, and alpha never changes the result;
  * to_rgb8 replicates a luma, drops alpha and keeps RGB8."""
import numpy as np
import pytest

from oracle import pyoracle_image as OI

LUMA8, LUMA_A8, RGB8, RGBA8, LUMA16, LUMA_A16, RGB16, RGBA16 = range(8)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _luma_np(rgb):
    """image 0.24 rgb_to_luma: (2126 R + 7152 G + 722 B) / 10000, u32 intermediates, truncating division"""
    r, g, b = (rgb[..., c].astype(np.uint32) for c in range(3))
    return (np.uint32(2126) * r + np.uint32(7152) * g + np.uint32(722) * b) // np.uint32(10000)


def test_luma8_and_luma16_exhaustive():
    v8 = np.arange(256, dtype=np.uint8).reshape(16, 16)
    assert np.array_equal(_bits(OI.from_dynamic(LUMA8, v8)), _bits(v8.astype(np.float32) / np.float32(255)))
    v16 = np.arange(65536, dtype=np.uint32).astype(np.uint16).reshape(256, 256)
    got = OI.from_dynamic(LUMA16, v16)
    assert np.array_equal(_bits(got), _bits(v16.astype(np.float32) / np.float32(65535)))
    assert got[0, 0] == 0.0 and got[-1, -1] == 1.0


@pytest.mark.parametrize("fmt,luma", [(LUMA_A8, LUMA8), (LUMA_A16, LUMA16)])
def test_luma_alpha_is_never_read(fmt, luma):
    dt = np.uint8 if fmt == LUMA_A8 else np.uint16
    rng = np.random.default_rng(fmt)
    v = rng.integers(0, np.iinfo(dt).max + 1, (37, 53), dtype=dt)
    want = OI.from_dynamic(luma, v)
    for alpha in (np.zeros_like(v), np.full_like(v, np.iinfo(dt).max), rng.integers(0, np.iinfo(dt).max + 1, v.shape, dtype=dt)):
        assert np.array_equal(_bits(OI.from_dynamic(fmt, np.stack([v, alpha], -1))), _bits(want))


@pytest.mark.parametrize("fmt", [RGB8, RGBA8, RGB16, RGBA16])
def test_rgb_equals_the_integer_transcription(fmt):
    dt, div = (np.uint8, np.float32(255)) if fmt in (RGB8, RGBA8) else (np.uint16, np.float32(65535))
    ch = 3 if fmt in (RGB8, RGB16) else 4
    mx = np.iinfo(dt).max
    rng = np.random.default_rng(10 + fmt)
    px = rng.integers(0, mx + 1, (61, 47, ch), dtype=dt)
    px[0, 0] = 0
    px[0, 1] = mx
    px[0, 2, :3] = (mx, 0, 0); px[0, 3, :3] = (0, mx, 0); px[0, 4, :3] = (0, 0, mx)
    got = OI.from_dynamic(fmt, px)
    want = _luma_np(px).astype(np.float32) / div
    assert np.array_equal(_bits(got), _bits(want))
    assert got[0, 0] == 0.0 and got[0, 1] == 1.0
    assert OI.rgb_to_luma(mx, mx, mx) == mx and OI.rgb_to_luma(255, 0, 0) == 54 and OI.rgb_to_luma(0, 255, 0) == 182


def test_gray_rgb_pixel_equals_luma_and_alpha_is_dropped():
    v8 = np.arange(256, dtype=np.uint8)
    v16 = np.arange(65536, dtype=np.uint32).astype(np.uint16)
    for v, luma, rgb, rgba in ((v8, LUMA8, RGB8, RGBA8), (v16, LUMA16, RGB16, RGBA16)):
        want = _bits(OI.from_dynamic(luma, v[None]))
        px = np.repeat(v[None, :, None], 3, -1)
        assert np.array_equal(_bits(OI.from_dynamic(rgb, px)), want)
        for a in (0, np.iinfo(v.dtype).max):
            assert np.array_equal(_bits(OI.from_dynamic(rgba, np.concatenate([px, np.full_like(px[..., :1], a)], -1))), want)


def test_to_rgb8_of_the_8_bit_formats():
    rng = np.random.default_rng(5)
    l = rng.integers(0, 256, (9, 11), dtype=np.uint8)
    a = rng.integers(0, 256, (9, 11), dtype=np.uint8)
    rgb = rng.integers(0, 256, (9, 11, 3), dtype=np.uint8)
    assert np.array_equal(OI.to_rgb8(LUMA8, l), np.repeat(l[..., None], 3, -1))
    assert np.array_equal(OI.to_rgb8(LUMA_A8, np.stack([l, a], -1)), np.repeat(l[..., None], 3, -1))
    assert np.array_equal(OI.to_rgb8(RGB8, rgb), rgb)
    assert np.array_equal(OI.to_rgb8(RGBA8, np.concatenate([rgb, a[..., None]], -1)), rgb)
    with pytest.raises(ValueError):
        OI.to_rgb8(LUMA16, l.astype(np.uint16))


def test_python_dynamic_image_checks_dtype_and_shape():
    import cv_b200
    D = cv_b200.DynamicImage
    assert D.luma8(np.zeros((4, 5), np.uint8)).format == 0 and D.rgba16(np.zeros((4, 5, 4), np.uint16)).format == 7
    for bad in (lambda: D.luma8(np.zeros((4, 5), np.uint16)), lambda: D.rgb16(np.zeros((4, 5, 3), np.uint8))):
        with pytest.raises(TypeError):
            bad()
    for bad in (lambda: D.rgb8(np.zeros((4, 5), np.uint8)), lambda: D.rgba8(np.zeros((4, 5, 3), np.uint8)),
                lambda: D.luma_a8(np.zeros((4, 5, 3), np.uint8)), lambda: D.luma16(np.zeros((0, 5), np.uint16))):
        with pytest.raises(ValueError):
            bad()
