"""akaze::image, the akaze crate's public image module, on the device (include/cvb200_filter.h, libcvb200_filter.so).

  gaussian_kernel(r, ks)              <- akaze::image::gaussian_kernel              (image.rs:349-374; host arithmetic)
  horizontal_filter(img, kernel)      <- akaze::image::horizontal_filter            (image.rs:202-251)
  vertical_filter(img, kernel)        <- akaze::image::vertical_filter              (image.rs:253-331)
  separable_filter(img, hk, vk)       <- akaze::image::separable_filter             (image.rs:333-340)
  gaussian_blur(img, r)               <- akaze::image::gaussian_blur                (image.rs:383-389)
  half_size(img)                      <- akaze::image::GrayFloatImage::half_size    (image.rs:154-199)

Images are float32 numpy arrays, one plane [H, W] or a batch of planes of one size [B, H, W] (one launch per pass for the batch); the
result has the same shape ([..., H // 2, W // 2] for half_size).  Results are bit-exact to the reference, zero-weighted tail taps of its
f32x4 layout included (see the header).  Kernels have an odd size of at most CVB_FILTER_MAX_TAPS (1023); other sizes raise CvbError
(EINVAL when even, EUNSUPPORTED when too long).  There is no CPU fallback: without a Hopper GPU the filters raise CvbError (ENODEV).
Device buffers go through the _dev entry points of the C ABI."""
import ctypes as C

import numpy as np

from ._lib import CvbError, default_context, load_filter_library

MAX_TAPS = 1023   # CVB_FILTER_MAX_TAPS


def bind(L):
    if getattr(L, "_filter_bound", False):
        return
    vp, u32, f32 = C.c_void_p, C.c_uint32, C.c_float
    L.cvb_gaussian_kernel.argtypes = [f32, u32, vp]
    for n in ("cvb_horizontal_filter", "cvb_vertical_filter"):
        getattr(L, n).argtypes = getattr(L, n + "_dev").argtypes = [vp, vp, u32, u32, u32, vp, u32, vp]
    L.cvb_separable_filter.argtypes = L.cvb_separable_filter_dev.argtypes = [vp, vp, u32, u32, u32, vp, u32, vp, u32, vp]
    L.cvb_gaussian_blur.argtypes = L.cvb_gaussian_blur_dev.argtypes = [vp, vp, u32, u32, u32, f32, vp]
    L.cvb_half_size.argtypes = L.cvb_half_size_dev.argtypes = [vp, vp, u32, u32, u32, vp]
    L._filter_bound = True


def lib():
    L = load_filter_library()
    bind(L)
    return L


def _planes(img):
    """img -> (C-contiguous float32 [B, H, W], the caller's shape)"""
    a = np.asarray(img)
    if a.dtype != np.float32:
        raise TypeError(f"images are float32, not {a.dtype}")
    if a.ndim not in (2, 3) or 0 in a.shape:
        raise ValueError(f"images are non-empty [H, W] or [B, H, W], not {a.shape}")
    return np.ascontiguousarray(a).reshape((-1,) + a.shape[-2:]), a.shape


def _taps(kernel):
    k = np.ascontiguousarray(kernel, np.float32)
    if k.ndim != 1:
        raise ValueError(f"a kernel is one-dimensional, not {k.shape}")
    return k


def _run(ctx, fn, img, *args, out_hw=None):
    a, shape = _planes(img)
    ctx = ctx if ctx is not None else default_context(0)
    B, H, W = a.shape
    oh, ow = out_hw(H, W) if out_hw else (H, W)
    out = np.empty((B, oh, ow), np.float32)
    ctx.check(getattr(lib(), fn)(ctx.handle, a.ctypes.data, B, W, H, *args, out.ctypes.data))
    return out.reshape(shape[:-2] + (oh, ow))


def gaussian_kernel(r, ks):
    """image.rs:349-374: ks f32 taps of a Gaussian of sigma r, divided by their sequential f32 sum (ks odd; r = 0 gives NaN taps)."""
    ks = int(ks)
    if ks < 0:
        raise ValueError("kernel size must be >= 0")
    out = np.empty(max(ks, 1), np.float32)
    rc = lib().cvb_gaussian_kernel(float(r), ks, out.ctypes.data)
    if rc != 0:
        raise CvbError(rc, f"gaussian_kernel: kernel size {ks} is not odd")
    return out[:ks]


def horizontal_filter(img, kernel, ctx=None):
    k = _taps(kernel)
    return _run(ctx, "cvb_horizontal_filter", img, k.ctypes.data, len(k))


def vertical_filter(img, kernel, ctx=None):
    k = _taps(kernel)
    return _run(ctx, "cvb_vertical_filter", img, k.ctypes.data, len(k))


def separable_filter(img, h_kernel, v_kernel, ctx=None):
    hk, vk = _taps(h_kernel), _taps(v_kernel)
    return _run(ctx, "cvb_separable_filter", img, hk.ctypes.data, len(hk), vk.ctypes.data, len(vk))


def gaussian_blur(img, r, ctx=None):
    """r > 0 (CvbError EINVAL otherwise); kernel size 2 * ceil(2 r) + 1, so r <= 255.5"""
    return _run(ctx, "cvb_gaussian_blur", img, float(r))


def half_size(img, ctx=None):
    return _run(ctx, "cvb_half_size", img, out_hw=lambda H, W: (H // 2, W // 2))


__all__ = ["gaussian_kernel", "horizontal_filter", "vertical_filter", "separable_filter", "gaussian_blur", "half_size", "MAX_TAPS"]
