"""The extractor's input as the reference takes it: image::DynamicImage's eight integer variants, converted on the device
(include/cvb200_image.h, libcvb200_image.so) as GrayFloatImage::from_dynamic (akaze/src/image.rs:45-109) converts them.

  DynamicImage.luma8(a) ... rgba16(a)   <- DynamicImage::ImageLuma8 ... ImageRgba16 (the pixels of ImageBuffer::as_bytes())

Akaze.extract / extract_batch, frame_features and two_view_frames take these and upload the frame's own bytes; plain numpy arrays keep
their f32 host conversion.  The RGB(A) luma is image 0.24's integer rgb_to_luma, restated from its published source (see the header)."""
import ctypes as C

import numpy as np

from ._lib import AkazeCfg, load_image_library

# cvb_pixel_format codes (include/cvb200_image.h): name -> (code, channels, dtype)
FORMATS = {
    "luma8": (0, 1, np.uint8), "luma_a8": (1, 2, np.uint8), "rgb8": (2, 3, np.uint8), "rgba8": (3, 4, np.uint8),
    "luma16": (4, 1, np.uint16), "luma_a16": (5, 2, np.uint16), "rgb16": (6, 3, np.uint16), "rgba16": (7, 4, np.uint16),
}


class DynamicImage:
    """One frame in one of image::DynamicImage's integer variants: `pixels` is [H, W] (luma) or [H, W, C] of uint8 / uint16, C-contiguous,
    i.e. the bytes of ImageBuffer::as_bytes() (16-bit channels in native byte order)."""

    def __init__(self, kind, pixels):
        code, ch, dt = FORMATS[kind]
        a = np.asarray(pixels)
        if a.dtype != dt:
            raise TypeError(f"DynamicImage.{kind} takes {np.dtype(dt).name} pixels, not {a.dtype}")
        if ch == 1 and a.ndim == 3 and a.shape[2] == 1:
            a = a[..., 0]
        want = 2 if ch == 1 else 3
        if a.ndim != want or (ch > 1 and a.shape[2] != ch) or a.shape[0] == 0 or a.shape[1] == 0:
            raise ValueError(f"DynamicImage.{kind} takes [H, W{'' if ch == 1 else f', {ch}'}] pixels, not {a.shape}")
        self.kind, self.format, self.pixels = kind, code, np.ascontiguousarray(a)

    @property
    def height(self):
        return self.pixels.shape[0]

    @property
    def width(self):
        return self.pixels.shape[1]

    @classmethod
    def luma8(cls, a):
        return cls("luma8", a)

    @classmethod
    def luma_a8(cls, a):
        return cls("luma_a8", a)

    @classmethod
    def rgb8(cls, a):
        return cls("rgb8", a)

    @classmethod
    def rgba8(cls, a):
        return cls("rgba8", a)

    @classmethod
    def luma16(cls, a):
        return cls("luma16", a)

    @classmethod
    def luma_a16(cls, a):
        return cls("luma_a16", a)

    @classmethod
    def rgb16(cls, a):
        return cls("rgb16", a)

    @classmethod
    def rgba16(cls, a):
        return cls("rgba16", a)

    def __repr__(self):
        return f"DynamicImage.{self.kind}({self.width}x{self.height})"


def is_dynamic(x):
    """a DynamicImage, or a non-empty list / tuple of them"""
    return isinstance(x, DynamicImage) or (isinstance(x, (list, tuple)) and len(x) > 0 and all(isinstance(i, DynamicImage) for i in x))


def stack(images):
    """frames of one size and format -> (format code, packed bytes of all frames, width, height)"""
    images = [images] if isinstance(images, DynamicImage) else list(images)
    f = images[0]
    for im in images[1:]:
        if im.kind != f.kind or im.pixels.shape != f.pixels.shape:
            raise ValueError(f"frames of one call share size and format: {f!r} and {im!r}")
    return f.format, np.ascontiguousarray(np.stack([im.pixels for im in images])), f.width, f.height


def bind(L):
    if getattr(L, "_image_bound", False):
        return
    vp, u32 = C.c_void_p, C.c_uint32
    L.cvb_gray_float_from_dynamic_dev.argtypes = [vp, u32, vp, u32, u32, u32, vp, vp]
    L.cvb_akaze_extract_dynamic_batch.argtypes = [vp, C.POINTER(AkazeCfg), u32, vp, u32, u32, u32, vp, vp, u32, vp]
    L.cvb_akaze_extract_dynamic_batch_dev.argtypes = [vp, C.POINTER(AkazeCfg), u32, vp, u32, u32, u32, vp, vp, u32, vp]
    L.cvb_frame_features_dynamic_batch.argtypes = [vp, vp, u32, vp, u32, u32, u32, vp, vp, vp, vp, vp, u32, vp]
    L.cvb_two_view_frames_dynamic_k1.argtypes = [vp, vp, u32, vp, u32, u32, u32, vp, vp, vp, vp, vp, u32, vp, vp, vp, vp, vp, vp, vp]
    L._image_bound = True


def lib():
    L = load_image_library()
    bind(L)
    return L


__all__ = ["DynamicImage", "FORMATS"]
