"""Host-side mirror of akaze::Akaze (akaze/src/lib.rs:109-185, 295-366) over the C ABI."""
import ctypes as C
from dataclasses import asdict, dataclass, replace

import numpy as np

from ._lib import CVB_ECAP, EVOLUTION_DTYPE, KP_DTYPE, AkazeCfg, Context, CvbError, default_context, load_stages_library
from .image import DynamicImage, is_dynamic
from .image import lib as _image_lib
from .image import stack as _stack_frames

PLANES = {"Lt": 0, "Lsmooth": 1, "Lx": 2, "Ly": 3, "Lflow": 4, "Ldet": 5}
STAGES = {"candidates": 0, "extrema": 1, "refined": 2, "sorted": 3}


@dataclass
class AkazeConfig:
    """The 11 public fields of akaze::Akaze with Akaze::default() values (lib.rs:169-185)."""
    maximum_features: int = -1          # usize::MAX
    num_sublevels: int = 4
    max_octave_evolution: int = 4
    base_scale_offset: float = 1.6
    initial_contrast: float = 0.001
    contrast_percentile: float = 0.7
    contrast_factor_num_bins: int = 300
    derivative_factor: float = 1.5
    detector_threshold: float = 0.001
    descriptor_channels: int = 3
    descriptor_pattern_size: int = 10

    def to_c(self):
        c = AkazeCfg()
        for f, _ in AkazeCfg._fields_:
            setattr(c, f, getattr(self, f))
        return c


class Akaze:
    """akaze::Akaze.  `Akaze(threshold)` == Akaze::new, plus `sparse()` / `dense()` (lib.rs:147-166)."""

    def __init__(self, detector_threshold=None, ctx=None, max_keypoints=32768, **fields):
        self.config = AkazeConfig(**fields)
        if detector_threshold is not None:
            self.config.detector_threshold = float(detector_threshold)
        self.ctx = ctx
        self.max_keypoints = int(max_keypoints)

    @classmethod
    def sparse(cls, **kw):
        return cls(0.01, **kw)

    @classmethod
    def dense(cls, **kw):
        return cls(0.0001, **kw)

    def _ctx(self):
        if self.ctx is None:
            self.ctx = default_context(0)
        return self.ctx

    # -- Akaze::extract (lib.rs:295): DynamicImage -> GrayFloatImage::from_dynamic (image.rs:45-109)
    def extract(self, image):
        """A DynamicImage is converted on the device (include/cvb200_image.h); a numpy array is converted here: uint8 / 255,
        uint16 / 65535, float32 as it is, [H, W] only."""
        if isinstance(image, DynamicImage):
            kps, descs = self.extract_batch([image])
            return kps[0], descs[0]
        image = np.asarray(image)
        if image.dtype == np.uint8:
            f = image.astype(np.float32) / np.float32(255)
        elif image.dtype == np.uint16:
            f = image.astype(np.float32) / np.float32(65535)
        elif image.dtype == np.float32:
            f = image
        else:
            raise TypeError("DynamicImage::grayscale() returned unexpected type")   # image.rs:107
        if f.ndim != 2:
            raise ValueError("expected a single-channel (luma) image")
        return self.extract_from_gray_float_image(f)

    # -- Akaze::extract_from_gray_float_image (lib.rs:309-339)
    def extract_from_gray_float_image(self, float_image):
        kps, descs = self.extract_batch(np.asarray(float_image, dtype=np.float32)[None])
        return kps[0], descs[0]

    def extract_batch(self, images):
        """B independent frames of one size in a single pass: [B, H, W] float32, or a list of DynamicImage of one size and format
        (uploaded as they are and converted on the device).  Returns lists of (keypoints, descriptors)."""
        if is_dynamic(images):
            return self._extract_dynamic(images)
        images = np.ascontiguousarray(images, dtype=np.float32)
        if images.ndim != 3:
            raise ValueError("images must be [B, H, W] float32")
        B, H, W = images.shape
        ctx = self._ctx()
        cap = self.max_keypoints
        kp = np.zeros((B, cap), dtype=KP_DTYPE)
        desc = np.zeros((B, cap, 64), dtype=np.uint8)
        n = np.zeros(B, dtype=np.uint32)
        cfg = self.config.to_c()
        rc = ctx.lib.cvb_akaze_extract_batch(ctx.handle, C.byref(cfg), images.ctypes.data, B, W, H, kp.ctypes.data,
                                             desc.ctypes.data, cap, n.ctypes.data)
        ctx.check(rc)
        return [kp[b, :n[b]].copy() for b in range(B)], [desc[b, :n[b]].copy() for b in range(B)]

    def _extract_dynamic(self, images):
        fmt, pixels, W, H = _stack_frames(images)
        B = pixels.shape[0]
        ctx = self._ctx()
        L = _image_lib()
        cap = self.max_keypoints
        kp = np.zeros((B, cap), dtype=KP_DTYPE)
        desc = np.zeros((B, cap, 64), dtype=np.uint8)
        n = np.zeros(B, dtype=np.uint32)
        cfg = self.config.to_c()
        ctx.check(L.cvb_akaze_extract_dynamic_batch(ctx.handle, C.byref(cfg), fmt, pixels.ctypes.data, B, W, H, kp.ctypes.data,
                                                    desc.ctypes.data, cap, n.ctypes.data))
        return [kp[b, :n[b]].copy() for b in range(B)], [desc[b, :n[b]].copy() for b in range(B)]

    # -- the staged surface (akaze/src/lib.rs:341-345; include/cvb200_stages.h)
    def create_scale_space(self, images):
        """allocate_evolutions + create_nonlinear_scale_space + detector_response of [H, W] or [B, H, W] frames, resident on the
        device: float32 as it is, uint8 / uint16 converted as `extract` converts them.  Returns a ScaleSpace, which any later call
        that rewrites this context's AKAZE planes (an extract, another scale space) makes stale."""
        images = np.asarray(images)
        if images.dtype == np.uint8:
            images = images.astype(np.float32) / np.float32(255)
        elif images.dtype == np.uint16:
            images = images.astype(np.float32) / np.float32(65535)
        elif images.dtype != np.float32:
            raise TypeError("images must be float32, uint8 or uint16")
        if images.ndim == 2:
            images = images[None]
        if images.ndim != 3:
            raise ValueError("images must be [H, W] or [B, H, W]")
        images = np.ascontiguousarray(images)
        B, H, W = images.shape
        ctx = self._ctx()
        L = load_stages_library()
        ticket = C.c_uint64()
        ctx.check(L.cvb_akaze_scale_space(ctx.handle, C.byref(self.config.to_c()), images.ctypes.data, B, W, H, C.byref(ticket)))
        return ScaleSpace(ctx, ticket.value, B, W, H, self.config)

    def find_image_keypoints(self, scale_space):
        """Akaze::find_image_keypoints (lib.rs:268-276) on a ScaleSpace: per frame, the keypoints in the reference's order, neither
        sorted nor truncated (maximum_features is ignored, as in the reference).  Detection runs with the config the scale space was
        built with (its detector response already depends on it), so this Akaze's detector fields must equal that config's:
        ValueError otherwise.  Only maximum_features and the descriptor fields may differ."""
        mine, built = _detector_fields(self.config), _detector_fields(scale_space.config)
        if mine != built:
            raise ValueError(f"detector config {mine} differs from the scale space's {built}: build the scale space with this Akaze")
        ctx, L = scale_space.ctx, load_stages_library()
        cap = max(self.max_keypoints, 1)
        while True:
            kp = np.zeros((scale_space.batch, cap), dtype=KP_DTYPE)
            n = np.zeros(scale_space.batch, dtype=np.uint32)
            rc = L.cvb_akaze_find_image_keypoints(ctx.handle, scale_space.ticket, kp.ctypes.data, cap, n.ctypes.data)
            if rc == CVB_ECAP and int(n.max()) > cap:
                cap = int(n.max())
                continue
            ctx.check(rc)
            return [kp[b, :n[b]].copy() for b in range(scale_space.batch)]

    def extract_descriptors(self, scale_space, keypoints_per_frame):
        """Akaze::extract_descriptors(&evolutions, &keypoints) (descriptors.rs:16-45) for one keypoint array per frame of the scale
        space (a bare array when it has one frame).  Only descriptor_channels and descriptor_pattern_size of this Akaze are read.
        Returns per-frame lists (keypoints kept, in input order; their [n, 64] uint8 descriptors)."""
        if isinstance(keypoints_per_frame, np.ndarray) and keypoints_per_frame.dtype == KP_DTYPE:
            keypoints_per_frame = [keypoints_per_frame]
        frames = [np.ascontiguousarray(k, dtype=KP_DTYPE).reshape(-1) for k in keypoints_per_frame]
        if len(frames) != scale_space.batch:
            raise ValueError(f"expected {scale_space.batch} keypoint arrays, got {len(frames)}")
        offsets = np.zeros(len(frames) + 1, np.uint32)
        offsets[1:] = np.cumsum([len(k) for k in frames])
        kp_in = np.concatenate(frames) if offsets[-1] else np.zeros(1, KP_DTYPE)
        total = max(int(offsets[-1]), 1)
        kp_out = np.zeros(total, KP_DTYPE)
        desc = np.zeros((total, 64), np.uint8)
        n = np.zeros(len(frames), np.uint32)
        ctx, L = scale_space.ctx, load_stages_library()
        ctx.check(L.cvb_akaze_extract_descriptors(ctx.handle, C.byref(self.config.to_c()), scale_space.ticket, kp_in.ctypes.data,
                                                  offsets.ctypes.data, kp_out.ctypes.data, desc.ctypes.data, n.ctypes.data))
        return ([kp_out[offsets[b]:offsets[b] + n[b]].copy() for b in range(len(frames))],
                [desc[offsets[b]:offsets[b] + n[b]].copy() for b in range(len(frames))])

    # -- introspection used by the parity tests (no reference counterpart)
    def debug_evolutions(self):
        ctx = self._ctx()
        n = C.c_uint32()
        ctx.check(ctx.lib.cvb_akaze_debug_num_evolutions(ctx.handle, C.byref(n)))
        out = []
        for i in range(n.value):
            v = [C.c_uint32() for _ in range(5)]
            ctx.check(ctx.lib.cvb_akaze_debug_evolution(ctx.handle, i, *[C.byref(x) for x in v]))
            out.append(dict(w=v[0].value, h=v[1].value, octave=v[2].value, sigma_size=v[3].value, n_fed_steps=v[4].value))
        return out

    def debug_plane(self, evolution, name, frame=0):
        ctx = self._ctx()
        info = self.debug_evolutions()[evolution]
        out = np.empty((info["h"], info["w"]), np.float32)
        ctx.check(ctx.lib.cvb_akaze_debug_plane(ctx.handle, frame, evolution, PLANES[name], out.ctypes.data))
        return out

    def debug_contrast(self, frame=0):
        ctx = self._ctx()
        k = C.c_double()
        ctx.check(ctx.lib.cvb_akaze_debug_contrast(ctx.handle, frame, C.byref(k)))
        return k.value

    def debug_stage(self, name, frame=0, cap=1 << 20):
        ctx = self._ctx()
        n = C.c_uint32()
        ctx.check(ctx.lib.cvb_akaze_debug_stage(ctx.handle, frame, STAGES[name], None, 0, C.byref(n)))
        out = np.zeros(max(n.value, 1), dtype=KP_DTYPE)
        ctx.check(ctx.lib.cvb_akaze_debug_stage(ctx.handle, frame, STAGES[name], out.ctypes.data, n.value, C.byref(n)))
        return out[:n.value]


def _detector_fields(config):
    """the AkazeConfig fields find_image_keypoints depends on: all but maximum_features (ignored by find), the two descriptor
    fields (read by describe only) and initial_contrast (never read, lib.rs:123,176)"""
    skip = {"maximum_features", "descriptor_channels", "descriptor_pattern_size", "initial_contrast"}
    return {f: v for f, v in asdict(config).items() if f not in skip}


class ScaleSpace:
    """A scale space resident in a context's AKAZE workspace (the device-side counterpart of akaze's Vec<EvolutionStep>):
    `ticket` names it in include/cvb200_stages.h, `evolutions` is its EvolutionStep table (EVOLUTION_DTYPE), `config` the
    AkazeConfig it was built with."""

    def __init__(self, ctx, ticket, batch, width, height, config):
        self.ctx, self.ticket, self.batch, self.width, self.height = ctx, ticket, batch, width, height
        self.config = replace(config)
        L = load_stages_library()
        n = C.c_uint32()
        ctx.check(L.cvb_akaze_evolutions(ctx.handle, ticket, None, 0, C.byref(n)))
        self.evolutions = np.zeros(n.value, EVOLUTION_DTYPE)
        if n.value:
            ctx.check(L.cvb_akaze_evolutions(ctx.handle, ticket, self.evolutions.ctypes.data, n.value, C.byref(n)))


__all__ = ["Akaze", "AkazeConfig", "CvbError", "Context", "ScaleSpace"]
