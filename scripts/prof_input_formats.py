"""Per-call time of the host-API extractor on 1080p batches from page-locked host frames, for the three inputs a caller has: the f32
plane (cvb_akaze_extract_batch, converted on the host beforehand), Luma8 and Rgb8 (cvb_akaze_extract_dynamic_batch, converted on the
device).  The three are alternated in one process and one context, each call timed on the host around a call that ends in a
synchronisation; the median of each is reported.  Then the kernel time of k_from_dynamic (LUMA8, RGB8, and LUMA8 with the RGB8 plane
of frame ingestion) from the per-kernel CUDA events of cvb_ctx_profile.  Reads the card's name and power limit in the same run.
Prints one line per configuration and one JSON line.
python scripts/prof_input_formats.py [rounds] [batch]"""
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import cv_b200  # noqa: E402
from cv_b200._lib import KP_DTYPE  # noqa: E402
from cv_b200.image import lib as image_lib  # noqa: E402
from tests.synth import synth_frame  # noqa: E402

ROUNDS = max(5, int(sys.argv[1]) if len(sys.argv) > 1 else 30)
B = max(1, int(sys.argv[2]) if len(sys.argv) > 2 else 4)
H, W = 1080, 1920


def pinned(shape, dtype):
    t = torch.empty(int(np.prod(shape)) * np.dtype(dtype).itemsize, dtype=torch.uint8, pin_memory=True)
    return t.numpy().view(dtype).reshape(shape)


luma = np.stack([np.round(synth_frame(40 + b) * 255).astype(np.uint8) for b in range(B)])
src = {"f32": pinned((B, H, W), np.float32), "luma8": pinned((B, H, W), np.uint8), "rgb8": pinned((B, H, W, 3), np.uint8)}
src["luma8"][:] = luma
src["f32"][:] = luma.astype(np.float32) / np.float32(255)
src["rgb8"][:] = np.repeat(luma[..., None], 3, -1)
ctx = cv_b200.Context(0)
L, IL = ctx.lib, image_lib()
ak = cv_b200.Akaze(ctx=ctx)
cfg = ak.config.to_c()
cap = 16384
kp, desc, n = pinned((B, cap), KP_DTYPE), pinned((B, cap, 64), np.uint8), pinned((B,), np.uint32)


def call(kind):
    if kind == "f32":
        rc = L.cvb_akaze_extract_batch(ctx.handle, C.byref(cfg), src[kind].ctypes.data, B, W, H, kp.ctypes.data, desc.ctypes.data, cap,
                                       n.ctypes.data)
    else:
        rc = IL.cvb_akaze_extract_dynamic_batch(ctx.handle, C.byref(cfg), 0 if kind == "luma8" else 2, src[kind].ctypes.data, B, W, H,
                                                kp.ctypes.data, desc.ctypes.data, cap, n.ctypes.data)
    ctx.check(rc)
    return n.copy()


counts = {k: call(k) for k in src}                      # warm-up: workspaces, graph capture; all three give the same keypoints
assert all(np.array_equal(counts["f32"], c) for c in counts.values()), counts
times = {k: [] for k in src}
for _ in range(ROUNDS):
    for k in src:
        t0 = time.perf_counter()
        call(k)
        times[k].append((time.perf_counter() - t0) * 1e3)
rows = []
for k, ts in times.items():
    upload = src[k].nbytes
    rows.append(dict(input=k, batch=B, ms_per_call=float(np.median(ts)), ms_min=float(np.min(ts)), upload_bytes=upload))
    print(f"extract {k:6s} B={B}: {np.median(ts):8.3f} ms/call median ({np.min(ts):.3f} min), upload {upload} B")

# k_from_dynamic alone, on device frames
dev = torch.device("cuda", 0)
d_luma = torch.from_numpy(src["luma8"]).to(dev)
d_rgb = torch.from_numpy(src["rgb8"]).to(dev)
gray = torch.empty(B * H * W, dtype=torch.float32, device=dev)
rgb8 = torch.empty(B * H * W * 3, dtype=torch.uint8, device=dev)
torch.cuda.synchronize()
kernel_rows = []
for name, fmt, px, out_rgb in (("luma8", 0, d_luma, None), ("rgb8", 2, d_rgb, None), ("luma8+rgb8 plane", 0, d_luma, rgb8)):
    conv = lambda: ctx.check(IL.cvb_gray_float_from_dynamic_dev(ctx.handle, fmt, px.data_ptr(), B, W, H, gray.data_ptr(),  # noqa: E731
                                                                out_rgb.data_ptr() if out_rgb is not None else None))
    conv()
    ctx.sync()
    ctx.profile(True)
    for _ in range(ROUNDS * 4):
        conv()
    ctx.sync()
    rep = ctx.profile_report()["k_from_dynamic"]
    ctx.profile(False)
    ms = rep["ms"] / rep["launches"]
    gbs = rep["bytes"] / rep["launches"] / (ms * 1e-3) / 1e9
    kernel_rows.append(dict(input=name, batch=B, kernel_ms=ms, bytes=rep["bytes"] / rep["launches"], GBps=gbs))
    print(f"k_from_dynamic {name:17s} B={B}: {ms:8.4f} ms/launch, {gbs:7.1f} GB/s of algorithmic bytes")
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(f"card: {gpu}")
print(json.dumps(dict(card=gpu, rounds=ROUNDS, batch=B, extract=rows, kernel=kernel_rows)))
ctx.close()
