"""Kernel and host-API time of akaze::image on the device (include/cvb200_filter.h): the reference's criterion cases (akaze/benches/
criterion.rs: horizontal and vertical filter of the KITTI frame with gaussian_kernel(1.0, 7) and gaussian_kernel(10.0, 71)), the
separable filter with both kernels, gaussian_blur(1.6) and half_size, on the KITTI frame (1392 x 512) and on a batch of 8 synthetic
1080p planes.
  kernel time: per-kernel CUDA events of cvb_ctx_profile over the _dev calls, >= 100 calls after warm-up, summed over a call's passes;
  host-API time: median over calls of the host form, each ending in its synchronisation (page-locked host planes);
  bounds: 8 w h B algorithmic bytes per filter pass over 3.35 TB/s of HBM3, and 2 * 4 ceil(ks / 4) + 3 unfused FP32 instructions per
  output over 132 SMs x 128 lanes at the card's maximum SM clock; the share is the larger bound over the kernel time;
  CPU: oracle/ref_filter.c, the C restatement of the reference's loops, single-threaded on the same planes (not the Rust criterion
  numbers, which are not recorded anywhere).
Reads the card's name, power limit and maximum SM clock in the same run.  Prints one line per case and one JSON line.
python scripts/prof_filters.py [launches]"""
import ctypes as C
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import cv_b200  # noqa: E402
from cv_b200 import filter as F  # noqa: E402
from oracle import pyoracle_filter as OF  # noqa: E402
from tests.common import kitti_frame  # noqa: E402
from tests.synth import synth_frame  # noqa: E402

LAUNCHES = max(100, int(sys.argv[1]) if len(sys.argv) > 1 else 200)
HOST_CALLS = 30
HBM = 3.35e12
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"], capture_output=True,
                     text=True).stdout.strip().splitlines()[0]
card, power, mhz = [s.strip() for s in gpu.split(",")]
SM_CLOCK = float(mhz) * 1e6
FP32_ISSUE = 132 * 128 * SM_CLOCK   # unfused FP32 instructions per second, one per lane per clock


def pinned(shape):
    t = torch.empty(int(np.prod(shape)), dtype=torch.float32, pin_memory=True)
    return t.numpy().reshape(shape)


planes = {"kitti 1392x512": kitti_frame("0000000000")[None],
          "8 x 1080p": np.stack([synth_frame(50 + b) for b in range(8)]).astype(np.float32)}
k7, k71 = F.gaussian_kernel(1.0, 7), F.gaussian_kernel(10.0, 71)
blur_ks = OF.blur_size(1.6)
ctx = cv_b200.Context(0)
L = F.lib()
dev = torch.device("cuda", 0)


def instr(ks):
    return 2 * 4 * math.ceil(ks / 4) + 3


# name -> (host entry, extra args, filter passes as kernel sizes (None: half_size), oracle)
CASES = [
    ("horizontal k7", "cvb_horizontal_filter", (k7.ctypes.data, 7), [7], lambda a: OF.horizontal_filter(a, k7)),
    ("horizontal k71", "cvb_horizontal_filter", (k71.ctypes.data, 71), [71], lambda a: OF.horizontal_filter(a, k71)),
    ("vertical k7", "cvb_vertical_filter", (k7.ctypes.data, 7), [7], lambda a: OF.vertical_filter(a, k7)),
    ("vertical k71", "cvb_vertical_filter", (k71.ctypes.data, 71), [71], lambda a: OF.vertical_filter(a, k71)),
    ("separable k7", "cvb_separable_filter", (k7.ctypes.data, 7, k7.ctypes.data, 7), [7, 7], lambda a: OF.separable_filter(a, k7, k7)),
    ("separable k71", "cvb_separable_filter", (k71.ctypes.data, 71, k71.ctypes.data, 71), [71, 71],
     lambda a: OF.separable_filter(a, k71, k71)),
    ("gaussian_blur 1.6", "cvb_gaussian_blur", (C.c_float(1.6),), [blur_ks, blur_ks], lambda a: OF.gaussian_blur(a, 1.6)),
    ("half_size", "cvb_half_size", (), None, OF.half_size),
]

rows = []
for pname, img in planes.items():
    B, H, W = img.shape
    src_h = pinned(img.shape)
    src_h[:] = img
    out_h = pinned(img.shape)
    src_d = torch.from_numpy(img).to(dev)
    out_d = torch.empty_like(src_d)
    torch.cuda.synchronize()
    for name, fn, args, passes, oracle in CASES:
        dev_call = lambda: ctx.check(getattr(L, fn + "_dev")(ctx.handle, src_d.data_ptr(), B, W, H, *args, out_d.data_ptr()))  # noqa: E731
        host_call = lambda: ctx.check(getattr(L, fn)(ctx.handle, src_h.ctypes.data, B, W, H, *args, out_h.ctypes.data))  # noqa: E731
        for _ in range(5):
            dev_call()
            host_call()
        ctx.sync()
        t0 = time.perf_counter()
        want = oracle(img)
        cpu_ms = (time.perf_counter() - t0) * 1e3
        got = out_h.reshape(-1)[:want.size].reshape(want.shape)
        assert got.tobytes() == want.tobytes(), f"{name} on {pname} differs from the oracle"
        ctx.profile(True)
        for _ in range(LAUNCHES):
            dev_call()
        ctx.sync()
        rep = ctx.profile_report()
        ctx.profile(False)
        kernel_ms = sum(r["ms"] for r in rep.values()) / LAUNCHES
        by_kernel = {k: r["ms"] / r["launches"] for k, r in rep.items()}
        ts = []
        for _ in range(HOST_CALLS):
            t0 = time.perf_counter()
            host_call()
            ts.append((time.perf_counter() - t0) * 1e3)
        if passes is None:
            nbytes = 4.0 * (W * H + (W // 2) * (H // 2)) * B
            t_hbm, t_fp = nbytes / HBM, 0.0
        else:
            nbytes = 8.0 * W * H * B * len(passes)
            t_hbm = nbytes / HBM
            t_fp = sum(W * H * B * instr(ks) for ks in passes) / FP32_ISSUE
        bound = "HBM" if t_hbm >= t_fp else "FP32 issue"
        share = max(t_hbm, t_fp) / (kernel_ms * 1e-3)
        rows.append(dict(planes=pname, case=name, kernel_ms=kernel_ms, kernels=by_kernel, host_ms_median=float(np.median(ts)),
                         host_ms_min=float(np.min(ts)), algorithmic_bytes=nbytes, GBps=nbytes / (kernel_ms * 1e-3) / 1e9,
                         fp32_instr_per_output=[instr(ks) for ks in passes] if passes else None, bound=bound, share_of_bound=share,
                         oracle_cpu_1thread_ms=cpu_ms))
        print(f"{pname:15s} {name:18s} kernel {kernel_ms * 1e3:9.2f} us  host {np.median(ts):8.3f} ms  "
              f"{nbytes / (kernel_ms * 1e-3) / 1e9:7.1f} GB/s  {share * 100:5.1f}% of the {bound} bound  "
              f"C oracle 1 thread {cpu_ms:9.2f} ms")
print(f"card: {card}, power limit {power} W, max SM clock {mhz} MHz")
print(json.dumps(dict(card=card, power_limit_w=float(power), max_sm_clock_mhz=float(mhz), launches=LAUNCHES, host_calls=HOST_CALLS,
                      rows=rows)))
ctx.close()
