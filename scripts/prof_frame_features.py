"""CUDA-event time of the frame-ingestion kernel (k_frame_features: K1 bearing + bicubic colour per keypoint) on B 1080p frames with
about 5 000 keypoints each, from the per-kernel events of cvb_ctx_profile.  Prints one JSON line with the card and its power limit.
python scripts/prof_frame_features.py [batch] [iterations]"""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import cv_b200  # noqa: E402
from cv_b200._lib import KP_DTYPE  # noqa: E402
from cv_b200.pair import IntrinsicsK1, bind  # noqa: E402
from tests.synth import synth_frame, warp_frame  # noqa: E402

B = int(sys.argv[1]) if len(sys.argv) > 1 else 16
iters = int(sys.argv[2]) if len(sys.argv) > 2 else 50
H, W, cap = 1080, 1920, 5000
dev = torch.device("cuda", 0)
base = [synth_frame(s) for s in (21, 22)]
gray = np.stack([warp_frame(base[i % 2], 100 + i) if i >= 2 else base[i] for i in range(B)])
rgb = np.stack([np.round(gray * 255).astype(np.uint8)] * 3, -1)
rgb[..., 1] = np.random.default_rng(3).integers(0, 256, gray.shape, dtype=np.uint8)
ctx = cv_b200.Context(0)
L = ctx.lib
bind(L)
g = torch.from_numpy(gray).to(dev)
c = torch.from_numpy(np.ascontiguousarray(rgb)).to(dev)
kp = torch.zeros(B * cap * KP_DTYPE.itemsize, dtype=torch.uint8, device=dev)
desc = torch.zeros(B * cap * 64, dtype=torch.uint8, device=dev)
n = torch.zeros(B, dtype=torch.int32, device=dev)
bear = torch.zeros(B * cap * 3, dtype=torch.float64, device=dev)
col = torch.zeros(B * cap * 3, dtype=torch.uint8, device=dev)
cfg = cv_b200.AkazeConfig(maximum_features=cap).to_c()
K = IntrinsicsK1(893.39010814, 898.32648616, 951.1310043, 555.13350077, 0.0, -0.28052513)
torch.cuda.synchronize()
ctx.check(L.cvb_akaze_extract_batch_dev(ctx.handle, C.byref(cfg), g.data_ptr(), B, W, H, kp.data_ptr(), desc.data_ptr(), cap, n.data_ptr()))


def features():
    ctx.check(L.cvb_frame_features_batch_dev(ctx.handle, kp.data_ptr(), n.data_ptr(), B, cap, c.data_ptr(), W, H, C.byref(K), bear.data_ptr(),
                                             col.data_ptr()))


for _ in range(5):
    features()
ctx.sync()
ctx.profile(True)
for _ in range(iters):
    features()
rep = ctx.profile_report()
ctx.profile(False)
ctx.timer_begin()
for _ in range(iters):
    features()
ms_back_to_back = ctx.timer_end() / iters
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout
r = rep["k_frame_features"]
print(json.dumps({"batch": B, "keypoints": n.cpu().tolist(), "k_frame_features_us_per_call": 1e3 * r["ms"] / r["launches"],
                  "back_to_back_us_per_call": 1e3 * ms_back_to_back, "iterations": iters, "gpu": q.strip().splitlines()[0] if q else None}))
