"""Device time of AKAZE's staged surface (include/cvb200_stages.h) against the one-call extractor, on 1080p synthetic frames
(tests/synth.py, Akaze::default(), threshold 0.001) at batch 1 and 8:
  extract            cvb_akaze_extract_batch_dev
  scale space + find cvb_akaze_scale_space_dev + cvb_akaze_find_image_keypoints_dev
  describe 5k / 50k  cvb_akaze_extract_descriptors_dev at 5 000 and 50 000 caller keypoints per frame (find's keypoints repeated and
                     jittered), on a resident scale space
  find + describe    scale space + find + describe of every found keypoint (extract's work without the sort and truncation)
Each case: CUDA events on the context's stream around `reps` back-to-back calls after a warm-up, median of 5 such windows.  Every
staged call is eager (no CUDA graph); extract replays its graph.  Reads the card's name and power limit in the same run.  Prints one
line per case and one JSON line.
python scripts/prof_akaze_stages.py [reps]"""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from cv_b200._lib import KP_DTYPE, load_stages_library  # noqa: E402
from cv_b200.akaze import AkazeConfig  # noqa: E402
from cv_b200.multi import make_context  # noqa: E402
from tests.synth import synth_frame  # noqa: E402

REPS = max(3, int(sys.argv[1]) if len(sys.argv) > 1 else 10)
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"], capture_output=True,
                     text=True).stdout.strip().splitlines()[0]
card, power = [s.strip() for s in gpu.split(",")]
ctx = make_context(0)
stream = ctx.torch_stream
L = load_stages_library()
dev = torch.device("cuda", 0)
cfg = AkazeConfig(detector_threshold=0.001).to_c()
H, W = 1080, 1920
CAP = 1 << 16


def event_ms(fn):
    fn()
    times = []
    for _ in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(stream):
            e0.record()
            for _ in range(REPS):
                fn()
            e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1) / REPS)
    return float(np.median(times))


rows = []
for B in (1, 8):
    imgs = torch.from_numpy(np.stack([synth_frame(100 + b) for b in range(B)])).to(dev)
    kp = torch.zeros(B * CAP * KP_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    desc = torch.zeros(B * CAP * 64, dtype=torch.uint8, device=dev)
    n = torch.zeros(B, dtype=torch.int32, device=dev)
    t = C.c_uint64()

    def extract():
        ctx.check(ctx.lib.cvb_akaze_extract_batch_dev(ctx.handle, C.byref(cfg), imgs.data_ptr(), B, W, H, kp.data_ptr(), desc.data_ptr(),
                                                      CAP, n.data_ptr()))

    def scale_space():
        ctx.check(L.cvb_akaze_scale_space_dev(ctx.handle, C.byref(cfg), imgs.data_ptr(), B, W, H, C.byref(t)))

    def find():
        ctx.check(L.cvb_akaze_find_image_keypoints_dev(ctx.handle, t.value, kp.data_ptr(), CAP, n.data_ptr()))

    scale_space()
    find()
    torch.cuda.synchronize()
    counts = n.cpu().numpy()
    found = kp.cpu().numpy().view(KP_DTYPE).reshape(B, CAP)
    rows.append(dict(case="extract", batch=B, ms=event_ms(extract)))
    rows.append(dict(case="scale space + find", batch=B, ms=event_ms(lambda: (scale_space(), find())), keypoints=int(counts.sum())))
    scale_space()
    rng = np.random.default_rng(0)
    for per in (5_000, 50_000):
        frames = []
        for b in range(B):
            src = found[b, :counts[b]]
            k = src[rng.integers(0, len(src), per)].copy()
            k["x"] += rng.uniform(-2, 2, per).astype(np.float32)
            k["y"] += rng.uniform(-2, 2, per).astype(np.float32)
            k["angle"] = rng.uniform(0, 2 * np.pi, per).astype(np.float32)
            frames.append(k)
        allk = np.concatenate(frames)
        kin = torch.from_numpy(allk.view(np.uint8).copy()).to(dev)
        offs = torch.from_numpy((np.arange(B + 1, dtype=np.int64) * per).astype(np.int32)).to(dev)
        kout = torch.zeros(len(allk) * KP_DTYPE.itemsize, dtype=torch.uint8, device=dev)
        dout = torch.zeros(len(allk) * 64, dtype=torch.uint8, device=dev)

        def describe(kin=kin, offs=offs, kout=kout, dout=dout, total=len(allk)):
            ctx.check(L.cvb_akaze_extract_descriptors_dev(ctx.handle, C.byref(cfg), t.value, kin.data_ptr(), offs.data_ptr(), total,
                                                          kout.data_ptr(), dout.data_ptr(), n.data_ptr()))
        rows.append(dict(case=f"describe {per // 1000}k/frame", batch=B, ms=event_ms(describe)))
    # find + describe of every found keypoint: find writes B x CAP slots, describe reads them packed (CSR), so the packed copy is
    # made once up front from find's (deterministic) output; the timed window runs scale space, find and describe
    packed = np.concatenate([found[b, :counts[b]] for b in range(B)])
    kin_found = torch.from_numpy(packed.view(np.uint8).copy()).to(dev)
    offs_found = torch.from_numpy(np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)).to(dev)
    kout = torch.zeros_like(kp)
    dout = torch.zeros_like(desc)

    def find_describe():
        scale_space()
        find()
        ctx.check(L.cvb_akaze_extract_descriptors_dev(ctx.handle, C.byref(cfg), t.value, kin_found.data_ptr(), offs_found.data_ptr(),
                                                      len(packed), kout.data_ptr(), dout.data_ptr(), n.data_ptr()))
    rows.append(dict(case="find + describe", batch=B, ms=event_ms(find_describe)))

flag = C.c_uint32()
ctx.check(ctx.lib.cvb_akaze_dev_overflow(ctx.handle, C.byref(flag)))
for r in rows:
    print(f"{r['case']:>22s}  B={r['batch']}  {r['ms']:8.3f} ms" + (f"  ({r['keypoints']} keypoints)" if "keypoints" in r else ""))
print(json.dumps(dict(card=card, power_limit_w=power, reps=REPS, overflow_flag=flag.value, rows=rows)))
