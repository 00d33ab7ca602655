"""Time of the similar-frame search on the device (include/cvb200_lsh.h) at cv-sfm's shape: 4096-bit frame hashes (words = 128), k = 512
(cv-sfm's default tracking_similar_frame_search_num).
  single query: one cvb_hash_knn_dev call per frame, as VSlam::add_frame makes it, over m = 1 000, 10 000 and 100 000 hashes resident on
    the device; the device time per call from CUDA events around back-to-back calls, and the host time of a call that ends in a
    synchronisation (median);
  batch: all-vs-all over 10 000 hashes (1e8 pairs), CUDA events around each call; pairs/s, and the share of the popcount bound:
    128 32-bit popcounts per pair over 132 SMs x 16 popcounts per clock at the card's maximum SM clock.
Results are checked against the oracle (a few rows of the batch) before they are timed.  Reads the card's name, power limit and maximum
SM clock in the same run.  Prints one line per case and one JSON line.
python scripts/prof_frame_search.py [calls]"""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from cv_b200.knn import _lsh_lib  # noqa: E402
from cv_b200.multi import make_context  # noqa: E402
from oracle import pyoracle_lsh as OL  # noqa: E402

CALLS = max(50, int(sys.argv[1]) if len(sys.argv) > 1 else 200)
WORDS, K = 128, 512
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"], capture_output=True,
                     text=True).stdout.strip().splitlines()[0]
card, power, mhz = [s.strip() for s in gpu.split(",")]
POPC_PER_S = 132 * 16 * float(mhz) * 1e6

ctx = make_context(0)
stream = ctx.torch_stream
L = _lsh_lib()
dev = torch.device("cuda", 0)
rng = np.random.default_rng(0)


def search(q_d, n, db_d, m, idx_d, dist_d):
    ctx.check(L.cvb_hash_knn_dev(ctx.handle, WORDS, q_d.data_ptr(), None, n, db_d.data_ptr(), None, m, K, idx_d.data_ptr(),
                                 dist_d.data_ptr()))


def event_ms(fn, reps):
    """device time per call: CUDA events on the context's stream around `reps` back-to-back calls"""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(stream):
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


rows = []
for m in (1_000, 10_000, 100_000):
    db = rng.integers(0, 256, (m, 4 * WORDS), dtype=np.uint8)
    db_d = torch.from_numpy(db).to(dev)
    q_d = db_d[m // 2:m // 2 + 1]
    idx_d = torch.empty((1, K), dtype=torch.int32, device=dev)
    dist_d = torch.empty_like(idx_d)
    torch.cuda.synchronize()
    call = lambda: search(q_d, 1, db_d, m, idx_d, dist_d)  # noqa: E731
    for _ in range(20):
        call()
    ctx.sync()
    want = OL.hash_knn(db[m // 2:m // 2 + 1], db, K)
    assert np.array_equal(idx_d.cpu().numpy().view(np.uint32), want[0]) and np.array_equal(dist_d.cpu().numpy().view(np.uint32), want[1])
    dev_ms = event_ms(call, CALLS)
    ts = []
    for _ in range(CALLS):
        t0 = time.perf_counter()
        call()
        ctx.sync()
        ts.append((time.perf_counter() - t0) * 1e3)
    rows.append(dict(case="single query", m=m, device_us_per_call=dev_ms * 1e3, host_us_median=float(np.median(ts)) * 1e3,
                     host_us_min=float(np.min(ts)) * 1e3, scanned_MB=m * 4 * WORDS / 1e6))
    print(f"single query  m {m:7d}  device {dev_ms * 1e3:8.1f} us/call  host (to synchronisation) median {np.median(ts) * 1e3:8.1f} us")

N = 10_000
db = rng.integers(0, 256, (N, 4 * WORDS), dtype=np.uint8)
db_d = torch.from_numpy(db).to(dev)
idx_d = torch.empty((N, K), dtype=torch.int32, device=dev)
dist_d = torch.empty_like(idx_d)
torch.cuda.synchronize()
call = lambda: search(db_d, N, db_d, N, idx_d, dist_d)  # noqa: E731
call()
ctx.sync()
check = rng.choice(N, 16, replace=False)
want = OL.hash_knn(db[check], db, K)
assert np.array_equal(idx_d.cpu().numpy().view(np.uint32)[check], want[0])
assert np.array_equal(dist_d.cpu().numpy().view(np.uint32)[check], want[1])
times = [event_ms(call, 1) for _ in range(10)]
batch_ms = float(np.median(times))
pairs = float(N) * N
share = pairs * WORDS / POPC_PER_S / (batch_ms * 1e-3)
rows.append(dict(case="all-vs-all", n=N, m=N, k=K, ms_median=batch_ms, ms_min=float(np.min(times)), pairs_per_s=pairs / (batch_ms * 1e-3),
                 share_of_popc_bound=share))
print(f"all-vs-all    {N} x {N}  {batch_ms:8.2f} ms  {pairs / (batch_ms * 1e-3):.3e} pairs/s  {share * 100:5.1f}% of the popcount bound")
print(f"card: {card}, power limit {power} W, max SM clock {mhz} MHz")
print(json.dumps(dict(card=card, power_limit_w=float(power), max_sm_clock_mhz=float(mhz), words=WORDS, k=K, calls=CALLS, rows=rows)))
ctx.close()
