"""wgmma Hamming k-NN (CVB_KNN_WGMMA=1) against the CPU oracle, then its time next to the mma.sync and popcount kernels."""
import json, os, sys, time
os.environ["CVB_KNN_WGMMA"] = "1"
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cv_b200
from oracle import pyoracle as O
from tests.synth import random_descriptors

ok = True
for n, m, k in [(1, 1, 1), (3, 2, 2), (5, 1, 2), (130, 257, 2), (128, 128, 2), (129, 127, 1), (1000, 999, 3), (77, 5000, 8), (5000, 5000, 2), (300, 20000, 2)]:
    q, db = random_descriptors(n, 10 + n), random_descriptors(m, 20 + m)
    idx, dist = cv_b200.hamming_knn(q, db, k)
    oi, od = O.hamming_knn(q, db, k)
    e = bool(np.array_equal(dist, od) and np.array_equal(idx, oi))
    ok &= e
    print(json.dumps({"n": n, "m": m, "k": k, "equal": e, "bad_rows": int((dist != od).any(1).sum())}), flush=True)
    if not e:
        r = int(np.where((dist != od).any(1) | (idx != oi).any(1))[0][0])
        print("first bad row", r, dist[r].tolist(), od[r].tolist(), idx[r].tolist(), oi[r].tolist(), flush=True)
base = random_descriptors(16, 3); db = np.concatenate([base] * 40); q = random_descriptors(64, 4); q[:16] = base
idx, dist = cv_b200.hamming_knn(q, db, 4); oi, od = O.hamming_knn(q, db, 4)
e = bool(np.array_equal(idx, oi) and np.array_equal(dist, od)); ok &= e
print(json.dumps({"ties": e}), flush=True)
import torch
dev = torch.device("cuda", 0)
a = torch.from_numpy(random_descriptors(5000, 1)).to(dev); b = torch.from_numpy(random_descriptors(5000, 2)).to(dev)
oi_ = torch.empty(5000 * 2, dtype=torch.int32, device=dev); od_ = torch.empty_like(oi_)
for mode in ("wgmma", "mma.sync", "popcount"):
    for v in ("CVB_KNN_WGMMA", "CVB_KNN_IMMA", "CVB_KNN_POPC"):
        os.environ.pop(v, None)
    os.environ[{"wgmma": "CVB_KNN_WGMMA", "mma.sync": "CVB_KNN_IMMA", "popcount": "CVB_KNN_POPC"}[mode]] = "1"
    ctx = cv_b200.Context(0)
    L = ctx.lib
    for _ in range(3):
        ctx.check(L.cvb_hamming_knn_dev(ctx.handle, a.data_ptr(), 5000, b.data_ptr(), 5000, 2, oi_.data_ptr(), od_.data_ptr()))
    ctx.sync()
    ctx.timer_begin()
    for _ in range(20):
        ctx.check(L.cvb_hamming_knn_dev(ctx.handle, a.data_ptr(), 5000, b.data_ptr(), 5000, 2, oi_.data_ptr(), od_.data_ptr()))
    ms = ctx.timer_end() / 20
    print(json.dumps({"mode": mode, "ms_5kx5k_incl_merge": ms, "Gcmp_per_s": 25e6 / (ms * 1e-3) / 1e9}), flush=True)
print("ALL_EQUAL", ok)
sys.exit(0 if ok else 1)
