"""Per-kernel CUDA-event times of one frame pair (extract x2 -> symmetric match -> bearings -> ARRSAC), single context, no overlap.
python scripts/prof_kernels.py [pairs]   (env CVB_TMA / CVB_KNN_WGMMA select the variants)"""
import ctypes as C, json, os, sys
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import cv_b200
from cv_b200._lib import KP_DTYPE
from cv_b200.geom import ArrsacCfg, Rng, _lib as geom_lib
from cv_b200.pair import Intrinsics, bind
from tests.synth import synth_frame, warp_frame

pairs = int(sys.argv[1]) if len(sys.argv) > 1 else 4
dev = torch.device("cuda", 0)
ctx = cv_b200.Context(0); L = ctx.lib; geom_lib(ctx); bind(L)
cap = 5000
frames = []
for i in range(2):
    a = synth_frame(i); frames.append(torch.from_numpy(np.stack([a, warp_frame(a, 1000 + i)])).to(dev))
cfg = cv_b200.AkazeConfig(maximum_features=cap).to_c()
K = Intrinsics(1000.0, 1000.0, 960.0, 540.0, 0.0)
ac = ArrsacCfg(); L.cvb_arrsac_default_cfg(C.byref(ac), 1e-7); ac.initialization_hypotheses = 8192; ac.max_candidate_hypotheses = 1024
rng = Rng(); L.cvb_rng_seed_xoshiro256pp(C.byref(rng), 0)
kp = torch.empty(2 * cap * KP_DTYPE.itemsize, dtype=torch.uint8, device=dev); desc = torch.zeros(2 * cap * 64, dtype=torch.uint8, device=dev)
n = torch.zeros(2, dtype=torch.int32, device=dev); pr = torch.zeros(cap * 2, dtype=torch.int32, device=dev); inl = torch.zeros(cap, dtype=torch.int32, device=dev)
cnt = torch.zeros(4, dtype=torch.int32, device=dev); model = torch.zeros(12, dtype=torch.float64, device=dev)
stats = (C.c_uint32 * 16)()
def one(i):
    img = frames[i % 2]
    ctx.check(L.cvb_akaze_extract_batch_dev(ctx.handle, C.byref(cfg), img.data_ptr(), 2, 1920, 1080, kp.data_ptr(), desc.data_ptr(), cap, n.data_ptr()))
    ctx.check(L.cvb_two_view_pair_dev(ctx.handle, kp.data_ptr(), desc.data_ptr(), n.data_ptr(), kp.data_ptr() + cap * KP_DTYPE.itemsize, desc.data_ptr() + cap * 64,
                                      n.data_ptr() + 4, cap, 24, C.byref(K), C.addressof(ac), C.addressof(rng), pr.data_ptr(), cap, cnt.data_ptr(), model.data_ptr(),
                                      inl.data_ptr(), cnt.data_ptr() + 4, cnt.data_ptr() + 8))
    ctx.check(L.cvb_arrsac_commit_rng(ctx.handle, C.addressof(rng), stats))
for i in range(3):
    one(i)
ctx.timer_begin()
for i in range(pairs):
    one(i)
ms_graph = ctx.timer_end() / pairs
ctx.profile(True)
for i in range(pairs):
    one(i)
rep = ctx.profile_report()
ctx.profile(False)
tot = sum(v["ms"] for v in rep.values())
print(json.dumps({"tma": os.environ.get("CVB_TMA"), "wgmma": os.environ.get("CVB_KNN_WGMMA"), "single_context_ms_per_pair": ms_graph,
                  "sum_kernel_ms_per_pair": tot / pairs, "counts": cnt.cpu().tolist(), "stats": [int(x) for x in stats]}))
for k, v in sorted(rep.items(), key=lambda kv: -kv[1]["ms"]):
    print(f"{k:28s} {v['ms'] / pairs:9.4f} ms/pair  {v['launches'] / pairs:7.1f} launches")
