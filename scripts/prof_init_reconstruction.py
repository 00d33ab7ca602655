"""Times cv-sfm's three-view initialisation on the device (include/cvb200_init.h: cvb_init_reconstruction_dev) against its C oracle on one
host thread (oracle/ref_init.c), for F = 8 and 31 options, in two cases: the first pair decides, and only the last pair decides (every
earlier pair shares no matches and is rejected for too few relative scales).  Device times are medians of CUDA-event timings after a
warm-up; then one profiled run (ctx.profile: CUDA events around each launch) gives the per-kernel times.  cv-sfm's default settings
(three_view_patience 65 536) unless --patience is given.  Prints one JSON line per row; with --out DIR it also writes
DIR/prof_init_reconstruction.json.

    python scripts/prof_init_reconstruction.py [--runs 5] [--patience N] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cv_b200._lib import default_context  # noqa: E402
from cv_b200.pair import InitSettings, init_reconstruction_dev  # noqa: E402
from oracle import pyoracle_init as OI  # noqa: E402
from tests.init_scenes import init_scene  # noqa: E402


def scene(F, late, per=300, shared=600):
    """F options with `per` own points each; the pair that decides (pair 0, or the last pair) also shares `shared` points"""
    rng = np.random.default_rng(F * 2 + late)
    n = F * per + shared
    seen = [list(range(f * per, (f + 1) * per)) for f in range(F)]
    for f in ((F - 2, F - 1) if late else (0, 1)):
        seen[f] += list(range(F * per, n))
    cap = 1 << int(np.ceil(np.log2(n)))
    return init_scene(rng, F, n_points=n, cap=cap, noise=1e-5, outliers=0.05, seen=[np.array(s) for s in seen])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--patience", type=int, default=1 << 16)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    ctx = default_context(0)
    cfg = dict(three_view_patience=a.patience)
    rows = []
    for F in (8, 31):
        for late in (False, True):
            sc = scene(F, late)
            arrs = OI.options_from_matches(F, sc["bearings"].shape[1], sc["matches"], sc["poses"])
            names = ("pairs", "n_pairs", "model", "inliers", "n_inliers", "found")
            dev = {k: torch.from_numpy(np.ascontiguousarray(v).view(np.int32) if v.dtype != np.float64 else v).cuda()
                   for k, v in zip(names, arrs)}
            bear = torch.from_numpy(sc["bearings"]).cuda()
            run = lambda: init_reconstruction_dev(ctx, bear, 0, sc["options"], dev, InitSettings(**cfg), stats=True)  # noqa: E731
            got = run()                                                                     # warm-up
            ts = []
            for _ in range(a.runs):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                run()
                e1.record()
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1))
            t0 = time.perf_counter()
            want = OI.init_reconstruction(sc["bearings"], 0, sc["options"], *arrs, OI.InitCfg(**cfg))
            t_oracle = (time.perf_counter() - t0) * 1e3
            torch.cuda.synchronize()
            ctx.profile(True)
            run()
            torch.cuda.synchronize()
            rep = ctx.profile_report()
            ctx.profile(False)
            st = got["stats"]
            dec = int(got["result"]["pair"])
            row = dict(F=F, case="last pair decides" if late else "first pair decides", pairs=F * (F - 1) // 2, decided_pair=dec,
                       status=int(got["result"]["status"]), same_decision_as_oracle=bool(got["result"]["pair"] == want["result"]["pair"] and
                                                                                         got["result"]["status"] == want["result"]["status"]),
                       device_ms_median=round(float(np.median(ts)), 3), device_ms_runs=[round(t, 3) for t in ts],
                       oracle_ms_one_thread=round(t_oracle, 1), optimiser_updates_decisive_pair=int(st[dec]["updates"]),
                       kernels={k: dict(launches=v["launches"], ms=round(v["ms"], 3)) for k, v in rep.items() if k.startswith("k_")})
            print(json.dumps(row), flush=True)
            rows.append(row)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "prof_init_reconstruction.json"), "w") as f:
            json.dump(dict(gpu=gpu, patience=a.patience, rows=rows), f, indent=1)
    print("gpu:", gpu)


if __name__ == "__main__":
    main()
