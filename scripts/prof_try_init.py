"""Times cv-sfm's reconstruction creation on the device (include/cvb200_try_init.h).  (1) add_reconstruction_dev at cap 1024, 4096 and
8192 with every frame full (3 cap features) and match lists over 40 % of the center's features; then one profiled run (ctx.profile: CUDA
events around each launch) gives the per-kernel times.  (2) try_init_dev against the same work done as before this module existed:
the two-view options and init_reconstruction on the device, the lists copied to the host, the snapshot built there (the C restatement of
add_reconstruction) and uploaded.  Times are medians of CUDA-event timings after a warm-up.  Prints the card's name and power limit from
the same run, and one JSON line per row; with --out DIR it also writes DIR/prof_try_init.json.

    python scripts/prof_try_init.py [--runs 7] [--patience 0] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cv_b200  # noqa: E402
from cv_b200._lib import default_context  # noqa: E402
from cv_b200.incorporate import snapshot_to_device  # noqa: E402
from cv_b200.pair import INIT_RESULT_DTYPE, InitSettings, _two_view_options_dev, init_reconstruction_dev  # noqa: E402
from cv_b200.try_init import add_reconstruction_dev, try_init_dev  # noqa: E402
from oracle import pyoracle_try_init as OT  # noqa: E402
from tests.try_init_scenes import descriptor_scene, frame_store, random_lists  # noqa: E402


def timed(fn, runs):
    fn()                                                                          # warm-up
    ts = []
    for _ in range(runs):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return round(float(np.median(ts)), 3), [round(t, 3) for t in ts]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--patience", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print("gpu:", gpu, flush=True)
    ctx = default_context(0)
    rows = []
    for cap in (1024, 4096, 8192):
        rng = np.random.default_rng(cap)
        k = int(0.4 * cap)
        comb, fm, sm = random_lists(rng, cap, cap, cap, k // 2, k // 2, k // 2)
        st = frame_store(rng, [cap, cap, cap], cap)
        t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()   # noqa: E731
        ds = dict(descriptors=t(st["descriptors"]), counts=t(st["counts"]), bearings=t(st["bearings"]), colors=t(st["colors"]))
        ir = np.zeros(1, INIT_RESULT_DTYPE)
        ir["n_combined"], ir["n_first_matches"], ir["n_second_matches"] = len(comb), len(fm), len(sm)
        pad = lambda x, c: t(np.concatenate([x, np.zeros((cap - len(x), c), np.uint32)]).view(np.int32))   # noqa: E731
        args = (t(ir.view(np.uint8)), pad(comb, 3), pad(fm, 2), pad(sm, 2))
        run = lambda: add_reconstruction_dev(ctx, ds, 0, 1, 2, *args)   # noqa: E731
        med, ts = timed(run, a.runs)
        torch.cuda.synchronize()
        ctx.profile(True)
        run()
        torch.cuda.synchronize()
        rep = ctx.profile_report()
        ctx.profile(False)
        row = dict(call="add_reconstruction_dev", cap=cap, features=3 * cap, landmarks=int(run()[1]["L"]), device_ms_median=med, device_ms_runs=ts,
                   kernels={k: dict(launches=v["launches"], ms=round(v["ms"], 3)) for k, v in rep.items() if k.startswith("k_")})
        print(json.dumps(row), flush=True)
        rows.append(row)
    # try_init against the init on the device followed by host glue and an upload
    sc = descriptor_scene(np.random.default_rng(5), 4, n_points=3000, cap=4096, noise=1e-6)
    st = sc["store"]
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()   # noqa: E731
    ds = dict(descriptors=t(st["descriptors"]), counts=t(st["counts"]), bearings=t(st["bearings"]), colors=t(st["colors"]))
    options = [1, 2, 3, 4]
    cfg = InitSettings(three_view_patience=a.patience, two_view_minimum_robust_matches=64)

    def device():
        ars = cv_b200.Arrsac(1e-6, cv_b200.Xoshiro256PlusPlus(0), ctx=ctx)
        return try_init_dev(ds, 0, options, ars, [cv_b200.Xoshiro256PlusPlus(s) for s in (1, 2, 3, 4)], settings=cfg)

    def glue():
        ars = cv_b200.Arrsac(1e-6, cv_b200.Xoshiro256PlusPlus(0), ctx=ctx)
        _, _, opts, two = _two_view_options_dev(ds, 0, options, ars, [cv_b200.Xoshiro256PlusPlus(s) for s in (1, 2, 3, 4)], 24)
        r = init_reconstruction_dev(ctx, ds["bearings"], 0, opts, two, cfg)
        res = r["result"]
        if res["status"] != 1:
            return None
        snap = OT.add_reconstruction(st["descriptors"], st["counts"], st["bearings"], st["colors"], 0, options[res["first"]],
                                     options[res["second"]], res["first_pose"], res["second_pose"], r["combined"], r["first_matches"],
                                     r["second_matches"])
        return snapshot_to_device(snap)

    status = device()["status"]
    md, tsd = timed(device, a.runs)
    mg, tsg = timed(glue, a.runs)
    row = dict(call="try_init_dev vs init on the device + host glue + upload", options=len(options), features_per_frame=3000, cap=4096,
               patience=a.patience, status=status, try_init_dev_ms_median=md, try_init_dev_ms_runs=tsd, init_glue_upload_ms_median=mg,
               init_glue_upload_ms_runs=tsg)
    print(json.dumps(row), flush=True)
    rows.append(row)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "prof_try_init.json"), "w") as f:
            json.dump(dict(gpu=gpu, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
