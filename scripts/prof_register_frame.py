"""Measures cv-sfm's frame registration on the device (include/cvb200_register.h) on the seeded scenes of tests/register_scenes.py at 8
and 32 matched views: the host-clock median of cvb_register_frame per call (the call ends in a synchronise; uploads and copies back
included), the device time of its three stages from the context's profiling scopes (matching: the k-NN and the glue up to matches_3d;
consensus: ARRSAC and the inlier take; filter: the optimiser, consistency and final passes), and one run of the single-threaded C oracle,
which restates the reference loop for loop.  The card's name and power limit are read in the same run.

    python scripts/prof_register_frame.py [--out FILE]    # every row is printed as a JSON line; --out also writes them as one file
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError) as e:
        raise SystemExit(f"no GPU: {e}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, nargs="*", default=[8, 32])
    ap.add_argument("--per-view", type=int, default=3000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = card()
    import cv_b200
    from oracle import pyoracle as O
    from oracle import pyoracle_register as OR
    from tests import register_scenes as RS
    ctx = cv_b200.Context(0)
    rows = []
    for V in a.views:
        s = RS.scene(V=V, per_view=a.per_view, seed=100 + V, outliers=0.15, merges=20, doubly=10, step=0.3 if V <= 8 else 0.12)
        run = lambda: cv_b200.register_frame(ctx, *RS.args(s), cv_b200.Arrsac(1e-5, cv_b200.Xoshiro256PlusPlus(7), ctx), stats=True)
        status, _, matches, st, _ = run()
        ts = []
        for _ in range(a.reps):
            t = time.perf_counter()
            run()
            ts.append(time.perf_counter() - t)
        ctx.profile(True)
        run()
        rep = ctx.profile_report()
        ctx.profile(False)
        t = time.perf_counter()
        want = OR.register_frame(*RS.args(s), O.arrsac_cfg(1e-5), O.rng_xoshiro(7))
        t_oracle = time.perf_counter() - t
        row = dict(gpu=gpu, views=V, new_features=len(s["new_descriptors"]), status=status, subsets=int(st["subsets"]),
                   inliers=int(st["inliers"]), final_matches=len(matches), oracle_status=want["status"],
                   oracle_final_matches=len(want["matches"]), device_call_ms=1e3 * float(np.median(ts)),
                   stage_ms={k: round(rep[k]["ms"], 3) for k in ("register_match", "register_consensus", "register_filter") if k in rep},
                   oracle_ms=1e3 * t_oracle)
        print(json.dumps(row), flush=True)
        rows.append(row)
    if a.out:
        with open(a.out, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
