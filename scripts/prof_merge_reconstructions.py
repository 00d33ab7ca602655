"""Times one reconstruction merge (include/cvb200_merge.h) at 8+8 and 32+32 views on the device: merge_reconstructions_dev end to end,
incorporate_reconstruction_dev (the move and its constraint calls) alone, and the single-threaded C oracle chain.  Prints the card's
name and power limit from the same run.  Run from the repository root: python scripts/prof_merge_reconstructions.py"""
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cv_b200  # noqa: E402
from cv_b200.incorporate import snapshot_to_device  # noqa: E402
from cv_b200.merge import incorporate_reconstruction_dev, merge_reconstructions_dev  # noqa: E402
from oracle import pyoracle as O  # noqa: E402
from oracle import pyoracle_merge as OM  # noqa: E402
from tests import merge_scenes as MS  # noqa: E402


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("device:", q)
    ctx = cv_b200.Context(0)
    for n in (8, 32):
        sc = MS.split(V=2 * n, k=n - 1, seed=4, per_view=800 if n <= 8 else 500, step=0.3 if n <= 8 else 0.1)
        R, t = sc["iso"]
        wt = np.concatenate([R.T.reshape(9), -R.T @ t])
        lm = MS.true_landmark_map(sc)
        dd, sd = snapshot_to_device(sc["dest"]), snapshot_to_device(sc["src"])
        wtd, lmd = torch.from_numpy(wt).cuda(), torch.from_numpy(lm.view(np.int32)).cuda()
        times, mv = [], []
        for i in range(6):
            ars = cv_b200.Arrsac(1e-5, cv_b200.Xoshiro256PlusPlus(5), ctx)
            torch.cuda.synchronize(); t0 = time.perf_counter()
            r = merge_reconstructions_dev(ctx, dd, sd, sc["s_view"], sc["dest_view_matches"], ars)
            torch.cuda.synchronize(); times.append(time.perf_counter() - t0)
            torch.cuda.synchronize(); t0 = time.perf_counter()
            m = incorporate_reconstruction_dev(ctx, dd, sd, wtd, lmd)
            torch.cuda.synchronize(); mv.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        w = OM.merge_reconstructions(sc["dest"], sc["src"], sc["s_view"], sc["dest_view_matches"], O.arrsac_cfg(1e-5), O.rng_xoshiro(5))
        to = time.perf_counter() - t0
        print(f"{n}+{n} views: merge {r['status']} (oracle {w['status']}), median of 5 after warm-up: merge_reconstructions_dev "
              f"{1e3 * np.median(times[1:]):.1f} ms, incorporate_reconstruction_dev {1e3 * np.median(mv[1:]):.1f} ms "
              f"({int(m['result']['constraint_calls'])} constraint call(s), {int(m['result']['refused_views'])} refused); C oracle chain {to:.2f} s")


if __name__ == "__main__":
    main()
