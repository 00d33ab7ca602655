"""Times cv-sfm's frame incorporation on one GPU (include/cvb200_incorporate.h): incorporate_frame_dev on register scenes of 8, 32 and 128
views against the same work done as separate calls (register_frame, a host add_view on numpy, generate_view_constraints,
optimize_reconstruction, a host replay of its edits, with the uploads each call makes), and add_view_dev / apply_optimization_dev alone on
the 512-view, 1.1 M-observation scene.  Prints one JSON line per measurement, the card's name and power limit included; writes them to a
file only when --out is given.

    python scripts/prof_incorporate_frame.py [--reps 5] [--out FILE]
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

import cv_b200  # noqa: E402
from cv_b200.incorporate import add_view_dev, apply_optimization_dev, incorporate_frame_dev, snapshot_to_device  # noqa: E402
from tests import incorporate_scenes as IS  # noqa: E402
from tests import register_scenes as RS  # noqa: E402
from tests.test_gpu_incorporate import _np_add_view, _np_replay  # noqa: E402


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    name, power = [x.strip() for x in q.splitlines()[0].split(",")]
    return name, power


def _median_ms(fn, reps):
    t = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t)), float(np.min(t)), float(np.max(t))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    name, power = _card()
    ctx = cv_b200.Context(0)
    lines = []
    keys = ("poses", "view_offsets", "view_landmarks", "bearings", "landmark_offsets", "observations")
    for V, per_view, step in ((8, 1500, 0.3), (32, 1500, 0.12), (128, 1500, 0.12)):
        s = RS.scene(V=V, per_view=per_view, seed=71, outliers=0.1, step=step)
        snap = IS.snapshot(s, 71)
        sd = snapshot_to_device(snap)
        nd, nb = torch.from_numpy(s["new_descriptors"]).cuda(), torch.from_numpy(s["new_bearings"]).cuda()
        nc = torch.from_numpy(np.zeros((len(s["new_bearings"]), 3), np.uint8)).cuda()
        status = []

        def fused():
            r = incorporate_frame_dev(ctx, sd, nd, nb, s["view_matches"], cv_b200.Arrsac(1e-5, cv_b200.Xoshiro256PlusPlus(9), ctx), new_colors=nc)
            status.append(r["status"])

        def separate():
            ars = cv_b200.Arrsac(1e-5, cv_b200.Xoshiro256PlusPlus(9), ctx)
            st, pose, m = cv_b200.register_frame(ctx, *(s[k] for k in RS.SNAP_KEYS), s["new_descriptors"], s["new_bearings"],
                                                 s["view_matches"], ars)
            if st != "ok":
                return
            a = _np_add_view(snap, np.concatenate([pose[0].reshape(9), pose[1]]), s["new_bearings"], m)
            cons = cv_b200.generate_view_constraints(ctx, *(a[k] for k in keys), [V])
            if not cons["results"][0]["accepted"]:
                return
            allc = np.concatenate([snap["constraints"], cons["constraints"][0]])
            a["constraints"] = allc
            o = cv_b200.optimize_reconstruction(ctx, *(a[k] for k in keys), allc)
            if int(o["result"]["status"]) == 0:
                _np_replay(a, o["poses"], o["view_state"], o["obs_state"])

        fused()
        f = _median_ms(fused, args.reps)
        p = _median_ms(separate, max(2, args.reps // 2))
        lines.append(dict(bench="incorporate_frame", views=V, observations=len(snap["observations"]), status=status[-1],
                          fused_ms=f[0], fused_min_ms=f[1], fused_max_ms=f[2], separate_ms=p[0], separate_min_ms=p[1], separate_max_ms=p[2],
                          gpu=name, power_limit=power))
        print(json.dumps(lines[-1]), flush=True)
    from tests.scale_scenes import sliding_scene
    s, _ = sliding_scene(512, per_view=2700, seed=3, noise=1e-4, singles=560)
    snap = dict(s, descriptors=None, colors=None, constraints=IS.chain_constraints(512, 3))
    sd = snapshot_to_device(snap)
    N = 2700
    rng = np.random.default_rng(0)
    nb = torch.from_numpy(rng.normal(size=(N, 3))).cuda()
    m = IS.random_matches(snap, N, seed=1, n_match=N // 2, merges=100)
    md = torch.from_numpy(m.view(np.uint8).reshape(-1, 12).copy()).cuda()
    pose = torch.from_numpy(snap["poses"][0].copy()).cuda()
    vs, os_ = IS.random_states(snap, seed=7, removed=9, split=0.02)
    vsd, osd = torch.from_numpy(vs).cuda(), torch.from_numpy(os_).cuda()
    a = _median_ms(lambda: add_view_dev(ctx, sd, pose, nb, md), args.reps)
    b = _median_ms(lambda: apply_optimization_dev(ctx, sd, sd["poses"], vsd, osd), args.reps)
    for nm, t in (("add_view_dev", a), ("apply_optimization_dev", b)):
        lines.append(dict(bench=nm, views=512, observations=len(snap["observations"]), ms=t[0], min_ms=t[1], max_ms=t[2], gpu=name,
                          power_limit=power, note="wall time of the Python call: tensor allocation, two small read-backs and the kernels"))
        print(json.dumps(lines[-1]), flush=True)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write("\n".join(json.dumps(x) for x in lines) + "\n")


if __name__ == "__main__":
    main()
