"""Times cv_b200.generate_view_constraints (include/cvb200_constraints.h) on synthetic reconstructions, the CPU oracle on the same inputs,
and the adaptive three-view optimiser A/B: the warp-per-problem kernel (cvb_three_view_adaptive_optimize_l2_dev) against the CTA-per-problem
k_three_view_opt (cvb_three_view_optimize_l2, adaptive) on batches of the same shape as the call's selected problems, outputs asserted
equal.  Prints the card's name and power limit, then one JSON line per case (medians of --reps runs after a warm-up).

    python scripts/prof_view_constraints.py [--reps 3] [--oracle-threads 0] [--out DIR]
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


def med(f, reps):
    f()
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        f()
        ts.append(time.perf_counter() - t)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--oracle-threads", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import cv_b200
    from cv_b200.constraints import ConstraintSettings, generate_view_constraints, three_view_adaptive_optimize_l2_dev
    from cv_b200.optimize import _lib as opt_lib
    from tests.constraint_scenes import scene
    from oracle.pyoracle_constraints import ConstraintsCfg, view_constraints
    print(json.dumps({"card": card()}), flush=True)
    ctx = cv_b200.Context(0)
    dev = torch.device("cuda", 0)
    lines = []

    def emit(d):
        print(json.dumps(d), flush=True)
        lines.append(d)

    threads = a.oracle_threads or os.cpu_count()
    for V in (32, 128):
        s, _, _ = scene(V, points=20 * V + 400, seed=V, noise=2e-4, outliers=0.02, fov_cos=0.8)
        for name, qs in (("one_view", [V // 2]), ("all_views", list(range(V)))):
            full = med(lambda: generate_view_constraints(ctx, **s, queries=qs), a.reps)
            rest = med(lambda: generate_view_constraints(ctx, **s, queries=qs, settings=ConstraintSettings(constraint_patience=0)), a.reps)
            r = generate_view_constraints(ctx, **s, queries=qs, stats=True)
            sizes = [int(m) for c in r["constraints"] for m in c["landmarks"]]
            t = time.perf_counter()
            o = view_constraints(**s, queries=qs, cfg=ConstraintsCfg(), threads=threads)
            t_or = time.perf_counter() - t
            same = all(np.array_equal(x["views"], y["views"]) for x, y in zip(r["constraints"], o["constraints"]))
            emit(dict(case=f"V{V}_{name}", views=V, queries=len(qs), features=int(len(s["view_landmarks"])),
                      landmarks=int(len(s["landmark_offsets"]) - 1), problems=len(sizes), device_s=full, device_patience0_s=rest,
                      device_optimiser_s=full - rest, oracle_s=t_or, oracle_threads=threads, oracle_views_equal=bool(same)))
            if not sizes:
                continue
            # A/B on a batch of the same shape: B problems with the selected problems' landmark counts
            rng = np.random.default_rng(V)
            B = len(sizes)
            off = np.zeros(B + 1, np.uint32)
            off[1:] = np.cumsum(sizes)
            obs = rng.normal(0, 1, (int(off[-1]), 3, 3)) + np.array([0, 0, 5.0])
            obs /= np.linalg.norm(obs, axis=2, keepdims=True)
            obs = np.ascontiguousarray(obs.reshape(-1, 9))
            poses = np.zeros((B, 2, 12))
            poses[:, :, [0, 4, 8]] = 1.0
            poses[:, 0, 9] = 1.0
            poses[:, 1, 9] = 2.0
            poses[:, :, 10:] = rng.normal(0, 0.1, (B, 2, 2))
            poses = np.ascontiguousarray(poses.reshape(-1, 12))
            it = 4096
            _, L = opt_lib(ctx)
            want = np.zeros_like(poses)
            wupd = np.zeros(B, np.uint32)

            def cta():
                ctx.check(L.cvb_three_view_optimize_l2(ctx.handle, poses.ctypes.data, B, 1, 0.0, it, obs.ctypes.data, off.ctypes.data,
                                                       want.ctypes.data, wupd.ctypes.data))
            tp, to, tf = (torch.from_numpy(poses).to(dev), torch.from_numpy(obs).to(dev), torch.from_numpy(off.astype(np.int32)).to(dev))
            res = {}

            def warp():
                res["out"] = three_view_adaptive_optimize_l2_dev(ctx, tp, to, tf, it)
            t_cta, t_warp = med(cta, a.reps), med(warp, a.reps)
            assert res["out"][0].cpu().numpy().tobytes() == want.tobytes()
            emit(dict(case=f"V{V}_{name}_optimiser_ab", problems=B, landmarks=int(off[-1]), iterations=it, k_three_view_opt_s=t_cta,
                      k_three_view_opt_warp_s=t_warp, speedup=t_cta / t_warp, outputs_equal=True))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "prof_view_constraints.jsonl"), "w") as f:
            f.write(json.dumps({"card": card()}) + "\n")
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
