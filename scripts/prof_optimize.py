"""Kernel time of cv-optimize's pose optimizers on the device, L1 (include/cvb200_opt.h) next to L2 (include/cvb200.h), from the
per-kernel CUDA events of cvb_ctx_profile: B in {1, 16, 132} problems of 2 048 landmarks each at a fixed iteration cap, one CTA per
problem (132 = one CTA per SM of an H100 SXM).  Also times the CPU oracle on one host thread for one problem, and reads the card's name
and power limit in the same run.  Prints one line per configuration and one JSON line.
python scripts/prof_optimize.py [iterations] [launches]"""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import cv_b200  # noqa: E402
from oracle import pyoracle as O  # noqa: E402
from oracle import pyoracle_opt as P  # noqa: E402
from tests.geom_util import perturb_pose, pnp_scene, three_view_scene  # noqa: E402

ITERS = int(sys.argv[1]) if len(sys.argv) > 1 else 500
LAUNCHES = int(sys.argv[2]) if len(sys.argv) > 2 else 5
N = 2048
EPS, RATE_L1, RATE_L2 = 1e-12, 0.01, 1e-3     # rates at which these scenes run to the cap rather than to the patience rule

rng = np.random.default_rng(2048)
single, three = [], []
for b in range(132):
    R, t, bearings, world, _ = pnp_scene(rng, N, noise=2e-4)
    single.append((perturb_pose(rng, (R, t), 2e-3, 5e-3), bearings, world))
    truth, obs = three_view_scene(rng, N, noise=1e-4)
    three.append(([perturb_pose(rng, p, 3e-3, 5e-3) for p in truth], obs))

ctx = cv_b200.Context(0)
rows = []


def run(name, kernel, B, call):
    call()                                              # warm-up: module load, workspace allocation
    ctx.sync()
    ctx.profile(True)
    t0 = time.perf_counter()
    for _ in range(LAUNCHES):
        upd = call()
    ctx.sync()
    wall = (time.perf_counter() - t0) / LAUNCHES * 1e3
    rep = ctx.profile_report()
    ctx.profile(False)
    ms = rep[kernel]["ms"] / rep[kernel]["launches"]
    mean_upd = float(np.mean(upd))
    row = dict(name=name, kernel=kernel, B=B, landmarks=N, iterations=ITERS, mean_updates=mean_upd, kernel_ms=ms, call_ms=wall,
               us_per_iteration=ms * 1e3 / max(mean_upd, 1.0))
    rows.append(row)
    print(f"{name:6s} B={B:3d}  {kernel:22s} {ms:9.3f} ms/launch  ({row['us_per_iteration']:.2f} us per iteration, "
          f"{mean_upd:.0f} updates, call {wall:.3f} ms)")


for B in (1, 16, 132):
    poses = [s[0] for s in single[:B]]
    bearings = np.concatenate([s[1] for s in single[:B]]); world = np.concatenate([s[2] for s in single[:B]])
    off = np.arange(B + 1) * N
    run("sv-l1", "k_single_view_opt_l1", B, lambda: cv_b200.single_view_simple_optimize_l1_batch(
        poses, EPS, RATE_L1, ITERS, bearings, world, off, ctx=ctx)[1])
    run("sv-l2", "k_single_view_opt", B, lambda: cv_b200.single_view_simple_optimize_l2_batch(
        poses, RATE_L2, ITERS, bearings, world, off, ctx=ctx)[1])
    pairs = [s[0] for s in three[:B]]
    obs = np.concatenate([s[1] for s in three[:B]])
    run("tv-l1", "k_three_view_opt_l1", B, lambda: cv_b200.three_view_simple_optimize_l1_batch(
        pairs, EPS, RATE_L1, ITERS, obs, off, ctx=ctx)[1])
    run("tv-l2", "k_three_view_opt", B, lambda: cv_b200.three_view_optimize_l2_batch(
        pairs, RATE_L2, ITERS, obs, off, ctx=ctx)[1])

# the oracle on one host thread, one problem of N landmarks (-O3, landmark order)
cpu = {}
(p0, b0, w0), (q0, o0) = single[0], three[0]
for name, f in (("sv-l1", lambda: P.single_view_optimize_l1(p0, EPS, RATE_L1, ITERS, b0, w0)[2]),
                ("sv-l2", lambda: O.single_view_optimize_l2(p0, RATE_L2, ITERS, b0, w0)[2]),
                ("tv-l1", lambda: P.three_view_optimize_l1(q0, EPS, RATE_L1, ITERS, o0)[1]),
                ("tv-l2", lambda: O.three_view_optimize_l2(q0, RATE_L2, ITERS, o0)[1])):
    t0 = time.perf_counter()
    upd = f()
    ms = (time.perf_counter() - t0) * 1e3
    cpu[name] = dict(ms_per_problem=ms, updates=upd)
    print(f"{name:6s} oracle, one host thread: {ms:9.1f} ms per problem ({upd} updates)")

q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout
card = q.strip().splitlines()[0] if q.strip() else "unknown"
print(f"card: {card}")
print(json.dumps(dict(card=card, gpu=rows, cpu_oracle=cpu)))
