"""Kernel time of every triangulator of include/cvb200_tri.h on a track-sized workload, from the per-kernel CUDA events of
cvb_ctx_profile, against the CPU oracle on one host thread.  Observations methods: L seeded landmarks of 2-8 views each
(k_triangulate); relative methods: L (pose, a, b) triples with one pose per triple (k_triangulate_relative).  Also prints the
distribution of SineL1's refinement iterations (from the oracle, whose results equal the device's bit for bit), because a warp waits
for its slowest landmark.  Writes one JSON line with the card name and power limit read in the same run.
python scripts/prof_triangulate.py [landmarks] [launches]"""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import cv_b200  # noqa: E402
from cv_b200.geom import POSE_DTYPE  # noqa: E402
from oracle import pyoracle_tri as T  # noqa: E402

L = int(sys.argv[1]) if len(sys.argv) > 1 else 200_000
launches = int(sys.argv[2]) if len(sys.argv) > 2 else 10
ORACLE_L = min(L, 20_000)     # the oracle is timed on the first landmarks / triples only


def rodrigues(v):
    th = np.linalg.norm(v, axis=1, keepdims=True)
    k = v / th
    K = np.zeros((len(v), 3, 3))
    K[:, 0, 1], K[:, 0, 2], K[:, 1, 0], K[:, 1, 2], K[:, 2, 0], K[:, 2, 1] = -k[:, 2], k[:, 1], k[:, 2], -k[:, 0], -k[:, 1], k[:, 0]
    s, c = np.sin(th)[:, :, None], np.cos(th)[:, :, None]
    return np.eye(3)[None] + s * K + (1 - c) * K @ K


def unit(x):
    return x / np.linalg.norm(x, axis=-1, keepdims=True)


rng = np.random.default_rng(2024)
# a track: 2-8 views of every landmark, cameras within a few units of the origin, points 4-40 units ahead, 1e-3 bearing noise
counts = rng.integers(2, 9, L)
off = np.zeros(L + 1, np.uint32); off[1:] = np.cumsum(counts)
nobs = int(off[-1])
X = np.repeat(rng.uniform([-10, -10, 4], [10, 10, 40], (L, 3)), counts, axis=0)
R = rodrigues(rng.normal(0, 0.1, (nobs, 3)))
t = rng.normal(0, 1.0, (nobs, 3))
poses = np.zeros(nobs, POSE_DTYPE); poses["r"] = R.reshape(-1, 9); poses["t"] = t
bearings = unit(np.einsum("nij,nj->ni", R, X) + t + rng.normal(0, 1e-3, (nobs, 3)))
Xr = rng.uniform([-10, -10, 4], [10, 10, 40], (L, 3))
Rr = rodrigues(rng.normal(0, 0.1, (L, 3))); tr = rng.normal(0, 1.0, (L, 3))
rposes = np.zeros(L, POSE_DTYPE); rposes["r"] = Rr.reshape(-1, 9); rposes["t"] = tr
ra = unit(Xr + rng.normal(0, 1e-3, (L, 3)))
rb = unit(np.einsum("nij,nj->ni", Rr, Xr) + tr + rng.normal(0, 1e-3, (L, 3)))

ctx = cv_b200.Context(0)
res = {"landmarks": L, "observations": nobs, "launches": launches, "oracle_items": ORACLE_L, "methods": {}}
for cls in (cv_b200.LinearEigenTriangulator, cv_b200.SineL1Triangulator, cv_b200.MeanMeanTriangulator, cv_b200.RelativeDltTriangulator,
            cv_b200.AngularL1Triangulator, cv_b200.AngularLInfinityTriangulator):
    tri = cls()
    ocfg = T.triangulator(tri.cfg.method, tri.cfg.epsilon, tri.cfg.max_iterations, tri.cfg.optimization_rate)
    rel = tri.cfg.method >= T.RELATIVE_DLT
    for form in (["relative"] if rel else ["observations", "relative"]):
        if form == "observations":
            run = lambda: tri.triangulate_batch(poses, bearings, off, ctx)      # noqa: E731
            kname = "k_triangulate"
            t0 = time.perf_counter(); _, ook, its = T.triangulate_observations_batch(ocfg, poses, bearings, off[:ORACLE_L + 1]); t_or = time.perf_counter() - t0
        else:
            run = lambda: tri.triangulate_relative_batch(rposes, ra, rb, ctx)   # noqa: E731
            kname = "k_triangulate_relative"
            t0 = time.perf_counter(); _, ook = T.triangulate_relative_batch(ocfg, rposes[:ORACLE_L], ra[:ORACLE_L], rb[:ORACLE_L]); t_or = time.perf_counter() - t0
        _, ok = run()                                                           # warm-up
        ctx.sync()
        ctx.profile(True)
        t0 = time.perf_counter()
        for _ in range(launches):
            run()
        t_call = (time.perf_counter() - t0) / launches
        rep = ctx.profile_report()
        ctx.profile(False)
        k = rep[kname]
        ms = k["ms"] / k["launches"]
        res["methods"][f"{type(tri).__name__}.{form}"] = {
            "kernel_ms": round(ms, 4), "kernel_ns_per_item": round(1e6 * ms / L, 2), "call_ms_host_to_host": round(1e3 * t_call, 3),
            "ok_fraction": round(float(ok.mean()), 4), "oracle_1thread_ns_per_item": round(1e9 * t_or / ORACLE_L, 1),
            "oracle_over_kernel": round((1e9 * t_or / ORACLE_L) / (1e6 * ms / L), 1)}
        if tri.cfg.method == T.SINE_L1 and form == "observations":
            _, _, its = T.triangulate_observations_batch(ocfg, poses, bearings, off)
            refined = its[its > 0]
            res["sine_l1_iterations"] = {"refined_landmarks": int(len(refined)), "mean": round(float(refined.mean()), 1),
                                         "percentiles_10_50_90_99": [int(np.percentile(refined, q)) for q in (10, 50, 90, 99)],
                                         "at_max_iterations": int((refined == tri.cfg.max_iterations).sum()),
                                         # a warp of 32 consecutive landmarks runs as long as its slowest lane
                                         "warp_busy_fraction": round(float(its[: len(its) // 32 * 32].reshape(-1, 32).mean(1).sum()
                                                                           / its[: len(its) // 32 * 32].reshape(-1, 32).max(1).sum()), 3)}
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout
res["gpu"] = q.strip().splitlines()[0] if q else None
print(json.dumps(res))
