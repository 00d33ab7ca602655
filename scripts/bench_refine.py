"""Secondary measurement for SURVEY.md section 8f rows 2-3: python scripts/bench_refine.py  (one JSON line)
GPU: host API wall clock incl. all copies.  CPU: the C restatement (oracle/), single thread, on a bounded sample."""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import cv_b200  # noqa: E402
from oracle import pyoracle as O  # noqa: E402
from tests.geom_util import perturb_pose, pnp_scene, rot_from_scaled_axis, three_view_scene, unit  # noqa: E402

rng = np.random.default_rng(0)
out = {}

# ---- single-view L2 refinement: cv-sfm's sizes (<= 2048 matches, rate 1e-3), fixed iteration count
N, IT = 2048, 2000
probs = []
for b in range(132):
    R, t, bearings, world, _ = pnp_scene(rng, N, noise=2e-4)
    probs.append((perturb_pose(rng, (R, t), 2e-3, 5e-3), bearings, world))
for B in (1, 16, 132):
    poses = [p[0] for p in probs[:B]]
    bearings = np.concatenate([p[1] for p in probs[:B]]); world = np.concatenate([p[2] for p in probs[:B]])
    off = np.arange(B + 1) * N
    cv_b200.single_view_simple_optimize_l2_batch(poses, 1e-3, 10, bearings, world, off)
    t0 = time.perf_counter()
    _, upd = cv_b200.single_view_simple_optimize_l2_batch(poses, 1e-3, IT, bearings, world, off)
    dt = time.perf_counter() - t0
    out[f"single_view_gpu_B{B}"] = {"ms": dt * 1e3, "updates": int(upd.sum()), "us_per_iteration": dt * 1e6 / max(int(upd.max()), 1),
                                    "landmark_iterations_per_s": float(upd.sum()) * N / dt}
t0 = time.perf_counter()
_, _, uw = O.single_view_optimize_l2(probs[0][0], 1e-3, IT, probs[0][1], probs[0][2])
dt = time.perf_counter() - t0
out["single_view_cpu_B1"] = {"ms": dt * 1e3, "updates": int(uw), "us_per_iteration": dt * 1e6 / max(uw, 1), "landmark_iterations_per_s": uw * N / dt}

# ---- three-view L2 refinement: 1024 landmarks (cv-sfm three_view_optimization_landmarks)
N3, IT3 = 1024, 1000
p3 = []
for b in range(132):
    truth, obs = three_view_scene(rng, N3, noise=1e-4)
    p3.append(([perturb_pose(rng, p, 3e-3, 5e-3) for p in truth], obs))
for B in (1, 132):
    starts = [p[0] for p in p3[:B]]; obs = np.concatenate([p[1] for p in p3[:B]]); off = np.arange(B + 1) * N3
    cv_b200.three_view_optimize_l2_batch(starts, 1e-3, 10, obs, off)
    t0 = time.perf_counter()
    _, upd = cv_b200.three_view_optimize_l2_batch(starts, 1e-3, IT3, obs, off)
    dt = time.perf_counter() - t0
    out[f"three_view_gpu_B{B}"] = {"ms": dt * 1e3, "updates": int(upd.sum()), "us_per_iteration": dt * 1e6 / max(int(upd.max()), 1),
                                   "landmark_iterations_per_s": float(upd.sum()) * N3 / dt}
t0 = time.perf_counter()
_, uw = O.three_view_optimize_l2(p3[0][0], 1e-3, IT3, p3[0][1])
dt = time.perf_counter() - t0
out["three_view_cpu_B1"] = {"ms": dt * 1e3, "updates": int(uw), "us_per_iteration": dt * 1e6 / max(uw, 1), "landmark_iterations_per_s": uw * N3 / dt}

# ---- observation losses: 100k landmarks x 4 observations
L, K = 100000, 4
X = np.stack([rng.uniform(-2, 2, L), rng.uniform(-2, 2, L), rng.uniform(3, 9, L)], 1)
views = [(rot_from_scaled_axis(rng.uniform(-1, 1, 3) * 0.2), rng.uniform(-0.6, 0.6, 3)) for _ in range(K)]
poses = np.zeros(L * K, cv_b200.geom.POSE_DTYPE)
bearings = np.zeros((L * K, 3))
for k, (R, t) in enumerate(views):
    poses["r"][k::K] = R.reshape(9); poses["t"][k::K] = t
    bearings[k::K] = unit(X @ R.T + t + rng.normal(0, 1e-3, (L, 3)))
off = np.arange(L + 1) * K
cv_b200.observation_losses(poses[:4000], bearings[:4000], off[:1001])
t0 = time.perf_counter(); got = cv_b200.observation_losses(poses, bearings, off); dt = time.perf_counter() - t0
out["observation_losses_gpu"] = {"ms": dt * 1e3, "observations_per_s": L * K / dt}
S = 5000
t0 = time.perf_counter()
for l in range(S):
    O.observation_losses([views[k] for k in range(K)], bearings[l * K:(l + 1) * K])
dt = time.perf_counter() - t0
out["observation_losses_cpu"] = {"ms": dt * 1e3, "observations_per_s": S * K / dt, "sample": f"{S} landmarks, incl. ctypes call overhead"}
print(json.dumps(out))
