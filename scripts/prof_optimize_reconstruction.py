"""Times cv_b200.optimize_reconstruction (include/cvb200_reconstruction.h) on synthetic reconstructions of 32, 128 and 512 views with about
64 constraints per view, and the CPU oracle on the same inputs (on all the host's threads).  Per scene: the whole call at cv-sfm's defaults
(1 024 Jacobi steps, then the filter), the filter alone (optimization_iterations = 0), their difference per step, the oracle's time, and
whether the device's statuses, states and counts equal the oracle's.  The per-step time is compared with the least a design that launches
each step's two stages would pay: two tiny kernels per step replayed from one CUDA graph.  Prints the card's name and power limit, then one
JSON line per case (medians of --reps runs after a warm-up).

The scenes are built vectorised (a forward-moving camera, points seen by the views whose frustum holds them, noisy bearings), and the
constraints from the true relative poses of nearby view triples times a small random isometry, so that building them does not dominate.

    python scripts/prof_optimize_reconstruction.py [--reps 3] [--oracle-threads 0] [--out DIR]
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


def rodrigues(w):
    """[n, 3] scaled axes -> [n, 3, 3]"""
    a = np.linalg.norm(w, axis=1)[:, None, None]
    k = w / np.maximum(a[:, :, 0], 1e-300)
    K = np.zeros((len(w), 3, 3))
    K[:, 0, 1], K[:, 0, 2], K[:, 1, 2] = -k[:, 2], k[:, 1], -k[:, 0]
    K = K - K.transpose(0, 2, 1)
    return np.eye(3) + np.sin(a) * K + (1 - np.cos(a)) * K @ K


def build(V, per_view=64, window=12, points_per_view=24, seed=0):
    from oracle.pyoracle_reconstruction import CONSTRAINT_DTYPE
    rng = np.random.default_rng(seed)
    v = np.arange(V)
    R = rodrigues(np.stack([0.01 * np.cos(0.7 * v), 0.02 * v + 0.01 * np.sin(v), np.zeros(V)], 1))
    c = np.stack([0.25 * v, 0.05 * np.sin(0.5 * v), np.zeros(V)], 1)
    t = -np.einsum("vij,vj->vi", R, c)
    N = points_per_view * V
    X = np.stack([rng.uniform(-2, 0.25 * V + 2, N), rng.uniform(-2, 2, N), rng.uniform(3, 8, N)], 1)
    cam = np.einsum("vij,nj->vni", R, X) + t[:, None, :]                       # [V, N, 3]
    b = cam / np.linalg.norm(cam, axis=2, keepdims=True)
    seen = b[:, :, 2] > 0.8
    keep = seen.sum(0) >= 1
    b, seen = b[:, keep], seen[:, keep]
    b = b + rng.normal(0, 2e-4, b.shape)
    b /= np.linalg.norm(b, axis=2, keepdims=True)
    L = seen.shape[1]
    vo = np.zeros(V + 1, np.uint32)
    vo[1:] = np.cumsum(seen.sum(1))
    vl = np.concatenate([np.nonzero(seen[x])[0] for x in range(V)]).astype(np.uint32)
    bear = np.concatenate([b[x, seen[x]] for x in range(V)])
    feat = np.zeros((V, L), np.int64)
    for x in range(V):
        feat[x, seen[x]] = np.arange(int(seen[x].sum()))
    lv, ll = np.nonzero(seen.T)                                                 # landmark-major, views ascending
    lo = np.zeros(L + 1, np.uint32)
    lo[1:] = np.cumsum(seen.sum(0))
    ob = np.stack([ll, feat[ll, lv]], 1).astype(np.uint32)
    poses = np.concatenate([R.reshape(V, 9), t], 1)
    # perturbed starting poses; constraints from the true poses of nearby triples times a small isometry
    Rp = rodrigues(rng.normal(0, 2e-3, (V, 3))) @ R
    tp = np.einsum("vij,vj->vi", rodrigues(rng.normal(0, 2e-3, (V, 3))), t) + rng.normal(0, 2e-3, (V, 3))
    start = np.concatenate([Rp.reshape(V, 9), tp], 1)
    tri = []
    for x in range(V):
        near = [u for u in range(max(0, x - window), min(V, x + window + 1)) if u != x]
        pairs = [(p, q) for i, p in enumerate(near) for q in near[i + 1:]]
        for k in rng.permutation(len(pairs))[:per_view]:
            tri.append(sorted([x, *pairs[k]]))
    tri = np.array(tri)
    cons = np.zeros(len(tri), CONSTRAINT_DTYPE)
    cons["views"] = tri
    cons["landmarks"] = 32
    for k in range(2):
        a, o = tri[:, 0], tri[:, k + 1]
        Rr = R[o] @ R[a].transpose(0, 2, 1)
        tr = t[o] - np.einsum("nij,nj->ni", Rr, t[a])
        Rn = rodrigues(rng.normal(0, 1e-4, (len(tri), 3)))
        cons["poses"][:, k]["r"] = (Rn @ Rr).reshape(-1, 9)
        cons["poses"][:, k]["t"] = np.einsum("nij,nj->ni", Rn, tr) + rng.normal(0, 1e-4, (len(tri), 3))
    snap = dict(poses=start, view_offsets=vo, view_landmarks=vl, bearings=bear, landmark_offsets=lo, observations=ob)
    return snap, cons, poses


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--oracle-threads", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import cv_b200
    from cv_b200.reconstruction import ReconstructionSettings, optimize_reconstruction
    from oracle.pyoracle_reconstruction import ReconCfg
    from oracle.pyoracle_reconstruction import optimize_reconstruction as ref_optimize
    name = card()
    print(json.dumps({"card": name}), flush=True)
    ctx = cv_b200.Context(0)
    lines = [{"card": name}]

    def emit(d):
        print(json.dumps(d), flush=True)
        lines.append(d)

    # the least a launch-per-stage design pays per step: two tiny kernels, replayed from one CUDA graph of 1 024 steps
    x = torch.zeros(1, device="cuda")
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        x.add_(1)
    torch.cuda.synchronize()
    with torch.cuda.graph(g, stream=s):
        for _ in range(2 * 1024):
            x.add_(1)

    def replay():
        g.replay()
        torch.cuda.synchronize()
    emit(dict(case="graph_two_launches_per_step", per_step_s=med(replay, a.reps) / 1024))
    threads = a.oracle_threads or os.cpu_count()
    for V in (32, 128, 512):
        snap, cons, _ = build(V, seed=V)
        run = (lambda **kw: optimize_reconstruction(ctx, **snap, constraints=cons, settings=ReconstructionSettings(**kw)))
        full = med(run, a.reps)
        filt = med(lambda: run(optimization_iterations=0), a.reps)
        d = run()
        t = time.perf_counter()
        o = ref_optimize(snap["poses"], snap["view_offsets"], snap["bearings"], snap["landmark_offsets"], snap["observations"], cons,
                         cfg=ReconCfg(), threads=threads)
        t_or = time.perf_counter() - t
        same = (d["result"].tobytes() == o["result"].tobytes() and np.array_equal(d["view_state"], o["view_state"]) and
                np.array_equal(d["obs_state"], o["obs_state"]))
        r = d["result"]
        emit(dict(case=f"V{V}", views=V, constraints=len(cons), edges=6 * len(cons), landmarks=int(len(snap["landmark_offsets"]) - 1),
                  observations=int(snap["landmark_offsets"][-1]), status=int(r["status"]), small_angle_updates=int(r["small_angle_updates"]),
                  observations_split=int(r["observations_split"]), device_s=full, device_filter_s=filt, device_per_step_s=(full - filt) / 1024,
                  oracle_s=t_or, oracle_threads=threads, oracle_discrete_equal=bool(same),
                  max_pose_diff=float(np.abs(d["poses"] - o["poses"]).max())))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "prof_optimize_reconstruction.jsonl"), "w") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
