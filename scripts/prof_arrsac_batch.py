"""Batched device ARRSAC (include/cvb200_batch.h) against B sequential single calls on one context, for B in {1, 2, 4, 8, 16, 31, 64}
(64 = CVB_ARRSAC_BATCH_MAX: the undecided-predicate queue is split 64 ways).

Workloads: (a) the bench pair's matches under B different generators, vslam-sandbox's two-view configuration
(Arrsac(1e-7).initialization_hypotheses(8192).max_candidate_hypotheses(1024) + EightPoint); (b) B distinct synthetic two-view scenes
of 64 to 5 000 matches and 10-60 % outliers, same configuration; (c) P3P at the single-view configuration
(Arrsac(1e-5).initialization_hypotheses(16384).max_candidate_hypotheses(1024).estimations_per_block(256)) on B synthetic scenes.
Both sides run from device buffers, graphs captured (one warm-up pass of each shape, then five timed runs); times are CUDA-event
medians of the enqueue-to-commit span, so they include the host's raw-draw generation; the host time until the enqueueing call
returns is reported on its own: in the timed runs the graph is replayed, so that is the raw-draw generation plus one graph launch.
Then, in a separate profiled pass (ctx.profile: eager launches, CUDA events around each launch), the per-kernel device time of B = 31
sequential calls and of one batch of 31 on (a).  Last, the fused path: F x cvb_two_view_pair_k1_dev against one
cvb_two_view_options_dev over a center frame and F in {1, 4, 8, 16, 31} warped synthetic option frames.
    python scripts/prof_arrsac_batch.py [--out DIR]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import cv_b200  # noqa: E402
from cv_b200._lib import load_batch_library  # noqa: E402
from cv_b200.geom import Rng  # noqa: E402
from tests.geom_util import pnp_scene, two_view_scene  # noqa: E402
from tests.synth import synth_frame, warp_frame  # noqa: E402

BS = (1, 2, 4, 8, 16, 31, 64)


def _states(seeds):
    return (Rng * len(seeds))(*[cv_b200.Xoshiro256PlusPlus(s).state for s in seeds])


def _results(model, inl, ninl, found):
    """per problem: None, or (pose bytes, inlier indices) -- the outputs up to each count"""
    model, inl, ninl, found = model.cpu().numpy(), inl.cpu().numpy(), ninl.cpu().numpy(), found.cpu().numpy()
    return [(model[i].tobytes(), inl[i, :ninl[i]].tolist()) if found[i] else None for i in range(len(found))]


class Runner:
    def __init__(self, ctx, cfg, kind, probs):
        self.ctx, self.cfg, self.kind, self.B = ctx, cfg, kind, len(probs)
        self.n_max = max(len(p[0]) for p in probs)
        bc = 4 if kind == 1 else 3
        a = np.zeros((self.B * self.n_max, 3)); b = np.zeros((self.B * self.n_max, bc))
        for i, (pa, pb) in enumerate(probs):
            a[i * self.n_max:i * self.n_max + len(pa)] = pa; b[i * self.n_max:i * self.n_max + len(pb)] = pb
        self.a, self.b = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
        self.n = torch.tensor([len(p[0]) for p in probs], dtype=torch.int32).cuda()
        self.sa, self.sb, self.sn = self.a[:self.n_max].clone(), self.b[:self.n_max].clone(), self.n[:1].clone()
        self.model = torch.zeros(self.B * 12, dtype=torch.float64, device="cuda")
        self.inl = torch.zeros(self.B * self.n_max, dtype=torch.int32, device="cuda")
        self.ninl = torch.zeros(self.B, dtype=torch.int32, device="cuda"); self.found = torch.zeros(self.B, dtype=torch.int32, device="cuda")
        self.smodel, self.sinl = self.model[:12].clone(), self.inl[:self.n_max].clone()
        self.sninl, self.sfound = self.ninl[:1].clone(), self.found[:1].clone()
        self.L, self.BL = cv_b200.load_library(), load_batch_library()
        self.L.cvb_arrsac_eight_point_dev.argtypes = [C.c_void_p] * 5 + [C.c_uint32] + [C.c_void_p] * 3 + [C.c_uint32] + [C.c_void_p] * 2
        self.L.cvb_arrsac_p3p_dev.argtypes = self.L.cvb_arrsac_eight_point_dev.argtypes
        self.L.cvb_arrsac_commit_rng.argtypes = [C.c_void_p] * 3

    def batch(self, st):
        t0 = time.perf_counter()
        self.ctx.check(self.BL.cvb_arrsac_batch_dev(self.ctx.handle, C.addressof(self.cfg), self.kind, 5, self.a.data_ptr(), self.b.data_ptr(),
                                                    self.n.data_ptr(), self.n_max, self.B, C.addressof(st), self.model.data_ptr(),
                                                    self.inl.data_ptr(), self.n_max, self.ninl.data_ptr(), self.found.data_ptr()))
        self.host_ms = (time.perf_counter() - t0) * 1e3
        self.ctx.check(self.BL.cvb_arrsac_commit_rng_batch(self.ctx.handle, C.addressof(st), self.B, None))

    def sequential(self, st):
        # every call reads one slot (problem i's rows copied there first), so all calls share one graph-cache key, as a caller that
        # reuses its buffers would
        fn = self.L.cvb_arrsac_eight_point_dev if self.kind == 0 else self.L.cvb_arrsac_p3p_dev
        self.host_ms = 0.0
        for i in range(self.B):
            self.sa.copy_(self.a[i * self.n_max:(i + 1) * self.n_max]); self.sb.copy_(self.b[i * self.n_max:(i + 1) * self.n_max])
            self.sn.copy_(self.n[i:i + 1])
            torch.cuda.synchronize()                     # the copies run on torch's stream, the call on the context's
            t0 = time.perf_counter()
            self.ctx.check(fn(self.ctx.handle, C.addressof(self.cfg), self.sa.data_ptr(), self.sb.data_ptr(), self.sn.data_ptr(), self.n_max,
                              C.addressof(st[i]), self.smodel.data_ptr(), self.sinl.data_ptr(), self.n_max, self.sninl.data_ptr(),
                              self.sfound.data_ptr()))
            self.host_ms += (time.perf_counter() - t0) * 1e3
            torch.cuda.synchronize()
            self.model[12 * i:12 * i + 12].copy_(self.smodel); self.inl[i * self.n_max:(i + 1) * self.n_max].copy_(self.sinl)
            self.ninl[i:i + 1].copy_(self.sninl); self.found[i:i + 1].copy_(self.sfound)
            self.ctx.check(self.L.cvb_arrsac_commit_rng(self.ctx.handle, C.addressof(st[i]), None))

    def time(self, fn, seeds, reps=5):
        ts, hs = [], []
        for r in range(reps + 2):                    # two warm-up passes: the first runs eagerly, the second captures the graphs
            st = _states(seeds)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(torch.cuda.current_stream())
            fn(st)
            e1.record(torch.cuda.current_stream())
            torch.cuda.synchronize()
            if r >= 2:
                ts.append(e0.elapsed_time(e1)); hs.append(self.host_ms)
        res = (_results(self.model.view(self.B, 12), self.inl.view(self.B, self.n_max), self.ninl, self.found),
               [list(st[i].s) for i in range(self.B)])
        return float(np.median(ts)), float(np.median(hs)), res


def profile(ctx, pair):
    """per-kernel ms of 31 sequential single calls and of one batch of 31 on the bench pair (eager, profiled)"""
    ars = cv_b200.Arrsac(1e-7, cv_b200.Xoshiro256PlusPlus(0), ctx=ctx).initialization_hypotheses(8192).max_candidate_hypotheses(1024)
    R = Runner(ctx, ars.cfg, 0, [pair] * 31)
    out = {}
    for name, fn in (("sequential", R.sequential), ("batch", R.batch)):
        fn(_states(list(range(31))))                       # warm-up
        torch.cuda.synchronize()
        ctx.profile(True)
        fn(_states(list(range(31))))
        torch.cuda.synchronize()
        rep = ctx.profile_report()
        ctx.profile(False)
        out[name] = {k: dict(launches=v["launches"], ms=round(v["ms"], 3)) for k, v in rep.items() if k.startswith("k_ars")}
    return out


def fused(ctx):
    """F x cvb_two_view_pair_k1_dev against one cvb_two_view_options_dev (center frame 0, F warped synthetic frames)"""
    cap, Fmax = 4096, 31
    base = synth_frame(5, h=540, w=960, nblobs=2500)
    frames = np.stack([base] + [warp_frame(base, 300 + i, shift=(0.3 * i, -0.2 * i)) for i in range(Fmax)])
    cam = cv_b200.CameraIntrinsics(focals=(800.0, 800.0), principal_point=(480.0, 270.0))
    ak = cv_b200.Akaze(maximum_features=cap)
    feats = cv_b200.frame_features(ak, frames, (frames * 255).astype(np.uint8), cam)
    n_fr = len(frames)
    kp = np.zeros((n_fr, cap), cv_b200.KP_DTYPE); desc = np.zeros((n_fr, cap, 64), np.uint8); bear = np.zeros((n_fr, cap, 3))
    n = np.zeros(n_fr, np.int32)
    for f, d in enumerate(feats):
        k = len(d["keypoints"]); kp[f, :k] = d["keypoints"]; desc[f, :k] = d["descriptors"]; bear[f, :k] = d["bearings"]; n[f] = k
    kpd, descd, nd, beard = (torch.from_numpy(kp.view(np.uint8).reshape(n_fr, -1)).cuda(), torch.from_numpy(desc).cuda(), torch.from_numpy(n).cuda(),
                             torch.from_numpy(bear).cuda())
    L, BL = cv_b200.load_library(), load_batch_library()
    cv_b200.pair.bind(L)
    K = cv_b200.IntrinsicsK1.from_camera(cam)
    ars = cv_b200.Arrsac(1e-7, cv_b200.Xoshiro256PlusPlus(0), ctx=ctx).initialization_hypotheses(8192).max_candidate_hypotheses(1024)
    pairs = torch.zeros((Fmax, cap, 2), dtype=torch.int32, device="cuda"); npairs = torch.zeros(Fmax, dtype=torch.int32, device="cuda")
    model = torch.zeros((Fmax, 12), dtype=torch.float64, device="cuda"); inl = torch.zeros((Fmax, cap), dtype=torch.int32, device="cuda")
    ninl = torch.zeros(Fmax, dtype=torch.int32, device="cuda"); found = torch.zeros(Fmax, dtype=torch.int32, device="cuda")
    skp, sdesc, sn = kpd[0].clone(), descd[0].clone(), nd[:1].clone()
    spairs, snp, smodel, sinl = pairs[0].clone(), npairs[:1].clone(), model[0].clone(), inl[0].clone()
    sninl, sfound = ninl[:1].clone(), found[:1].clone()
    rows = []
    for F in (1, 4, 8, 16, 31):
        opts = np.arange(1, F + 1, dtype=np.uint32)

        def sep(st):
            # the option frame is copied into one slot first, so all calls share one graph-cache key
            for f in range(F):
                o = int(opts[f])
                skp.copy_(kpd[o]); sdesc.copy_(descd[o]); sn.copy_(nd[o:o + 1])
                torch.cuda.synchronize()                 # the copies run on torch's stream, the call on the context's
                ctx.check(L.cvb_two_view_pair_k1_dev(ctx.handle, kpd.data_ptr(), descd.data_ptr(), nd.data_ptr(), skp.data_ptr(),
                                                     sdesc.data_ptr(), sn.data_ptr(), cap, 24, C.byref(K),
                                                     C.addressof(ars.cfg), C.addressof(st[f]), spairs.data_ptr(), cap, snp.data_ptr(),
                                                     smodel.data_ptr(), sinl.data_ptr(), sninl.data_ptr(), sfound.data_ptr()))
                torch.cuda.synchronize()
                pairs[f].copy_(spairs); npairs[f:f + 1].copy_(snp); model[f].copy_(smodel); inl[f].copy_(sinl)
                ninl[f:f + 1].copy_(sninl); found[f:f + 1].copy_(sfound)
                ctx.check(L.cvb_arrsac_commit_rng(ctx.handle, C.addressof(st[f]), None))

        def one(st):
            ctx.check(BL.cvb_two_view_options_dev(ctx.handle, descd.data_ptr(), nd.data_ptr(), beard.data_ptr(), n_fr, cap, 0, opts.ctypes.data,
                                                  F, 24, C.addressof(ars.cfg), C.addressof(st), pairs.data_ptr(), npairs.data_ptr(),
                                                  model.data_ptr(), inl.data_ptr(), ninl.data_ptr(), found.data_ptr()))
            ctx.check(BL.cvb_arrsac_commit_rng_batch(ctx.handle, C.addressof(st), F, None))

        res = {}
        for name, fn in (("separate", sep), ("options", one)):
            ts = []
            for r in range(7):
                st = _states(list(range(F)))
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(torch.cuda.current_stream())
                fn(st)
                e1.record(torch.cuda.current_stream())
                torch.cuda.synchronize()
                if r >= 2:
                    ts.append(e0.elapsed_time(e1))
            res[name] = (float(np.median(ts)), _results(model[:F], inl[:F], ninl[:F], found[:F]), [list(st[i].s) for i in range(F)])
        rows.append(dict(workload="fused_two_view_options", F=F, separate_pair_k1_ms=round(res["separate"][0], 3),
                         options_ms=round(res["options"][0], 3), speedup=round(res["separate"][0] / res["options"][0], 2),
                         same_results=res["separate"][1:] == res["options"][1:]))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--bs", default=",".join(map(str, BS)))
    args = ap.parse_args()
    bs = [int(x) for x in args.bs.split(",")]
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("GPU:", gpu)
    z = np.load(os.path.join(ROOT, "tests", "golden", "bench_pair0.npz"))
    pair = (z["ba"], z["bb"])
    rng = np.random.default_rng(2024)
    sizes = np.linspace(64, 5000, 31).astype(int)
    scenes = []
    for i, n in enumerate(sizes):
        _, _, a, b, _ = two_view_scene(rng, int(n), outlier_frac=0.1 + 0.5 * ((i * 7) % 31) / 30, noise=5e-5)
        scenes.append((a, b))
    pnp = []
    for i in range(64):
        _, _, a, b, _ = pnp_scene(rng, 2000, outlier_frac=0.2, noise=1e-4)
        pnp.append((a, b))
    rows = []
    ctx = cv_b200.Context(0)
    try:
        for wl in ("a_bench_pair", "b_synthetic", "c_p3p"):
            if wl == "c_p3p":
                ars = cv_b200.Arrsac(1e-5, cv_b200.Xoshiro256PlusPlus(0), ctx=ctx).initialization_hypotheses(16384).max_candidate_hypotheses(1024).estimations_per_block(256)
                kind = 1
            else:
                ars = cv_b200.Arrsac(1e-7, cv_b200.Xoshiro256PlusPlus(0), ctx=ctx).initialization_hypotheses(8192).max_candidate_hypotheses(1024)
                kind = 0
            for B in bs:
                if wl == "b_synthetic" and B > len(scenes):
                    continue
                probs = [pair] * B if wl == "a_bench_pair" else (scenes[:B] if wl == "b_synthetic" else pnp[:B])
                seeds = list(range(B))
                R = Runner(ctx, ars.cfg, kind, probs)
                t_seq, h_seq, r_seq = R.time(R.sequential, seeds)
                t_bat, h_bat, r_bat = R.time(R.batch, seeds)
                row = dict(workload=wl, B=B, sequential_ms=round(t_seq, 3), batch_ms=round(t_bat, 3), speedup=round(t_seq / t_bat, 2),
                           same_results=r_seq == r_bat, host_enqueue_ms_sequential=round(h_seq, 3), host_enqueue_ms_batch=round(h_bat, 3))
                rows.append(row)
                print(json.dumps(row), flush=True)
        rows.append(dict(profile_31=profile(ctx, pair)))
        print(json.dumps(rows[-1]), flush=True)
        for row in fused(ctx):
            rows.append(row)
            print(json.dumps(row), flush=True)
    finally:
        ctx.close()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "prof_arrsac_batch.json"), "w") as f:
            json.dump(dict(gpu=gpu, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
