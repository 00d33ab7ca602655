"""Consensus scoring on the bench's frame pair (tests/golden/bench_pair0.npz, 3 811 matches, vslam-sandbox configuration):
per-kernel CUDA-event times of the ARRSAC kernels (one context, eager launches, no overlap) and the predicates the
CameraToCamera filter left undecided, by scoring phase, per pair.  Prints the card's name and power limit beside the numbers.
python scripts/prof_score.py [pairs]"""
import json, os, re, subprocess, sys, tempfile
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import cv_b200

pairs = int(sys.argv[1]) if len(sys.argv) > 1 else 8
z = np.load(os.path.join(ROOT, "tests", "golden", "bench_pair0.npz"))
a, b = z["ba"], z["bb"]
ctx = cv_b200.Context(0)


def run(seed):
    ars = cv_b200.Arrsac(1e-7, cv_b200.Xoshiro256PlusPlus(seed), ctx=ctx).initialization_hypotheses(8192).max_candidate_hypotheses(1024)
    return ars.model_inliers(cv_b200.EightPoint(), a, b)


for s in range(2):
    run(s)
# the driver reports its counters on stderr under CVB_ARS_DEBUG=1: capture file descriptor 2 around the profiled runs
os.environ["CVB_ARS_DEBUG"] = "1"
err = tempfile.TemporaryFile()
saved = os.dup(2)
os.dup2(err.fileno(), 2)
try:
    ctx.profile(True)
    for s in range(pairs):
        run(s)
    rep = ctx.profile_report()
    ctx.profile(False)
finally:
    os.dup2(saved, 2)
    os.close(saved)
del os.environ["CVB_ARS_DEBUG"]
err.seek(0)
lines = [l for l in err.read().decode().splitlines() if l.startswith("[arrsac]")]
queued = [tuple(int(x) for x in re.search(r"queued: initial (\d+) block (\d+)", l).groups()) for l in lines]
iters = [int(re.search(r"block iterations (\d+)", l).group(1)) for l in lines]
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
ars = {k: v for k, v in rep.items() if k.startswith("k_ars_")}
tot = sum(v["ms"] for v in ars.values())
print(json.dumps({"card": card, "pairs": pairs, "matches": len(a),
                  "arrsac_kernel_ms_per_pair": tot / pairs,
                  "undecided_initial_per_pair": float(np.mean([q[0] for q in queued])) if queued else None,
                  "undecided_block_per_pair": float(np.mean([q[1] for q in queued])) if queued else None,
                  "block_iterations_per_pair": float(np.mean(iters)) if iters else None,
                  "kernels": {k: {"ms_per_pair": v["ms"] / pairs, "launches_per_pair": v["launches"] / pairs, "share_of_arrsac": v["ms"] / tot}
                              for k, v in sorted(ars.items(), key=lambda kv: -kv[1]["ms"])}}, indent=1))
