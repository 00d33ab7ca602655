"""How much of the ARRSAC block loop's scoring early rejection skips, on the bench's frame pair (tests/golden/bench_pair0.npz,
vslam-sandbox configuration: Arrsac(1e-7).initialization_hypotheses(8192).max_candidate_hypotheses(1024) + EightPoint, seed 0).

The device counts the block loop's 32-datum units (CVB_ARS_DEBUG): kept-row units, new-model units, new-model units written 0
instead of scored because the model can no longer beat the bar, and blocks whose new samples were not estimated at all (worst >=
acc_hi: no new model can beat the bar).  One JSON line: those counts (units as predicates, x 32), the skipped share of all
block-scoring predicates, and the block loop kernels' CUDA-event time per call with early rejection on and forced off
(CVB_ARS_EARLY_REJECT=0; the blocks without estimation are the same either way).

    python scripts/prof_block_scoring.py [calls]
"""
import json, os, re, sys, tempfile
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import cv_b200

CALLS = int(sys.argv[1]) if len(sys.argv) > 1 else 5
DEBUG = re.compile(r"block units: kept (\d+) new (\d+) skipped (\d+) \| blocks worst0 \d+ bar<32 \d+ not estimated (\d+)")
z = np.load(os.path.join(ROOT, "tests", "golden", "bench_pair0.npz"))
a, b = z["ba"], z["bb"]


def measure(early):
    """(kept, new, skipped) units of one call, k_ars_score_block ms per call, inlier count"""
    os.environ["CVB_ARS_EARLY_REJECT"] = "1" if early else "0"
    os.environ["CVB_ARS_DEBUG"] = "1"
    ctx = cv_b200.Context(0)
    with tempfile.TemporaryFile("w+") as f:      # the library writes its debug line to fd 2
        sys.stderr.flush()
        saved = os.dup(2)
        os.dup2(f.fileno(), 2)
        try:
            ars = cv_b200.Arrsac(1e-7, cv_b200.Xoshiro256PlusPlus(0), ctx=ctx).initialization_hypotheses(8192).max_candidate_hypotheses(1024)
            r = ars.model_inliers(cv_b200.EightPoint(), a, b)          # warm-up (module load, workspaces)
            ctx.profile(True)
            for _ in range(CALLS):
                ars.rng = cv_b200.Xoshiro256PlusPlus(0)
                ars.model_inliers(cv_b200.EightPoint(), a, b)
            rep = ctx.profile_report()
            ctx.profile(False)
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        f.seek(0)
        units = [tuple(int(x) for x in m) for m in DEBUG.findall(f.read())]
    ctx.close()
    assert len(units) == CALLS + 1 and len({u[:2] + u[3:] for u in units}) == 1, units
    skipped = sum(u[2] for u in units[1:]) / CALLS             # which units are skipped depends on the warps' timing: the mean
    return (units[-1][0], units[-1][1], skipped, units[-1][3]), rep, len(r[2])


(kept, new, skipped, bar0), rep_on, inl_on = measure(True)
(kept0, new0, skipped0, bar00), rep_off, inl_off = measure(False)
assert (kept, new, bar0) == (kept0, new0, bar00) and skipped0 == 0 and inl_on == inl_off
BLOCK = ("k_ars_estimate_block", "k_ars_score_block", "k_ars_resolve_block", "k_ars_book")
print(json.dumps({
    "pair": "tests/golden/bench_pair0.npz", "matches": len(a), "inliers": inl_on, "calls": CALLS,
    "blocks_not_estimated": bar0,
    "kept_row_predicates": 32 * kept, "new_model_predicates": 32 * new, "skipped_predicates": 32 * skipped,
    "skipped_share_of_new": skipped / new if new else 0.0, "skipped_share_of_block_scoring": skipped / (kept + new) if kept + new else 0.0,
    "block_loop_ms_per_call": {k: {"early_rejection": rep_on[k]["ms"] / CALLS if k in rep_on else 0.0,
                                   "forced_off": rep_off[k]["ms"] / CALLS if k in rep_off else 0.0} for k in BLOCK},
    "timing": "CUDA events around each launch (ctx.profile: eager launches, one context, no overlap)"}))
