"""cv-sfm's device constraints (include/cvb200_constraints.h) and reconstruction optimisation (include/cvb200_reconstruction.h) at the
sizes where their launch plans split the work, against the CPU oracles (oracle/ref_constraints.c, oracle/ref_reconstruction.c):

  - cvb_view_constraints_dev over several phase-B sub-chunks (its per-sub-chunk workspace is kept below CON_CHUNK_BYTES = 256 MiB), with
    both optimisers in one call, and over two phase-A chunks; every query also equals the same query run alone;
  - queries wide enough that the block-stride loops of k_con_lists / k_con_select (256 threads) and k_con_order's bitonic sort (1 024
    threads) wrap;
  - k_rec_steps with more edges, and more views, than a grid of every H100 SM at full residency has threads or warps;
  - several optimisation rounds that end KEPT, and a round whose last step removes views.

Each test asserts that its plan was reached: profiler launch counts for the chunks and sub-chunks, the returned statistics for the wide
queries, and sizes for the wraps.  The CPU tests check the scenes' layout and restate the driver's chunk arithmetic (geom.cu,
view_constraints_dev's bytes_a and bytes_b); if CON_CHUNK_BYTES or the workspace layout changes, they show which sizes to update."""
import functools

import numpy as np
import pytest

import cv_b200
from cv_b200.constraints import ConstraintSettings, check_snapshot, generate_view_constraints
from cv_b200.reconstruction import KEPT, OBS_SPLIT, VIEW_NON_FINITE, ReconstructionSettings, check_reconstruction, optimize_reconstruction
from oracle.pyoracle_constraints import ConstraintsCfg, view_constraints
from oracle.pyoracle_reconstruction import ReconCfg
from oracle.pyoracle_reconstruction import optimize_reconstruction as ref_optimize
from oracle.pyoracle_tri import LINEAR_EIGEN, SINE_L1, triangulator
from tests.reconstruction_scenes import args
from tests.scale_scenes import constraints, perturbed, sliding_scene

TRIS = {LINEAR_EIGEN: cv_b200.LinearEigenTriangulator, SINE_L1: cv_b200.SineL1Triangulator}

# ------------------------------------------------------------------------------------------------ the driver's chunk arithmetic
CON_CHUNK_BYTES = 256 << 20
CON_QUERY_BYTES = 19 * 4          # sizeof(ConQuery)
POSE_BYTES = 12 * 8               # sizeof(cvb_pose)
H100_RESIDENT_THREADS = 2048 * 132  # threads per SM x SMs of an H100 SXM, the most any H100 holds resident


def _pow2(x):
    n = 1
    while n < x:
        n <<= 1
    return n


def bytes_a(n_features, V):
    """phase A, per query: its robust list, the three V-sized arrays and its ConQuery"""
    return 4 * (int(n_features) + 3 * V) + CON_QUERY_BYTES


def bytes_b(K, R, V, max_c, opt_max):
    """phase B, per query of K kept coviews and R robust landmarks: bitsets, pair keys, counts and order, visited words, the selection
    sort buffer, and max_c problems of opt_max rows (rows, packed rows, poses in and out, counts, views, offsets, updates, scale)"""
    K, R = int(K), int(R)
    P = K * (K - (K > 0)) // 2
    return (4 * (K * ((R + 31) // 32) + 2 * P + (V + 31) // 32) + 8 * (_pow2(P) + _pow2(R)) +
            max_c * (2 * 8 * 9 * max(opt_max, 1) + 4 * POSE_BYTES + 4 * 6 + 8) + 16 * 256)


def greedy_chunks(sizes):
    """the driver's split: a chunk takes queries while they fit CON_CHUNK_BYTES, and always at least one.  Returns the chunk lengths."""
    out, s0 = [], 0
    while s0 < len(sizes):
        s1, used = s0, 0
        while s1 < len(sizes) and (s1 == s0 or used + sizes[s1] <= CON_CHUNK_BYTES):
            used += sizes[s1]
            s1 += 1
        out.append(s1 - s0)
        s0 = s1
    return out


# ------------------------------------------------------------------------------------------------ scenes
# Phase-B sub-chunks: at optimization_maximum_landmarks = 512 a query needs ~4.77 MB, so 56 fill a sub-chunk; 113 queries give 56, 56
# and 1, and the last sub-chunk's 64 problems run on k_three_view_opt (B <= SMs) while the full ones run on k_three_view_opt_warp.
SUB = dict(V=64, per_view=1500, seed=3, queries=113, opt_max=512)
# Phase-A chunks: 4 096 views, ~45 features a view (3 V words a query dominate), 6 000 queries: a chunk holds ~5 436 of them.
CHUNK_A = dict(V=4096, per_view=60, fov_cos=0.9, seed=5, queries=6000)
# Wide queries: 40 far points seen by all 300 views make every other view a kept coview (K = 299, 44 551 triples).
WIDE = dict(V=300, per_view=400, far=40, seed=4, queries=[150, 0, 299, 150])


@functools.lru_cache(maxsize=None)
def _sub_scene():
    s, _ = sliding_scene(SUB["V"], per_view=SUB["per_view"], seed=SUB["seed"], noise=2e-4, outliers=0.02)
    rng = np.random.default_rng(7)
    V = SUB["V"]
    q = rng.permutation(np.concatenate([np.arange(V), rng.integers(0, V, SUB["queries"] - V)]))   # every view, repeats, shuffled
    return s, q


@functools.lru_cache(maxsize=None)
def _chunk_a_scene():
    s, _ = sliding_scene(CHUNK_A["V"], per_view=CHUNK_A["per_view"], fov_cos=CHUNK_A["fov_cos"], seed=CHUNK_A["seed"], noise=2e-4,
                         outliers=0.02)
    q = np.random.default_rng(9).integers(0, CHUNK_A["V"], CHUNK_A["queries"])
    return s, q


@functools.lru_cache(maxsize=None)
def _wide_scene():
    s, _ = sliding_scene(WIDE["V"], per_view=WIDE["per_view"], far=WIDE["far"], seed=WIDE["seed"], noise=2e-4, outliers=0.02)
    return s, np.asarray(WIDE["queries"])


def _recon(V, per_view, cons_per_view, seed, noise=1e-4, outliers=0.0):
    """a snapshot with its poses perturbed from the truth, and noisy constraints of the true poses"""
    s, true = sliding_scene(V, per_view=per_view, seed=seed, noise=noise, outliers=outliers)
    s["poses"] = perturbed(true, 2e-3, 2e-3, seed + 100)
    return s, constraints(true, per_view=cons_per_view, window=6, noise_rot=1e-4, noise_trans=1e-4, seed=seed)


# Pose graph: (a) 2 000 views with 24 constraints each, 6 C edges above H100_RESIDENT_THREADS; (b) 8 500 views with 3 constraints each,
# one warp per view above H100_RESIDENT_THREADS / 32 warps.  Both need more CTAs of 256 threads than can be resident.
WRAPS = {"edges": dict(V=2000, per_view=20, cons_per_view=24, seed=1), "views": dict(V=8500, per_view=10, cons_per_view=3, seed=2)}


@functools.lru_cache(maxsize=None)
def _wrap_scene(name):
    return _recon(**WRAPS[name])


# ------------------------------------------------------------------------------------------------ CPU: the scenes and the arithmetic
def _views_ascending(s):
    lo, ob = s["landmark_offsets"], s["observations"]
    return all(np.all(np.diff(ob[lo[l]:lo[l + 1], 0].astype(np.int64)) > 0) for l in range(len(lo) - 1))


def test_scenes_pass_the_snapshot_check_and_keep_the_layout():
    for s, q in (_sub_scene(), _chunk_a_scene(), _wide_scene()):
        assert check_snapshot(s["view_offsets"], s["view_landmarks"], s["landmark_offsets"], s["observations"], q) == 0
    for name in WRAPS:
        s, c = _wrap_scene(name)
        assert check_reconstruction(s["view_offsets"], s["view_landmarks"], s["landmark_offsets"], s["observations"], c) == 0
    s, _ = _sub_scene()
    assert _views_ascending(s)
    nl = np.diff(s["landmark_offsets"].astype(np.int64))
    assert (nl == 1).sum() >= 4 * SUB["V"] and nl.max() > 3           # single-observation landmarks and long tracks
    vo, vl = s["view_offsets"], s["view_landmarks"]
    assert not all(np.all(np.diff(vl[vo[v]:vo[v + 1]].astype(np.int64)) > 0) for v in range(SUB["V"]))   # shuffled features


def test_restated_chunk_arithmetic_reaches_three_sub_chunks_and_two_chunks():
    """bytes_b has a floor that does not depend on the query: at opt_max 512 at most 56 queries fit a sub-chunk, so 113 queries take at
    least 3.  The exact split, from the oracle's coviews and robust landmarks (the device's, bit for bit), is 56 + 56 + 1.  Phase A's
    sizes are known on the host: 6 000 queries of the 4 096-view scene take 2 chunks."""
    V, om = SUB["V"], SUB["opt_max"]
    per = CON_CHUNK_BYTES // bytes_b(0, 0, V, 64, om)
    assert per == 56 and -(-SUB["queries"] // per) >= 3
    s, q = _sub_scene()
    o = view_constraints(**s, queries=q, cfg=ConstraintsCfg(optimization_maximum_landmarks=om, constraint_patience=0))
    split = greedy_chunks([bytes_b(k, r, V, 64, om) for k, r in zip(o["stats"]["coviews"], o["stats"]["robust_landmarks"])])
    assert split == [56, 56, 1], split
    s, q = _chunk_a_scene()
    nf = np.diff(s["view_offsets"].astype(np.int64))
    split = greedy_chunks([bytes_a(nf[x], CHUNK_A["V"]) for x in q])
    assert len(split) == 2 and min(split) > 500, split


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def ctx():
    return cv_b200.Context(0)


def _profiled(ctx, fn):
    ctx.profile(True)
    try:
        out = fn()
        rep = ctx.profile_report()
    finally:
        ctx.profile(False)
    return out, rep


def _same_constraints(d, o):
    assert d["results"].tobytes() == o["results"].tobytes()
    assert d["stats"].tobytes() == o["stats"].tobytes()
    assert len(d["constraints"]) == len(o["constraints"])
    for cd, co in zip(d["constraints"], o["constraints"]):
        assert cd.tobytes() == co.tobytes()


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.gpu
@pytest.mark.parametrize("method", [LINEAR_EIGEN, SINE_L1])
def test_constraints_across_phase_b_sub_chunks(ctx, method):
    s, q = _sub_scene()
    kw = dict(optimization_maximum_landmarks=SUB["opt_max"], constraint_patience=0)
    dc = ConstraintSettings(**kw)
    d, rep = _profiled(ctx, lambda: generate_view_constraints(ctx, **s, queries=q, settings=dc, triangulator=TRIS[method](), stats=True))
    o = view_constraints(**s, queries=q, cfg=ConstraintsCfg(**kw), tri=triangulator(method))
    _same_constraints(d, o)
    split = greedy_chunks([bytes_b(k, r, SUB["V"], 64, SUB["opt_max"]) for k, r in zip(d["stats"]["coviews"], d["stats"]["robust_landmarks"])])
    assert len(split) >= 3 and split[-1] * 64 <= _sms() < split[0] * 64, split
    assert rep["k_con_lists"]["launches"] == 1
    assert rep["k_con_triples"]["launches"] == rep["k_con_finish"]["launches"] == len(split)
    assert rep["k_three_view_opt"]["launches"] >= 1 and rep["k_three_view_opt_warp"]["launches"] >= 1
    assert all(r["n_constraints"] == 64 for r in d["results"])
    assert max(c["landmarks"].max() for c in d["constraints"]) > 256          # k_con_select's row loop wraps too
    for i, x in enumerate(q):
        one = generate_view_constraints(ctx, **s, queries=[x], settings=dc, triangulator=TRIS[method](), stats=True)
        assert one["results"].tobytes() == d["results"][i:i + 1].tobytes(), i
        assert one["stats"].tobytes() == d["stats"][i:i + 1].tobytes(), i
        assert one["constraints"][0].tobytes() == d["constraints"][i].tobytes(), i


@pytest.mark.gpu
def test_constraints_across_phase_a_chunks(ctx):
    """The oracle takes well under a second here, so every query is compared with it."""
    s, q = _chunk_a_scene()
    dc = ConstraintSettings(constraint_patience=0)
    d, rep = _profiled(ctx, lambda: generate_view_constraints(ctx, **s, queries=q, settings=dc, stats=True))
    o = view_constraints(**s, queries=q, cfg=ConstraintsCfg(constraint_patience=0))
    _same_constraints(d, o)
    nf = np.diff(s["view_offsets"].astype(np.int64))
    assert rep["k_con_lists"]["launches"] == len(greedy_chunks([bytes_a(nf[x], CHUNK_A["V"]) for x in q])) == 2
    assert sum(r["n_constraints"] for r in d["results"]) > len(q) and d["results"]["accepted"].sum() > 100


@pytest.mark.gpu
def test_wide_queries(ctx):
    s, q = _wide_scene()
    dc = ConstraintSettings(constraint_patience=0)
    d = generate_view_constraints(ctx, **s, queries=q, settings=dc, stats=True)
    st = d["stats"]
    assert np.any((st["coviews"] > 256) & (st["robust_landmarks"] > 256) & (st["triples"] > 1024)), st
    o = view_constraints(**s, queries=q, cfg=ConstraintsCfg(constraint_patience=0))
    _same_constraints(d, o)
    assert all(r["n_constraints"] == 64 for r in d["results"])


def _run_recon(ctx, s, cons, **kw):
    d = optimize_reconstruction(ctx, s["poses"], s["view_offsets"], s["view_landmarks"], s["bearings"], s["landmark_offsets"],
                                s["observations"], cons, settings=ReconstructionSettings(**kw))
    o = ref_optimize(*args(s), cons, cfg=ReconCfg(**kw), tri=triangulator(LINEAR_EIGEN))
    return d, o


def _same_recon(d, o, tol=1e-8):
    """tests/test_gpu_reconstruction.py's contract: statuses, states and counts equal, poses within tol"""
    for f in d["result"].dtype.names:
        assert d["result"][f] == o["result"][f], (f, d["result"], o["result"])
    assert np.array_equal(d["view_state"], o["view_state"])
    assert np.array_equal(d["obs_state"], o["obs_state"])
    fin = np.isfinite(o["poses"])
    assert np.array_equal(fin, np.isfinite(d["poses"]))
    assert np.abs(d["poses"][fin] - o["poses"][fin]).max(initial=0.0) <= tol


@pytest.mark.gpu
@pytest.mark.parametrize("steps", [1, 16])
@pytest.mark.parametrize("name", sorted(WRAPS))
def test_pose_graph_wraps_past_a_resident_grid(ctx, name, steps):
    s, cons = _wrap_scene(name)
    V, E = len(s["view_offsets"]) - 1, 6 * len(cons)
    resident = max(H100_RESIDENT_THREADS, 2048 * _sms())
    if name == "edges":
        assert E > resident                 # the edge loop wraps, and needs more CTAs than can be resident
    else:
        assert V * 32 > resident            # the one-warp-per-view loop wraps, likewise
    d, o = _run_recon(ctx, s, cons, optimization_iterations=steps)
    assert o["result"]["status"] == KEPT and o["result"]["views_removed"] == 0
    _same_recon(d, o)


@pytest.mark.gpu
@pytest.mark.parametrize("rounds", [2, 3])
@pytest.mark.parametrize("V", [64, 256])
def test_rounds_that_stay_kept(ctx, V, rounds):
    """Round 2 on rebuilds the edge CSR from the carried state half, its filter skips what round 1 split, and the split count adds up.
    Bearing noise of 2e-3 puts observations near maximum_cosine_distance, so that the moved poses split more of them in later rounds."""
    s, cons = _recon(V, 150, 8, seed=V, noise=2e-3, outliers=0.02)
    first = ref_optimize(*args(s), cons, cfg=ReconCfg(optimization_iterations=64), tri=triangulator(LINEAR_EIGEN))
    assert first["result"]["observations_split"] > 0
    d, o = _run_recon(ctx, s, cons, optimization_iterations=64, reconstruction_optimization_iterations=rounds)
    assert o["result"]["status"] == KEPT and o["result"]["round"] == rounds
    assert o["result"]["observations_split"] > first["result"]["observations_split"]
    _same_recon(d, o)


@pytest.mark.gpu
def test_round_ending_with_removed_views_then_more_rounds(ctx):
    """One step per round: the views of a constraint with an infinite translation are removed on round 1's last step; rounds 2 and 3
    drop their constraints and observations and run on without the reference's panic"""
    s, cons = _recon(64, 150, 8, seed=11, outliers=0.02)
    bad = int(np.nonzero(cons["views"][:, 0] == 30)[0][0])
    cons["poses"][bad, 1]["t"][0] = np.inf
    d, o = _run_recon(ctx, s, cons, optimization_iterations=1, reconstruction_optimization_iterations=3)
    assert o["result"]["status"] == KEPT and o["result"]["round"] == 3 and o["result"]["views_removed"] >= 3
    assert (o["view_state"] == VIEW_NON_FINITE).sum() >= 3 and (o["obs_state"] == OBS_SPLIT).any()
    _same_recon(d, o)
