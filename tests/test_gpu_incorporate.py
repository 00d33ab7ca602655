"""GPU: cv_b200.add_view / apply_optimization / incorporate_frame (include/cvb200_incorporate.h) against the C oracle of the two CSR edits
(oracle/ref_incorporate.c) and the oracle chain of oracle/pyoracle_incorporate.py, and incorporate_frame against the composition of the
existing public calls.

The edits move integers and copy rows, so they are held bit for bit.  The chain's poses come from the registration's and the optimisation's
FP64 arithmetic on the device, which agrees with the oracles to rounding: poses are held to 1e-8 after optimisation steps, and everything
else -- statuses, states, counts, maps, every other array of the snapshot -- must be equal; at optimization_iterations = 0 the poses are
equal too."""
import ctypes as C

import numpy as np
import pytest
import torch

import cv_b200
from cv_b200._lib import CvbError, load_incorporate_library
from cv_b200.incorporate import (add_view_dev, apply_optimization_dev, incorporate_frame_dev, snapshot_to_device, snapshot_to_host)
from oracle import pyoracle as O
from oracle import pyoracle_constraints as OC
from oracle import pyoracle_incorporate as OI
from oracle import pyoracle_reconstruction as OREC
from oracle import pyoracle_register as OR
from oracle.pyoracle_tri import LINEAR_EIGEN, MEAN_MEAN, SINE_L1, triangulator as o_tri

from . import incorporate_scenes as IS
from . import register_scenes as RS

pytestmark = pytest.mark.gpu

TRIS = {LINEAR_EIGEN: cv_b200.LinearEigenTriangulator, SINE_L1: cv_b200.SineL1Triangulator, MEAN_MEAN: cv_b200.MeanMeanTriangulator}
NONPOSE = ("view_offsets", "view_landmarks", "bearings", "descriptors", "colors", "landmark_offsets", "observations")


@pytest.fixture(scope="module")
def ctx():
    return cv_b200.Context(0)


def _pose(s):
    R, t = s["true_pose"]
    return np.concatenate([R.reshape(9), t])


def _new_colors(s):
    return np.random.default_rng(1).integers(0, 256, (len(s["new_bearings"]), 3), dtype=np.uint8)


@pytest.mark.parametrize("V,seed", [(8, 1), (32, 2)])
def test_add_view_and_apply_equal_the_oracle(ctx, V, seed):
    s = RS.scene(V=V, per_view=1500, seed=seed, merges=30, shared_merges=10, doubly=10, step=0.3 if V == 8 else 0.12)
    snap = IS.snapshot(s, seed, IS.chain_constraints(V, seed))
    N = len(s["new_bearings"])
    m = IS.random_matches(snap, N, seed=seed, n_match=N // 2, merges=25)
    assert (m["landmark_b"] != IS.NONE).sum() >= 10
    nc = _new_colors(s)
    got = cv_b200.add_view(ctx, snap, _pose(s), s["new_bearings"], m, s["new_descriptors"], nc)
    want = OI.add_view(snap, _pose(s), s["new_bearings"], m, s["new_descriptors"], nc)
    IS.snap_equal(got, want)
    assert got["landmark_map"].tobytes() == want["landmark_map"].tobytes() and got["merges"] == want["merges"]
    IS.sanity(got)
    for k in range(3):
        vs, os_ = IS.random_states(got, seed=seed + k, removed=1 + k, split=0.05 * k)
        P = got["poses"] + 1e-3 * k
        g = cv_b200.apply_optimization(ctx, got, P, vs, os_)
        w = OI.apply_optimization(got, P, vs, os_)
        IS.snap_equal(g, w)
        assert g["view_map"].tobytes() == w["view_map"].tobytes() and g["landmark_map"].tobytes() == w["landmark_map"].tobytes()
        IS.sanity(g)
    # without descriptors and colours
    bare = dict(snap, descriptors=None, colors=None)
    g = cv_b200.add_view(ctx, bare, _pose(s), s["new_bearings"], m)
    w = OI.add_view(bare, _pose(s), s["new_bearings"], m)
    IS.snap_equal(g, w)


def test_apply_on_the_512_view_scene(ctx):
    """512 views and more than 1.1 M observations (the scene of DESIGN 4m), random states."""
    from .scale_scenes import sliding_scene
    s, _ = sliding_scene(512, per_view=2700, seed=3, noise=1e-4, singles=560)
    snap = dict(s, descriptors=None, colors=None, constraints=IS.chain_constraints(512, 3))
    assert len(snap["observations"]) > 1_100_000
    vs, os_ = IS.random_states(snap, seed=7, removed=9, split=0.02)
    g = cv_b200.apply_optimization(ctx, snap, snap["poses"], vs, os_)
    w = OI.apply_optimization(snap, snap["poses"], vs, os_)
    IS.snap_equal(g, w)
    assert g["view_map"].tobytes() == w["view_map"].tobytes() and g["landmark_map"].tobytes() == w["landmark_map"].tobytes()


# ---- incorporate_frame against the oracle chain -----------------------------------------------------------------------------------------
def _settings(reg=None, con=None, rec=None):
    return (dict(reg or {}), dict(con or {}), dict(rec or {}))


def _run_both(ctx, snap, s, seed=5, method=LINEAR_EIGEN, reg=None, con=None, rec=None, view_matches=None):
    reg, con, rec = _settings(reg, con, rec)
    vm = s["view_matches"] if view_matches is None else view_matches
    nc = _new_colors(s) if snap.get("colors") is not None else None
    ars = cv_b200.Arrsac(1e-5, cv_b200.Xoshiro256PlusPlus(seed), ctx)
    got = cv_b200.incorporate_frame(ctx, snap, s["new_descriptors"], s["new_bearings"], vm, ars, new_colors=nc,
                                    register_settings=cv_b200.RegisterSettings(**reg), constraint_settings=cv_b200.ConstraintSettings(**con),
                                    reconstruction_settings=cv_b200.ReconstructionSettings(**rec), triangulator=TRIS[method]())
    orng = O.rng_xoshiro(seed)
    want = OI.incorporate_frame(snap, s["new_descriptors"], s["new_bearings"], vm, O.arrsac_cfg(1e-5), orng, new_colors=nc,
                                register_cfg=OR.RegisterCfg(**reg), constraints_cfg=OC.ConstraintsCfg(**con), recon_cfg=OREC.ReconCfg(**rec),
                                tri=o_tri(method))
    assert list(ars.rng.state.s) == list(orng.s)
    return got, want


def _assert_chain(got, want, exact_poses=False):
    assert got["status"] == want["status"], (got["status"], want["status"])
    r = got["result"]
    assert OR.STATUS_NAMES[int(r["reg"]["status"])] == want["register"]["status"]
    if want["register"]["status"] == "ok":
        assert np.array_equal(got["matches"], want["register"]["matches"])
    if want["constraints"] is not None:
        wc = want["constraints"]["results"][0]
        assert int(r["con"]["n_constraints"]) == int(wc["n_constraints"]) and int(r["con"]["accepted"]) == int(wc["accepted"])
    if want["recon"] is not None:
        wr = want["recon"]["result"]
        for k in ("status", "round", "step", "views_removed", "robust_before", "robust_after", "observations_split"):
            assert int(r["recon"][k]) == int(wr[k]), k
    assert np.array_equal(got["view_map"], want["view_map"]) and np.array_equal(got["landmark_map"], want["landmark_map"])
    assert got["new_view"] == want["new_view"]
    if want["snapshot"] is None:
        assert got["snapshot"] is None and int(r["counts"]["V"]) == 0
        return
    g, w = got["snapshot"], want["snapshot"]
    IS.snap_equal(g, w, keys=NONPOSE)
    IS.sanity(g)
    assert len(g["constraints"]) == len(w["constraints"])
    assert np.array_equal(g["constraints"]["views"], w["constraints"]["views"])
    assert np.array_equal(g["constraints"]["landmarks"], w["constraints"]["landmarks"])
    if exact_poses:
        assert g["poses"].tobytes() == w["poses"].tobytes()
    else:
        assert np.abs(g["poses"] - w["poses"]).max() < 1e-8
    for x in ("r", "t"):
        assert np.abs(g["constraints"]["poses"][x] - w["constraints"]["poses"][x]).max(initial=0) < 1e-8


def _scene71(**kw):
    s = RS.scene(V=8, per_view=1500, seed=71, outliers=0.1, **kw)
    return IS.snapshot(s, 71), s


def test_kept_equals_the_oracle_chain(ctx):
    snap, s = _scene71()
    got, want = _run_both(ctx, snap, s)
    assert want["status"] == "kept"
    _assert_chain(got, want)
    assert got["new_view"] == 8 and len(got["snapshot"]["constraints"]) > 0


def test_kept_bit_for_bit_without_steps(ctx):
    snap, s = _scene71()
    got, want = _run_both(ctx, snap, s, rec=dict(optimization_iterations=0))
    assert want["status"] == "kept"
    _assert_chain(got, want, exact_poses=True)


def test_kept_with_a_view_in_no_constraint_removed(ctx):
    # two constraints at most cover six of the nine views; the rest have no edges and the optimisation removes them
    snap, s = _scene71()
    got, want = _run_both(ctx, snap, s, con=dict(optimization_maximum_three_view_constraints=2, optimization_minimum_new_constraints=1))
    assert want["status"] == "kept" and int(want["recon"]["result"]["views_removed"]) > 0
    _assert_chain(got, want)
    assert (got["view_map"] == IS.NONE).any()


def test_rejected_keeps_the_merges(ctx):
    s = RS.scene(V=10, per_view=2000, seed=14, merges=40, shared_merges=15, doubly=25, outliers=0.1)
    snap = IS.snapshot(s, 14, IS.chain_constraints(10, 14))
    got, want = _run_both(ctx, snap, s, con=dict(optimization_minimum_new_constraints=1000, optimization_robust_covisibility_minimum_landmarks=10 ** 6))
    assert want["status"] == "rejected"
    _assert_chain(got, want, exact_poses=True)
    assert int(got["result"]["counts"]["L"]) < len(snap["landmark_offsets"]) - 1      # merged pairs stay merged
    assert (got["matches"]["landmark_b"] != IS.NONE).any()


def test_removed_filter(ctx):
    snap, s = _scene71()
    got, want = _run_both(ctx, snap, s, rec=dict(minimum_robust_landmarks=10 ** 7))
    assert want["status"] == "removed_filter"
    _assert_chain(got, want)


@pytest.mark.parametrize("status,kw,scene_kw", [
    ("few_robust_landmarks", dict(single_view_minimum_landmarks=100000), dict()),
    ("few_matches", dict(single_view_minimum_robust_landmarks=100000), dict()),
    ("filter_half", dict(maximum_cosine_distance=1e-14, maximum_sine_distance=1e-14), dict(noise=1e-3)),
    ("final_half", dict(single_view_filter_loop_iterations=1, maximum_cosine_distance=1e-14, maximum_sine_distance=1e-14), dict(noise=1e-3)),
    ("final_robust_half", dict(single_view_filter_loop_iterations=0, maximum_cosine_distance=1e-14, maximum_sine_distance=1e-14),
     dict(noise=1e-3)),
    ("no_consensus", dict(), dict(outliers=1.0)),
])
def test_not_registered_gives_the_input_back(ctx, status, kw, scene_kw):
    s = RS.scene(V=6, per_view=800, seed=41, **scene_kw)
    snap = IS.snapshot(s, 41, IS.chain_constraints(6, 41))
    got, want = _run_both(ctx, snap, s, reg=kw)
    assert want["register"]["status"] == status and want["status"] == "not_registered"
    _assert_chain(got, want, exact_poses=True)
    IS.snap_equal(got["snapshot"], snap)


def test_register_panic(ctx):
    s = RS.scene(V=6, per_view=800, seed=42)
    snap = IS.snapshot(s, 42)
    got, want = _run_both(ctx, snap, s, view_matches=np.array([], np.uint32))
    assert want["status"] == "register_panic"
    _assert_chain(got, want)
    assert (got["view_map"] == IS.NONE).all() and (got["landmark_map"] == IS.NONE).all()


@pytest.mark.parametrize("method", [SINE_L1, MEAN_MEAN])
def test_other_triangulators(ctx, method):
    snap, s = _scene71()
    got, want = _run_both(ctx, snap, s, method=method)
    _assert_chain(got, want)


# ---- against the composition of the existing public calls ------------------------------------------------------------------------------
def _np_add_view(snap, pose, new_bearings, matches):
    """add_view on the numpy CSR in the header's pinned orders"""
    vo, vl, lo, ob = (np.asarray(snap[k]).astype(np.int64) for k in ("view_offsets", "view_landmarks", "landmark_offsets", "observations"))
    ob = ob.reshape(-1, 2)
    V, L, N = len(vo) - 1, len(lo) - 1, len(new_bearings)
    lms = [[tuple(x) for x in ob[lo[l]:lo[l + 1]]] for l in range(L)]
    match = {int(m["feature"]): (int(m["landmark_a"]), int(m["landmark_b"])) for m in matches}
    dead = set()
    for f in range(N):
        if f in match:
            a, b = match[f]
            if b != IS.NONE:
                lms[a] += lms[b]
                dead.add(b)
            lms[a].append((V, f))
    new_of = {}
    for f in range(N):
        if f not in match:
            lms.append([(V, f)])
            new_of[f] = len(lms) - 1
    keep = [l for l in range(len(lms)) if l not in dead]
    idx = {l: i for i, l in enumerate(keep)}
    for f, (a, b) in match.items():
        if b != IS.NONE:
            idx[b] = idx[a]
    lmap = np.array([idx[l] for l in range(L)], np.uint32)
    newv = [idx[match[f][0]] if f in match else idx[new_of[f]] for f in range(N)]
    out_lo = np.concatenate([[0], np.cumsum([len(lms[l]) for l in keep])]).astype(np.uint32)
    out_ob = np.array([o for l in keep for o in lms[l]], np.uint32).reshape(-1, 2)
    return dict(poses=np.concatenate([snap["poses"], np.asarray(pose).reshape(1, 12)]),
                view_offsets=np.append(snap["view_offsets"], int(vo[-1]) + N).astype(np.uint32),
                view_landmarks=np.concatenate([lmap[vl], newv]).astype(np.uint32), bearings=np.concatenate([snap["bearings"], new_bearings]),
                landmark_offsets=out_lo, observations=out_ob, constraints=snap["constraints"])


def _np_replay(snap, poses, vs, os_):
    """optimize_reconstruction's edits on the numpy CSR in the header's pinned orders"""
    vo, vl, lo, ob = (np.asarray(snap[k]).astype(np.int64) for k in ("view_offsets", "view_landmarks", "landmark_offsets", "observations"))
    ob = ob.reshape(-1, 2)
    V, L = len(vo) - 1, len(lo) - 1
    kv = np.where(vs == 0)[0]
    vmap = np.full(V, IS.NONE, np.uint32)
    vmap[kv] = np.arange(len(kv))
    lms, owner = [], {}
    lmap = np.full(L, IS.NONE, np.uint32)
    for l in range(L):
        k = [o for o in range(lo[l], lo[l + 1]) if os_[o] == 0]
        if k:
            lmap[l] = len(lms)
            lms.append(k)
    for o in np.where(os_ == 1)[0]:
        lms.append([o])
    for i, k in enumerate(lms):
        for o in k:
            owner[o] = i
    nvl = []
    for v in kv:
        for f in range(vo[v + 1] - vo[v]):
            o = next(o for o in range(lo[vl[vo[v] + f]], lo[vl[vo[v] + f] + 1]) if ob[o, 0] == v)
            nvl.append(owner[o])
    c = snap["constraints"]
    keepc = np.array([all(vs[w] == 0 for w in x) for x in c["views"]], bool) if len(c) else np.zeros(0, bool)
    nc = c[keepc].copy()
    if len(nc):
        nc["views"] = vmap[nc["views"]]
    rows = np.concatenate([np.arange(vo[v], vo[v + 1]) for v in kv]) if len(kv) else np.zeros(0, np.int64)
    return dict(poses=np.asarray(poses)[kv], view_offsets=np.concatenate([[0], np.cumsum(vo[kv + 1] - vo[kv])]).astype(np.uint32),
                view_landmarks=np.array(nvl, np.uint32), bearings=snap["bearings"][rows],
                landmark_offsets=np.concatenate([[0], np.cumsum([len(k) for k in lms])]).astype(np.uint32),
                observations=np.stack([vmap[ob[[o for k in lms for o in k], 0]], ob[[o for k in lms for o in k], 1]], 1).astype(np.uint32),
                constraints=nc), vmap, lmap


def test_equals_the_composition_of_public_calls(ctx):
    snap, s = _scene71()
    snap = dict(snap, colors=None)
    ars = cv_b200.Arrsac(1e-5, cv_b200.Xoshiro256PlusPlus(9), ctx)
    got = cv_b200.incorporate_frame(ctx, snap, s["new_descriptors"], s["new_bearings"], s["view_matches"], ars)
    assert got["status"] == "kept"
    ars2 = cv_b200.Arrsac(1e-5, cv_b200.Xoshiro256PlusPlus(9), ctx)
    status, pose, matches = cv_b200.register_frame(ctx, *(s[k] for k in RS.SNAP_KEYS), s["new_descriptors"], s["new_bearings"],
                                                   s["view_matches"], ars2)
    assert status == "ok" and np.array_equal(matches, got["matches"])
    a = _np_add_view(snap, np.concatenate([pose[0].reshape(9), pose[1]]), s["new_bearings"], matches)
    keys = ("poses", "view_offsets", "view_landmarks", "bearings", "landmark_offsets", "observations")
    V = len(a["view_offsets"]) - 1
    cons = cv_b200.generate_view_constraints(ctx, *(a[k] for k in keys), [V - 1])
    assert cons["results"][0]["accepted"]
    allc = np.concatenate([snap["constraints"], cons["constraints"][0]])
    a["constraints"] = allc
    out = cv_b200.optimize_reconstruction(ctx, *(a[k] for k in keys), allc)
    e, vmap, lmap = _np_replay(a, out["poses"], out["view_state"], out["obs_state"])
    g = got["snapshot"]
    for k in keys + ("constraints",):
        assert np.ascontiguousarray(g[k]).tobytes() == np.ascontiguousarray(e[k]).tobytes(), k
    assert np.array_equal(got["view_map"], vmap[:V - 1])


# ---- a sequence on device tensors ------------------------------------------------------------------------------------------------------
def test_sequence_on_device_tensors(ctx):
    s0 = RS.scene(V=8, per_view=1500, seed=71, outliers=0.1)
    snap = IS.snapshot(s0, 71)
    sd = snapshot_to_device(snap)
    host = snap
    seed = 20
    for k, nv in enumerate((4.35, 4.6, 4.85)):
        s = RS.scene(V=8, per_view=1500, seed=71, outliers=0.1, new_view=nv)
        V = len(host["view_offsets"]) - 1
        nc = _new_colors(s)
        ars = cv_b200.Arrsac(1e-5, cv_b200.Xoshiro256PlusPlus(seed + k), ctx)
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
        got = incorporate_frame_dev(ctx, sd, dev(s["new_descriptors"]), dev(s["new_bearings"]), np.arange(V, dtype=np.uint32), ars,
                                    new_colors=dev(nc))
        orng = O.rng_xoshiro(seed + k)
        want = OI.incorporate_frame(host, s["new_descriptors"], s["new_bearings"], np.arange(V, dtype=np.uint32), O.arrsac_cfg(1e-5), orng,
                                    new_colors=nc)
        assert list(ars.rng.state.s) == list(orng.s)
        assert got["status"] == want["status"] == "kept", (k, got["status"], want["status"])
        g = snapshot_to_host(got["snapshot"])
        IS.snap_equal(g, want["snapshot"], keys=NONPOSE)
        assert np.abs(g["poses"] - want["snapshot"]["poses"]).max() < 1e-8
        assert np.array_equal(got["landmark_map"].cpu().numpy().view(np.uint32), want["landmark_map"])
        IS.sanity(g)
        # the oracle continues from the device's snapshot so that pose rounding cannot accumulate between the two
        sd, host = got["snapshot"], g
    ex = cv_b200.export_reconstruction(ctx, host["poses"], host["view_offsets"], host["view_landmarks"], host["bearings"],
                                       host["landmark_offsets"], host["observations"], host["colors"])
    assert len(ex["points"]) > 100 and len(ex["cameras"]) == len(host["view_offsets"]) - 1


# ---- other forms -----------------------------------------------------------------------------------------------------------------------
def test_dev_forms_equal_host_forms_and_repeat(ctx):
    s = RS.scene(V=8, per_view=1000, seed=5, merges=20)
    snap = IS.snapshot(s, 5, IS.chain_constraints(8, 5))
    N = len(s["new_bearings"])
    m = IS.random_matches(snap, N, seed=5, merges=10)
    nc = _new_colors(s)
    host = cv_b200.add_view(ctx, snap, _pose(s), s["new_bearings"], m, s["new_descriptors"], nc)
    sd = snapshot_to_device(snap)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    for _ in range(2):
        out, lmap, c = add_view_dev(ctx, sd, dev(_pose(s)), dev(s["new_bearings"]), dev(m.view(np.uint8).reshape(-1, 12)),
                                    dev(s["new_descriptors"]), dev(nc))
        IS.snap_equal(snapshot_to_host(out), host)
        assert np.array_equal(lmap.cpu().numpy().view(np.uint32), host["landmark_map"])
    vs, os_ = IS.random_states(host, seed=3, removed=2, split=0.05)
    h2 = cv_b200.apply_optimization(ctx, host, host["poses"], vs, os_)
    for _ in range(2):
        o2, vmap, lmap2, c2 = apply_optimization_dev(ctx, out, out["poses"], dev(vs), dev(os_))
        IS.snap_equal(snapshot_to_host(o2), h2)
        assert np.array_equal(vmap.cpu().numpy().view(np.uint32), h2["view_map"])
    # the host chain twice from the same generator state gives the same bits
    snap71, s71 = _scene71()
    r = [cv_b200.incorporate_frame(ctx, snap71, s71["new_descriptors"], s71["new_bearings"], s71["view_matches"],
                                   cv_b200.Arrsac(1e-5, cv_b200.Xoshiro256PlusPlus(3), ctx), new_colors=_new_colors(s71)) for _ in range(2)]
    assert r[0]["status"] == r[1]["status"] == "kept"
    IS.snap_equal(r[0]["snapshot"], r[1]["snapshot"])
    assert r[0]["result"].tobytes() == r[1]["result"].tobytes()


def test_argument_errors(ctx):
    s = RS.scene(V=6, per_view=500, seed=8)
    snap = IS.snapshot(s, 8)
    N = len(s["new_bearings"])
    m = np.array([(0, 0, 0)], IS.MATCH_DTYPE)      # a == b
    with pytest.raises(CvbError):
        cv_b200.add_view(ctx, snap, _pose(s), s["new_bearings"], m, s["new_descriptors"], _new_colors(s))
    with pytest.raises(CvbError):                   # colours in the snapshot, none for the new frame
        cv_b200.add_view(ctx, snap, _pose(s), s["new_bearings"], np.zeros(0, IS.MATCH_DTYPE), s["new_descriptors"])
    V, no = len(snap["view_offsets"]) - 1, len(snap["observations"])
    with pytest.raises(CvbError):                   # a kept observation of a removed view
        cv_b200.apply_optimization(ctx, snap, snap["poses"], np.ones(V, np.uint8), np.zeros(no, np.uint8))
    with pytest.raises(CvbError):                   # triangulator method 3 is unsupported
        cv_b200.incorporate_frame(ctx, snap, s["new_descriptors"], s["new_bearings"], s["view_matches"],
                                  cv_b200.Arrsac(1e-5, cv_b200.Xoshiro256PlusPlus(1), ctx), new_colors=_new_colors(s),
                                  triangulator=cv_b200.RelativeDltTriangulator())
    with pytest.raises(ValueError):
        cv_b200.incorporate_frame(ctx, dict(snap, descriptors=None), s["new_descriptors"], s["new_bearings"], s["view_matches"],
                                  cv_b200.Arrsac(1e-5, cv_b200.Xoshiro256PlusPlus(1), ctx))
    sd = snapshot_to_device(snap)
    L = load_incorporate_library()
    rc = L.cvb_add_view_dev(ctx.handle, V, sd["poses"].data_ptr(), sd["view_offsets"].data_ptr(), sd["view_landmarks"].data_ptr(),
                            sd["bearings"].data_ptr(), None, None, int(snap["view_offsets"][-1]) + 1, len(snap["landmark_offsets"]) - 1,
                            sd["landmark_offsets"].data_ptr(), sd["observations"].data_ptr(), no, sd["poses"].data_ptr(),
                            sd["bearings"].data_ptr(), None, None, 1, None, 0, *([sd["poses"].data_ptr()] * 4), None, None,
                            *([sd["poses"].data_ptr()] * 4))
    assert rc == cv_b200._lib.CVB_EINVAL      # n_features disagrees with view_offsets[V]
    assert C.sizeof(C.c_uint32) == 4
