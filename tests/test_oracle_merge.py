"""CPU: the oracle of include/cvb200_merge.h (oracle/pyoracle_merge.py) on split scenes (tests/merge_scenes.py), and the refusals of the
host validator cvb_merge_check."""
import numpy as np
import pytest

from cv_b200.merge import check_merge
from oracle import pyoracle_constraints as OC
from oracle import pyoracle as O
from oracle import pyoracle_merge as OM
from oracle import pyoracle_reconstruction as OREC
from oracle import pyoracle_register as OR

from . import incorporate_scenes as IS
from . import merge_scenes as MS

NONE = MS.NONE


def _wt(sc):
    R, t = sc["iso"]
    return np.concatenate([R.T.reshape(9), -R.T @ t])   # S's world -> D's world


@pytest.fixture(scope="module")
def clean():
    return MS.split(V=12, k=5, seed=3, per_view=800, noise=0.0)


def test_noise_free_split_moves_back(clean):
    sc = clean
    m = OM.incorporate_reconstruction(sc["dest"], sc["src"], _wt(sc), MS.true_landmark_map(sc))
    s = m["snapshot"]
    IS.sanity(s)
    VD = len(sc["dest"]["view_offsets"]) - 1
    assert m["refused"] == 0 and list(m["src_view_map"]) == list(range(VD, VD + 6))
    assert np.abs(s["poses"][VD:] - sc["full"]["poses"][:6]).max() < 1e-9
    # every moved feature joins the D landmark of its original landmark where D observes it, and one created landmark otherwise
    full_vl = np.asarray(sc["full"]["view_landmarks"])
    fo = np.asarray(sc["full"]["view_offsets"])
    so = np.asarray(s["view_offsets"])
    created = {}
    for v in range(6):
        for f in range(fo[v + 1] - fo[v]):
            orig = int(full_vl[fo[v] + f])
            got = int(s["view_landmarks"][so[VD + v] + f])
            if sc["dest_lmap"][orig] != NONE:
                assert got == sc["dest_lmap"][orig]
            else:
                assert created.setdefault(orig, got) == got and got >= len(sc["dest"]["landmark_offsets"]) - 1


def test_source_constraints_are_not_read(clean):
    sc = clean
    a = OM.incorporate_reconstruction(sc["dest"], sc["src"], _wt(sc), MS.true_landmark_map(sc))
    src = dict(sc["src"], constraints=IS.chain_constraints(6, 9))
    b = OM.incorporate_reconstruction(sc["dest"], src, _wt(sc), MS.true_landmark_map(sc))
    IS.snap_equal(a["snapshot"], b["snapshot"])


def test_refuse_every_view(clean):
    sc = clean
    cfg = OC.ConstraintsCfg(optimization_maximum_three_view_constraints=2, optimization_minimum_new_constraints=3)
    m = OM.incorporate_reconstruction(sc["dest"], sc["src"], _wt(sc), MS.true_landmark_map(sc), constraints_cfg=cfg)
    IS.sanity(m["snapshot"])
    assert m["refused"] > 0
    assert (m["src_view_map"] == NONE).sum() == m["refused"]


# 8+8 views at covisibility 380 and 10 new constraints: views 0, 1, 2, 4 and 7 are refused and 3, 5, 6 accepted; removing view 4 lowers
# view 6's constraints from 19 to 15 and turns view 7 from accepted (11) to refused (8), and constraints that views 3 and 5 recorded
# with view 4 or 7 in them are dropped by the removals
REFUSING = dict(optimization_robust_covisibility_minimum_landmarks=380, optimization_minimum_new_constraints=10)


def test_refusals_change_later_views_and_drop_earlier_constraints():
    sc = MS.split(V=16, k=7, seed=3, per_view=800, step=0.3)
    cfg = OC.ConstraintsCfg(**REFUSING)
    lm = MS.true_landmark_map(sc)
    m = OM.incorporate_reconstruction(sc["dest"], sc["src"], _wt(sc), lm, constraints_cfg=cfg)
    IS.sanity(m["snapshot"])
    acc = [bool(r["accepted"]) for r in m["con_results"]]
    assert acc == [False, False, False, True, False, True, True, False]
    # the one call over every moved view (what the device runs first) disagrees with the sequential loop after the first refusal
    s, svm, _ = OM.move(sc["dest"], sc["src"], _wt(sc), lm)
    spec = OC.view_constraints(s["poses"], s["view_offsets"], s["view_landmarks"], s["bearings"], s["landmark_offsets"], s["observations"],
                               list(svm), cfg=cfg)["results"]
    assert [int(r["n_constraints"]) for r in spec[:4]] == [int(r["n_constraints"]) for r in m["con_results"][:4]]
    assert bool(spec[7]["accepted"]) and int(spec[6]["n_constraints"]) != int(m["con_results"][6]["n_constraints"])
    recorded = sum(int(r["n_constraints"]) for r in m["con_results"] if r["accepted"])
    assert len(m["snapshot"]["constraints"]) < recorded       # removals dropped constraints of earlier accepted views
    assert (m["src_view_map"] == NONE).sum() == m["refused"] == 5


def test_merge_moves_the_views_onto_the_known_isometry():
    sc = MS.split(V=12, k=5, seed=3, per_view=800, noise=0.0)
    r = _merge(sc, rec=dict(optimization_iterations=0))
    assert r["status"] == "merged"
    full = np.asarray(sc["full"]["poses"]).reshape(-1, 12)
    for v in range(5):   # the moved views of S, back in D's world
        assert np.abs(r["snapshot"]["poses"][r["src_view_map"][v]] - full[v]).max() < 1e-6, v
    assert np.abs(r["snapshot"]["poses"][r["dest_view"]] - full[5]).max() < 1e-6


def _merge(sc, reg=None, con=None, rec=None):
    return OM.merge_reconstructions(sc["dest"], sc["src"], sc["s_view"], sc["dest_view_matches"], O.arrsac_cfg(1e-5), O.rng_xoshiro(5),
                                    register_cfg=OR.RegisterCfg(**(reg or {})), constraints_cfg=OC.ConstraintsCfg(**(con or {})),
                                    recon_cfg=OREC.ReconCfg(**(rec or {})))


@pytest.mark.parametrize("status,kw", [
    ("merged", {}),
    ("not_registered", dict(reg=dict(single_view_minimum_landmarks=100000))),
    ("rejected", dict(con=dict(optimization_minimum_new_constraints=1000, optimization_robust_covisibility_minimum_landmarks=10 ** 6))),
    ("removed_filter", dict(rec=dict(minimum_robust_landmarks=10 ** 7))),
])
def test_every_status(status, kw):
    sc = MS.split(V=12, k=5, seed=4, per_view=800, garbage=3)
    r = _merge(sc, **kw)
    assert r["status"] == status
    if r["snapshot"] is not None:
        IS.sanity(r["snapshot"])
    if status == "rejected":   # the merges of add_view stay
        L = len(sc["dest"]["landmark_offsets"]) - 1
        assert len(r["snapshot"]["landmark_offsets"]) - 1 == L - int((r["register"]["matches"]["landmark_b"] != NONE).sum())
    if status == "merged":
        assert r["dest_view"] is not None and r["src_view_map"][sc["s_view"]] == r["dest_view"]


def test_check_refusals(clean):
    sc = clean
    d, s = sc["dest"], sc["src"]
    LS, LD = len(s["landmark_offsets"]) - 1, len(d["landmark_offsets"]) - 1
    ok = MS.true_landmark_map(sc)
    assert check_merge(d, s, 5, ok) == 0 and check_merge(d, s, NONE, ok) == 0 and check_merge(d, s, 5) == 0
    assert check_merge(d, s, 6, ok) != 0                       # s_view / skip_view >= V_S
    assert check_merge(d, s, NONE) != 0                        # no s_view
    bad = ok.copy(); bad[0] = LD
    assert check_merge(d, s, 5, bad) != 0                      # an entry >= L_D
    dup = np.full(LS, NONE, np.uint32); dup[:2] = 0
    assert check_merge(d, s, 5, dup) != 0                      # not injective
    assert check_merge(d, dict(s, colors=None), 5, ok) != 0    # colours on one side only
    broken = dict(s, view_landmarks=np.asarray(s["view_landmarks"]).copy())
    broken["view_landmarks"][0] = LS
    assert check_merge(d, broken, 5, ok) != 0                  # a malformed snapshot
