"""CPU-only: properties of the oracle of include/cvb200_reconstruction.h (oracle/ref_reconstruction.c) on the synthetic reconstructions and
edge cases of tests/reconstruction_scenes.py: the fixed point, convergence in relative pose, both exp branches at |delta|^2 either side of
f64::EPSILON, removal without edges, the apply_constraints removal, the panic stop, the filter's keep-first and keep-last splits, the
two-observation sine test at its threshold, dropped observations, acceptance at minimum_robust_landmarks, two rounds, C = 0 and V < 3."""
import ctypes as C

import numpy as np

from oracle import pyoracle_reconstruction as R
from oracle.pyoracle_reconstruction import ReconCfg, optimize_reconstruction
from tests.reconstruction_scenes import CASES, args, inv, mul, py_pose_inverse, py_pose_mul, recon_scene


def _run(name, **over):
    s, cons, kw = CASES[name]()
    kw.update(over)
    return s, cons, optimize_reconstruction(*args(s), cons, cfg=ReconCfg(**kw))


def test_exact_constraints_are_a_fixed_point():
    s, _, o = _run("fixed_point")
    assert o["result"]["status"] == 0 and o["result"]["step"] == 0
    assert np.abs(o["poses"] - s["poses"]).max() <= 1e-12


def test_perturbed_poses_converge_in_relative_pose():
    s, true, cons = recon_scene(12, points=200, noise=0.0, per_view=6, window=4, noise_rot=0.0, noise_trans=0.0)
    o = optimize_reconstruction(*args(s), cons, cfg=ReconCfg(minimum_robust_landmarks=0))
    rel = (lambda P, a, b: mul(P[b], inv(P[a])))
    before = max(np.abs(rel(s["poses"], a, a + 1) - rel(true, a, a + 1)).max() for a in range(11))
    after = max(np.abs(rel(o["poses"], a, a + 1) - rel(true, a, a + 1)).max() for a in range(11))
    assert after < 1e-3 * before


def test_both_exp_branches_either_side_of_epsilon():
    _, _, below = _run("exp_below")
    _, _, above = _run("exp_above")
    assert below["result"]["small_angle_updates"] == above["result"]["small_angle_updates"] + 1
    assert np.abs(below["poses"] - above["poses"]).max() < 1e-12


def test_a_view_without_edges_is_removed_and_the_others_go_on():
    s, _, o = _run("no_edges")
    assert list(o["view_state"]) == [0, 0, 0, 1] and o["result"]["status"] == 0 and o["result"]["views_removed"] == 1
    vo, ob = s["view_offsets"], s["observations"]
    assert np.array_equal(o["obs_state"] == 2, ob[:, 0] == 3)     # the removed view's observations are dropped
    assert np.abs(o["poses"] - s["poses"]).max() <= 1e-12 and np.array_equal(o["poses"][3], s["poses"][3])


def test_two_updated_views_remove_the_reconstruction():
    s, _, o = _run("two_updated")
    r = o["result"]
    assert (r["status"], r["round"], r["step"]) == (1, 0, 0)
    assert not o["view_state"].any() and np.array_equal(o["poses"], s["poses"])   # the failing step is not applied


def test_infinite_constraint_translation_panics_when_steps_remain():
    _, _, o = _run("panic")
    r = o["result"]
    assert (r["status"], r["round"], r["step"]) == (3, 0, 1)
    assert list(o["view_state"]) == [0, 0, 2, 2, 2, 0]


def test_infinite_constraint_translation_removes_views_on_the_last_step():
    s, _, o = _run("panic_on_last_step")
    assert o["result"]["status"] == 0 and list(o["view_state"]) == [0, 0, 2, 2, 2, 0]
    assert np.array_equal(o["obs_state"] == 2, np.isin(s["observations"][:, 0], [2, 3, 4]))


def test_second_round_drops_the_constraints_of_removed_views():
    # had the second round kept the constraint (0, 1, 2), views 0 and 1 would reach the removed view 2 and panic
    _, _, two = _run("two_rounds")
    assert two["result"]["status"] == 0 and two["result"]["round"] == 2 and list(two["view_state"]) == [0, 0, 2, 2, 2, 0]


def test_untriangulable_landmark_keeps_its_first_observation():
    s, _, o = _run("negated_landmark")
    l = s["negated"]
    lo = s["landmark_offsets"]
    st = o["obs_state"][lo[l]:lo[l + 1]]
    assert st[0] == 0 and (st[1:] == 1).all()


def test_all_inconsistent_observations_keep_the_last():
    s, _, o = _run("all_inconsistent")
    lo = s["landmark_offsets"]
    n = 0
    for l in range(len(lo) - 1):
        st = o["obs_state"][lo[l]:lo[l + 1]]
        if len(st) >= 3:
            assert list(st) == [1] * (len(st) - 1) + [0]
            n += 1
    assert n > 0 and o["result"]["robust_after"] == 0


def test_two_observation_sine_test_at_its_threshold():
    s, _, cons = recon_scene(16, seed=3)
    P = s["poses"]
    lo, ob, vo, B = s["landmark_offsets"], s["observations"], s["view_offsets"], s["bearings"]
    l = next(i for i in range(len(lo) - 1) if lo[i + 1] - lo[i] == 2)
    (v0, f0), (v1, f1) = ob[lo[l]], ob[lo[l] + 1]
    tot = py_pose_mul([float(x) for x in P[v1]], py_pose_inverse([float(x) for x in P[v0]]))
    a = [float(x) for x in B[vo[v0] + f0]]
    fb = [tot[3 * r] * a[0] + tot[3 * r + 1] * a[1] + tot[3 * r + 2] * a[2] for r in range(3)]
    d = (C.c_double * 3)
    lib = R._lib()
    lib.ref_epipolar_loss.argtypes = [C.c_void_p] * 3
    lib.ref_epipolar_loss.restype = C.c_double
    loss = lib.ref_epipolar_loss(d(*tot[9:]), d(*fb), d(*[float(x) for x in B[vo[v1] + f1]]))
    at = optimize_reconstruction(*args(s), cons, cfg=ReconCfg(optimization_iterations=0, maximum_sine_distance=loss))
    above = optimize_reconstruction(*args(s), cons, cfg=ReconCfg(optimization_iterations=0, maximum_sine_distance=np.nextafter(loss, 1.0)))
    assert list(at["obs_state"][lo[l]:lo[l + 1]]) == [0, 1]     # not below the threshold: split_landmark keeps the first
    assert list(above["obs_state"][lo[l]:lo[l + 1]]) == [0, 0]


def test_acceptance_at_minimum_robust_landmarks():
    s, _, cons = recon_scene(16, seed=3)
    n = optimize_reconstruction(*args(s), cons, cfg=ReconCfg(optimization_iterations=0, minimum_robust_landmarks=0))["result"]["robust_after"]
    assert n > 0
    at = optimize_reconstruction(*args(s), cons, cfg=ReconCfg(optimization_iterations=0, minimum_robust_landmarks=n))["result"]
    below = optimize_reconstruction(*args(s), cons, cfg=ReconCfg(optimization_iterations=0, minimum_robust_landmarks=n + 1))["result"]
    assert at["status"] == 0 and (below["status"], below["round"], below["step"]) == (2, 0, 0)


def test_no_constraints_and_fewer_than_three_views():
    for name in ("empty", "two_views"):
        s, _, o = _run(name)
        assert (o["result"]["status"], o["result"]["step"]) == (1, 0) and not o["view_state"].any(), name
        assert np.array_equal(o["poses"], s["poses"])
    for name in ("empty_filter_only", "two_views_filter_only"):
        _, _, o = _run(name)
        assert o["result"]["status"] == 0 and o["result"]["robust_after"] > 0, name
