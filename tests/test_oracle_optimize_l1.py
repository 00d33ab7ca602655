"""CPU checks of the oracle of cv-optimize's L1 (Weiszfeld) optimizers (oracle/ref_optimize_l1.c): the properties the algorithms must
have, the reference's quirks against a numpy transcription of the two functions, and the drift between the reference's summation
order and the device's, which sets the tolerance of tests/test_gpu_optimize_l1.py."""
import numpy as np

from oracle import pyoracle as O
from oracle import pyoracle_opt as P
from tests import opt_l1_cases as K
from tests.geom_util import perturb_pose, pnp_scene, rot_angle, rot_from_scaled_axis, three_view_scene, unit


def _mean_residual(pose, bearings, world):
    return np.mean([O.residual_w2c(pose[0], pose[1], bearings[i], world[i]) for i in range(len(bearings))])


def _max_diff(a, b):
    return max(np.abs(np.asarray(x) - np.asarray(y)).max() for x, y in zip(a, b))


def test_exact_pose_is_a_fixed_point():
    # At a zero-residual pose the gradients are rounding noise, so their normalised directions are arbitrary, but the Weiszfeld
    # weights bound the step: |delta.t| <= rate * tscale * eps and |delta.r| <= rate * eps per iteration.  rate * eps * iterations
    # stays below 1e-10 here for both epsilons.
    rng = np.random.default_rng(10)
    R, t, bearings, world, _ = pnp_scene(rng, 300)
    truth, obs = three_view_scene(rng, 200)
    for eps in (1e-12, 1e-6):
        Re, te, upd = P.single_view_optimize_l1((R, t), eps, 1e-4, 10, bearings, world)
        assert upd == 10 and _max_diff((Re, te), (R, t)) < 1e-10, eps
        out, upd = P.three_view_optimize_l1(truth, eps, 1e-4, 10, obs)
        assert upd == 10 and max(_max_diff(out[v], truth[v]) for v in range(2)) < 1e-10, eps


def test_perturbed_start_improves():
    rng = np.random.default_rng(11)
    R, t, bearings, world, _ = pnp_scene(rng, 300, noise=2e-4)
    start = perturb_pose(rng, (R, t), 2e-3, 5e-3)
    r0 = _mean_residual(start, bearings, world)
    for eps in (1e-12, 1e-6):
        Rr, tr, _ = P.single_view_optimize_l1(start, eps, 0.1, 300, bearings, world)
        assert _mean_residual((Rr, tr), bearings, world) < 0.2 * r0, eps
    # three view: the epipolar gradients move the rotations; the translation directions barely move (as with the L2 optimizer)
    truth, obs = three_view_scene(rng, 200, noise=1e-4)
    start3 = [perturb_pose(rng, p, 3e-3, 0.0) for p in truth]
    err = lambda poses: sum(rot_angle(p[0], q[0]) for p, q in zip(poses, truth))   # noqa: E731
    out, _ = P.three_view_optimize_l1(start3, 1e-12, 0.1, 3000, obs)
    assert err(out) < err(start3), (err(out), err(start3))


def test_iteration_cap_and_patience():
    rng = np.random.default_rng(12)
    R, t, bearings, world, _ = pnp_scene(rng, 300, noise=2e-4)
    start = perturb_pose(rng, (R, t), 2e-3, 5e-3)
    assert P.single_view_optimize_l1(start, 1e-12, 0.1, 200, bearings, world)[2] == 200         # the cap (:71-75)
    upd = P.single_view_optimize_l1(start, 1e-12, 1.0, 100000, bearings, world)[2]
    assert 200 < upd < 100000                                                                    # patience: 50 without a new best
    Rz, tz, uz = P.single_view_optimize_l1(start, 1e-12, 0.1, 0, bearings, world)                # no iterations: untouched
    assert uz == 0 and np.array_equal(Rz, start[0]) and np.array_equal(tz, start[1])
    truth, obs = three_view_scene(rng, 200, noise=1e-4)
    start3 = [perturb_pose(rng, p, 3e-3, 5e-3) for p in truth]
    assert P.three_view_optimize_l1(start3, 1e-12, 0.1, 100, obs)[1] == 100
    upd3 = P.three_view_optimize_l1(start3, 1e-12, 1.0, 100000, obs)[1]
    assert 100 < upd3 < 100000


def test_empty_input_returns_the_pose_bit_for_bit():
    rng = np.random.default_rng(13)
    pose = perturb_pose(rng, (rot_from_scaled_axis([0.1, -0.2, 0.3]), np.array([0.3, -0.1, 0.7])), 1e-2, 1e-2)
    R, t, upd = P.single_view_optimize_l1(pose, 1e-12, 0.1, 100, np.zeros((0, 3)), np.zeros((0, 4)))
    assert upd == 0 and R.tobytes() == pose[0].tobytes() and t.tobytes() == pose[1].tobytes()
    poses = [pose, perturb_pose(rng, pose, 1e-2, 1e-2)]
    out, upd = P.three_view_optimize_l1(poses, 1e-12, 0.1, 100, np.zeros((0, 3, 3)))
    assert upd == 0 and all(out[v][k].tobytes() == poses[v][k].tobytes() for v in range(2) for k in range(2))   # no double inversion


# ---- numpy transcription of single_view_optimizer.rs:16-78 and three_view_optimizer.rs:23-124 (cv-core so3.rs for the tangents)
def _tangent_new(v):
    return np.zeros(3) if np.isnan(v).any() else v


def _normalize(v):
    with np.errstate(invalid="ignore", divide="ignore"):
        return v / np.sqrt(v @ v)


def _isometry_mul(dt, dr, R, t):
    Rd = rot_from_scaled_axis(dr)
    return Rd @ R, Rd @ dt + Rd @ t


def _weiszfeld_delta(terms, tscale, eps, rate, count_zero_weights=True):
    l1t, l1r, ts, rs = np.zeros(3), np.zeros(3), 0.0, 0.0
    with np.errstate(divide="ignore"):
        for tg, rg in terms:
            if count_zero_weights or (tg @ tg > 0 and rg @ rg > 0):
                ts += 1.0 / (np.sqrt(tg @ tg) + tscale * eps)
                rs += 1.0 / (np.sqrt(rg @ rg) + eps)
            l1t = l1t + _tangent_new(_normalize(tg)); l1r = l1r + _tangent_new(_normalize(rg))
        return l1t * rate * (1.0 / ts), l1r * rate * (1.0 / rs), np.sqrt(l1t @ l1t), np.sqrt(l1r @ l1r)


def _np_single_view_l1(pose, eps, rate, iterations, bearings, world, count_zero_weights=True):
    R, t = np.array(pose[0]), np.array(pose[1])
    if len(bearings) == 0:
        return R, t, 0
    best, stall, upd = [np.inf, np.inf], 0, 0
    for it in range(iterations):
        terms = []
        for b, w in zip(bearings, world):
            q = np.append(R @ w[:3] + t * w[3], w[3])
            if np.signbit(q[3]):
                q = -q
            q = q / np.sqrt(q[:3] @ q[:3])
            if q[3] == 0.0:                                   # landmark_delta: None
                continue
            p = q[:3] / q[3]
            terms.append((_tangent_new((p @ b) * b - p), _tangent_new(np.cross(_normalize(p), b))))
        dt, dr, nt, nr = _weiszfeld_delta(terms, np.sqrt(t @ t), eps, rate, count_zero_weights)
        stall += 1
        for k, v in enumerate((nt, nr)):
            if best[k] > v:
                best[k], stall = v, 0
        if stall >= 50:
            break
        R, t = _isometry_mul(dt, dr, R, t); upd += 1
    return R, t, upd


def _np_three_view_l1(poses, eps, rate, iterations, obs):
    if len(obs) == 0:
        return [tuple(p) for p in poses], 0
    P_ = [(p[0].T, -p[0].T @ p[1]) for p in poses]
    best, stall, upd = [[np.inf, np.inf], [np.inf, np.inf]], 0, 0
    for it in range(iterations):
        tscale = np.sqrt(P_[0][1] @ P_[0][1]) + np.sqrt(P_[1][1] @ P_[1][1])
        terms = [[], []]
        for o in obs:
            g = O.three_view_gradients(o[0], P_[0][0] @ o[1], P_[0][1], P_[1][0] @ o[2], P_[1][1])
            terms[0].append((g[0:3], g[3:6])); terms[1].append((g[6:9], g[9:12]))
        deltas = [_weiszfeld_delta(terms[v], tscale, eps, rate) for v in range(2)]
        stall += 1
        for v in range(2):
            for k in range(2):
                if best[v][k] > deltas[v][2 + k]:
                    best[v][k], stall = deltas[v][2 + k], 0
        if stall >= 50:
            break
        P_ = [_isometry_mul(deltas[v][0], deltas[v][1], *P_[v]) for v in range(2)]; upd += 1
    return [(p[0].T, -p[0].T @ p[1]) for p in P_], upd


def _quirk_scene(rng, n=6):
    """pose (I, (0.5, 0, 0)) and n noisy landmarks, plus one landmark whose camera point (0, 0, 2) lies exactly on its bearing (an
    exactly zero gradient) and one world point at infinity (w = 0, skipped)"""
    pose = (np.eye(3), np.array([0.5, 0.0, 0.0]))
    C = np.stack([rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), rng.uniform(2, 5, n)], 1)
    bearings = unit(C + rng.normal(0, 2e-2, C.shape))
    world = np.concatenate([C - pose[1], np.ones((n, 1))], 1)
    bearings = np.concatenate([bearings, [[0.0, 0.0, 1.0], unit([0.2, 0.1, 1.0])]])
    world = np.concatenate([world, [[-0.5, 0.0, 2.0, 1.0], [1.0, 0.5, 3.0, 0.0]]])
    return pose, bearings, world


def test_single_view_quirks_match_a_numpy_transcription():
    rng = np.random.default_rng(14)
    pose, bearings, world = _quirk_scene(rng)
    for eps in (1e-3, 1e-6):
        for iters in (1, 5, 60):
            Rw, tw, uw = _np_single_view_l1(pose, eps, 0.5, iters, bearings, world)
            Ro, to, uo = P.single_view_optimize_l1(pose, eps, 0.5, iters, bearings, world)
            assert uo == uw and _max_diff((Ro, to), (Rw, tw)) < 1e-12, (eps, iters)
    # the w = 0 landmark adds nothing: dropping it changes no bit
    Rd, td, _ = P.single_view_optimize_l1(pose, 1e-3, 0.5, 5, bearings[:-1], world[:-1])
    Ro, to, _ = P.single_view_optimize_l1(pose, 1e-3, 0.5, 5, bearings, world)
    assert Rd.tobytes() == Ro.tobytes() and td.tobytes() == to.tobytes()
    # the zero-gradient landmark adds 1/(tscale eps) and 1/eps to the weights although its l1 term is zero
    Rn, tn, _ = _np_single_view_l1(pose, 1e-3, 0.5, 1, bearings, world, count_zero_weights=False)
    Ro, to, _ = P.single_view_optimize_l1(pose, 1e-3, 0.5, 1, bearings, world)
    assert _max_diff((Ro, to), (Rn, tn)) > 1e-6


def test_three_view_quirks_match_a_numpy_transcription():
    rng = np.random.default_rng(15)
    truth, obs = three_view_scene(rng, 8, noise=1e-2)
    obs = np.concatenate([obs, np.zeros((1, 3, 3))])       # zero bearings: both gradients are NaN, zeroed, and still weighted
    start = [perturb_pose(rng, p, 3e-3, 5e-3) for p in truth]
    for eps in (1e-3, 1e-6):
        for iters in (1, 5, 60):
            want, uw = _np_three_view_l1(start, eps, 0.5, iters, obs)
            got, uo = P.three_view_optimize_l1(start, eps, 0.5, iters, obs)
            assert uo == uw and max(_max_diff(got[v], want[v]) for v in range(2)) < 1e-12, (eps, iters)


def test_device_order_drift_on_the_gpu_batches():
    """The oracle in landmark order against the oracle in the device's order on the GPU test's batches: the pose agreement and the
    update-count drift that tests/opt_l1_cases.py records and the GPU test allows."""
    drift, pose_diff = 0, 0.0
    poses, B, W, off = K.single_view_batch()
    for eps in K.EPSILONS:
        for iters in K.ITERATIONS:
            for k in range(len(poses)):
                s = slice(off[k], off[k + 1])
                a = P.single_view_optimize_l1(poses[k], eps, K.RATE, iters, B[s], W[s], P.LANDMARK_ORDER)
                b = P.single_view_optimize_l1(poses[k], eps, K.RATE, iters, B[s], W[s], P.DEVICE_ORDER)
                drift = max(drift, abs(a[2] - b[2])); pose_diff = max(pose_diff, _max_diff(a[:2], b[:2]))
    starts, obs, off = K.three_view_batch()
    for eps in K.EPSILONS:
        for iters in K.ITERATIONS:
            for k in range(len(starts)):
                a, ua = P.three_view_optimize_l1(starts[k], eps, K.RATE, iters, obs[k], P.LANDMARK_ORDER)
                b, ub = P.three_view_optimize_l1(starts[k], eps, K.RATE, iters, obs[k], P.DEVICE_ORDER)
                drift = max(drift, abs(ua - ub)); pose_diff = max(pose_diff, max(_max_diff(a[v], b[v]) for v in range(2)))
    print(f"landmark order vs device order: update drift {drift}, pose difference {pose_diff:.3g}")
    assert drift <= K.UPDATE_DRIFT and pose_diff < 1e-2 * K.POSE_TOL


def test_report_l1_against_l2_with_gross_outliers():
    """A measurement, not a property: L1 and L2 from the same start on a scene with 10 % gross outlier landmarks."""
    rng = np.random.default_rng(16)
    R, t, bearings, world, good = pnp_scene(rng, 500, outlier_frac=0.1, noise=2e-4)
    start = perturb_pose(rng, (R, t), 2e-3, 5e-3)
    rows = [("start", start)]
    Rl, tl, _ = P.single_view_optimize_l1(start, 1e-12, 1.0, 2000, bearings, world)
    rows.append(("l1 rate 1.0", (Rl, tl)))
    Rq, tq, _ = O.single_view_optimize_l2(start, 1e-3, 20000, bearings, world)
    rows.append(("l2 rate 1e-3", (Rq, tq)))
    for name, p in rows:
        print(f"{name}: rotation error {rot_angle(p[0], R):.3g} rad, translation error {np.linalg.norm(p[1] - t):.3g}, "
              f"inlier residual {_mean_residual(p, bearings[good], world[good]):.3g}")
    assert all(np.isfinite(p[0]).all() and np.isfinite(p[1]).all() for _, p in rows)
