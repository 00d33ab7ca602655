"""Seeded degenerate scenes for the minimal solvers and ARRSAC (plain numpy, f64).

What cv-sfm meets in ordinary use: a wall or floor filling the view (planar), a camera turning in place (rotation only), a tiny
baseline, a keypoint detected at two scales (repeated matches), landmarks triangulated from tiny parallax (w ~ 0), and rows that
a broken upstream stage fills with NaN, +-inf or zeros.  Two-view builders return (a, b) unit bearings, PnP builders (bearings,
world) with world in Projective::from_point form; outliers (20-30 % unless stated) are correspondences permuted among themselves,
so an outlier is still a plausible bearing."""
import numpy as np

from tests.geom_util import pnp_scene, rot_from_euler, rot_from_scaled_axis, two_view_scene, unit, world_homog

# the 2D image points and planar world grid of lambda-twist/tests/consensus.rs:68-134 ("endless loop": repeated bearings)
ENDLESS_LOOP_IMAGE = [(0.3070512144698557, 0.19317668016026052), (0.3208462966353674, 0.20741702947913013),
                      (0.3070512144698557, 0.19317668016026052), (0.3208462966353674, 0.20741702947913013),
                      (0.3208462966353674, 0.20741702947913013), (0.3070512144698557, 0.19317668016026052),
                      (0.26619553978146293, 0.15033756455213498), (0.3494806979265859, 0.18264329458710366),
                      (0.32132193890323213, 0.15408143785084824)]
ENDLESS_LOOP_WORLD = [(1.0, 1.0, 0.0), (1.0, 1.5, 0.0), (3.0, 1.0, 0.0), (1.0, 2.0, 0.0), (2.0, 2.0, 0.0), (3.0, 2.0, 0.0),
                      (1.0, 3.0, 0.0), (2.0, 3.0, 0.0), (3.0, 3.0, 0.0)]

POISON_KINDS = ("nan", "+inf", "-inf", "zero", "z0", "zneg")


def _c(*xs):
    return tuple(np.ascontiguousarray(x, np.float64) for x in xs)


def _permute_outliers(rng, x, frac):
    n = len(x)
    bad = rng.choice(n, int(n * frac), replace=False)
    x[bad] = x[rng.permutation(bad)]
    return bad


def _two_view(rng, P, R, t, noise, outlier_frac):
    a, b = unit(P), unit(P @ R.T + t)
    if noise:
        a = unit(a + rng.normal(0, noise, a.shape)); b = unit(b + rng.normal(0, noise, b.shape))
    _permute_outliers(rng, b, outlier_frac)
    return _c(a, b)


def planar(seed, n, noise=0.0, outlier_frac=0.25):
    """all points on the tilted plane z = 5 + 0.3 x: over all rows the eight-point design has a 3-dimensional null space"""
    rng = np.random.default_rng(seed)
    R = rot_from_scaled_axis(rng.uniform(-1, 1, 3) * 0.1); t = unit(rng.uniform(-1, 1, 3))
    x, y = rng.uniform(-2, 2, n), rng.uniform(-2, 2, n)
    return _two_view(rng, np.stack([x, y, 5.0 + 0.3 * x], 1), R, t, noise, outlier_frac)


def rotation_only(seed, n, outlier_frac=0.25):
    """t = 0: every essential of the sample is degenerate, the design again has a 3-dimensional null space"""
    rng = np.random.default_rng(seed)
    R = rot_from_scaled_axis(rng.uniform(-1, 1, 3) * 0.1)
    P = np.stack([rng.uniform(-2, 2, n), rng.uniform(-2, 2, n), rng.uniform(3, 9, n)], 1)
    return _two_view(rng, P, R, np.zeros(3), 0.0, outlier_frac)


def small_baseline(seed, n, baseline=1e-5, noise=0.0, outlier_frac=0.25):
    rng = np.random.default_rng(seed)
    R = rot_from_scaled_axis(rng.uniform(-1, 1, 3) * 0.1); t = baseline * unit(rng.uniform(-1, 1, 3))
    P = np.stack([rng.uniform(-2, 2, n), rng.uniform(-2, 2, n), rng.uniform(3, 9, n)], 1)
    return _two_view(rng, P, R, t, noise, outlier_frac)


def repeated(seed, n, noise=1e-4, outlier_frac=0.25):
    """n rows made of ~n/2.5 correspondences, each present 2 or 3 times, shuffled; returns (a, b, source index of every row)"""
    rng = np.random.default_rng(seed)
    reps = rng.integers(2, 4, n)
    reps = reps[:np.searchsorted(np.cumsum(reps), n) + 1]
    _, _, a, b, _ = two_view_scene(rng, len(reps), outlier_frac=outlier_frac, noise=noise)
    src = rng.permutation(np.repeat(np.arange(len(reps)), reps))[:n]
    return a[src].copy(), b[src].copy(), src


def five_point_cap_samples():
    """600 five-point samples of planar(1, 400, noise=1e-4); two of them give the 40-pose cap of the reference's solver"""
    rng = np.random.default_rng(8)
    return np.array([rng.choice(400, 5, replace=False) for _ in range(600)], np.uint32)


def pnp_planar(seed, n, noise=0.0, outlier_frac=0.25):
    """world points on z = 0"""
    rng = np.random.default_rng(seed)
    R = rot_from_euler(*rng.uniform(-0.3, 0.3, 3)); t = rng.uniform(-0.5, 0.5, 3) + np.array([0.0, 0.0, 8.0])
    W = np.stack([rng.uniform(-3, 3, n), rng.uniform(-3, 3, n), np.zeros(n)], 1)
    bear = unit(W @ R.T + t)
    if noise:
        bear = unit(bear + rng.normal(0, noise, bear.shape))
    _permute_outliers(rng, bear, outlier_frac)
    return _c(bear, world_homog(W))


def pnp_collinear(seed, n, n_line, outlier_frac=0.25):
    """the first n_line landmarks lie on the world line s (1, 1/2, 1/4).  The power-of-two ratios survive Projective::from_point and
    back exactly, so any three of them are collinear to the last bit and inv3 of the P3P frame fails; returns (bearings, world)"""
    rng = np.random.default_rng(seed)
    R, t, bear, world, _ = pnp_scene(rng, n, outlier_frac=outlier_frac, noise=1e-4)
    s = rng.uniform(-3, 3, n_line)
    W = s[:, None] * np.array([1.0, 0.5, 0.25])
    world[:n_line] = world_homog(W)
    bear[:n_line] = unit(W @ R.T + t + np.array([0.0, 0.0, 6.0]))       # in front of the camera; P3P only sees the world side fail
    return _c(bear, world)


def pnp_at_infinity(seed, n, frac=0.1, outlier_frac=0.2):
    """a fraction of the landmarks at w = 0 (half) and w = 1e-300 (half); returns (bearings, world, indices of those rows)"""
    rng = np.random.default_rng(seed)
    _, _, bear, world, _ = pnp_scene(rng, n, outlier_frac=outlier_frac, noise=1e-4)
    k = rng.choice(n, int(n * frac), replace=False)
    world[k[:len(k) // 2], 3] = 0.0
    world[k[len(k) // 2:], 3] = 1e-300
    return bear, world, k


def pnp_duplicated(seed, n, outlier_frac=0.25):
    """every landmark observed two or three times (identical rows), shuffled"""
    rng = np.random.default_rng(seed)
    reps = rng.integers(2, 4, n)
    reps = reps[:np.searchsorted(np.cumsum(reps), n) + 1]
    _, _, bear, world, _ = pnp_scene(rng, len(reps), outlier_frac=outlier_frac, noise=1e-4)
    src = rng.permutation(np.repeat(np.arange(len(reps)), reps))[:n]
    return _c(bear[src], world[src])


def endless_loop():
    """lambda-twist/tests/consensus.rs:68-134: (bearings, world), nine landmarks on z = 0 with repeated bearings"""
    bearings = unit(np.array([[x, y, 1.0] for x, y in ENDLESS_LOOP_IMAGE]))
    return _c(bearings, world_homog(np.array(ENDLESS_LOOP_WORLD)))


def poison(x, rows, kinds=POISON_KINDS):
    """a copy of x with rows[i] replaced by a row of kind kinds[i % len(kinds)]: NaN, +inf or -inf in one component, the zero vector,
    a unit bearing with z = 0, a unit bearing with z < 0 (component 2 is z)"""
    x = np.array(x, np.float64, copy=True)
    for i, r in enumerate(rows):
        kind = kinds[i % len(kinds)]
        if kind == "nan":
            x[r, i % 3] = np.nan
        elif kind == "+inf":
            x[r, i % 3] = np.inf
        elif kind == "-inf":
            x[r, i % 3] = -np.inf
        elif kind == "zero":
            x[r] = 0.0
        elif kind == "z0":
            x[r, :3] = unit(np.array([x[r, 0], x[r, 1], 0.0]) + [1e-3, 0.0, 0.0])
        elif kind == "zneg":
            x[r, 2] = -abs(x[r, 2])
        else:
            raise ValueError(kind)
    return x


def two_view_poisoned(seed, n, n_poison=24, outlier_frac=0.25):
    """a general scene with n_poison rows of a and b poisoned (every kind in both views); returns (a, b, poisoned rows)"""
    rng = np.random.default_rng(seed)
    _, _, a, b, _ = two_view_scene(rng, n, outlier_frac=outlier_frac, noise=1e-4)
    rows = rng.choice(n, n_poison, replace=False)
    half = n_poison // 2
    return poison(a, rows[:half]), poison(b, rows[half:]), rows


def pnp_poisoned(seed, n, n_poison=24, outlier_frac=0.2):
    """a general PnP scene with poisoned bearing rows and NaN / inf world rows; returns (bearings, world, poisoned rows)"""
    rng = np.random.default_rng(seed)
    _, _, bear, world, _ = pnp_scene(rng, n, outlier_frac=outlier_frac, noise=1e-4)
    rows = rng.choice(n, n_poison, replace=False)
    half = n_poison // 2
    return poison(bear, rows[:half]), poison(world, rows[half:], kinds=("nan", "+inf", "-inf", "zero")), rows


def design_matrix(a, b):
    """the eight-point epipolar rows over all matches, with the reference's b / a.z (eight-point/src/lib.rs:16)"""
    ap = a / a[:, 2:3]
    bp = b / a[:, 2:3]
    return (ap[:, :, None] * bp[:, None, :]).reshape(len(a), 9)
