"""Seeded inputs shared by the cv-pinhole tests (tests/test_oracle_pinhole.py on the CPU, tests/test_gpu_pinhole.py on the GPU)."""
import numpy as np

from tests.geom_util import rot_from_euler, rot_from_scaled_axis, skew, unit


def reprojection_batch(rng, n=12000):
    """n (CameraToCamera pose, a, b) triples; the kinds i % 10 cover a point behind A and behind B, +0.0 and -0.0 z, zero baseline
    (w = 0), parallel bearings, NaN and zero bearings.  -> (Rs[n, 3, 3], ts[n, 3], a[n, 3], b[n, 3])"""
    Rs, ts, As, Bs = [], [], [], []
    for i in range(n):
        kind = i % 10
        X = rng.uniform([-3, -3, 2], [3, 3, 12])
        R = rot_from_scaled_axis(rng.normal(0, 0.2, 3))
        t = np.zeros(3) if kind == 1 else rng.normal(0, 1.0, 3)        # kind 1: zero baseline
        if kind == 2:
            X[2] = -X[2]                                                 # behind A, in front along a
        if kind == 3:
            X = R.T @ (np.array([X[0], X[1], -X[2]]) - t)                # behind B
        a = unit(X + rng.normal(0, 1e-3, 3)); b = unit(R @ X + t + rng.normal(0, 1e-3, 3))
        if kind == 4:
            b = R @ a                                                    # parallel bearings
        if kind == 5:
            (a if i % 20 == 5 else b)[:] = np.nan
        if kind == 6:
            (a if i % 20 == 6 else b)[:] = 0.0
        if kind == 7:
            (a if i % 20 == 7 else b)[2] = 0.0                           # +0.0 z
        if kind == 8:
            (a if i % 20 == 8 else b)[2] = -0.0                          # -0.0 z
        Rs.append(R); ts.append(t); As.append(a); Bs.append(b)
    return np.array(Rs), np.array(ts), np.array(As), np.array(Bs)


def essential_batch(rng, m=4096):
    """m 3x3 matrices: [t]x R of random poses, the same with noise, exactly rank-one and zero matrices (no decomposition), scaled and
    random ones"""
    Es = []
    for j in range(m):
        kind = j % 8
        R = rot_from_scaled_axis(rng.normal(0, 0.5, 3)); t = rng.normal(0, 1.0, 3)
        E = skew(t) @ R
        if kind == 1:
            E = E + rng.normal(0, 1e-3, (3, 3))
        if kind == 2:
            E = np.zeros((3, 3)); E[:, j % 3] = rng.normal(size=3)       # exactly rank one: s1 = 0
        if kind == 3:
            E = np.zeros((3, 3))
        if kind == 4:
            E = E * 10.0 ** rng.uniform(-6, 6)
        if kind == 5:
            E = rng.normal(size=(3, 3))
        Es.append(E)
    return np.array(Es)


def random_rs_scene(rng):
    """eight-point/tests/random.rs:14-36: a random pose and 16 points with Vector3::new_random() (uniform [0, 1) per component)"""
    R = rot_from_scaled_axis(rng.random(3) * np.pi * 2.0 * 0.2)
    t = rng.random(3)
    A = rng.random((16, 3)) * 2.0
    A[:, 0] -= 1.0; A[:, 1] -= 1.0; A[:, 2] += 3.0
    return unit(A), unit(A @ R.T + t)


DOC_POSE = (rot_from_euler(0.2, 0.3, 0.4), np.array([-0.8, 0.4, 0.5]))     # essential.rs:96-99, 171-174, 200-203
