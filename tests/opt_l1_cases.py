"""The problem batches of the L1 optimizer tests, shared by the CPU test of the oracle (tests/test_oracle_optimize_l1.py) and the GPU
test (tests/test_gpu_optimize_l1.py), so that the tolerance the GPU test uses is the one measured on the CPU for the same problems."""
import numpy as np

from tests.geom_util import perturb_pose, pnp_scene, three_view_scene

SINGLE_SIZES = (300, 2048, 1, 0, 37, 1000)      # landmarks per problem; 0 returns the pose untouched
THREE_SIZES = (200, 1024, 3, 0)                 # the sizes of the L2 test (tests/test_gpu_optimize.py)
ITERATIONS = (1, 150, 4000)
EPSILONS = (1e-12, 1e-6)
RATE = 0.1

# The device adds the per-iteration sums in another order than the reference.  Once a run has converged to the noise floor, the
# patience rule (50 iterations without a new best |l1sum|) reacts to that rounding, so the update counts can differ a lot while the
# poses agree.  Measured between the oracle in landmark order and in the device's order over the batches below, at every
# ITERATIONS x EPSILONS (tests/test_oracle_optimize_l1.py::test_device_order_drift_on_the_gpu_batches): at most 92 updates (the
# 37-landmark problem at eps = 1e-12 and 4000 iterations stops after 526 and 618 updates; its poses agree to 1.3e-11), every other
# problem 0; poses agree to 1.4e-11.  The GPU test allows UPDATE_DRIFT updates and POSE_TOL on every pose element.
UPDATE_DRIFT = 128
POSE_TOL = 1e-8


def single_view_batch(seed=0):
    """-> (start poses, bearings[n,3], world[n,4], offsets); every 41st landmark of a problem has w = 0 (a point at infinity, which
    landmark_delta skips)"""
    rng = np.random.default_rng(seed)
    poses, B, W, off = [], [], [], [0]
    for n in SINGLE_SIZES:
        if n:
            R, t, bearings, world, _ = pnp_scene(rng, n, noise=2e-4)
            world = world.copy()
            world[20::41, 3] = 0.0
        else:
            R, t, bearings, world = np.eye(3), np.zeros(3), np.zeros((0, 3)), np.zeros((0, 4))
        poses.append(perturb_pose(rng, (R, t), 2e-3, 5e-3)); B.append(bearings); W.append(world); off.append(off[-1] + n)
    return poses, np.concatenate(B), np.concatenate(W), off


def three_view_batch(seed=1):
    """-> (start pose pairs, [observations[n,3,3] per problem], offsets)"""
    rng = np.random.default_rng(seed)
    starts, obs, off = [], [], [0]
    for n in THREE_SIZES:
        truth, o = three_view_scene(rng, max(n, 1), noise=1e-4)
        starts.append([perturb_pose(rng, p, 3e-3, 5e-3) for p in truth]); obs.append(o[:n]); off.append(off[-1] + n)
    return starts, obs, off
