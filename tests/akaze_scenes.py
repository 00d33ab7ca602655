"""Seeded frames that take AKAZE's keypoint stages (cv_b200/csrc/akaze.cu, stage_detect and stage_sort_describe) past their first plan,
for tests/test_gpu_akaze_dense.py.  tests/test_akaze_scenes.py checks, with the CPU oracle, that each frame lands on the intended side of
every limit below.

Each builder returns (image, config) where config holds the Akaze arguments the scene was designed for.  The counts in the docstrings
are the oracle's (oracle/ref_akaze.c): `candidates` is every 3x3 maximum above the threshold, `pair` the most candidates in two adjacent
classes (what k_suppress_smem keeps in its ring), `extrema` the keypoints left after duplicate suppression and the upper-scale filter (a
lower bound on the suppression's cache), `final` the keypoints with descriptors."""
import numpy as np

from tests.synth import synth_frame


def dense():
    """synth_frame(0) (1920x1080) at threshold 1e-4, no feature cap: 44 768 candidates, pair 13 700 (above the 8 192-entry ring, so
    the suppression falls back to k_suppress_par), 19 415 extrema (above 64 chunks of 256, so the chunk loops of k_filter_upper,
    k_rank_count and k_rank_scatter wrap).  Within the default capacities of a 1080p frame."""
    return synth_frame(0), dict(detector_threshold=1e-4, maximum_features=-1)


def _tile():
    # a 64x64 period is a multiple of 2^o for every octave o < 4, so every copy of the tile gives bit-identical responses
    return synth_frame(3, h=64, w=64, nblobs=12)


def tied():
    """A 64x64 tile repeated 17x30 and cut to 1920x1080, at 0.001: 13 340 keypoints with 34 distinct responses.  Pair 9 866, so the
    ties go through the suppression's fallback."""
    return np.ascontiguousarray(np.tile(_tile(), (17, 30))[:1080]), dict(detector_threshold=0.001, maximum_features=-1)


def tied_small():
    """The same tile repeated 8x10 (640x512), at 0.001: 1 569 keypoints with 35 distinct responses, pair 1 492: the ring path."""
    return np.ascontiguousarray(np.tile(_tile(), (8, 10))), dict(detector_threshold=0.001, maximum_features=-1)


def noise_vga():
    """640x480 uniform noise at 1e-4: 21 030 candidates, 10 176 extrema (more than the default 9 600 cached keypoints)."""
    return np.random.default_rng(1).random((480, 640), dtype=np.float32), dict(detector_threshold=1e-4, maximum_features=-1)


def noise_kitti():
    """1242x375 uniform noise at 1e-5: 40 005 candidates, 18 462 extrema (more than the default 14 554 cached keypoints)."""
    return np.random.default_rng(3).random((375, 1242), dtype=np.float32), dict(detector_threshold=1e-5, maximum_features=-1)


def lattice():
    """640x480 dot lattice (every 5th pixel of every 5th row is 1) over 1e-3 uniform noise, at threshold 0: 97 743 candidates (more
    than the default 38 400) and 31 390 extrema (more than the default 9 600 cached keypoints)."""
    img = np.zeros((480, 640), np.float32)
    img[::5, ::5] = 1.0
    img += np.float32(1e-3) * np.random.default_rng(5).random((480, 640), dtype=np.float32)
    return img, dict(detector_threshold=0.0, maximum_features=-1)


CAPACITY = {"noise_vga": noise_vga, "noise_kitti": noise_kitti, "lattice": lattice}
