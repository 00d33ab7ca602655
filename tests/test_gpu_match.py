"""GPU parity of the brute-force Hamming k-NN against the CPU oracle (bit-exact indices and distances)."""
import numpy as np
import pytest

import cv_b200
from oracle import pyoracle as O
from tests.common import GOLDEN, lowe_matches
from tests.synth import random_descriptors

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n,m,k", [(1, 1, 1), (3, 2, 2), (5, 1, 2), (130, 257, 2), (1000, 999, 3), (77, 5000, 8), (5000, 5000, 2)])
def test_knn_matches_oracle(n, m, k):
    q, db = random_descriptors(n, 10 + n), random_descriptors(m, 20 + m)
    idx, dist = cv_b200.hamming_knn(q, db, k)
    oi, od = O.hamming_knn(q, db, k)
    assert np.array_equal(dist, od)
    assert np.array_equal(idx, oi)


def test_ties_resolve_to_lower_index():
    # many duplicates -> many equal distances; the earlier database index must come first
    base = random_descriptors(16, 3)
    db = np.concatenate([base] * 40)           # every descriptor appears 40 times
    q = random_descriptors(64, 4)
    q[:16] = base
    idx, dist = cv_b200.hamming_knn(q, db, 4)
    oi, od = O.hamming_knn(q, db, 4)
    assert np.array_equal(idx, oi) and np.array_equal(dist, od)
    assert (dist[:16, 0] == 0).all() and (idx[:16, 0] == np.arange(16)).all() and (idx[:16, 1] == np.arange(16) + 16).all()


def test_reference_golden_match_count():
    import os
    g = np.load(os.path.join(GOLDEN, "oracle_kitti_sparse.npz"))
    idx, dist = cv_b200.hamming_knn(g["desc0"], g["desc14"], 2)
    assert lowe_matches(dist) == 11            # akaze/tests/estimate_pose.rs:59
    assert np.array_equal(idx, g["knn_idx"]) and np.array_equal(dist, g["knn_dist"])


def test_linear_knn_interface_and_symmetric_matching():
    a, b = random_descriptors(700, 1), random_descriptors(650, 2)
    b[:300] = a[100:400]
    b[:300, 5] ^= 1                             # near-duplicates -> confident matches
    knn = cv_b200.LinearKnn(b)
    nb = knn.knn(a[100], 2)
    assert nb[0] == (0, 1) and len(nb) == 2
    pairs = cv_b200.symmetric_matching(a, b, 24)
    # host restatement of cv-sfm/src/lib.rs:3097-3133 on oracle k-NN tables
    fi, fd = O.hamming_knn(a, b, 2)
    ri, rd = O.hamming_knn(b, a, 2)
    fwd = np.where(fd[:, 0] + 24 <= fd[:, 1], fi[:, 0].astype(np.int64), -1)
    rev = np.where(rd[:, 0] + 24 <= rd[:, 1], ri[:, 0].astype(np.int64), -1)
    want = [[i, int(j)] for i, j in enumerate(fwd) if j >= 0 and rev[j] == i]
    assert pairs.tolist() == want and len(want) >= 300
    assert np.array_equal(cv_b200.matching(a, b, 24), fwd)


def test_large_problem_properties():
    # full BASELINE size through properties: distances ascending, self-match distance 0 at own index
    d = random_descriptors(20000, 9)
    idx, dist = cv_b200.hamming_knn(d[:5000], d, 2)
    assert (dist[:, 0] == 0).all() and (idx[:, 0] == np.arange(5000)).all()
    assert (dist[:, 1] >= dist[:, 0]).all()
    x = np.unpackbits(d[:5000] ^ d[idx[:, 1]], axis=1).sum(1)
    assert np.array_equal(x.astype(np.uint32), dist[:, 1])


def test_landmark_matches_against_loop_restatement():
    """cv-sfm register_frame_subset's matching stage (cv-sfm/src/lib.rs:1468-1576) over three views."""
    rng = np.random.default_rng(11)
    n_land = 400
    proto = rng.integers(0, 256, (n_land, 64), dtype=np.uint8)
    proto[:, 60] &= 0x3F; proto[:, 61:] = 0                        # 486-bit descriptors

    def noisy(d, flips):
        d = d.copy()
        for r in range(len(d)):
            for bit in rng.choice(486, flips, replace=False):
                d[r, bit >> 3] ^= 1 << (bit & 7)
        return d
    views, landmark_views, obs_count = [], {l: set() for l in range(n_land + 40)}, {l: 0 for l in range(n_land + 40)}
    for v in range(3):
        ids = rng.choice(n_land, 250, replace=False)
        desc = noisy(proto[ids], 12)
        ids = ids.copy()
        if v > 0:
            ids[:20] = n_land + np.arange(20) + 20 * (v - 1)       # the same points tracked as separate landmarks: merge candidates
        views.append((desc, ids))
        for l in ids:
            landmark_views[int(l)].add(v); obs_count[int(l)] += 1
    new = noisy(proto[rng.choice(n_land, 300, replace=False)], 10)
    got = cv_b200.landmark_matches(new, views, 24, landmark_views, obs_count)
    want = O.landmark_matches_ref(new, views, 24, landmark_views, obs_count)
    assert got == want
    assert sum(len(m[0]) == 1 for m in got) > 100 and sum(len(m[0]) == 2 for m in got) > 3
    assert cv_b200.landmark_matches(new, views, 24) == O.landmark_matches_ref(new, views, 24)


@pytest.mark.parametrize("mode", ["wgmma", "imma", "popc"])
def test_three_matcher_kernels_agree_with_oracle(mode, monkeypatch):
    """wgmma (default), legacy mma.sync int8 and popcount kernels: identical k-NN tables, ragged sizes included"""
    for k_ in ("CVB_KNN_WGMMA", "CVB_KNN_IMMA", "CVB_KNN_POPC"):
        monkeypatch.delenv(k_, raising=False)
    monkeypatch.setenv({"wgmma": "CVB_KNN_WGMMA", "imma": "CVB_KNN_IMMA", "popc": "CVB_KNN_POPC"}[mode], "1")
    ctx = cv_b200.Context(0)          # the kernel choice is latched per context at its first k-NN call
    for n, m, k in [(1, 1, 1), (129, 127, 2), (300, 1000, 3), (1000, 300, 2), (640, 2049, 8)]:
        q, db = random_descriptors(n, 100 + n), random_descriptors(m, 200 + m)
        idx, dist = cv_b200.hamming_knn(q, db, k, ctx=ctx)
        oi, od = O.hamming_knn(q, db, k)
        assert np.array_equal(dist, od) and np.array_equal(idx, oi), (mode, n, m, k)
    ctx.close()


def test_hash_bag_is_nearest_codeword_bag_of_words():
    """HammingHasher::hash_bag (hamming-lsh, cv-sfm/src/lib.rs:672) restated: every feature sets its nearest codeword's bit."""
    code = random_descriptors(4096, 77)            # same shape as cv-sfm/src/codewords.rs (4 096 x 64 bytes -> 512-byte hash)
    feats = random_descriptors(3000, 78)
    feats[:50] = code[100:150]; feats[:50, 7] ^= 3  # near-duplicates of known codewords
    got = cv_b200.HammingHasher(code).hash_bag(feats)
    oi, _ = O.hamming_knn(feats, code, 1)
    want = np.zeros(512, np.uint8)
    for ix in oi[:, 0]:
        want[ix >> 3] |= 1 << (ix & 7)
    assert np.array_equal(got, want)
    assert all((got[ix >> 3] >> (ix & 7)) & 1 for ix in range(100, 150))
    assert np.array_equal(cv_b200.HammingHasher(code).hash_bag(np.zeros((0, 64), np.uint8)), np.zeros(512, np.uint8))
