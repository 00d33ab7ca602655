"""The frames of tests/akaze_scenes.py against the limits of AKAZE's keypoint stages, with the CPU oracle's counts.

The limits are restated from cv_b200/csrc: build_workspace's default capacities (capc candidates, capk cached keypoints), the ring of
k_suppress_smem (SUP_CAPS entries for two adjacent classes) and the chunk span of k_filter_upper / k_rank_count / k_rank_scatter (at most
64 chunks of 256 cached keypoints).  When one of them changes, these tests show which scene no longer reaches its path."""
import functools

import numpy as np
import pytest

from oracle import pyoracle as O
from tests import akaze_scenes as S

SUP_CAPS = 8192     # k_suppress_smem's ring (akaze_kernels.cuh)
NT = 256            # threads (keypoints) per chunk
MAX_CHUNKS = 64     # stage_detect / stage_sort_describe: ichunks = min(cdiv(capk, NT), 64)


def capc(P):
    return min(max(P // 8, 4096), 1 << 20)


def capk(P):
    return min(max(P // 32, 4096), 1 << 17)


def chunk_span(P):
    """cached keypoints the chunk grid covers before its loops wrap"""
    return NT * min(-(-capk(P) // NT), MAX_CHUNKS)


def pair(cand):
    """the most candidates in two adjacent classes: what k_suppress_smem holds in its ring"""
    cnt = np.bincount(cand["class_id"].astype(np.int64))
    return int(max(cnt[e] + (cnt[e - 1] if e else 0) for e in range(len(cnt))))


@functools.lru_cache(maxsize=None)
def counts(name):
    img, cfg = getattr(S, name)()
    o = O.Akaze(**cfg)
    kps, _ = o.extract(img)
    cand = o.stage("candidates")
    return dict(P=img.size, candidates=len(cand), pair=pair(cand), extrema=len(o.stage("extrema")), final=len(kps),
                distinct=len(np.unique(kps["response"])))


def test_limits_restated():
    assert (capc(1920 * 1080), capk(1920 * 1080)) == (259200, 64800)
    assert (capc(640 * 480), capk(640 * 480)) == (38400, 9600)
    assert (capc(1242 * 375), capk(1242 * 375)) == (58218, 14554)
    assert chunk_span(1920 * 1080) == 16384


def test_dense_falls_back_and_wraps_within_default_capacities():
    c = counts("dense")
    assert (c["candidates"], c["pair"], c["extrema"]) == (44768, 13700, 19415)
    assert c["pair"] > SUP_CAPS and c["extrema"] > chunk_span(c["P"])
    assert c["candidates"] <= capc(c["P"]) and c["extrema"] <= capk(c["P"])


def test_tied_frames_take_both_suppression_paths():
    big, small = counts("tied"), counts("tied_small")
    assert (big["final"], big["distinct"], big["pair"]) == (13340, 34, 9866)
    assert (small["final"], small["distinct"], small["pair"]) == (1569, 35, 1492)
    assert big["pair"] > SUP_CAPS >= small["pair"]
    assert big["candidates"] <= capc(big["P"]) and big["extrema"] <= capk(big["P"])


@pytest.mark.parametrize("name,exceeds", [("noise_vga", "k"), ("noise_kitti", "k"), ("lattice", "ck")])
def test_capacity_frames_exceed_the_default_capacities(name, exceeds):
    c = counts(name)
    assert (c["candidates"] > capc(c["P"])) == ("c" in exceeds)
    # the extrema are a lower bound on the suppression's cache, so these frames overflow it
    assert c["extrema"] > capk(c["P"])
    want = {"noise_vga": (21030, 10176, 10169), "noise_kitti": (40005, 18462, 18441), "lattice": (97743, 31390, 31379)}[name]
    assert (c["candidates"], c["extrema"], c["final"]) == want
