"""GPU: the similar-frame search (include/cvb200_lsh.h, cv_b200/csrc/lsh.cu) equals the oracle (oracle/ref_lsh.c) bit for bit.

  * shapes: words 1, 2, 16, 127, 128 x k 1 .. 1024 around the warp, tile and power-of-two edges x database sizes 0, 1, k - 1, k, k + 1,
    the 64-row tile edges, the split edges, and ~200 000; one query (cv-sfm's call) and ~2 000;
  * distance extremes (0 and 32 * words, complements) and ties: few distinct codes, all-zero databases, equal distances on both sides
    of the k-th place and across split boundaries;
  * the device form with counts below their maxima (decoy rows behind them, output rows past the count untouched) and NULL counts;
  * on 64-byte codes with k <= 8 the result equals the descriptor matcher cvb_hamming_knn;
  * repeated calls in one context and in fresh contexts give the same bytes;
  * cv-sfm's add-frame flow: hashes from cvb_hash_bag_dev written into consecutive rows of one device database, each searched with a
    device count; every frame finds itself at distance 0, and FrameHashIndex gives the same answer."""
import numpy as np
import pytest

import cv_b200
from cv_b200.knn import _lsh_lib
from oracle import pyoracle_lsh as L
from tests.synth import random_descriptors

pytestmark = pytest.mark.gpu

MISS = 0xFFFFFFFF
FILL = 0xA5A5A5A5
WORDS = (1, 2, 16, 127, 128)
KS = (1, 2, 8, 9, 31, 32, 33, 511, 512, 513, 1023, 1024)
TILE = 64                        # database rows per tile of k_lsh_scan


def _codes(rng, m, words, distinct=None):
    if distinct is None:
        return rng.integers(0, 256, (m, 4 * words), dtype=np.uint8)
    palette = rng.integers(0, 256, (distinct, 4 * words), dtype=np.uint8)
    return palette[rng.integers(0, distinct, m)]


def _same(got, want, what):
    assert np.array_equal(got[0], want[0]), (what, "idx", np.flatnonzero((got[0] != want[0]).ravel())[:8])
    assert np.array_equal(got[1], want[1]), (what, "dist")


def _check(q, db, k, what):
    got = cv_b200.hash_knn(q, db, k)
    _same(got, L.hash_knn(q, db, k), what)
    return got


def _dev(a):
    import torch
    a = np.ascontiguousarray(a)
    if a.dtype == np.uint32:
        a = a.view(np.int32)
    return torch.from_numpy(a.copy()).to("cuda:0")


def _host(t, dtype=np.uint32):
    return t.cpu().numpy().view(dtype)


def _knn_dev(ctx, words, qd, n_dev, n_max, dbd, m_dev, m_max, k, out_rows=None):
    """cvb_hash_knn_dev into FILL-initialised outputs of max(n_max, out_rows) rows; returns the host copies"""
    import torch
    rows = max(n_max, out_rows or 0)
    idx, dist = _dev(np.full((rows, k), FILL, np.uint32)), _dev(np.full((rows, k), FILL, np.uint32))
    torch.cuda.synchronize()
    ctx.check(_lsh_lib().cvb_hash_knn_dev(ctx.handle, words, qd.data_ptr(), n_dev.data_ptr() if n_dev is not None else None, n_max,
                                          dbd.data_ptr(), m_dev.data_ptr() if m_dev is not None else None, m_max, k, idx.data_ptr(),
                                          dist.data_ptr()))
    ctx.sync()
    return _host(idx), _host(dist)


SPLIT = 16 * TILE                # fewest database rows per split (knn_launch: min(2 * SMs, ceil(m / SPLIT)) splits)


def _split_edges(words):
    """database sizes for one query at which the split plan changes: one split to two and three, and the most splits (264 on 132 SMs)"""
    edges = [SPLIT - 1, SPLIT, SPLIT + 1, 2 * SPLIT + 1]
    return edges + ([SPLIT * 264 - 1, SPLIT * 264 + 1] if words <= 16 else [])


@pytest.mark.parametrize("words", WORDS)
@pytest.mark.parametrize("k", KS)
def test_shapes_one_query(words, k):
    rng = np.random.default_rng(1000 * words + k)
    q = rng.integers(0, 256, (1, 4 * words), dtype=np.uint8)
    sizes = sorted({0, 1, k - 1, k, k + 1, TILE - 1, TILE, TILE + 1, 2 * TILE + 1})
    if words in (1, 128) or k in (512, 1024):
        sizes += _split_edges(words)
    for m in sizes:
        db = _codes(rng, m, words, distinct=3 if m % 2 else None)
        _check(q, db, k, (words, k, m))


@pytest.mark.parametrize("words,k", [(128, 512), (128, 1024), (1, 1024), (2, 33), (16, 8)])
def test_large_database(words, k):
    rng = np.random.default_rng(words + k)
    db = _codes(rng, 200_003, words)
    q = np.concatenate([db[[5, 199_999]], rng.integers(0, 256, (1, 4 * words), dtype=np.uint8)])
    idx, dist = _check(q[:1], db, k, (words, k, "200k"))
    assert idx[0, 0] == 5 and dist[0, 0] == 0
    _check(q, db, k, (words, k, "200k, 3 queries"))


@pytest.mark.parametrize("words,k", [(128, 512), (128, 1024), (127, 33), (16, 8), (1, 9), (2, 511)])
def test_many_queries(words, k):
    rng = np.random.default_rng(7 * words + k)
    m = 3000 if words >= 127 else 5000
    db = _codes(rng, m, words, distinct=50 if words < 16 else None)
    q = np.concatenate([db[rng.integers(0, m, 1000)], _codes(rng, 1003, words)])
    _check(q, db, k, (words, k, "2003 queries"))


@pytest.mark.parametrize("words", WORDS)
def test_distance_extremes(words):
    rng = np.random.default_rng(words)
    q = rng.integers(0, 256, (3, 4 * words), dtype=np.uint8)
    db = np.concatenate([~q, _codes(rng, 700, words), q, ~q])
    for k in (1, 8, 512, 1024):
        idx, dist = _check(q, db, k, (words, k, "extremes"))
        assert (dist[:, 0] == 0).all() and (idx[:, 0] == np.arange(703, 706)).all()
    idx, dist = _check(q, np.concatenate([~q, ~q]), 1024, (words, "complements"))
    for i in range(3):                                           # a query's two complements are its farthest rows
        assert (dist[i, 4:6] == 32 * words).all() and list(idx[i, 4:6]) == [i, i + 3] and (dist[i, 6:] == MISS).all()


@pytest.mark.parametrize("words", [1, 16, 128])
@pytest.mark.parametrize("k", [1, 33, 512, 1024])
def test_ties(words, k):
    rng = np.random.default_rng(words * 3 + k)
    for m in (k + 1, 3 * k + 17, 40_000):
        # all-zero database (frames without features): every distance equal; the lowest indices win, across every split
        zeros = np.zeros((m, 4 * words), np.uint8)
        idx, dist = _check(np.zeros((2, 4 * words), np.uint8), zeros, k, (words, k, m, "zeros"))
        assert (idx == np.arange(k)).all() and (dist == 0).all()
        # equal distances straddling the k-th place, scattered over the database and so over split boundaries
        q = rng.integers(0, 256, (1, 4 * words), dtype=np.uint8)
        db = _codes(rng, m, words)
        near = q.copy()
        near[0, 0] ^= 3
        where = np.sort(rng.choice(m, size=min(m, k + 5), replace=False))
        db[where] = near
        idx, dist = _check(q, db, k, (words, k, m, "straddle"))
        assert np.array_equal(idx[0], where[:k]) and (dist[0] == 2).all()
        # few distinct codes
        _check(_codes(rng, 4, words), _codes(rng, m, words, distinct=4), k, (words, k, m, "few codes"))


@pytest.mark.parametrize("words,k", [(128, 512), (16, 8), (1, 1024), (127, 33)])
def test_device_counts(words, k):
    ctx = cv_b200.Context(0)
    rng = np.random.default_rng(words * k)
    n_max, n_cnt, m_max, m_cnt = 37, 23, 3100, 1234
    q = _codes(rng, n_max, words)
    db = _codes(rng, m_max, words)
    db[m_cnt:] = q[rng.integers(0, n_max, m_max - m_cnt)]      # decoys at distance 0 behind the count
    qd, dbd = _dev(q), _dev(db)
    idx, dist = _knn_dev(ctx, words, qd, _dev(np.array([n_cnt], np.uint32)), n_max, dbd, _dev(np.array([m_cnt], np.uint32)), m_max, k)
    _same((idx[:n_cnt], dist[:n_cnt]), L.hash_knn(q[:n_cnt], db[:m_cnt], k), (words, k, "counts"))
    assert (idx[n_cnt:] == FILL).all() and (dist[n_cnt:] == FILL).all()
    # counts above their maxima are clamped to them
    idx, dist = _knn_dev(ctx, words, qd, _dev(np.array([10 * n_max], np.uint32)), n_max, dbd, _dev(np.array([10 ** 9], np.uint32)),
                         m_max, k)
    _same((idx, dist), L.hash_knn(q, db, k), (words, k, "clamped counts"))
    # NULL counts: n_max / m_max
    idx, dist = _knn_dev(ctx, words, qd, None, n_max, dbd, None, m_max, k)
    _same((idx, dist), L.hash_knn(q, db, k), (words, k, "NULL counts"))
    # zero counts: nothing written / every slot empty
    idx, dist = _knn_dev(ctx, words, qd, _dev(np.array([0], np.uint32)), n_max, dbd, None, m_max, k)
    assert (idx == FILL).all() and (dist == FILL).all()
    idx, dist = _knn_dev(ctx, words, qd, None, n_max, dbd, _dev(np.array([0], np.uint32)), m_max, k)
    assert (idx == MISS).all() and (dist == MISS).all()


def test_device_form_rejects_misaligned_arrays():
    ctx = cv_b200.Context(0)
    buf = _dev(np.zeros(4096, np.uint8))
    out = _dev(np.zeros(64, np.uint32))
    p, o = buf.data_ptr(), out.data_ptr()
    for args in ((p + 4, p, o, o + 128), (p, p + 8, o, o + 128), (p, p, o + 4, o + 128), (p, p, o, o + 132)):
        rc = _lsh_lib().cvb_hash_knn_dev(ctx.handle, 1, args[0], None, 1, args[1], None, 4, 4, args[2], args[3])
        assert rc == cv_b200._lib.CVB_EINVAL, args


@pytest.mark.parametrize("k", range(1, 9))
def test_equals_descriptor_matcher(k):
    """64-byte codes are BitArray<64>: the same search as cvb_hamming_knn, bit for bit"""
    for seed, (n, m) in enumerate(((1, 5000), (300, 4097), (129, 7))):
        q, db = random_descriptors(n, 10 * k + seed), random_descriptors(m, 20 * k + seed)
        db[::7] = db[0]                                          # ties
        got = cv_b200.hash_knn(q, db, k)
        want = cv_b200.hamming_knn(q, db, k)
        _same(got, want, (k, n, m))


def test_deterministic_across_calls_and_contexts():
    rng = np.random.default_rng(5)
    q = _codes(rng, 9, 128, distinct=2)
    db = _codes(rng, 50_000, 128, distinct=6)
    first = cv_b200.hash_knn(q, db, 1024)
    for ctx in (None, None, cv_b200.Context(0), cv_b200.Context(0)):
        again = cv_b200.hash_knn(q, db, 1024, ctx=ctx)
        assert first[0].tobytes() == again[0].tobytes() and first[1].tobytes() == again[1].tobytes()
    _same(first, L.hash_knn(q, db, 1024), "determinism")


def _host_hash(feats, code):
    """HammingHasher::hash_bag on the host: each feature sets the bit of its nearest codeword, the lower on ties"""
    out = np.zeros(len(code) // 8, np.uint8)
    if len(feats):
        d = np.bitwise_count(feats.view(np.uint64)[:, None, :] ^ code.view(np.uint64)[None, :, :]).sum(-1)
        for ix in d.argmin(axis=1):
            out[ix >> 3] |= np.uint8(1 << (ix & 7))
    return out


def test_cv_sfm_add_frame_flow():
    """VSlam::add_frame's order: hash the frame into row m of the database (cvb_hash_bag_dev), then search with that row and the count
    m + 1 on the device (cvb_hash_knn_dev)."""
    import torch
    from tests.common import kitti_frame
    ak = cv_b200.Akaze.sparse()
    frames = [ak.extract_from_gray_float_image(kitti_frame(n))[1] for n in ("0000000000", "0000000014")]
    assert all(len(f) > 100 for f in frames)
    frames += [random_descriptors(n, 900 + n) for n in (5, 300, 2000)]
    frames += [np.zeros((0, 64), np.uint8), frames[0][:50], np.zeros((0, 64), np.uint8), frames[0]]   # empty frames and repeats
    code = random_descriptors(4096, 77)                          # the shape of cv-sfm's codeword table
    ctx = ak.ctx
    words, k, cap = 128, 512, 16
    db = _dev(np.full((cap, 4 * words), 0x5A, np.uint8))         # rows past the count are decoys
    cd = _dev(code)
    hashes = []
    index = cv_b200.FrameHashIndex(words)
    for m, feats in enumerate(frames):
        fd = _dev(feats if len(feats) else np.zeros((1, 64), np.uint8))
        row = db[m]
        torch.cuda.synchronize()
        nd = _dev(np.array([len(feats)], np.uint32))             # kept alive until the call has run
        ctx.check(ctx.lib.cvb_hash_bag_dev(ctx.handle, fd.data_ptr(), nd.data_ptr(), max(len(feats), 1), cd.data_ptr(), 4096,
                                           row.data_ptr()))
        m_dev = _dev(np.array([m + 1], np.uint32))
        idx, dist = _knn_dev(ctx, words, row, None, 1, db, m_dev, cap, k)
        h = _host_hash(feats, code)
        assert np.array_equal(_host(row, np.uint8), h), m
        hashes.append(h)
        want = L.hash_knn(h[None], np.stack(hashes), k)
        _same((idx, dist), want, ("frame", m))
        first_same = next(i for i, x in enumerate(hashes) if np.array_equal(x, h))
        assert dist[0, 0] == 0 and idx[0, 0] == first_same, m
        assert m in idx[0, :m + 1] and dist[0, list(idx[0]).index(m)] == 0
        index.insert(h, f"frame{m}")
        got = index.knn_values(h, k)
        assert got == [(int(d), f"frame{i}") for i, d in zip(want[0][0], want[1][0]) if i != MISS], m
    assert first_same == 0                                       # the last frame repeats frame 0, which is listed first


def test_frame_hash_index_grows_and_takes_device_rows():
    import torch
    rng = np.random.default_rng(11)
    hashes = _codes(rng, 300, 128, distinct=40)
    index = cv_b200.FrameHashIndex(128, capacity=4)
    for i, h in enumerate(hashes):
        if i % 2:
            index.insert_dev(torch.from_numpy(h.copy()).to("cuda:0"), i)
        else:
            index.insert(h, i)
    assert len(index) == 300
    for qi in (0, 1, 299):
        want = L.hash_knn(hashes[qi:qi + 1], hashes, 512)
        assert index.knn_values(hashes[qi], 512) == [(int(d), int(i)) for i, d in zip(want[0][0], want[1][0]) if i != MISS]
