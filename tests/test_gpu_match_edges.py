"""GPU: the brute-force Hamming matcher (cv_b200/csrc/match.cu, match_wgmma.cuh) where its kernels can go wrong.

  * a plain NumPy brute force (popcount of the XOR over uint64 words, the k smallest by np.lexsort((index, distance)), 0xffffffff
    where the database runs out) equals the C oracle on every case; the wgmma, mma.sync and popcount kernels equal it bit for bit;
  * descriptor families: single-bit bases (each query bit must meet its own database bit), all-zero / all-one / complement
    extremes (distances 0 and 512: the key 512 << 22 sets bit 31), AKAZE-shaped rows of extreme popcount, and equal-distance
    copies on both sides of every tile and split edge (the lower index wins);
  * every template instance k = 1..8 at query counts around the 8/16/64/128-row boundaries, database sizes around the tiles,
    and database sizes whose last split holds one row;
  * database indices past 2^22 (a key keeps 22 bits of a split-local index; the merge adds the split's base);
  * the device-count entry points cvb_hamming_knn_dev_counts, cvb_match_symmetric_dev, cvb_match_symmetric_pairs_dev and
    cvb_hash_bag_dev, with counts below, at and above their maxima and decoys behind the counts."""
import functools
import os

import numpy as np
import pytest

import cv_b200
from cv_b200.pair import bind as bind_pair_abi
from oracle import pyoracle as O
from tests.synth import random_descriptors

pytestmark = pytest.mark.gpu

MISS = 0xFFFFFFFF                 # an empty k-NN slot, and "no match" in the symmetric flags
FILL = 0xA5A5A5A5                 # what an output word holds when the entry must not write it
IDX_MASK = (1 << 22) - 1          # the split-local index bits of a (distance << 22 | index) key
KERNELS = {"wgmma": "CVB_KNN_WGMMA", "imma": "CVB_KNN_IMMA", "popc": "CVB_KNN_POPC"}
TILE = {"wgmma": 128, "imma": 32, "popc": 128}      # database rows per tile of each kernel


def _cdiv(a, b):
    return -(-a // b)


# ---------------------------------------------------------------------------------------------------------------------------
# the reference

def ref_knn(q, db, k):
    """LinearKnn{Hamming}.knn for every query by brute force: (idx[n, k], dist[n, k]) uint32."""
    q, db = np.ascontiguousarray(q, np.uint8), np.ascontiguousarray(db, np.uint8)
    idx = np.full((len(q), k), MISS, np.uint32)
    dist = np.full((len(q), k), MISS, np.uint32)
    m = len(db)
    if m == 0:
        return idx, dist
    qw, dw = q.view(np.uint64), db.view(np.uint64)
    kk = min(k, m)
    step = max(1, (1 << 19) // m)
    for s in range(0, len(q), step):
        d = np.bitwise_count(qw[s:s + step, None, :] ^ dw[None, :, :]).sum(-1, dtype=np.uint32)
        for r, dr in enumerate(d):
            cand = np.flatnonzero(dr <= np.partition(dr, kk - 1)[kk - 1])    # every row that can be among the k smallest
            top = cand[np.lexsort((cand, dr[cand]))[:kk]]
            idx[s + r, :kk] = top
            dist[s + r, :kk] = dr[top]
    return idx, dist


def expected_knn(q, db, k):
    """The brute force, checked against the C oracle."""
    want = ref_knn(q, db, k)
    oi, od = O.hamming_knn(q, db, k)
    assert np.array_equal(want[0], oi) and np.array_equal(want[1], od), "NumPy brute force != C oracle"
    return want


def ref_symmetric(a, b, better_by):
    """cv-sfm symmetric_matching (cv-sfm/src/lib.rs:3097-3133) restated as a loop: per a, its b or MISS."""
    n, m = len(a), len(b)
    out = np.full(n, MISS, np.uint32)
    if n < 2 or m < 2:
        return out
    fi, fd = expected_knn(a, b, 2)
    ri, rd = expected_knn(b, a, 2)
    for i in range(n):
        if int(fd[i, 0]) + better_by <= int(fd[i, 1]):
            j = int(fi[i, 0])
            if int(rd[j, 0]) + better_by <= int(rd[j, 1]) and int(ri[j, 0]) == i:
                out[i] = j
    return out


def ref_pairs(a, b, better_by):
    flags = ref_symmetric(a, b, better_by)
    return [(i, int(j)) for i, j in enumerate(flags) if j != MISS]


def ref_hash_bag(feats, code):
    """HammingHasher::hash_bag (cv-sfm/src/lib.rs:672): each feature sets the bit of its nearest codeword, the lower on ties."""
    out = np.zeros(len(code) // 8, np.uint8)
    if len(feats):
        for ix in expected_knn(feats, code, 1)[0][:, 0]:
            out[ix >> 3] |= np.uint8(1 << (ix & 7))
    return out


def layout(kernel, n, m, sms):
    """(splits, chunk): how knn_dev in match.cu splits m database rows for n queries on a device with `sms` SMs."""
    if kernel == "wgmma" and m > 0:
        splits, tile = min(max(1, sms // _cdiv(n, 128)), max(1, _cdiv(m, 128))), 128
    elif kernel == "imma" and m > 0:
        splits, tile = min(max(1, sms * 4 // _cdiv(n, 64)), max(1, _cdiv(m, 64))), 32
    else:
        m = max(m, 1)
        splits, tile = min(max(1, _cdiv(sms * 4, _cdiv(n, 128))), max(1, _cdiv(m, 256))), 128
    chunk = _cdiv(_cdiv(m, splits), tile) * tile
    while chunk > IDX_MASK:
        splits *= 2
        chunk = _cdiv(_cdiv(m, splits), tile) * tile
    return _cdiv(m, chunk), chunk


# ---------------------------------------------------------------------------------------------------------------------------
# descriptors

def _pack(bits):
    """bool [n, 512] -> [n, 64] uint8: bit i is bit i & 7 of byte i >> 3 (BitArray<64>)."""
    return np.packbits(np.asarray(bits, bool).reshape(-1, 512), axis=1, bitorder="little")


def _with_bits(positions):
    b = np.zeros(512, bool)
    b[list(positions)] = True
    return b


def _flip(d, bits):
    d = d.copy()
    for b in bits:
        d[b >> 3] ^= np.uint8(1 << (b & 7))
    return d


def _flip_random(d, rng, count, live=486):
    return _flip(d, rng.choice(live, count, replace=False))


def fam_basis(kernel, sms):
    """Database row i has only bit i set.  A query with bit set S is |S| - 1 from the rows in S and |S| + 1 from the others, so the
    top-k is S in ascending order, then the lowest indices outside S."""
    rng = np.random.default_rng(1)
    sets = [[i] for i in range(512)]
    sets += [sorted(rng.choice(512, s, replace=False)) for s in (0, 1, 2, 3, 5, 8, 9, 17, 64, 255, 256, 257, 486, 510, 511, 512)
             for _ in range(3)]
    q = _pack([_with_bits(S) for S in sets])
    db = _pack(np.eye(512, dtype=bool))
    idx = np.empty((len(sets), 8), np.uint32)
    dist = np.empty((len(sets), 8), np.uint32)
    for r, S in enumerate(sets):
        inside = {int(i) for i in S}
        order = sorted(inside)[:8] + [i for i in range(8 + len(inside)) if i not in inside]
        idx[r] = order[:8]
        dist[r] = [len(S) - 1 if i in inside else len(S) + 1 for i in order[:8]]
    return [("basis", q, db, (idx, dist))]


def fam_basis_dual(kernel, sms):
    """The database is one descriptor x with bit i flipped in row i: x is 1 from every row (pure index order), x ^ e_j is 0 from
    row j and 2 from the rest, x ^ e_j ^ e_l is 1 from rows j and l and 3 from the rest."""
    rng = np.random.default_rng(2)
    x = rng.integers(0, 256, 64, dtype=np.uint8)
    db = np.stack([_flip(x, [i]) for i in range(512)])
    flips = [[]] + [[j] for j in range(512)] + [sorted(rng.choice(512, 2, replace=False)) for _ in range(40)]
    q = np.stack([_flip(x, f) for f in flips])
    idx = np.empty((len(flips), 8), np.uint32)
    dist = np.empty((len(flips), 8), np.uint32)
    for r, f in enumerate(flips):
        f = [int(i) for i in f]
        order = f + [i for i in range(10) if i not in f]
        idx[r] = order[:8]
        dist[r] = [(len(f) - 1 if i in f else len(f) + 1) for i in order[:8]]
    return [("basis_dual", q, db, (idx, dist))]


def fam_extremes(kernel, sms):
    """Distances 0 and 512: all-zero against all-zero (pure index order), all-one against all-zero, complement pairs, and one
    database mixing 0- and 512-distance rows."""
    zeros, ones = np.zeros((300, 64), np.uint8), np.full((300, 64), 0xFF, np.uint8)
    idx = np.tile(np.arange(8, dtype=np.uint32), (3, 1))
    cases = [("zero_vs_zero", zeros[:3], zeros, (idx, np.zeros((3, 8), np.uint32))),
             ("one_vs_zero", ones[:3], zeros, (idx, np.full((3, 8), 512, np.uint32)))]
    rng = np.random.default_rng(3)
    r = rng.integers(0, 256, (150, 64), dtype=np.uint8)
    cases.append(("complements", np.concatenate([r[::7], ~r[::5], zeros[:1], ones[:1]]), np.concatenate([r, ~r]), None))
    mixed = ones.copy()
    mixed[[5, 31, 32, 127, 128, 299]] = 0
    cases.append(("mixed_0_512", np.concatenate([zeros[:2], ones[:2], r[:20]]), mixed, None))
    return cases


def fam_akaze(kernel, sms):
    """AKAZE-shaped: 486 live bits (byte 60 & 0x3F, bytes 61..63 zero), rows with 0..3 and 483..486 bits set among random ones."""
    rng = np.random.default_rng(4)

    def rows(pops):
        return _pack([_with_bits(rng.choice(486, p, replace=False)) for p in pops])
    edge = [0, 0, 1, 1, 2, 3, 483, 484, 485, 485, 486, 486]
    db = rows(edge + list(rng.integers(0, 487, 700)) + edge)
    q = rows(edge + [5, 240, 243, 246, 481] + list(rng.integers(0, 487, 200)))
    assert not (db[:, 61:].any() or (db[:, 60] & 0xC0).any())
    return [("akaze", q, db, None)]


def fam_planted(kernel, sms):
    """A few prototypes; two copies of each with the same number (0..3) of flipped bits sit on the two sides of one tile or split
    edge of the layout `kernel` picks (the last pair ends in the database's last row), against a random background.  The query
    is the prototype, so the lower index must come first across every edge."""
    cases = []
    for n, m in ((17, 1000), (129, sms * 128 + 1), (300, 2 * sms * 128 + 1)):
        rng = np.random.default_rng(n + m)
        splits, chunk = layout(kernel, n, m, sms)
        tile = TILE[kernel]
        if m > 1000:
            assert splits > 1, (kernel, n, m, splits, chunk)
        last = (splits - 1) * chunk
        last_tile = last + (m - 1 - last) // tile * tile
        edges = []
        for e in sorted({31, 127, tile - 1, chunk - 1, chunk + tile - 1, last - 1, last_tile - 1, m - 2}):
            if e >= 0 and e + 1 < m and (not edges or e > edges[-1] + 1):
                edges.append(e)
        db = random_descriptors(m, 5 + m)
        q = random_descriptors(n, 6 + n)
        protos = random_descriptors(len(edges), 7)
        for j, e in enumerate(edges):
            db[e] = _flip_random(protos[j], rng, j % 4)
            db[e + 1] = _flip_random(protos[j], rng, j % 4)
            q[j] = protos[j]
        cases.append((f"planted_n{n}_m{m}_splits{splits}_chunk{chunk}", q, db, None))
    return cases


FAMILIES = {"basis": fam_basis, "basis_dual": fam_basis_dual, "extremes": fam_extremes, "akaze": fam_akaze, "planted": fam_planted}


@functools.lru_cache(maxsize=None)
def family_cases(family, kernel, sms):
    """[(label, q, db, idx8, dist8)]: the top-8 of the brute force, checked against the oracle and, where the family states one,
    against its closed form (the top-k for k < 8 is its prefix)."""
    out = []
    for label, q, db, closed in FAMILIES[family](kernel, sms):
        idx, dist = expected_knn(q, db, 8)
        if closed is not None:
            assert np.array_equal(idx, closed[0]) and np.array_equal(dist, closed[1]), label
        out.append((label, q, db, idx, dist))
    return out


@functools.lru_cache(maxsize=None)
def grid_case(m, nq, m_all):
    """Queries and a database of m rows for the shape tests (the first n queries are the n-query case; the top-k is the prefix of
    the top-8).  Database rows are random or prototypes with 0..3 flipped bits, so distances tie across every tile and split;
    queries are prototypes, copies of the database's middle and last rows, near copies of random rows, and random rows."""
    rng = np.random.default_rng(9)
    protos = random_descriptors(6, 10)
    base = _db_all(m_all)
    db = base[:m].copy()
    q = random_descriptors(nq, 11)
    q[1:7] = protos
    if m:
        for r, row in ((0, m - 1), (7, m // 2), (8, max(m - 2, 0))):
            q[r] = db[row]
        for r in range(16, nq, 16):
            q[r] = _flip_random(db[int(rng.integers(m))], rng, int(rng.integers(0, 3)))
    idx, dist = expected_knn(q, db, 8)
    return q, db, idx, dist


@functools.lru_cache(maxsize=None)
def _db_all(m_all):
    rng = np.random.default_rng(12)
    protos = random_descriptors(6, 10)
    db = random_descriptors(m_all, 13)
    for j in range(m_all):
        if j % 3:
            db[j] = _flip_random(protos[j % 6], rng, j % 4)
    return db


# ---------------------------------------------------------------------------------------------------------------------------
# fixtures and helpers

@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def kernel_ctx():
    """kernel name -> a Context latched to that kernel (each context reads its kernel from the environment at its first k-NN)."""
    made = {}

    def get(kernel):
        if kernel not in made:
            saved = {v: os.environ.pop(v, None) for v in KERNELS.values()}
            os.environ[KERNELS[kernel]] = "1"
            try:
                ctx = cv_b200.Context(0)
                cv_b200.hamming_knn(np.zeros((1, 64), np.uint8), np.zeros((1, 64), np.uint8), 1, ctx=ctx)
            finally:
                for v, val in saved.items():
                    os.environ.pop(v, None)
                    if val is not None:
                        os.environ[v] = val
            made[kernel] = ctx
        return made[kernel]
    yield get
    for ctx in made.values():
        ctx.close()


def assert_knn(got, want_idx, want_dist, what):
    idx, dist = got
    k = idx.shape[1]
    bad = np.flatnonzero((idx != want_idx[:, :k]).any(1) | (dist != want_dist[:, :k]).any(1))
    assert bad.size == 0, (f"{what}: {bad.size} of {len(idx)} rows differ; first is row {bad[0]}: idx {idx[bad[0]].tolist()} "
                           f"dist {dist[bad[0]].tolist()}, want idx {want_idx[bad[0], :k].tolist()} dist {want_dist[bad[0], :k].tolist()}")


def _dev(a):
    import torch
    a = np.ascontiguousarray(a)
    if a.dtype == np.uint32:
        a = a.view(np.int32)
    return torch.from_numpy(a.copy()).to("cuda:0")


def _host(t, dtype=np.uint32):
    return t.cpu().numpy().view(dtype)


def _u32(v):
    """A device count.  Keep the tensor alive across the call: a freed one's block is handed to the next allocation."""
    return _dev(np.array([v], np.uint32))


def _run(ctx, fn, *args):
    import torch
    torch.cuda.synchronize()
    ctx.check(fn(ctx.handle, *args))
    ctx.sync()


N_GRID = (1, 7, 8, 9, 15, 16, 17, 63, 64, 65, 127, 128, 129, 257)
N_SPLIT = tuple(n for n in N_GRID if n <= 128)


# ---------------------------------------------------------------------------------------------------------------------------
# the k-NN tables

@pytest.mark.parametrize("k", range(1, 9))
@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("kernel", list(KERNELS))
def test_descriptor_families(kernel_ctx, sms, kernel, family, k):
    ctx = kernel_ctx(kernel)
    for label, q, db, idx, dist in family_cases(family, kernel, sms):
        assert_knn(cv_b200.hamming_knn(q, db, k, ctx=ctx), idx, dist, f"{kernel} k={k} n={len(q)} m={len(db)} {label}")


@pytest.mark.parametrize("n", N_GRID)
@pytest.mark.parametrize("k", range(1, 9))
@pytest.mark.parametrize("kernel", list(KERNELS))
def test_query_and_database_counts(kernel_ctx, kernel, k, n):
    """Query counts around every kernel's 8/16/64/128-row boundaries against database sizes around its 32- and 128-row tiles."""
    ctx = kernel_ctx(kernel)
    for m in sorted({1, k - 1, k, k + 1, 31, 32, 33, 127, 128, 129, 257}):
        q, db, idx, dist = grid_case(m, max(N_GRID), 257)
        assert_knn(cv_b200.hamming_knn(q[:n], db, k, ctx=ctx), idx[:n], dist[:n], f"{kernel} k={k} n={n} m={m} grid")


@pytest.mark.parametrize("blocks", [1, 2])
@pytest.mark.parametrize("k", range(1, 9))
@pytest.mark.parametrize("kernel", list(KERNELS))
def test_split_whose_last_tile_holds_one_row(kernel_ctx, sms, kernel, k, blocks):
    """m = blocks * SMs * 128 + 1 with n <= 128: the database is split across the SMs and the last split holds one row."""
    ctx = kernel_ctx(kernel)
    m = blocks * sms * 128 + 1
    for n in N_SPLIT:
        splits, chunk = layout(kernel, n, m, sms)
        assert splits > 1, (kernel, n, m)
        if kernel != "imma":
            assert m - (splits - 1) * chunk == 1, (kernel, n, m, splits, chunk)
        q, db, idx, dist = grid_case(m, max(N_SPLIT), 2 * sms * 128 + 1)
        assert_knn(cv_b200.hamming_knn(q[:n], db, k, ctx=ctx), idx[:n], dist[:n],
                   f"{kernel} k={k} n={n} m={m} splits={splits} chunk={chunk} one-row split")


BIG_M = (1 << 22) + 300
BIG_PLANTED_ROWS = ((1 << 22) - 1, 1 << 22, (1 << 22) + 1, BIG_M - 1)
BIG_PLANTED_AT = (0, 777, 2048, 4095)          # query rows holding exact copies of those database rows
BIG_N_LEGACY = 4096                            # the mma.sync and popcount kernels take the first 4096 queries


@pytest.fixture(scope="module")
def big(sms):
    """2^22 + 300 random database rows (270 MB), SMs * 128 queries with four planted copies, and the reference top-2 of 32 of them."""
    rng = np.random.default_rng(22)
    db = np.frombuffer(rng.bytes(BIG_M * 64), np.uint8).reshape(BIG_M, 64)
    q = np.frombuffer(rng.bytes(sms * 128 * 64), np.uint8).reshape(-1, 64).copy()
    q[list(BIG_PLANTED_AT)] = db[list(BIG_PLANTED_ROWS)]
    rows = np.array(sorted(set(BIG_PLANTED_AT) | set(rng.choice(BIG_N_LEGACY, 28, replace=False).tolist())))
    idx, dist = expected_knn(q[rows], db, 2)
    return q, db, rows, idx, dist


@pytest.mark.parametrize("kernel", list(KERNELS))
def test_database_indices_past_2_pow_22(kernel_ctx, sms, big, kernel):
    q, db, rows, idx, dist = big
    n = sms * 128 if kernel == "wgmma" else BIG_N_LEGACY
    if kernel == "wgmma":
        # one CTA row per SM leaves one split, whose chunk is over 22 bits: the split is doubled
        assert _cdiv(BIG_M, 128) * 128 > IDX_MASK and layout(kernel, n, BIG_M, sms)[0] == 2
    got_idx, got_dist = cv_b200.hamming_knn(q[:n], db, 2, ctx=kernel_ctx(kernel))
    planted = list(BIG_PLANTED_AT)
    assert got_idx[planted, 0].tolist() == list(BIG_PLANTED_ROWS), kernel
    assert (got_dist[planted, 0] == 0).all(), kernel
    assert_knn((got_idx[rows], got_dist[rows]), idx, dist, f"{kernel} k=2 n={n} m={BIG_M}")


# ---------------------------------------------------------------------------------------------------------------------------
# the device-count entry points

@pytest.mark.parametrize("n_max,m_max,n_dev,m_dev,k", [
    (300, 700, 200, 500, 3), (300, 700, 300, 700, 3), (300, 700, 999, 5000, 3), (300, 700, 0, 700, 2), (300, 700, 300, 0, 2),
    (300, 700, 300, 1, 2), (257, 700, 129, 33, 8),
    (130, 20000, 130, 1500, 8),        # the splits past row 1500 are empty
])
@pytest.mark.parametrize("kernel", list(KERNELS))
def test_knn_dev_counts(kernel_ctx, kernel, n_max, m_max, n_dev, m_dev, k):
    """cvb_hamming_knn_dev_counts equals the host entry on the first min(count, max) rows; the database rows behind the count are
    copies of the queries (a read past it wins) and output rows from min(n_dev, n_max) on keep their fill."""
    ctx = kernel_ctx(kernel)
    slack = 16
    n, m = min(n_dev, n_max), min(m_dev, m_max)
    q = random_descriptors(n_max + slack, 30 + n_max)
    db = random_descriptors(m_max + slack, 31 + m_max)
    for i in range(min(n, m // 7)):
        db[7 * i] = _flip(q[i], [3])             # every query has a near copy among the live rows ...
    db[m:] = np.resize(q, (m_max + slack - m, 64))   # ... and an exact one behind the count
    want_idx, want_dist = cv_b200.hamming_knn(q[:n], db[:m], k, ctx=ctx)
    ri, rd = expected_knn(q[:n], db[:m], k)
    assert np.array_equal(want_idx, ri) and np.array_equal(want_dist, rd)
    qd, dbd, nd, md = _dev(q), _dev(db), _u32(n_dev), _u32(m_dev)
    idx = _dev(np.full((n_max + slack, k), FILL, np.uint32))
    dist = _dev(np.full((n_max + slack, k), FILL, np.uint32))
    _run(ctx, ctx.lib.cvb_hamming_knn_dev_counts, qd.data_ptr(), nd.data_ptr(), n_max, dbd.data_ptr(), md.data_ptr(), m_max, k,
         idx.data_ptr(), dist.data_ptr())
    gi, gd = _host(idx).reshape(-1, k), _host(dist).reshape(-1, k)
    assert_knn((gi[:n], gd[:n]), want_idx, want_dist, f"{kernel} k={k} n={n_dev}/{n_max} m={m_dev}/{m_max}")
    assert (gi[n:] == FILL).all() and (gd[n:] == FILL).all(), "rows past the query count were written"


def _planted_matches(n, m, seed, pairs):
    """Random a [n] and b [m]; b[j] is a[i] with one bit flipped for each (i, j) in `pairs`: confident symmetric matches."""
    a, b = random_descriptors(n, seed), random_descriptors(m, seed + 1)
    for i, j in pairs:
        b[j] = _flip(a[i], [(7 * i + j) % 486])
    return a, b


@pytest.mark.parametrize("n,m", [(1, 50), (50, 1), (1, 1), (2, 2), (300, 280), (1000, 1200)])
@pytest.mark.parametrize("kernel", list(KERNELS))
def test_match_symmetric_dev_flags(kernel_ctx, kernel, n, m):
    """cvb_match_symmetric_dev: one flag per a, equal to the restatement; n < 2 or m < 2 flags nothing."""
    ctx = kernel_ctx(kernel)
    rng = np.random.default_rng(n * m)
    k = min(n, m) // 3
    a, b = _planted_matches(n, m, 40, zip(rng.choice(n, k, replace=False), rng.choice(m, k, replace=False)))
    ad, bd = _dev(a), _dev(b)
    for better_by in (0, 1, 24, 512):
        want = ref_symmetric(a, b, better_by)
        out = _dev(np.full(n + 8, FILL, np.uint32))
        _run(ctx, ctx.lib.cvb_match_symmetric_dev, ad.data_ptr(), n, bd.data_ptr(), m, better_by, out.data_ptr())
        got = _host(out)
        assert np.array_equal(got[:n], want), (kernel, n, m, better_by)
        assert (got[n:] == FILL).all()
        if n < 2 or m < 2:
            assert (got[:n] == MISS).all()
        elif better_by == 24:
            assert (want != MISS).sum() >= k


def _pairs_dev(ctx, a, n_dev, b, m_dev, better_by, cap, n_max=None, m_max=None):
    """cvb_match_symmetric_pairs_dev on a and b (all their rows on the device); -> (pairs, *n_pairs, the words past the pairs)."""
    bind_pair_abi(ctx.lib)
    n_max = len(a) if n_max is None else n_max
    m_max = len(b) if m_max is None else m_max
    ad, bd, nd, md = _dev(a), _dev(b), _u32(n_dev), _u32(m_dev)
    pairs = _dev(np.full(2 * cap + 16, FILL, np.uint32))
    npairs = _u32(FILL)
    _run(ctx, ctx.lib.cvb_match_symmetric_pairs_dev, ad.data_ptr(), nd.data_ptr(), n_max, bd.data_ptr(), md.data_ptr(), m_max,
         better_by, pairs.data_ptr(), cap, npairs.data_ptr())
    np_ = int(_host(npairs)[0])
    got = _host(pairs)
    return [(int(got[2 * i]), int(got[2 * i + 1])) for i in range(min(np_, cap))], np_, got[2 * min(np_, cap):]


@pytest.mark.parametrize("n_dev,m_dev", [(400, 350), (500, 450), (10 ** 6, 10 ** 6), (1, 350), (400, 1), (2, 2)])
@pytest.mark.parametrize("kernel", list(KERNELS))
def test_symmetric_pairs_dev_counts(kernel_ctx, kernel, n_dev, m_dev):
    """Counts below, at and above the maxima (500, 450): rows behind the counts are exact copies of rows of the other side, so
    reading one changes the pairs."""
    ctx = kernel_ctx(kernel)
    n_max, m_max, slack = 500, 450, 32
    rng = np.random.default_rng(50)
    a, b = _planted_matches(n_max + slack, m_max + slack, 51, zip(rng.choice(400, 120, replace=False), rng.choice(350, 120, replace=False)))
    n, m = min(n_dev, n_max), min(m_dev, m_max)
    a[n:] = np.resize(b[m - 100 if m > 100 else 0:], (len(a) - n, 64))
    b[m:] = np.resize(a[:100], (len(b) - m, 64))
    want = ref_pairs(a[:n], b[:m], 24)
    got, npairs, rest = _pairs_dev(ctx, a, n_dev, b, m_dev, 24, n_max, n_max, m_max)
    assert npairs == len(want) and got == want, (kernel, n_dev, m_dev)
    assert (rest == FILL).all()
    if n >= 400 and m >= 350:
        assert len(want) >= 100


CARRY_PLANTED = (0, 1, 1022, 1023, 1024, 1025, 2047, 2048, 2999)


@functools.lru_cache(maxsize=None)
def _carry_case():
    rng = np.random.default_rng(60)
    ai = sorted(set(CARRY_PLANTED) | set(rng.choice(3000, 300, replace=False).tolist()))
    bj = rng.choice(2000, len(ai), replace=False)
    a, b = _planted_matches(3000, 2000, 61, zip(ai, bj))
    want = ref_pairs(a, b, 24)
    assert {i for i, _ in want} >= set(CARRY_PLANTED)
    return a, b, want


@pytest.mark.parametrize("cap", ["all", "all-1", "5", "0", "n"])
@pytest.mark.parametrize("kernel", list(KERNELS))
def test_symmetric_pairs_dev_compaction(kernel_ctx, kernel, cap):
    """3000 queries walk the compaction in chunks of 1024 with matches on both sides of each chunk edge; a cap below the count keeps
    the first cap pairs in ascending a and reports cap."""
    ctx = kernel_ctx(kernel)
    a, b, want = _carry_case()
    c = {"all": len(want), "all-1": len(want) - 1, "5": 5, "0": 0, "n": len(a)}[cap]
    got, npairs, rest = _pairs_dev(ctx, a, len(a), b, len(b), 24, c)
    assert npairs == min(c, len(want)) and got == want[:c], (kernel, cap)
    assert (rest == FILL).all()


@functools.lru_cache(maxsize=None)
def _better_by_case():
    """a 10 <-> b 20 are equal, with second neighbours at 30 bits on both sides (d1 - d0 = 30); a 3 is one bit from both b 5 and
    b 6 (d0 == d1, b 5 first)."""
    rng = np.random.default_rng(70)
    a, b = random_descriptors(64, 71), random_descriptors(64, 72)
    bits = rng.choice(486, 62, replace=False)
    b[20] = a[10]
    b[40] = _flip(a[10], bits[:30])
    a[50] = _flip(a[10], bits[30:60])
    b[5] = _flip(a[3], bits[60:61])
    b[6] = _flip(a[3], bits[61:62])
    return a, b


@pytest.mark.parametrize("better_by", [0, 1, 30, 31, 512, 513])
@pytest.mark.parametrize("kernel", list(KERNELS))
def test_symmetric_pairs_dev_better_by(kernel_ctx, kernel, better_by):
    """d0 + better_by <= d1 on both sides, at equality and one past it; 512 and 513 on a zero / all-ones pair (d0 = 0, d1 = 512)."""
    ctx = kernel_ctx(kernel)
    a, b = _better_by_case()
    want = ref_pairs(a, b, better_by)
    assert ((10, 20) in want) == (better_by <= 30) and ((3, 5) in want) == (better_by == 0)
    got, npairs, _ = _pairs_dev(ctx, a, len(a), b, len(b), better_by, len(a))
    assert npairs == len(want) and got == want, (kernel, better_by)
    z = np.stack([np.zeros(64, np.uint8), np.full(64, 0xFF, np.uint8)])
    want = ref_pairs(z, z, better_by)
    assert want == ([(0, 0), (1, 1)] if better_by <= 512 else [])
    got, npairs, _ = _pairs_dev(ctx, z, 2, z.copy(), 2, better_by, 4)
    assert npairs == len(want) and got == want, (kernel, better_by, "zero / all-ones")


@functools.lru_cache(maxsize=None)
def _hash_case(ncode):
    """(codewords, features, n_dev, bag of the first n_dev features, bag of all): the features behind n_dev are copies of codewords
    whose bit the first n_dev leave clear; a feature one bit away from two codewords on either side of a tile edge precedes them."""
    rng = np.random.default_rng(ncode)
    code = random_descriptors(ncode, 80 + ncode)
    n_dev = 8 if ncode == 32 else 600
    feats = random_descriptors(n_dev + 40, 81 + ncode)
    ties = [(0, 31), (15, 16)] if ncode == 32 else [(31, 32), (127, 128), (4095, 4096), (ncode - 2, ncode - 1)]
    ties = [(i, j) for i, j in ties if j < ncode]
    for t, (i, j) in enumerate(ties):
        bits = rng.choice(486, 2, replace=False)
        code[i], code[j] = _flip(feats[t], bits[:1]), _flip(feats[t], bits[1:])
    want = ref_hash_bag(feats[:n_dev], code)
    for i, j in ties:
        assert (want[i >> 3] >> (i & 7)) & 1 and not (want[j >> 3] >> (j & 7)) & 1, (ncode, i, j)
    clear = [c for c in range(ncode) if not (want[c >> 3] >> (c & 7)) & 1]
    feats[n_dev:] = code[np.resize(clear, len(feats) - n_dev)]
    return code, feats, n_dev, want, ref_hash_bag(feats, code)


@pytest.mark.parametrize("ncode", [32, 4096, 4128])
@pytest.mark.parametrize("kernel", list(KERNELS))
def test_hash_bag_dev(kernel_ctx, kernel, ncode):
    """cvb_hash_bag_dev: the restated bag for a device count below the maximum (the features behind it are copies of codewords whose
    bit is otherwise clear), at it, and 0 (an all-zero hash); equidistant codewords set only the lower index's bit."""
    ctx = kernel_ctx(kernel)
    code, feats, n_dev, want, want_all = _hash_case(ncode)
    n_max = len(feats)
    fd, cd = _dev(feats), _dev(code)
    for count, expect in ((n_dev, want), (n_max, want_all), (0, np.zeros(ncode // 8, np.uint8))):
        out, nd = _dev(np.full(ncode // 8 + 16, 0xA5, np.uint8)), _u32(count)
        _run(ctx, ctx.lib.cvb_hash_bag_dev, fd.data_ptr(), nd.data_ptr(), n_max, cd.data_ptr(), ncode, out.data_ptr())
        got = _host(out, np.uint8)
        assert np.array_equal(got[:ncode // 8], expect), (kernel, ncode, count)
        assert (got[ncode // 8:] == 0xA5).all()
