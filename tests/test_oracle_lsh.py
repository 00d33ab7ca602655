"""CPU-only: the oracle of include/cvb200_lsh.h (oracle/ref_lsh.c, LinearKnn's insertion at the partition point) equals a numpy brute
force -- distances from unpacked bits, order from a lexsort on (index, distance) -- for every width and k of interest, databases smaller
than, equal to and larger than k, and heavy ties: few distinct codes, all-zero hashes, duplicates on both sides of the k-th place."""
import numpy as np
import pytest

from oracle import pyoracle_lsh as L


def brute(q, db, k):
    """(idx, dist) [N, k]: ascending distance, lower index first; 0xffffffff past len(db)"""
    qb, dbb = np.unpackbits(q, axis=1), np.unpackbits(db, axis=1)
    idx = np.full((len(q), k), 0xFFFFFFFF, np.uint32)
    dist = np.full((len(q), k), 0xFFFFFFFF, np.uint32)
    for i in range(len(q)):
        d = (qb[i][None, :] != dbb).sum(axis=1)
        order = np.lexsort((np.arange(len(db)), d))[:k]
        idx[i, :len(order)] = order
        dist[i, :len(order)] = d[order]
    return idx, dist


def check(q, db, k):
    got = L.hash_knn(q, db, k)
    want = brute(q, db, k)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    return got


@pytest.mark.parametrize("words", [1, 16, 128])
@pytest.mark.parametrize("k", [1, 8, 512, 1024])
def test_oracle_equals_brute_force_below_at_and_above_k(words, k):
    rng = np.random.default_rng(words * 7919 + k)
    for m in (0, 1, k - 1, k, k + 1, 2 * k + 37):
        q = rng.integers(0, 256, (3, 4 * words), dtype=np.uint8)
        db = rng.integers(0, 256, (m, 4 * words), dtype=np.uint8)
        idx, dist = check(q, db, k)
        assert (idx[:, min(m, k):] == 0xFFFFFFFF).all() and (dist[:, min(m, k):] == 0xFFFFFFFF).all()


@pytest.mark.parametrize("words", [1, 16, 128])
@pytest.mark.parametrize("k", [1, 8, 512, 1024])
def test_oracle_ties(words, k):
    rng = np.random.default_rng(words + 31 * k)
    m = k + 300
    # few distinct codes: every distance is shared by hundreds of rows
    palette = rng.integers(0, 256, (5, 4 * words), dtype=np.uint8)
    db = palette[rng.integers(0, 5, m)]
    check(palette[[0, 3]], db, k)
    # all-zero hashes (frames without features): every row at distance 0 from a zero query
    zeros = np.zeros((m, 4 * words), np.uint8)
    idx, dist = check(zeros[:2], zeros, k)
    assert (dist == 0).all() and (idx == np.arange(k)).all()
    # duplicates straddling the k-th place: the k-th distance is shared by rows before and after it
    q = rng.integers(0, 256, (1, 4 * words), dtype=np.uint8)
    near = q.copy()
    near[0, 0] ^= 1                                              # distance 1
    db = rng.integers(0, 256, (m, 4 * words), dtype=np.uint8)
    where = np.sort(rng.choice(m, size=min(m, k + 20), replace=False))
    db[where] = near
    idx, dist = check(q, db, k)
    assert (dist[0] == 1).all() and np.array_equal(idx[0], where[:k])


def test_oracle_extreme_distances():
    for words in (1, 16, 128):
        q = np.random.default_rng(words).integers(0, 256, (2, 4 * words), dtype=np.uint8)
        db = np.concatenate([~q, q])                              # complements first, then the queries themselves
        idx, dist = check(q, db, 4)
        assert dist[0, 0] == 0 and idx[0, 0] == 2 and dist[0, -1] == 32 * words
