"""Host-side mirror of space::LinearKnn + bitarray::Hamming and the match filters built on it."""
import ctypes as C

import numpy as np

from ._lib import default_context


def _desc(a):
    a = np.ascontiguousarray(a, dtype=np.uint8)
    if a.ndim != 2 or a.shape[1] != 64:
        raise ValueError("descriptors must be [N, 64] uint8 (BitArray<64>)")
    return a


def hamming_knn(queries, database, k=2, ctx=None):
    """All-queries form of `LinearKnn{metric: Hamming, iter: database}.knn(q, k)`.

    Returns (index[N,k], distance[N,k]) uint32, ascending distance, ties -> lower index first
    (space 0.17 LinearKnn; call sites akaze/tests/estimate_pose.rs:82-86).  Missing neighbours
    (database smaller than k) are 0xffffffff.
    """
    q, db = _desc(queries), _desc(database)
    ctx = ctx or default_context(0)
    idx = np.empty((len(q), k), np.uint32)
    dist = np.empty((len(q), k), np.uint32)
    ctx.check(ctx.lib.cvb_hamming_knn(ctx.handle, q.ctypes.data, len(q), db.ctypes.data, len(db), k, idx.ctypes.data,
                                      dist.ctypes.data))
    return idx, dist


class LinearKnn:
    """space::LinearKnn { metric: Hamming, iter } -- `knn(query, num)` yields Neighbor{index, distance}."""

    def __init__(self, database, ctx=None):
        self.database = _desc(database)
        self.ctx = ctx

    def knn(self, query, num):
        idx, dist = hamming_knn(np.asarray(query, np.uint8).reshape(1, 64), self.database, num, self.ctx)
        return [(int(i), int(d)) for i, d in zip(idx[0], dist[0]) if i != 0xFFFFFFFF]

    def knn_batch(self, queries, num):
        return hamming_knn(queries, self.database, num, self.ctx)

    def nn(self, query):
        r = self.knn(query, 1)
        return r[0] if r else None


def lowe_ratio_matches(ds1, ds2, ratio=0.5, ctx=None):
    """akaze/tests/estimate_pose.rs:78-97 `match_descriptors`: 2-NN + Lowe ratio in f32, -> [(ix1, ix2), ...]."""
    idx, dist = hamming_knn(ds1, ds2, 2, ctx)
    ok = dist[:, 0].astype(np.float32) < dist[:, 1].astype(np.float32) * np.float32(ratio)
    return [(int(i), int(idx[i, 0])) for i in np.where(ok)[0]]


def matching(a, b, better_by=24, strict=False, ctx=None):
    """cv-sfm `matching` (cv-sfm/src/lib.rs:3097-3114: d0 + better_by <= d1); strict=True gives the
    tutorial rule d0 + 24 < d1 (chapter4 main.rs:99).  Returns an int64 array, -1 where None."""
    a, b = _desc(a), _desc(b)
    if len(a) < 2 or len(b) < 2:
        return np.zeros(0, np.int64)
    idx, dist = hamming_knn(a, b, 2, ctx)
    d0, d1 = dist[:, 0].astype(np.int64), dist[:, 1].astype(np.int64)
    good = (d0 + better_by < d1) if strict else (d0 + better_by <= d1)
    return np.where(good, idx[:, 0].astype(np.int64), -1)


def symmetric_matching(a, b, better_by=24, ctx=None):
    """cv-sfm `symmetric_matching` (cv-sfm/src/lib.rs:3116-3133): [[aix, bix], ...] in ascending aix."""
    a, b = _desc(a), _desc(b)
    ctx = ctx or default_context(0)
    cap = max(len(a), 1)
    pairs = np.empty((cap, 2), np.uint32)
    n = C.c_uint32()
    ctx.check(ctx.lib.cvb_match_symmetric(ctx.handle, a.ctypes.data, len(a), b.ctypes.data, len(b), better_by,
                                          pairs.ctypes.data, cap, C.byref(n)))
    return pairs[:n.value].astype(np.int64)


class HammingHasher:
    """hamming_lsh::HammingHasher<64, H>::new_with_codewords(codewords) (cv-sfm/src/lib.rs:205,216): `hash_bag(features)` sets, for
    every feature, the bit of its nearest codeword (first minimum on ties).  codewords: [H * 8, 64] uint8."""

    def __init__(self, codewords, ctx=None):
        self.codewords = _desc(codewords)
        if len(self.codewords) == 0 or len(self.codewords) % 32:
            raise ValueError("the number of codewords must be a positive multiple of 32")
        self.ctx = ctx

    def hash_bag(self, features):
        f = np.ascontiguousarray(features, np.uint8).reshape(-1, 64)
        ctx = self.ctx or default_context(0)
        out = np.zeros(len(self.codewords) // 8, np.uint8)
        ctx.check(ctx.lib.cvb_hash_bag(ctx.handle, f.ctypes.data, len(f), self.codewords.ctypes.data, len(self.codewords), out.ctypes.data))
        return out


# ---- exact k-NN over wide codes: cv-sfm's similar-frame search (include/cvb200_lsh.h, libcvb200_lsh.so) ----

MAX_WORDS = 128   # CVB_LSH_MAX_WORDS: 4096-bit codes, cv-sfm's frame hash
MAX_K = 1024      # CVB_LSH_MAX_K


def _lsh_lib():
    from ._lib import load_lsh_library
    L = load_lsh_library()
    if not getattr(L, "_lsh_bound", False):
        vp, u32 = C.c_void_p, C.c_uint32
        L.cvb_hash_knn.argtypes = [vp, u32, vp, u32, vp, u32, u32, vp, vp]
        L.cvb_hash_knn_dev.argtypes = [vp, u32, vp, vp, u32, vp, vp, u32, u32, vp, vp]
        L._lsh_bound = True
    return L


def _codes(a, name):
    a = np.asarray(a)
    if a.dtype != np.uint8:
        raise TypeError(f"{name} are uint8 codes, not {a.dtype}")
    if a.ndim != 2 or a.shape[1] == 0 or a.shape[1] % 4 or a.shape[1] > 4 * MAX_WORDS:
        raise ValueError(f"{name} are [N, 4 * words] uint8 with 1 <= words <= {MAX_WORDS}, not {a.shape}")
    return np.ascontiguousarray(a)


def hash_knn(queries, database, k, ctx=None):
    """Exact k-NN of every query among the database codes: `LinearKnn{metric: Hamming, iter: database}.knn(q, k)` over
    BitArray<4 * words>, the search behind cv-sfm's `lsh_to_frame.knn_values` (cv-sfm/src/lib.rs:597-668).

    queries [N, 4 * words], database [M, 4 * words]: uint8 (cvb_hash_bag's byte layout), words <= 128; 1 <= k <= 1024.
    Returns (index[N, k], distance[N, k]) uint32 in ascending distance, ties -> lower database index first; 0xffffffff past M.
    Parity with the reference is unpinned: cv-sfm's HGG is approximate, and LinearKnn leaves the order of ties beyond k = 20 to
    pdqsort; here ties are always in index order."""
    q, db = _codes(queries, "queries"), _codes(database, "database")
    if q.shape[1] != db.shape[1]:
        raise ValueError(f"queries and database differ in width: {q.shape[1]} != {db.shape[1]} bytes")
    ctx = ctx or default_context(0)
    idx = np.empty((len(q), k), np.uint32)
    dist = np.empty((len(q), k), np.uint32)
    ctx.check(_lsh_lib().cvb_hash_knn(ctx.handle, q.shape[1] // 4, q.ctypes.data, len(q), db.ctypes.data, len(db), k, idx.ctypes.data,
                                      dist.ctypes.data))
    return idx, dist


class FrameHashIndex:
    """cv-sfm's `lsh_to_frame: HggLite<Hamming, BitArray<512>, FrameKey>` (cv-sfm/src/lib.rs:207) answered exactly on the device:
    `insert(lsh, value)` (lib.rs:684) and `knn_values(lsh, num) -> [(distance, value), ...]` (lib.rs:597-668), nearest first, ties in
    insertion order.  The hashes live in one device buffer that doubles when full; `insert_dev` appends a hash that is already on the
    device (such as a row cvb_hash_bag_dev wrote) without a host round trip.  Values stay on the host, in insertion order.

    The index runs on its own context, whose stream torch also sees (`self.stream`); a device row given to insert_dev is read on that
    stream.  The filtering cv-sfm applies after the search (recent frames, same-feed threshold, take) stays with the caller."""

    def __init__(self, words=MAX_WORDS, device=0, capacity=64):
        import torch
        from .multi import make_context
        if not 1 <= words <= MAX_WORDS:
            raise ValueError(f"words must be 1..{MAX_WORDS}")
        self.words = words
        self.ctx = make_context(device)
        self.stream = self.ctx.torch_stream
        self.device = torch.device("cuda", device)
        with torch.cuda.stream(self.stream):
            self._db = torch.zeros((max(capacity, 1), 4 * words), dtype=torch.uint8, device=self.device)
        self._values = []

    def __len__(self):
        return len(self._values)

    def _slot(self):
        import torch
        m = len(self._values)
        if m == len(self._db):
            with torch.cuda.stream(self.stream):
                grown = torch.zeros((2 * len(self._db), 4 * self.words), dtype=torch.uint8, device=self.device)
                grown[:m].copy_(self._db)
            self._db = grown
        return self._db[m]

    def insert(self, lsh, value):
        import torch
        h = np.ascontiguousarray(lsh, np.uint8).reshape(-1)
        if h.size != 4 * self.words:
            raise ValueError(f"a hash is {4 * self.words} bytes, not {h.size}")
        with torch.cuda.stream(self.stream):
            self._slot().copy_(torch.from_numpy(h).to(self.device, non_blocking=False))
        self._values.append(value)

    def insert_dev(self, row, value):
        """row: a uint8 cuda tensor of 4 * words bytes on the index's device."""
        import torch
        if not (isinstance(row, torch.Tensor) and row.is_cuda and row.dtype == torch.uint8 and row.numel() == 4 * self.words):
            raise ValueError(f"insert_dev takes a uint8 cuda tensor of {4 * self.words} bytes")
        with torch.cuda.stream(self.stream):
            self._slot().copy_(row.reshape(-1))
        self._values.append(value)

    def knn_values(self, lsh, num):
        """The `num` nearest hashes as [(distance, value), ...], nearest first, equal distances in insertion order."""
        import torch
        h = np.ascontiguousarray(lsh, np.uint8).reshape(-1)
        if h.size != 4 * self.words:
            raise ValueError(f"a hash is {4 * self.words} bytes, not {h.size}")
        m = len(self._values)
        with torch.cuda.stream(self.stream):
            q = torch.from_numpy(h).to(self.device).reshape(1, -1)
            idx = torch.empty((1, num), dtype=torch.int32, device=self.device)
            dist = torch.empty((1, num), dtype=torch.int32, device=self.device)
            self.ctx.check(_lsh_lib().cvb_hash_knn_dev(self.ctx.handle, self.words, q.data_ptr(), None, 1, self._db.data_ptr(), None, m,
                                                       num, idx.data_ptr(), dist.data_ptr()))
            ix, ds = idx.cpu().numpy().view(np.uint32)[0], dist.cpu().numpy().view(np.uint32)[0]
        return [(int(d), self._values[int(i)]) for i, d in zip(ix, ds) if i != 0xFFFFFFFF]
