"""ctypes binding of the CPU oracle of include/cvb200_lsh.h (oracle/ref_lsh.c in oracle/_build/libcvb_oracle_lsh.so, built by
oracle/lsh.mk): space::LinearKnn over Hamming codes of 32 * words bits, ties in index order.

TEST INFRASTRUCTURE ONLY, like oracle/pyoracle.py.  Codes are uint8 [N, 4 * words].
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "libcvb_oracle_lsh.so")

_L = None


def build(force=False):
    srcs = [os.path.join(_HERE, f) for f in ("ref_lsh.c", "lsh.mk")]
    if not force and os.path.exists(_LIB_PATH) and all(os.path.getmtime(_LIB_PATH) >= os.path.getmtime(s) for s in srcs):
        return _LIB_PATH
    subprocess.check_call(["make", "-s", "-C", _HERE, "-f", "lsh.mk"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


def _lib():
    global _L
    if _L is None:
        build()
        L = C.CDLL(_LIB_PATH)
        u32, vp = C.c_uint32, C.c_void_p
        L.ref_hash_knn.argtypes = [u32, vp, u32, vp, u32, u32, vp, vp]
        L.ref_hash_knn.restype = None
        _L = L
    return _L


def hash_knn(queries, database, k):
    """(idx[N, k], dist[N, k]) uint32: the k nearest database rows of every query, ascending distance, ties -> lower index first;
    0xffffffff where the database has fewer than k rows."""
    q = np.ascontiguousarray(queries, np.uint8)
    db = np.ascontiguousarray(database, np.uint8)
    assert q.ndim == 2 and db.ndim == 2 and q.shape[1] == db.shape[1] and q.shape[1] % 4 == 0
    words = q.shape[1] // 4
    idx = np.empty((len(q), k), np.uint32)
    dist = np.empty((len(q), k), np.uint32)
    _lib().ref_hash_knn(words, q.ctypes.data, len(q), db.ctypes.data, len(db), k, idx.ctypes.data, dist.ctypes.data)
    return idx, dist
