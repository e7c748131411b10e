"""ctypes binding of the search.Searcher oracle (oracle/knn_oracle.c).  TEST INFRASTRUCTURE ONLY: imported by tests/
and tests/tools, never by the product package.  Built next to liborc.so by __graft_entry__.build()."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "knn_oracle.c")
_SO = os.path.join(_HERE, "_build", "libknn_orc.so")
CFLAGS = ["-O2", "-std=c99", "-fPIC", "-fopenmp", "-ffp-contract=off", "-Wall", "-Wextra", "-shared"]


def build(force=False):
    if not force and os.path.exists(_SO) and os.path.getmtime(_SO) >= os.path.getmtime(_SRC):
        return _SO
    os.makedirs(os.path.dirname(_SO), exist_ok=True)
    tmp = _SO + ".tmp.%d" % os.getpid()
    try:
        subprocess.check_call(["/usr/bin/gcc"] + CFLAGS + ["-o", tmp, _SRC, "-lm"])
        os.replace(tmp, _SO)
    finally:
        if os.path.exists(tmp):
            os.unlink(tmp)
    return _SO


_lib = None
_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int32)


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        L.orc_knn_norm.restype = C.c_double
        L.orc_knn_norm.argtypes = [_dp, C.c_int]
        L.orc_knn_cosine.restype = C.c_double
        L.orc_knn_cosine.argtypes = [_dp, _dp, C.c_double, C.c_double, C.c_int]
        L.orc_knn_search.restype = None
        L.orc_knn_search.argtypes = [C.POINTER(C.c_float), C.c_long, C.c_int, _dp, _ip, C.c_long, C.c_int, _ip, _dp, _ip]
        _lib = L
    return _lib


def norm(v):
    v = np.ascontiguousarray(v, np.float64)
    return lib().orc_knn_norm(v.ctypes.data_as(_dp), v.size)


def cosine(v1, v2):
    a = np.ascontiguousarray(v1, np.float64); b = np.ascontiguousarray(v2, np.float64)
    return lib().orc_knn_cosine(a.ctypes.data_as(_dp), b.ctypes.data_as(_dp), norm(a), norm(b), a.size)


def search(table, queries, k, ignore=None):
    """search.go's Search over the float32 table [N, D] for float64 queries [nq, D]; ignore: per query a row to skip
    (-1: none).  Returns (rows [nq, k] int32, sims [nq, k] float64, counts [nq] int32), empty slots -1 / 0."""
    t = np.ascontiguousarray(table, np.float32)
    q = np.ascontiguousarray(queries, np.float64)
    q = q.reshape(1, -1) if q.ndim == 1 else q
    N, D = t.shape
    assert q.shape[1] == D
    nq = q.shape[0]
    ig = None if ignore is None else np.ascontiguousarray(np.broadcast_to(ignore, (nq,)), np.int32)
    rows = np.empty((nq, k), np.int32); sims = np.empty((nq, k), np.float64); cnt = np.empty(nq, np.int32)
    lib().orc_knn_search(t.ctypes.data_as(C.POINTER(C.c_float)), N, D, q.ctypes.data_as(_dp),
                         None if ig is None else ig.ctypes.data_as(_ip), nq, k, rows.ctypes.data_as(_ip),
                         sims.ctypes.data_as(_dp), cnt.ctypes.data_as(_ip))
    return rows, sims, cnt
