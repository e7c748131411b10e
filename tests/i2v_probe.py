"""Builds and loads tests/cuda/i2v_probe.cu: ctypes entry points that launch the item2vec kernels of
go-ctr_b200/csrc/item2vec.cuh (the header itself, not a copy) on arrays the test owns."""
import ctypes as C
import importlib.util
import os
import shutil
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cuda", "i2v_probe.cu")
CSRC = os.path.join(ROOT, "go-ctr_b200", "csrc")
SO = os.path.join(ROOT, "tests", "cuda", "_build", "libi2v_probe.so")
DEPS = [SRC, os.path.join(CSRC, "item2vec.cuh"), os.path.join(CSRC, "common.cuh")]


def _nvcc():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    return nvcc if os.path.exists(nvcc) else shutil.which("nvcc")


def _library_flags():
    spec = importlib.util.spec_from_file_location("_ctr_b200_build", os.path.join(ROOT, "go-ctr_b200", "build.py"))
    mod = importlib.util.module_from_spec(spec); spec.loader.exec_module(mod)
    return list(mod.NVCC_FLAGS)


def build_probe(force=False):
    """Compiles the probe with the library's own flags when it is missing or older than its sources.  Returns
    (path, ptxas -v log or None when nothing was compiled).  Without nvcc an existing library is used as it is."""
    nvcc = _nvcc()
    fresh = os.path.exists(SO) and all(os.path.getmtime(SO) >= os.path.getmtime(d) for d in DEPS)
    if nvcc is None:
        if not os.path.exists(SO):
            raise RuntimeError("no nvcc and no %s: build the probe where nvcc is (pytest tests/test_i2v_pair_model_cpu.py)" % SO)
        return SO, None
    if fresh and not force:
        return SO, None
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    tmp = SO + ".tmp.%d" % os.getpid()                      # built aside and renamed, like go-ctr_b200/build.py
    cmd = [nvcc] + _library_flags() + ["-Xptxas", "-v", "-I", CSRC, "-o", tmp, SRC]
    try:
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0:
            raise RuntimeError("probe build failed:\n" + r.stdout)
        os.replace(tmp, SO)
    finally:
        if os.path.exists(tmp):
            os.unlink(tmp)
    return SO, r.stdout


_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build_probe()[0])
        L.i2v_probe_error.restype = C.c_char_p
        L.i2v_probe_paths.restype = C.c_longlong
        _lib = L
    return _lib


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def skipgram(a, grid, block=256):
    """One launch of k_i2v_skipgram_hs<D/4> on a tests.i2v_pair_model.Launch.  Returns (syn0, syn1, counters[3])."""
    L = lib()
    V, D = a.syn0.shape; nn = a.syn1.shape[0]
    doc = np.ascontiguousarray(a.doc, np.int32); z = np.ascontiguousarray(a.z, np.float64)
    poff = np.ascontiguousarray(a.poff, np.int64); pnode = np.ascontiguousarray(a.pnode, np.int32); pcode = np.ascontiguousarray(a.pcode, np.uint8)
    assert a.syn0.dtype == np.float32 and a.syn1.dtype == np.float32 and z.size == V and poff.size == V + 1
    s0 = np.array(a.syn0, np.float32, order="C"); s1 = np.array(a.syn1, np.float32, order="C")
    lr = np.ascontiguousarray(a.lr_tab, np.float32); ns = np.ascontiguousarray(a.node_scale, np.float32); ws = np.ascontiguousarray(a.word_scale, np.float32)
    assert ns.size == nn and ws.size == V
    ctr = np.zeros(3, np.uint64)
    rc = L.i2v_probe_skipgram(_p(doc, C.c_int), C.c_long(doc.size), _p(z, C.c_double), C.c_int(V), _p(poff, C.c_longlong), _p(pnode, C.c_int),
                              _p(pcode, C.c_ubyte), _p(s0, C.c_float), _p(s1, C.c_float), C.c_int(nn), C.c_int(D), C.c_int(a.W),
                              _p(lr, C.c_float), C.c_int(lr.size), C.c_int(a.upd), _p(ns, C.c_float), _p(ws, C.c_float),
                              C.c_uint(a.seed), C.c_int(a.iter), C.c_int(a.hot_base), C.c_int(a.hot_n), C.c_long(a.pos_begin), C.c_long(a.pos_end),
                              C.c_int(grid), C.c_int(block), _p(ctr, C.c_ulonglong))
    if rc != 0:
        raise RuntimeError(L.i2v_probe_error().decode())
    return s0, s1, [int(x) for x in ctr]


def tables(cnt, subsample, ceff, total, node_val):
    """k_i2v_word_tables + k_i2v_node_scale.  Returns (z float64 [V], word_scale float32 [V], node_scale float32 [nn])."""
    L = lib()
    cnt = np.ascontiguousarray(cnt, np.uint64); nv = np.ascontiguousarray(node_val, np.int64)
    z = np.empty(cnt.size, np.float64); ws = np.empty(cnt.size, np.float32); ns = np.empty(nv.size, np.float32)
    rc = L.i2v_probe_tables(_p(cnt, C.c_ulonglong), C.c_int(cnt.size), C.c_double(subsample), C.c_double(ceff), C.c_double(total),
                            _p(nv, C.c_longlong), C.c_int(nv.size), _p(z, C.c_double), _p(ws, C.c_float), _p(ns, C.c_float))
    if rc != 0:
        raise RuntimeError(L.i2v_probe_error().decode())
    return z, ws, ns


def paths(parent, code, cnt, max_depth):
    """Both passes of k_i2v_paths and the scan between them.  Returns (poff [V+1], pnode, pcode)."""
    L = lib()
    parent = np.ascontiguousarray(parent, np.int32); code = np.ascontiguousarray(code, np.uint8); cnt = np.ascontiguousarray(cnt, np.uint64)
    V = cnt.size
    assert parent.size == 2 * V - 1 and code.size == 2 * V - 1
    cap = V * min(max_depth, 2 * V) + 1
    poff = np.empty(V + 1, np.int64); pnode = np.empty(cap, np.int32); pcode = np.empty(cap, np.uint8)
    n = L.i2v_probe_paths(_p(parent, C.c_int), _p(code, C.c_ubyte), _p(cnt, C.c_ulonglong), C.c_int(V), C.c_int(max_depth),
                          _p(poff, C.c_longlong), _p(pnode, C.c_int), _p(pcode, C.c_ubyte), C.c_longlong(cap))
    if n < 0:
        raise RuntimeError(L.i2v_probe_error().decode())
    return poff, pnode[:n].copy(), pcode[:n].copy()
