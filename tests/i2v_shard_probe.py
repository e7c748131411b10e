"""Builds and loads tests/cuda/i2v_shard_probe.cu: ctypes entry points that run ctr_item_emb_train's numbering steps and
its row scatter from go-ctr_b200/csrc/item2vec.cuh and idmap.cuh (the headers themselves, not copies) on device buffers
the test owns.  Arguments are torch tensors on the GPU (or None for a null pointer); every call synchronises the device."""
import ctypes as C
import os
import subprocess

from tests import shard_probe as sp

ROOT = sp.ROOT
SRC = os.path.join(ROOT, "tests", "cuda", "i2v_shard_probe.cu")
SO = os.path.join(ROOT, "tests", "cuda", "_build", "libi2v_shard_probe.so")
DEPS = [SRC] + [os.path.join(sp.CSRC, h) for h in ("idmap.cuh", "item2vec.cuh", "ubcache.cuh", "common.cuh")]

_lib = None


def build_probe(force=False):
    """Compiles the probe with the library's own flags when it is missing or older than its sources.  Returns
    (path, ptxas -v log or None when nothing was compiled).  Without nvcc an existing library is used as it is."""
    nvcc = sp._nvcc()
    fresh = os.path.exists(SO) and all(os.path.getmtime(SO) >= os.path.getmtime(d) for d in DEPS)
    if nvcc is None:
        if not os.path.exists(SO):
            raise RuntimeError("no nvcc and no %s: build the probe where nvcc is (pytest tests/test_i2v_shard_cpu.py)" % SO)
        return SO, None
    if fresh and not force:
        return SO, None
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    tmp = SO + ".tmp.%d" % os.getpid()                      # built aside and renamed, like go-ctr_b200/build.py
    cmd = [nvcc] + sp._library_flags() + ["-Xptxas", "-v", "-I", sp.CSRC, "-o", tmp, SRC]
    try:
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0:
            raise RuntimeError("probe build failed:\n" + r.stdout)
        os.replace(tmp, SO)
    finally:
        if os.path.exists(tmp):
            os.unlink(tmp)
    return SO, r.stdout


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build_probe()[0])
        L.i2v_shard_probe_error.restype = C.c_char_p
        _lib = L
    return _lib


def _vp(t):
    return C.c_void_p(sp.ptr(t))


def _ll(v):
    return C.c_longlong(int(v))


def _check(rc):
    if rc != 0:
        raise RuntimeError(lib().i2v_shard_probe_error().decode())


def build_map(ids, keys, vals, flags):
    _check(lib().i2v_shard_probe_map(_vp(ids), _ll(ids.numel()), _vp(keys), _vp(vals), C.c_ulonglong(keys.numel()), _vp(flags)))


def local(keys, vals, ids, R, rank, rows, row_tag, side_ids, side_pos):
    """one rank's first tags and side list; returns the number of its distinct side ids"""
    u = C.c_int()
    _check(lib().i2v_shard_probe_local(_vp(keys), _vp(vals), C.c_ulonglong(keys.numel()), _vp(ids), _ll(ids.numel()), _ll(R), rank, _vp(rows),
                                       _vp(row_tag), _vp(side_ids), _vp(side_pos), C.byref(u)))
    return u.value


def merge(g_ids, g_pos, stride, cnt, side_id, side_tag):
    arr = (C.c_int * len(cnt))(*cnt)
    u = C.c_int()
    _check(lib().i2v_shard_probe_merge(_vp(g_ids), _vp(g_pos), _ll(stride), arr, len(cnt), _vp(side_id), _vp(side_tag), C.byref(u)))
    return u.value


def order(keys, vals, row_tag, R, side_id, side_tag, u, world, word_of_row, word_of_side, vocab_ids):
    V = C.c_int()
    _check(lib().i2v_shard_probe_order(_vp(keys), _vp(vals), C.c_ulonglong(keys.numel()), _vp(row_tag), _ll(R), _vp(side_id), _vp(side_tag), _ll(u),
                                       world, _vp(word_of_row), _vp(word_of_side), _vp(vocab_ids), C.byref(V)))
    return V.value


def doc(d, ids, word_of_row, side_id, u, word_of_side):
    _check(lib().i2v_shard_probe_doc(_vp(d), _vp(ids), _ll(ids.numel()), _vp(word_of_row), _vp(side_id), _ll(u), _vp(word_of_side)))


def scatter(syn0, word_of_row, R, D, world, rank, tab):
    _check(lib().i2v_shard_probe_scatter(_vp(syn0), _vp(word_of_row), _ll(R), D, world, rank, _vp(tab)))
