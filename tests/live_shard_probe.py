"""Builds and loads tests/cuda/live_shard_probe.cu: ctypes entry points that launch the collective live-table kernels of
go-ctr_b200/csrc/idmap.cuh, item2vec.cuh, attn.cuh and vmm.cuh (the headers themselves, not copies) on device buffers the
test owns.  Arguments are torch tensors on the GPU (or None for a null pointer); every call synchronises the device."""
import ctypes as C
import os

from tests import shard_probe as sp

ROOT = sp.ROOT
SRC = os.path.join(ROOT, "tests", "cuda", "live_shard_probe.cu")
SO = os.path.join(ROOT, "tests", "cuda", "_build", "liblive_shard_probe.so")
DEPS = [SRC] + [os.path.join(sp.CSRC, h) for h in ("attn.cuh", "idmap.cuh", "item2vec.cuh", "vmm.cuh", "common.cuh")]

_lib = None


def build_probe():
    """Compiles the probe with the library's own flags when it is missing or older than its sources."""
    nvcc = sp._nvcc()
    fresh = os.path.exists(SO) and all(os.path.getmtime(SO) >= os.path.getmtime(d) for d in DEPS)
    if fresh or nvcc is None:
        if not os.path.exists(SO):
            raise RuntimeError("no nvcc and no %s" % SO)
        return SO
    import subprocess
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    tmp = SO + ".tmp.%d" % os.getpid()
    try:
        r = subprocess.run([nvcc] + sp._library_flags() + ["-I", sp.CSRC, "-o", tmp, SRC], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0:
            raise RuntimeError("probe build failed:\n" + r.stdout)
        os.replace(tmp, SO)
    finally:
        if os.path.exists(tmp):
            os.unlink(tmp)
    return SO


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build_probe())
        L.live_probe_error.restype = C.c_char_p
        _lib = L
    return _lib


def _vp(t):
    return C.c_void_p(sp.ptr(t))


def _check(rc):
    if rc != 0:
        raise RuntimeError(lib().live_probe_error().decode())


def number(keys, vals, ids, rows, out_ids, out_pos):
    """one rank's numbering (keys None: no map); returns (ids without a row, distinct missing ids)"""
    m, u = C.c_longlong(), C.c_int()
    cap = keys.numel() if keys is not None else 0
    _check(lib().live_probe_number(_vp(keys), _vp(vals), C.c_ulonglong(cap), _vp(ids), C.c_longlong(ids.numel()), _vp(rows), _vp(out_ids),
                                   _vp(out_pos), C.byref(m), C.byref(u)))
    return m.value, u.value


def order(ids, pos, u, out_ids):
    _check(lib().live_probe_order(_vp(ids), _vp(pos), u, _vp(out_ids)))


def merge(g_ids, g_pos, stride, cnt, out_ids):
    arr = (C.c_int * len(cnt))(*cnt)
    u = C.c_int()
    _check(lib().live_probe_merge(_vp(g_ids), _vp(g_pos), C.c_longlong(stride), arr, len(cnt), _vp(out_ids), C.byref(u)))
    return u.value


def add(old_keys, old_vals, keys, vals, fresh, u, R, flags):
    oc = old_keys.numel() if old_keys is not None else 0
    _check(lib().live_probe_add(_vp(old_keys), _vp(old_vals), C.c_ulonglong(oc), _vp(keys), _vp(vals), C.c_ulonglong(keys.numel()),
                                _vp(fresh), u, R, _vp(flags)))


def dump(keys, vals, ids):
    _check(lib().live_probe_dump(_vp(keys), _vp(vals), C.c_ulonglong(keys.numel()), _vp(ids)))


def lookup(keys, vals, ids, rows):
    _check(lib().live_probe_lookup(_vp(keys), _vp(vals), C.c_ulonglong(keys.numel()), _vp(ids), C.c_longlong(ids.numel()), _vp(rows)))


def digest(keys, vals, out):
    _check(lib().live_probe_digest(_vp(keys), _vp(vals), C.c_ulonglong(keys.numel()), _vp(out)))


def write(t, rows, data, world=1, rank=0, mo=None, vo=None, hot=None, hot_k=0, hm=None, hv=None):
    _check(lib().live_probe_write(_vp(t), C.c_longlong(t.stride(0)), _vp(rows), _vp(data), C.c_longlong(rows.numel()), data.shape[1], world, rank,
                                  _vp(mo), _vp(vo), _vp(hot), hot_k, _vp(hm), _vp(hv)))


def grow(host, want, dev=0):
    """vmm_grow_rows on a shard filled from host [rows, width] float32: (grown [want, width], old bytes, new bytes, granule)"""
    import numpy as np
    rows, width = host.shape
    out = np.empty((want, width), np.float32)
    ob, nb, g = C.c_longlong(), C.c_longlong(), C.c_longlong()
    _check(lib().live_probe_grow(host.ctypes.data_as(C.c_void_p), C.c_longlong(rows), C.c_longlong(want), C.c_longlong(width * 4), dev,
                                 out.ctypes.data_as(C.c_void_p), C.byref(ob), C.byref(nb), C.byref(g)))
    return out, ob.value, nb.value, g.value
