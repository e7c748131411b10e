"""Builds and loads tests/cuda/auc_dist_probe.cu: ctypes entry points that run the per-rank steps of ctr_roc_auc_dist
and ctr_group_auc_dist (go-ctr_b200/csrc/auc.cuh itself, not a copy) for W ranks emulated as W shards of one device.
Arguments are torch tensors on the GPU; rank r's samples are [cuts[r], cuts[r + 1]).  Every call synchronises the
device."""
import ctypes as C
import os
import subprocess

import numpy as np

from tests import shard_probe

ROOT = shard_probe.ROOT
SRC = os.path.join(ROOT, "tests", "cuda", "auc_dist_probe.cu")
SO = os.path.join(ROOT, "tests", "cuda", "_build", "libauc_dist_probe.so")
DEPS = [SRC] + [os.path.join(shard_probe.CSRC, h) for h in ("auc.cuh", "common.cuh", "owner.cuh")]


def build_probe(force=False):
    """Compiles the probe with the library's own flags when it is missing or older than its sources.  Returns
    (path, ptxas -v log or None when nothing was compiled).  Without nvcc an existing library is used as it is."""
    nvcc = shard_probe._nvcc()
    fresh = os.path.exists(SO) and all(os.path.getmtime(SO) >= os.path.getmtime(d) for d in DEPS)
    if nvcc is None:
        if not os.path.exists(SO):
            raise RuntimeError("no nvcc and no %s: build the probe where nvcc is (pytest tests/test_auc_dist_probe_cpu.py)" % SO)
        return SO, None
    if fresh and not force:
        return SO, None
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    tmp = SO + ".tmp.%d" % os.getpid()                      # built aside and renamed, like go-ctr_b200/build.py
    cmd = [nvcc] + shard_probe._library_flags() + ["-Xptxas", "-v", "-I", shard_probe.CSRC, "-o", tmp, SRC]
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
        L.auc_dist_probe_error.restype = C.c_char_p
        _lib = L
    return _lib


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def roc(pred, y, cuts):
    """(auc, stats): stats[:W] runs sent by each rank, stats[W:2W] merged runs each rank owns, then area2, P, N"""
    W = len(cuts) - 1
    cc = np.ascontiguousarray(cuts, np.int64)
    auc = C.c_double(0)
    stats = np.zeros(2 * W + 3, np.uint64)
    rc = lib().auc_dist_probe_roc(_p(pred), _p(y), cc.ctypes.data_as(C.c_void_p), W, C.byref(auc), stats.ctypes.data_as(C.c_void_p))
    if rc != 0:
        raise RuntimeError(lib().auc_dist_probe_error().decode())
    return auc.value, stats


def gauc(pred, y, group, cuts, outs):
    """(gauc, n_groups, n_used, recv) with the per-group arrays written to outs (torch tensors on the GPU: group, n,
    pos, auc; room for every group)"""
    W = len(cuts) - 1
    cc = np.ascontiguousarray(cuts, np.int64)
    g = C.c_double(0); ng = C.c_longlong(0); nu = C.c_longlong(0)
    recv = np.zeros(W, np.int64)
    rc = lib().auc_dist_probe_gauc(_p(pred), _p(y), _p(group), cc.ctypes.data_as(C.c_void_p), W, C.byref(g), C.byref(ng), C.byref(nu),
                                   _p(outs["group"]), _p(outs["n"]), _p(outs["pos"]), _p(outs["auc"]), recv.ctypes.data_as(C.c_void_p))
    if rc != 0:
        raise RuntimeError(lib().auc_dist_probe_error().decode())
    return g.value, ng.value, nu.value, recv
