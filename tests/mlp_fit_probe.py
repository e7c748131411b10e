"""Builds and loads tests/cuda/mlp_fit_probe.cu: a ctypes entry point that launches the key-fed fit's minibatch gather of
go-ctr_b200/csrc/attn.cuh (the header itself, not a copy) on device buffers the test owns.  Arguments are torch tensors
on the GPU (or None for a null pointer); the kernel runs on the default stream and every call synchronises the device.
Row sources are tests/shard_probe.py Rows."""
import ctypes as C
import os
import subprocess

from tests import shard_probe

ROOT = shard_probe.ROOT
SRC = os.path.join(ROOT, "tests", "cuda", "mlp_fit_probe.cu")
SO = os.path.join(ROOT, "tests", "cuda", "_build", "libmlp_fit_probe.so")
DEPS = [SRC] + [os.path.join(shard_probe.CSRC, h) for h in ("attn.cuh", "common.cuh")]


def build_probe(force=False):
    """Compiles the probe with the library's own flags when it is missing or older than its sources.  Returns
    (path, ptxas -v log or None when nothing was compiled).  Without nvcc an existing library is used as it is."""
    nvcc = shard_probe._nvcc()
    fresh = os.path.exists(SO) and all(os.path.getmtime(SO) >= os.path.getmtime(d) for d in DEPS)
    if nvcc is None:
        if not os.path.exists(SO):
            raise RuntimeError("no nvcc and no %s: build the probe where nvcc is (pytest tests/test_mlp_fit_probe_cpu.py)" % SO)
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
        L.mlp_fit_probe_error.restype = C.c_char_p
        _lib = L
    return _lib


def gather(r, peer, dims, bi, X, rows):
    """X[:rows] = the float64 rows of samples bi[:rows] (bi an int64 tensor; a slice starts a later minibatch)"""
    uP, S, D, cF = dims
    rc = lib().mlp_fit_probe_gather(C.byref(r), int(peer), uP, S, D, cF, C.c_void_p(bi.data_ptr()), C.c_void_p(X.data_ptr()),
                                    C.c_longlong(X.stride(0)), rows)
    if rc != 0:
        raise RuntimeError(lib().mlp_fit_probe_error().decode())
