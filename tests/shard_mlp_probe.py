"""Builds and loads tests/cuda/shard_mlp_probe.cu: ctypes entry points that launch the float64 MLP's serving kernels of
go-ctr_b200/csrc/attn.cuh, mlp64.cuh and rec.cuh (the headers themselves, not copies) on device buffers the test owns.
Arguments are torch tensors on the GPU (or None for a null pointer); the kernels run on the default stream and every
call synchronises the device.  Row sources are tests/shard_probe.py Rows."""
import ctypes as C
import os
import subprocess

from tests import shard_probe

ROOT = shard_probe.ROOT
SRC = os.path.join(ROOT, "tests", "cuda", "shard_mlp_probe.cu")
SO = os.path.join(ROOT, "tests", "cuda", "_build", "libshard_mlp_probe.so")
DEPS = [SRC] + [os.path.join(shard_probe.CSRC, h) for h in ("attn.cuh", "rec.cuh", "knn.cuh", "mlp64.cuh", "common.cuh")]


def build_probe(force=False):
    """Compiles the probe with the library's own flags when it is missing or older than its sources.  Returns
    (path, ptxas -v log or None when nothing was compiled).  Without nvcc an existing library is used as it is."""
    nvcc = shard_probe._nvcc()
    fresh = os.path.exists(SO) and all(os.path.getmtime(SO) >= os.path.getmtime(d) for d in DEPS)
    if nvcc is None:
        if not os.path.exists(SO):
            raise RuntimeError("no nvcc and no %s: build the probe where nvcc is (pytest tests/test_shard_mlp_probe_cpu.py)" % SO)
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
        L.shard_mlp_probe_error.restype = C.c_char_p
        _lib = L
    return _lib


def _vp(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def _ll(v):
    return C.c_longlong(int(v))


def _check(rc):
    if rc != 0:
        raise RuntimeError(lib().shard_mlp_probe_error().decode())


class Net:
    """a network's shape for the probe: units [n_layers], the hidden and output activations"""

    def __init__(self, units, hidden_act=0, out_act=1):
        self.units = (C.c_int * 8)(*units)
        self.n = len(units)
        self.hidden_act, self.out_act = hidden_act, out_act


def gather(r, peer, dims, X, B):
    uP, S, D, cF = dims
    _check(lib().shard_mlp_probe_gather(C.byref(r), int(peer), uP, S, D, cF, _vp(X), _ll(X.stride(0)), B))


def prefix(peer, params, net, urow, uP, r, hist, S, D, pre):
    _check(lib().shard_mlp_probe_prefix(int(peer), _vp(params), net.n, net.units, net.hidden_act, net.out_act, _vp(urow), uP, C.byref(r),
                                        _vp(hist), S, D, _vp(pre)))


def score(smem_w, params, net, pre, pcols, emb, ifeat, n_ifeat, fworld, frank, D, cF, row0, n, ctas, acts, z):
    _check(lib().shard_mlp_probe_score(int(smem_w), _vp(params), net.n, net.units, net.hidden_act, net.out_act, _vp(pre), pcols, _vp(emb),
                                       _ll(emb.stride(0)), _vp(ifeat), _ll(0 if ifeat is None else ifeat.stride(0)), _ll(n_ifeat), fworld, frank,
                                       D, cF, _ll(row0), n, ctas, _vp(acts), _vp(z)))


def scan(z, n, row0, world, rank, rps, excl, nex, seen, k, run_s, run_r, out_s, out_row):
    _check(lib().shard_mlp_probe_scan(_vp(z), n, row0, world, rank, rps, _vp(excl), nex, _vp(seen), k, _vp(run_s), _vp(run_r), _vp(out_s),
                                      _vp(out_row)))


def merge(in_s, in_row, slices, k, qstride, sstride, n, out_row, out_s, out_count=None):
    _check(lib().shard_mlp_probe_merge(_vp(in_s), _vp(in_row), slices, k, _ll(qstride), _ll(sstride), n, _vp(out_row), _vp(out_s), _vp(out_count)))


def target_logits(z, n, row0, world, rank, rows, m, tl, seen, flag):
    _check(lib().shard_mlp_probe_target_logits(_vp(z), n, row0, world, rank, _vp(rows), m, _vp(tl), _vp(seen), _vp(flag)))


def sort(rows, tl, tls, world, m, n_items, excl, nex, flag, place, nvalid, ss, sr, bins):
    _check(lib().shard_mlp_probe_sort(_vp(rows), _vp(tl), tls, world, m, _ll(n_items), _vp(excl), nex, _vp(flag), _vp(place), _vp(nvalid),
                                      _vp(ss), _vp(sr), _vp(bins)))


def count(z, n, row0, world, rank, excl, nex, seen, ss, sr, nvalid, bins):
    _check(lib().shard_mlp_probe_count(_vp(z), n, row0, world, rank, _vp(excl), nex, _vp(seen), _vp(ss), _vp(sr), _vp(nvalid), _vp(bins)))


def finish(rows, tl, tls, world, place, m, n_items, bins, out_rank, out_logit):
    _check(lib().shard_mlp_probe_finish(_vp(rows), _vp(tl), tls, world, _vp(place), m, _ll(n_items), _vp(bins), _vp(out_rank), _vp(out_logit)))
