"""Builds and loads tests/cuda/shard_seen_probe.cu: ctypes entry points that launch the CTR_EXCLUDE_SEEN kernels of
go-ctr_b200/csrc/ubcache.cuh and rec.cuh (the headers themselves, not copies) on device buffers the test owns.  Arguments
are torch tensors on the GPU (or None for a null pointer); the kernels run on the default stream and every call
synchronises the device."""
import ctypes as C
import os
import subprocess

from tests import shard_probe

ROOT = shard_probe.ROOT
SRC = os.path.join(ROOT, "tests", "cuda", "shard_seen_probe.cu")
SO = os.path.join(ROOT, "tests", "cuda", "_build", "libshard_seen_probe.so")
DEPS = [SRC] + [os.path.join(shard_probe.CSRC, h) for h in ("rec.cuh", "ubcache.cuh", "knn.cuh", "mlp64.cuh", "attn.cuh", "common.cuh")]


def build_probe(force=False):
    """Compiles the probe with the library's own flags when it is missing or older than its sources.  Returns
    (path, ptxas -v log or None when nothing was compiled).  Without nvcc an existing library is used as it is."""
    nvcc = shard_probe._nvcc()
    fresh = os.path.exists(SO) and all(os.path.getmtime(SO) >= os.path.getmtime(d) for d in DEPS)
    if nvcc is None:
        if not os.path.exists(SO):
            raise RuntimeError("no nvcc and no %s: build the probe where nvcc is (pytest tests/test_shard_seen_probe_cpu.py)" % SO)
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
        L.shard_seen_probe_error.restype = C.c_char_p
        _lib = L
    return _lib


def _vp(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def _ll(v):
    return C.c_longlong(int(v))


def _check(rc):
    if rc != 0:
        raise RuntimeError(lib().shard_seen_probe_error().decode())


def build_seen(cache, u, max_ts, hist, S, n_items, world, rank, n_local, seen):
    """cache: (off, ts, items) device tensors, or None for a rank without a cache"""
    off, ts, items = cache if cache is not None else (None, None, None)
    n_users = 0 if off is None else off.numel() - 1
    ne = 0 if ts is None else ts.numel()
    _check(lib().shard_seen_probe_build(_vp(off), _vp(ts), _vp(items), _ll(n_users), _ll(ne), u, _ll(max_ts), _vp(hist), S, _ll(n_items),
                                        world, rank, _ll(n_local), _vp(seen)))


def scan(one, z, n, row0, world, rank, rps, seen, k, run_s, run_r, out_s, out_row):
    _check(lib().shard_seen_probe_scan(int(one), _vp(z), n, row0, world, rank, rps, _vp(seen), k, _vp(run_s), _vp(run_r), _vp(out_s), _vp(out_row)))


def merge(in_s, in_row, slices, k, qstride, sstride, n, out_row, out_s, out_count=None):
    _check(lib().shard_seen_probe_merge(_vp(in_s), _vp(in_row), slices, k, _ll(qstride), _ll(sstride), n, _vp(out_row), _vp(out_s), _vp(out_count)))


def target_logits(z, n, row0, world, rank, rows, m, tl, seen, flag):
    _check(lib().shard_seen_probe_target_logits(_vp(z), n, row0, world, rank, _vp(rows), m, _vp(tl), _vp(seen), _vp(flag)))


def sort(one, rows, tl, tls, world, m, n_items, flag, seen, place, nvalid, ss, sr, bins):
    _check(lib().shard_seen_probe_sort(int(one), _vp(rows), _vp(tl), tls, world, m, _ll(n_items), _vp(flag), _vp(seen), _vp(place), _vp(nvalid),
                                       _vp(ss), _vp(sr), _vp(bins)))


def count(one, z, n, row0, world, rank, seen, ss, sr, nvalid, bins):
    _check(lib().shard_seen_probe_count(int(one), _vp(z), n, row0, world, rank, _vp(seen), _vp(ss), _vp(sr), _vp(nvalid), _vp(bins)))


def finish(rows, tl, tls, world, place, m, n_items, bins, out_rank, out_logit):
    _check(lib().shard_seen_probe_finish(_vp(rows), _vp(tl), tls, world, _vp(place), m, _ll(n_items), _vp(bins), _vp(out_rank), _vp(out_logit)))
