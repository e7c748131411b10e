"""Builds and loads tests/cuda/shard_probe.cu: ctypes entry points that launch the row-sharded kernels of
go-ctr_b200/csrc/attn.cuh, knn.cuh and rec.cuh (the headers themselves, not copies) on device buffers the test owns.
Arguments are torch tensors on the GPU (or None for a null pointer); the kernels run on the default stream and every
call synchronises the device."""
import ctypes as C
import importlib.util
import os
import shutil
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cuda", "shard_probe.cu")
CSRC = os.path.join(ROOT, "go-ctr_b200", "csrc")
SO = os.path.join(ROOT, "tests", "cuda", "_build", "libshard_probe.so")
DEPS = [SRC] + [os.path.join(CSRC, h) for h in ("attn.cuh", "knn.cuh", "rec.cuh", "mlp64.cuh", "common.cuh")]
MAX_PEERS = 8


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
            raise RuntimeError("no nvcc and no %s: build the probe where nvcc is (pytest tests/test_shard_probe_cpu.py)" % SO)
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


class Rows(C.Structure):
    """ProbeRows of shard_probe.cu: what a RowSrc is built from."""
    _fields_ = ([(n, C.c_longlong) for n in ("emb", "ufeat", "ifeat", "user_row", "item_row", "hist", "rows_cache", "hot_tab")]
                + [("peer_emb", C.c_longlong * MAX_PEERS), ("peer_ifeat", C.c_longlong * MAX_PEERS)]
                + [(n, C.c_longlong) for n in ("lde", "ldu", "ldi")]
                + [(n, C.c_int) for n in ("nvalid", "n_emb", "n_user", "n_ifeat", "world", "ifeat_sharded", "hot_k", "pad")])


class Adam(C.Structure):
    _fields_ = [("peer_adam", C.c_longlong * MAX_PEERS), ("rows", C.c_longlong), ("hot_touch", C.c_longlong)]


class RowAdam(C.Structure):
    _fields_ = [(n, C.c_float) for n in ("lr", "b1", "b2", "eps", "c1", "c2", "inv_batch")]


_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build_probe()[0])
        L.shard_probe_error.restype = C.c_char_p
        _lib = L
    return _lib


def ptr(t):
    """device address of a tensor (0 for None)"""
    return 0 if t is None else t.data_ptr()


def _vp(t):
    return C.c_void_p(ptr(t))


def _check(rc):
    if rc != 0:
        raise RuntimeError(lib().shard_probe_error().decode())


def rows(emb=None, lde=0, ufeat=None, ldu=0, ifeat=None, ldi=0, user_row=None, item_row=None, hist=None, rows_cache=None,
         hot_tab=None, peer_emb=(), peer_ifeat=(), nvalid=0, n_emb=0, n_user=0, n_ifeat=0, world=1, ifeat_sharded=0, hot_k=0):
    r = Rows()
    r.emb, r.ufeat, r.ifeat = ptr(emb), ptr(ufeat), ptr(ifeat)
    r.user_row, r.item_row, r.hist, r.rows_cache, r.hot_tab = ptr(user_row), ptr(item_row), ptr(hist), ptr(rows_cache), ptr(hot_tab)
    for j, t in enumerate(peer_emb):
        r.peer_emb[j] = ptr(t)
    for j, t in enumerate(peer_ifeat):
        r.peer_ifeat[j] = ptr(t)
    r.lde, r.ldu, r.ldi = lde, ldu, ldi
    r.nvalid, r.n_emb, r.n_user, r.n_ifeat = nvalid, n_emb, n_user, n_ifeat
    r.world, r.ifeat_sharded, r.hot_k = world, ifeat_sharded, hot_k
    return r


def num_sms():
    return lib().shard_probe_num_sms()


def lanes(bwd, peer, D):
    lpr, vpl = C.c_int(), C.c_int()
    _check(lib().shard_probe_lanes(int(bwd), int(peer), D, C.byref(lpr), C.byref(vpl)))
    return lpr.value, vpl.value


def grad_layout(nrows, lde):
    """ShardGrad of shard_grad_layout(nrows, lde): dict(flag_off, list_off, grad_off, bytes)"""
    out = (C.c_longlong * 4)()
    lib().shard_probe_grad_layout(C.c_longlong(nrows), C.c_longlong(lde), out)
    return dict(zip(("flag_off", "list_off", "grad_off", "bytes"), list(out)))


def fwd_idx(r, model, dims, att, X0, Kp, B, peer, lane_peer=None):
    uP, S, D, cF = dims
    lane_peer = peer if lane_peer is None else lane_peer
    _check(lib().shard_probe_fwd_idx(C.byref(r), model, uP, S, D, cF, _vp(att), _vp(X0), C.c_long(X0.stride(0)), Kp, B,
                                     int(peer), int(lane_peer)))


def bwd_idx(r, model, dims, att, dX, B, peer, datt, dUb=None, dIt=None, neg_lr=1.0, hot_acc=None, hot_rows=0, hot_reps=0, adam=None):
    uP, S, D, cF = dims
    _check(lib().shard_probe_bwd_idx(C.byref(r), model, uP, S, D, cF, _vp(att), _vp(dX), C.c_long(dX.stride(0)), B, int(peer),
                                     _vp(datt), _vp(dUb), _vp(dIt), C.c_float(neg_lr), _vp(hot_acc), hot_rows, hot_reps,
                                     C.byref(adam) if adam is not None else None))


def hot_fold(hot_sum, hot_acc, hot_k, hot_reps, D):
    _check(lib().shard_probe_hot_fold(_vp(hot_sum), _vp(hot_acc), hot_k, hot_reps, D))


def hot_apply_sgd(hot_tab, hot_sum, n):
    _check(lib().shard_probe_hot_apply_sgd(_vp(hot_tab), _vp(hot_sum), C.c_longlong(n)))


def hot_adam(hot_tab, hsum, touch, mo, vo, hot_k, D, ra):
    _check(lib().shard_probe_hot_adam(_vp(hot_tab), _vp(hsum), _vp(touch), _vp(mo), _vp(vo), hot_k, D, C.byref(ra)))


def shard_adam(gbuf, nrows, tab, mo, vo, lde, D, ra):
    _check(lib().shard_probe_shard_adam(_vp(gbuf), C.c_longlong(nrows), _vp(tab), _vp(mo), _vp(vo), C.c_longlong(lde), D, C.byref(ra)))


def hot_pull(r, hot_tab, hot_k, D):
    _check(lib().shard_probe_hot_pull(C.byref(r), _vp(hot_tab), hot_k, D))


def hot_writeback(shard, lde, hot_tab, hot_k, D, world, rank):
    _check(lib().shard_probe_hot_writeback(_vp(shard), C.c_longlong(lde), _vp(hot_tab), hot_k, D, world, rank))


def hot_own(hot, shard, lde, hot_k, D, world, rank):
    _check(lib().shard_probe_hot_own(_vp(hot), _vp(shard), C.c_longlong(lde), hot_k, D, world, rank))


def fwd_user(r, model, dims, att, user, hist, i0, rank, X0, Kp, B, peer):
    uP, S, D, cF = dims
    _check(lib().shard_probe_fwd_user(C.byref(r), model, uP, S, D, cF, _vp(att), user, _vp(hist), i0, rank, _vp(X0),
                                      C.c_long(X0.stride(0)), Kp, B, int(peer)))


def gather_rows_f64(r, rows_, D, out):
    _check(lib().shard_probe_gather_rows_f64(C.byref(r), _vp(rows_), rows_.numel(), D, _vp(out)))


def knn_scan(tab, nrows, world, rank, D, nq, k, rows_per_slice, slices, out_sim, out_row, qvec=None, qrow=None, excl=None):
    _check(lib().shard_probe_knn_scan(_vp(tab), C.c_longlong(tab.stride(0)), C.c_longlong(nrows), world, rank, D, _vp(qvec), _vp(qrow),
                                      _vp(excl), nq, k, C.c_longlong(rows_per_slice), slices, _vp(out_sim), _vp(out_row),
                                      int(qrow is not None)))


def knn_merge(key, in_sim, in_row, slices, k, qstride, sstride, n, out_row, out_sim, out_count=None):
    """key 0: SimKey (float64 similarities), 1: LogitKey (float32 logits)"""
    _check(lib().shard_probe_knn_merge(key, _vp(in_sim), _vp(in_row), slices, k, C.c_longlong(qstride), C.c_longlong(sstride), n,
                                       _vp(out_row), _vp(out_sim), _vp(out_count)))


def rec_scan(z, n, row0, world, rank, rows_per_slice, excl, nex, k, out_s, out_row, run_s=None, run_r=None):
    _check(lib().shard_probe_rec_scan(_vp(z), n, row0, world, rank, rows_per_slice, _vp(excl), nex, k, _vp(run_s), _vp(run_r),
                                      _vp(out_s), _vp(out_row)))
