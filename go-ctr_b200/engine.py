"""ctypes binding of libctr_b200.so (include/ctr_b200.h).  This is the same C ABI the cgo shim
binds (go/ctrb200/ctrb200.go); Python is only the test / bench harness language here because the
image has no Go toolchain.  There is no CPU fallback: if the shared library is missing or no H100
is present, construction raises."""
import ctypes as C
import os

import numpy as np

from . import build as _build

__all__ = ["Engine", "Config", "MLPClassifier", "MLPRegressor", "MlpConfig", "MlpOptions", "StepStats", "CtrError", "load_library", "MODEL_YOUTUBE", "MODEL_DIN_COS",
           "MODEL_DIN_EUC", "TABLE_USER_FEAT", "TABLE_ITEM_FEAT", "TABLE_ITEM_EMB", "TABLE_FROZEN", "TABLE_SGD",
           "TABLE_SGD_DETERMINISTIC", "TABLE_ADAM", "GEMM_AUTO", "GEMM_FP32", "GEMM_TCGEN05_3XTF32", "EXPORTS", "IDMAP_USER", "IDMAP_ITEM", "ENOTFOUND", "EINVAL", "ESTATE", "rank_metrics",
           "EXCLUDE_NONE", "EXCLUDE_WINDOW", "EXCLUDE_SEEN", "AVERAGE", "MULTIOUTPUT", "ERROR_KIND"]

MODEL_YOUTUBE, MODEL_DIN_COS, MODEL_DIN_EUC = 0, 1, 2
TABLE_USER_FEAT, TABLE_ITEM_FEAT, TABLE_ITEM_EMB = 0, 1, 2
TABLE_FROZEN, TABLE_SGD, TABLE_SGD_DETERMINISTIC, TABLE_ADAM = 0, 1, 2, 3
GEMM_AUTO, GEMM_FP32, GEMM_TCGEN05_3XTF32 = 0, 1, 2
IDMAP_USER, IDMAP_ITEM = 0, 1
EINVAL, ESTATE, ENOTFOUND = 1, 5, 7
EXCLUDE_NONE, EXCLUDE_WINDOW, EXCLUDE_SEEN = 0, 1, 2
AVERAGE = {"macro": 0, "micro": 1, "weighted": 2}                                 # CTR_AVERAGE_*
MULTIOUTPUT = {"raw_values": 0, "uniform_average": 1, "variance_weighted": 2}      # CTR_MULTIOUTPUT_*
ERROR_KIND = {"squared": 0, "absolute": 1}                                        # CTR_ERROR_*

# every symbol include/ctr_b200.h declares (tests check the .so exports all of them)
EXPORTS = ["ctr_abi_version", "ctr_config_default", "ctr_create", "ctr_destroy", "ctr_last_error",
           "ctr_init_weights", "ctr_set_weights", "ctr_get_weights", "ctr_table_upload", "ctr_table_download", "ctr_table_fill",
           "ctr_gather_rows", "ctr_train_dense", "ctr_predict_dense", "ctr_train_step_idx", "ctr_train_idx", "ctr_train_keys", "ctr_predict_idx",
           "ctr_train_step_idx_dev", "ctr_predict_idx_dev", "ctr_last_cost", "ctr_sync", "ctr_get_stream",
           "ctr_set_stream", "ctr_launch_count", "ctr_profile_enable", "ctr_profile_get", "ctr_profile_reset",
           "ctr_profile_dump", "ctr_debug_grads_idx", "ctr_ubcache_upload", "ctr_ubcache_window", "ctr_ubcache_window_dev", "ctr_ubcache_append", "ctr_ubcache_set", "ctr_ubcache_download", "ctr_idmap_build", "ctr_idmap_lookup", "ctr_idmap_lookup_dev",
           "ctr_idmap_insert", "ctr_idmap_download", "ctr_table_write_rows",
           "ctr_batch_predict_keys", "ctr_checkpoint_save", "ctr_checkpoint_load", "ctr_roc_auc", "ctr_group_auc", "ctr_roc_auc_dist", "ctr_group_auc_dist", "ctr_roc_curve", "ctr_pr_curve", "ctr_average_precision", "ctr_group_average_precision", "ctr_accuracy_score", "ctr_confusion_matrix", "ctr_precision_recall_fscore", "ctr_r2_score", "ctr_mean_error", "ctr_knn_search", "ctr_recommend_topk", "ctr_rank_items", "ctr_recommend_topk_ex", "ctr_rank_items_ex", "ctr_rank_metrics", "ctr_i2v_config_default", "ctr_i2v_paths", "ctr_i2v_train", "ctr_i2v_train_dist", "ctr_item_emb_train", "ctr_item_emb_vocab", "ctr_comm_unique_id", "ctr_comm_init",
           "ctr_mlp_config_default", "ctr_mlp_options_default", "ctr_mlp_create", "ctr_mlp_create_ex", "ctr_mlp_destroy", "ctr_mlp_last_error", "ctr_mlp_fit", "ctr_mlp_predict",
           "ctr_mlp_get_params", "ctr_mlp_set_params", "ctr_mlp_fit_keys", "ctr_mlp_fit_keys_dist", "ctr_mlp_predict_keys",
           "ctr_mlp_recommend_topk", "ctr_mlp_rank_items", "ctr_mlp_recommend_topk_ex", "ctr_mlp_rank_items_ex", "ctr_mlp_get_classes", "ctr_mlp_set_classes", "ctr_mlp_regressor_create", "ctr_mlp_predict_f64",
           "ctr_mlp_score", "ctr_mlp_accuracy", "ctr_mlp_get_output", "ctr_mlp_set_output"]


def _exclusion(n, max_ts, exclude_history, exclude_seen):
    """(mode, cuts [n] int64 or None) of the _ex calls: exclude_seen implies exclude_history; max_ts (a scalar or [n];
    None: 0, every event) is only read under exclude_seen."""
    if not exclude_seen:
        return (EXCLUDE_WINDOW if exclude_history else EXCLUDE_NONE), None
    t = np.asarray(0 if max_ts is None else max_ts, np.int64)
    if t.ndim == 0:
        t = np.full(n, t, np.int64)
    if t.shape != (n,):
        raise ValueError("max_ts holds %d cuts for %d keys" % (t.size, n))
    return EXCLUDE_SEEN, np.ascontiguousarray(t)


class CtrError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("ctr_b200 error %d: %s" % (code, msg))
        self.code = code


class Config(C.Structure):
    _fields_ = [("model", C.c_int32), ("uP", C.c_int32), ("S", C.c_int32), ("D", C.c_int32), ("cF", C.c_int32),
                ("H0", C.c_int32), ("H1", C.c_int32), ("batch", C.c_int32), ("pred_batch", C.c_int32),
                ("lr", C.c_float), ("l2", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float), ("eps", C.c_float),
                ("dropout0", C.c_float), ("dropout1", C.c_float), ("seed", C.c_uint32),
                ("table_opt", C.c_int32), ("table_lr", C.c_float), ("gemm", C.c_int32), ("device", C.c_int32),
                ("rank", C.c_int32), ("world", C.c_int32), ("reserved", C.c_int32 * 8)]


class MlpConfig(C.Structure):
    _fields_ = [("n_layers", C.c_int32), ("units", C.c_int32 * 8), ("hidden_act", C.c_int32), ("batch", C.c_int32), ("max_iter", C.c_int32),
                ("n_iter_no_change", C.c_int32), ("shuffle", C.c_int32), ("adaptive", C.c_int32), ("warm_start", C.c_int32), ("seed", C.c_uint32),
                ("device", C.c_int32), ("alpha", C.c_double), ("lr_init", C.c_double), ("beta1", C.c_double), ("beta2", C.c_double),
                ("eps", C.c_double), ("tol", C.c_double)]


class MlpOptions(C.Structure):
    _fields_ = [("solver", C.c_int32), ("lr_schedule", C.c_int32), ("nesterov", C.c_int32), ("reserved0", C.c_int32),
                ("power_t", C.c_double), ("momentum", C.c_double), ("weight_decay", C.c_double), ("reserved", C.c_double * 5)]


class StepStats(C.Structure):
    _fields_ = [("cost", C.c_float), ("ms_device", C.c_float), ("launches", C.c_int32), ("reserved", C.c_int32)]


_lib = None
_fp = C.POINTER(C.c_float)
_lp = C.POINTER(C.c_int64)
_ip = C.POINTER(C.c_int32)


def load_library():
    """Loads the in-tree libctr_b200.so.  Raises if it has not been built (no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_build.SO):
        raise ImportError("libctr_b200.so is not built: run `python __graft_entry__.py build` "
                          "(this package has no CPU fallback)")
    L = C.CDLL(_build.SO)
    L.ctr_last_error.restype = C.c_char_p
    L.ctr_last_error.argtypes = [C.c_void_p]
    L.ctr_get_stream.restype = C.c_void_p
    L.ctr_get_stream.argtypes = [C.c_void_p]
    L.ctr_launch_count.restype = C.c_int64
    L.ctr_launch_count.argtypes = [C.c_void_p]
    L.ctr_destroy.argtypes = [C.c_void_p]
    L.ctr_destroy.restype = None
    L.ctr_config_default.restype = None
    L.ctr_mlp_last_error.restype = C.c_char_p
    L.ctr_mlp_last_error.argtypes = [C.c_void_p]
    L.ctr_mlp_destroy.argtypes = [C.c_void_p]
    L.ctr_mlp_destroy.restype = None
    L.ctr_mlp_config_default.restype = None
    L.ctr_mlp_options_default.restype = None
    _lib = L
    return L


def _f(a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    return a, a.ctypes.data_as(_fp)


_dp = C.POINTER(C.c_double)


def _d(a):
    a = np.ascontiguousarray(a, dtype=np.float64)
    return a, a.ctypes.data_as(_dp)


def _targets(y_true, y_pred):
    """(y_true, y_pred) as float64 [n, n_out] arrays of the same shape; a vector is one column"""
    t = np.asarray(y_true, np.float64); p = np.asarray(y_pred, np.float64)
    if t.shape != p.shape:
        raise ValueError("y_true and y_pred differ in shape: %s, %s" % (t.shape, p.shape))
    if t.ndim == 1:
        t, p = t[:, None], p[:, None]
    if t.ndim != 2:
        raise ValueError("expected [n] or [n, n_out] targets, got shape %s" % (t.shape,))
    return np.ascontiguousarray(t), np.ascontiguousarray(p)


def _weights(weight, n):
    if weight is None:
        return None, None
    w = np.ascontiguousarray(weight, np.float64).reshape(-1)
    if w.size != n:
        raise ValueError("weight has %d entries for %d samples" % (w.size, n))
    return w, w.ctypes.data_as(_dp)


def _mode(table, v, what):
    """a mode given by name (the reference's strings) or as the C enum's integer, which is passed through"""
    if isinstance(v, str):
        if v not in table:
            raise ValueError("%s must be one of %s, got %r" % (what, sorted(table), v))
        return table[v]
    return int(v)


def _i(a):
    a = np.ascontiguousarray(a, dtype=np.int32)
    return a, a.ctypes.data_as(_ip)


def default_config(model, **kw):
    cfg = Config()
    load_library().ctr_config_default(C.byref(cfg), C.c_int(model))
    for k, v in kw.items():
        if not hasattr(cfg, k):
            raise AttributeError(k)
        setattr(cfg, k, v)
    return cfg


class Engine:
    """One engine handle == one DinNet / YoutubeDnn plus its HBM tables (din.go:171, dnn.go:119)."""

    def __init__(self, cfg):
        self.L = load_library()
        self.cfg = cfg
        self.h = C.c_void_p()
        rc = self.L.ctr_create(C.byref(cfg), C.byref(self.h))
        if rc != 0:
            raise CtrError(rc, self.L.ctr_last_error(None).decode())
        self.inn = cfg.uP + 2 * cfg.D + cfg.cF

    def close(self):
        if getattr(self, "h", None) and self.h.value:
            self.L.ctr_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc != 0:
            raise CtrError(rc, self.L.ctr_last_error(self.h).decode())

    # ---- weights (Marshal layout, din.go:41-52)
    def init_weights(self, seed):
        self._ck(self.L.ctr_init_weights(self.h, C.c_uint32(seed)))

    def set_weights(self, mlp0, mlp1, mlp2, att0=None):
        c = self.cfg
        a0, p0 = _f(mlp0); a1, p1 = _f(mlp1); a2, p2 = _f(mlp2)
        assert a0.size == self.inn * c.H0 and a1.size == c.H0 * c.H1 and a2.size == c.H1
        if att0 is not None:
            a3, p3 = _f(att0); assert a3.size == c.S
        else:
            p3 = None
        self._ck(self.L.ctr_set_weights(self.h, p0, p1, p2, p3))

    def get_weights(self):
        c = self.cfg
        w0 = np.empty((self.inn, c.H0), np.float32); w1 = np.empty((c.H0, c.H1), np.float32)
        w2 = np.empty((c.H1, 1), np.float32); at = np.empty(c.S, np.float32)
        self._ck(self.L.ctr_get_weights(self.h, w0.ctypes.data_as(_fp), w1.ctypes.data_as(_fp),
                                        w2.ctypes.data_as(_fp), at.ctypes.data_as(_fp)))
        return w0, w1, w2, at

    # ---- tables
    def table_upload(self, which, rows):
        a, p = _f(rows)
        self._ck(self.L.ctr_table_upload(self.h, C.c_int(which), p, C.c_int64(a.shape[0]), C.c_int32(a.shape[1])))

    def table_fill(self, which, nrows, width, seed=0, dist=0, scale=1.0):
        self._ck(self.L.ctr_table_fill(self.h, C.c_int(which), C.c_int64(nrows), C.c_int32(width), C.c_uint32(seed),
                                       C.c_int32(dist), C.c_float(scale)))

    def table_download(self, which, nrows, width):
        out = np.zeros((nrows, width), np.float32)
        self._ck(self.L.ctr_table_download(self.h, C.c_int(which), out.ctypes.data_as(_fp), C.c_int64(nrows), C.c_int32(width)))
        return out

    def gather_rows(self, user_row, item_row, hist):
        c = self.cfg
        u, up = _i(user_row); it, ip = _i(item_row); hs, hp = _i(hist)
        B = u.size
        X = np.empty((B, c.uP + c.S * c.D + c.D + c.cF), np.float32)
        self._ck(self.L.ctr_gather_rows(self.h, up, ip, hp, C.c_int64(B), X.ctypes.data_as(_fp)))
        return X

    # ---- dense X (model.Train / model.Predict)
    def train_dense(self, X, Y, ranges, epochs, early_stop=0):
        Xa, Xp = _f(X); Ya, Yp = _f(Y)
        r = (C.c_int32 * 8)(*[int(v) for v in ranges])
        cost = C.c_float(0); ep = C.c_int32(0)
        self._ck(self.L.ctr_train_dense(self.h, Xp, Yp, C.c_int64(Xa.shape[0]), C.c_int32(Xa.shape[1]), r,
                                        C.c_int32(epochs), C.c_int32(early_stop), C.byref(cost), C.byref(ep)))
        return ep.value, cost.value

    def predict_dense(self, X, ranges):
        Xa, Xp = _f(X)
        r = (C.c_int32 * 8)(*[int(v) for v in ranges])
        out = np.empty(Xa.shape[0], np.float32)
        self._ck(self.L.ctr_predict_dense(self.h, Xp, C.c_int64(Xa.shape[0]), C.c_int32(Xa.shape[1]), r, out.ctypes.data_as(_fp)))
        return out

    # ---- index fast path
    def train_step_idx(self, user_row, item_row, hist, label):
        u, up = _i(user_row); it, ip = _i(item_row); hs, hp = _i(hist); y, yp = _f(label)
        st = StepStats()
        self._ck(self.L.ctr_train_step_idx(self.h, up, ip, hp, yp, C.c_int32(u.size), C.byref(st)))
        return st

    def train_step_idx_ptr(self, up, ip, hp, yp, B, stats=None):
        """Raw host pointers (ints) — pinned buffers owned by the caller (bench e2e leg)."""
        self._ck(self.L.ctr_train_step_idx(self.h, C.c_void_p(up), C.c_void_p(ip), C.c_void_p(hp), C.c_void_p(yp),
                                           C.c_int32(B), C.byref(stats) if stats is not None else None))

    def train_step_idx_dev(self, d_user, d_item, d_hist, d_label, B):
        """Device pointers (ints, e.g. torch.Tensor.data_ptr()); asynchronous."""
        self._ck(self.L.ctr_train_step_idx_dev(self.h, C.c_void_p(d_user), C.c_void_p(d_item), C.c_void_p(d_hist),
                                               C.c_void_p(d_label), C.c_int32(B)))

    def train_idx(self, user_row, item_row, hist, label):
        """One pass over n samples in batches of cfg.batch (pipelined H2D); returns the batch costs."""
        u, up = _i(user_row); it, ip = _i(item_row); hs, hp = _i(hist); y, yp = _f(label)
        nb = (u.size + self.cfg.batch - 1) // self.cfg.batch
        costs = np.empty(nb, np.float32)
        self._ck(self.L.ctr_train_idx(self.h, up, ip, hp, yp, C.c_int64(u.size), costs.ctypes.data_as(_fp)))
        return costs

    def train_idx_ptr(self, up, ip, hp, yp, n, costs_ptr=None):
        """Raw host pointers (pinned buffers owned by the caller)."""
        self._ck(self.L.ctr_train_idx(self.h, C.c_void_p(up), C.c_void_p(ip), C.c_void_p(hp), C.c_void_p(yp), C.c_int64(n),
                                      C.c_void_p(costs_ptr) if costs_ptr else None))

    def train_keys(self, user_ids, item_ids, ts, label, epochs=1, early_stop=0):
        """recommend.Train over sample keys (rcmd.go:197-246); returns (epochs_run, last_cost, rows_used)."""
        u = np.ascontiguousarray(user_ids, np.int64); i = np.ascontiguousarray(item_ids, np.int64); t = np.ascontiguousarray(ts, np.int64)
        y, yp = _f(label)
        assert u.size == i.size == t.size == y.size
        cost = C.c_float(0); ep = C.c_int32(0); used = C.c_int64(0)
        self._ck(self.L.ctr_train_keys(self.h, u.ctypes.data_as(_lp), i.ctypes.data_as(_lp), t.ctypes.data_as(_lp), yp, C.c_int64(u.size),
                                       C.c_int32(epochs), C.c_int32(early_stop), C.byref(cost), C.byref(ep), C.byref(used)))
        return ep.value, cost.value, used.value

    def predict_idx(self, user_row, item_row, hist):
        u, up = _i(user_row); it, ip = _i(item_row); hs, hp = _i(hist)
        out = np.empty(u.size, np.float32)
        self._ck(self.L.ctr_predict_idx(self.h, up, ip, hp, C.c_int64(u.size), out.ctypes.data_as(_fp)))
        return out

    def predict_idx_dev(self, d_user, d_item, d_hist, B, d_out=None):
        self._ck(self.L.ctr_predict_idx_dev(self.h, C.c_void_p(d_user), C.c_void_p(d_item), C.c_void_p(d_hist),
                                            C.c_int32(B), C.c_void_p(d_out) if d_out else None))

    def last_cost(self):
        c = C.c_float(0)
        self._ck(self.L.ctr_last_cost(self.h, C.byref(c)))
        return c.value

    def sync(self):
        self._ck(self.L.ctr_sync(self.h))

    @property
    def stream(self):
        return self.L.ctr_get_stream(self.h)

    def set_stream(self, ptr):
        self._ck(self.L.ctr_set_stream(self.h, C.c_void_p(ptr)))

    def launch_count(self):
        return int(self.L.ctr_launch_count(self.h))

    def profile(self, on):
        self._ck(self.L.ctr_profile_enable(self.h, C.c_int(int(on))))

    def profile_reset(self):
        self._ck(self.L.ctr_profile_reset(self.h))

    def profile_dump(self):
        buf = C.create_string_buffer(1 << 16)
        self._ck(self.L.ctr_profile_dump(self.h, buf, C.c_int64(len(buf))))
        out = {}
        for line in buf.value.decode().splitlines():
            name, ms, n = line.split()
            out[name] = (float(ms), int(n))
        return out

    def debug_grads_idx(self, user_row, item_row, hist, label, training=False):
        c = self.cfg
        u, up = _i(user_row); it, ip = _i(item_row); hs, hp = _i(hist); y, yp = _f(label)
        B = u.size
        g0 = np.empty((self.inn, c.H0), np.float32); g1 = np.empty((c.H0, c.H1), np.float32)
        g2 = np.empty((c.H1, 1), np.float32); ga = np.empty(c.S, np.float32)
        dUb = np.empty((B, c.S, c.D), np.float32); dIt = np.empty((B, c.D), np.float32)
        p = np.empty(B, np.float32); z = np.empty(B, np.float32); cost = C.c_float(0)
        self._ck(self.L.ctr_debug_grads_idx(self.h, up, ip, hp, yp, C.c_int32(B), C.c_int32(int(training)),
                                            g0.ctypes.data_as(_fp), g1.ctypes.data_as(_fp), g2.ctypes.data_as(_fp),
                                            ga.ctypes.data_as(_fp), dUb.ctypes.data_as(_fp), dIt.ctypes.data_as(_fp),
                                            p.ctypes.data_as(_fp), z.ctypes.data_as(_fp), C.byref(cost)))
        return dict(cost=cost.value, dW0=g0, dW1=g1, dW2=g2, datt=ga, dUb=dUb, dIt=dIt, p=p, logit=z)

    def comm_unique_id(self):
        buf = C.create_string_buffer(256); n = C.c_int32(256)
        rc = self.L.ctr_comm_unique_id(buf, C.byref(n))
        if rc != 0:
            raise CtrError(rc, "ctr_comm_unique_id failed (NCCL not loadable?)")
        return bytes(buf.raw[:n.value])

    def comm_init(self, uid):
        self._ck(self.L.ctr_comm_init(self.h, C.c_char_p(uid), C.c_int32(len(uid))))

    def ubcache_upload(self, offsets, ts, item_rows):
        off = np.ascontiguousarray(offsets, np.int64); t = np.ascontiguousarray(ts, np.int64); it = np.ascontiguousarray(item_rows, np.int32)
        self._ck(self.L.ctr_ubcache_upload(self.h, off.ctypes.data_as(C.POINTER(C.c_int64)), t.ctypes.data_as(C.POINTER(C.c_int64)),
                                           it.ctypes.data_as(_ip), C.c_int64(off.size - 1), C.c_int64(t.size)))

    def ubcache_window(self, user_row, max_ts):
        u, up = _i(user_row); t = np.ascontiguousarray(max_ts, np.int64)
        out = np.empty((u.size, self.cfg.S), np.int32)
        self._ck(self.L.ctr_ubcache_window(self.h, up, t.ctypes.data_as(C.POINTER(C.c_int64)), C.c_int32(u.size), out.ctypes.data_as(_ip)))
        return out

    def ubcache_window_dev(self, d_user, d_max_ts, B, d_hist):
        """ubcache_window on device pointers (ints, e.g. torch.Tensor.data_ptr()): d_user [B] int32, d_max_ts [B] int64
        → d_hist [B, S] int32; asynchronous on the engine stream."""
        self._ck(self.L.ctr_ubcache_window_dev(self.h, C.c_void_p(d_user), C.c_void_p(d_max_ts), C.c_int32(B), C.c_void_p(d_hist)))

    def ubcache_append(self, user_rows, ts, item_rows):
        """Appends events to the device ubcache (ctr_ubcache_append): equal timestamps keep the most recent arrival first."""
        u, up = _i(user_rows); t = np.ascontiguousarray(ts, np.int64); it, ip = _i(item_rows)
        assert u.size == t.size == it.size
        self._ck(self.L.ctr_ubcache_append(self.h, up, t.ctypes.data_as(_lp), ip, C.c_int64(u.size)))

    def ubcache_set(self, user_rows, offsets, ts, item_rows):
        """Replaces the whole sequences of distinct users (ctr_ubcache_set); user_rows[k]'s events are
        [offsets[k], offsets[k+1]) of ts / item_rows, time-descending.  An empty sequence deletes the user's history."""
        u, up = _i(user_rows); off = np.ascontiguousarray(offsets, np.int64); t = np.ascontiguousarray(ts, np.int64); it, ip = _i(item_rows)
        assert off.size == u.size + 1 and t.size == it.size
        self._ck(self.L.ctr_ubcache_set(self.h, up, off.ctypes.data_as(_lp), t.ctypes.data_as(_lp), ip, C.c_int64(u.size), C.c_int64(t.size)))

    def ubcache_download(self):
        """The live ubcache as (offsets [n_users+1], ts [n], item_rows [n])."""
        nu = C.c_int64(0); n = C.c_int64(0)
        self._ck(self.L.ctr_ubcache_download(self.h, None, None, None, C.c_int64(0), C.c_int64(0), C.byref(nu), C.byref(n)))
        off = np.empty(nu.value + 1, np.int64); t = np.empty(n.value, np.int64); it = np.empty(n.value, np.int32)
        self._ck(self.L.ctr_ubcache_download(self.h, off.ctypes.data_as(_lp), t.ctypes.data_as(_lp), it.ctypes.data_as(_ip),
                                             C.c_int64(nu.value), C.c_int64(n.value), C.byref(nu), C.byref(n)))
        return off, t, it

    def idmap_build(self, which, ids):
        a = np.ascontiguousarray(ids, np.int64)
        self._ck(self.L.ctr_idmap_build(self.h, C.c_int(which), a.ctypes.data_as(_lp), C.c_int64(a.size)))

    def idmap_lookup(self, which, ids):
        a = np.ascontiguousarray(ids, np.int64)
        out = np.empty(a.size, np.int32)
        self._ck(self.L.ctr_idmap_lookup(self.h, C.c_int(which), a.ctypes.data_as(_lp), C.c_int64(a.size), out.ctypes.data_as(_ip)))
        return out

    def idmap_lookup_dev(self, which, d_ids, n, d_rows):
        """idmap_lookup on device pointers (ints): d_ids [n] int64 → d_rows [n] int32, -1 for an unknown id;
        asynchronous on the engine stream."""
        self._ck(self.L.ctr_idmap_lookup_dev(self.h, C.c_int(which), C.c_void_p(d_ids), C.c_int64(n), C.c_void_p(d_rows)))

    def idmap_insert(self, which, ids):
        """Adds ids to a live map (ctr_idmap_insert): ids it lacks get the next rows in order of first occurrence, ids it
        holds keep theirs.  Returns the row of every id.  With the item map, extends `item_ids` (the row -> id list
        serving.Recommend maps rows back through) when the engine carries one.  With world > 1 the call is collective:
        every rank passes its own ids (possibly none) and every map ends as one GPU's insert of the ranks' ids concatenated
        in rank order; maps that differ across ranks, or a refused id on any rank, raise CtrError on every rank."""
        a = np.ascontiguousarray(ids, np.int64)
        out = np.empty(a.size, np.int32)
        self._ck(self.L.ctr_idmap_insert(self.h, C.c_int(which), a.ctypes.data_as(_lp), C.c_int64(a.size), out.ctypes.data_as(_ip)))
        known = getattr(self, "item_ids", None)
        if which == IDMAP_ITEM and known is not None and self.cfg.world > 1:
            self.item_ids = self.idmap_download(IDMAP_ITEM)       # other ranks' ids may have taken rows too
        elif which == IDMAP_ITEM and known is not None:
            known = np.asarray(known, np.int64)
            fresh = out >= known.size
            if fresh.any():
                new_rows, first = np.unique(out[fresh], return_index=True)
                self.item_ids = np.concatenate([known, a[fresh][first]])
                assert self.item_ids.size == new_rows[-1] + 1
        return out

    def idmap_download(self, which):
        """The ids of a map in row order (ctr_idmap_download): ids[r] is the id of row r.  Local on every rank (the maps
        of a multi-GPU handle are identical)."""
        n = C.c_int64(0)
        self._ck(self.L.ctr_idmap_download(self.h, C.c_int(which), None, C.c_int64(0), C.byref(n)))
        out = np.empty(n.value, np.int64)
        self._ck(self.L.ctr_idmap_download(self.h, C.c_int(which), out.ctypes.data_as(_lp), C.c_int64(n.value), C.byref(n)))
        return out

    def table_write_rows(self, which, rows, data):
        """Writes rows of a live table in HBM (ctr_table_write_rows): row rows[i] = data[i]; a row past the end grows
        the table (the gap reads as zero).  ITEM_EMB's written rows restart their row-Adam moments at zero.  With world
        > 1 the call is collective: every rank passes its own (rows, data), possibly none, and the table ends as one
        GPU's write of the ranks' lists concatenated in rank order; a row named twice anywhere raises CtrError on every
        rank.  A row-sharded table sends each row to its owner; a shard that outgrows its allocation is reallocated at
        twice its rows."""
        r, rp = _i(np.atleast_1d(rows))
        d, dp = _f(data)
        if r.size:
            d = d.reshape(r.size, -1) if d.size else d.reshape(r.size, 0)
            width = d.shape[1]
        else:           # a rank with nothing to write in a collective call: the table's width, not that of an empty array
            width = d.shape[1] if d.ndim == 2 else {TABLE_USER_FEAT: self.cfg.uP, TABLE_ITEM_FEAT: self.cfg.cF, TABLE_ITEM_EMB: self.cfg.D}.get(which, 0)
        self._ck(self.L.ctr_table_write_rows(self.h, C.c_int(which), rp, dp, C.c_int64(r.size), C.c_int32(width)))

    def item_emb_train(self, item_ids, cfg=None, sync_every=None, **kw):
        """recommend.Train's embedding stage into ITEM_EMB (ctr_item_emb_train): item2vec over the int64 item stream,
        words numbered by first appearance on the device, row r of ITEM_EMB = the vector of the item the item map sends
        to r (zeros when it never occurs).  cfg: an item2vec.I2vConfig (default: i2v_default_config(dim=D, **kw)).
        Returns (vocab_ids [V] int64: the item id of every word in word-id order, I2vStats).

        With world > 1 the call is collective: every rank passes its own shard of the stream (possibly empty) and ends as
        one GPU would after the same call on the ranks' shards concatenated in rank order, except that the vectors come
        from local SGD with the replicas averaged every sync_every centre positions (cfg.reserved[1]; None or 0: 4 Mi) and
        the stats are this rank's.  vocab_ids is the whole vocabulary on every rank: when other ranks' unmapped ids make
        it longer than this rank could size it, the rest is read back (ctr_item_emb_vocab)."""
        from .item2vec import I2vConfig, I2vStats, i2v_default_config
        cfg = I2vConfig.from_buffer_copy(cfg) if cfg is not None else i2v_default_config(**{"dim": self.cfg.D, **kw})
        if sync_every is not None:
            if isinstance(sync_every, (bool, np.bool_)) or not isinstance(sync_every, (int, np.integer)) or not 0 <= int(sync_every) < 2 ** 31:
                raise ValueError("sync_every must be an int in [0, 2^31), got %r" % (sync_every,))
            cfg.reserved[1] = int(sync_every)
        ids = np.ascontiguousarray(item_ids, np.int64).reshape(-1)
        cap = ids.size                          # one GPU: V <= n
        if self.cfg.world > 1:                  # every item-map row may be a word; only other ranks' unmapped ids can exceed it
            n = C.c_int64(0)
            if self.L.ctr_idmap_download(self.h, C.c_int(IDMAP_ITEM), None, C.c_int64(0), C.byref(n)) == 0:
                cap += n.value
        st = I2vStats(); V = C.c_int32(0)
        vocab = np.empty(max(cap, 1), np.int64)
        self._ck(self.L.ctr_item_emb_train(self.h, C.byref(cfg), ids.ctypes.data_as(_lp) if ids.size else None, C.c_int64(ids.size),
                                           vocab.ctypes.data_as(_lp), C.c_int64(cap), C.byref(V), C.byref(st)))
        if V.value > cap:
            vocab = np.empty(V.value, np.int64)
            self._ck(self.L.ctr_item_emb_vocab(self.h, vocab.ctypes.data_as(_lp), C.c_int64(vocab.size), C.byref(V)))
        return vocab[:V.value].copy(), st

    def batch_predict_keys(self, user_ids, item_ids, ts):
        """recommend.BatchPredict (rcmd.go:277-337) over Sample keys."""
        u = np.ascontiguousarray(user_ids, np.int64); i = np.ascontiguousarray(item_ids, np.int64); t = np.ascontiguousarray(ts, np.int64)
        assert u.size == i.size == t.size
        out = np.empty(u.size, np.float32)
        self._ck(self.L.ctr_batch_predict_keys(self.h, u.ctypes.data_as(_lp), i.ctypes.data_as(_lp), t.ctypes.data_as(_lp), C.c_int64(u.size),
                                                out.ctypes.data_as(_fp)))
        return out

    def checkpoint_save(self, path):
        self._ck(self.L.ctr_checkpoint_save(self.h, C.c_char_p(str(path).encode())))

    def checkpoint_load(self, path):
        self._ck(self.L.ctr_checkpoint_load(self.h, C.c_char_p(str(path).encode())))

    def roc_auc(self, pred, y):
        p, pp = _f(pred); t, tp = _f(y)
        auc = C.c_double(0)
        self._ck(self.L.ctr_roc_auc(self.h, pp, tp, C.c_int64(p.size), C.byref(auc)))
        return auc.value

    def group_auc(self, pred, y, group, per_group=False):
        """Grouped AUC (ctr_group_auc): RocAuc32 within each group (normally the user id), weighted by the groups'
        sample counts over the groups that hold both classes.  Returns (gauc, n_groups, n_used); with per_group=True
        also a dict of the ascending group ids and their n, positives and AUC (NaN for a group with one class)."""
        p, pp = _f(pred); t, tp = _f(y)
        gr = np.ascontiguousarray(group, np.int64)
        if not p.size == t.size == gr.size:
            raise ValueError("pred, y and group differ in length: %d, %d, %d" % (p.size, t.size, gr.size))
        gauc = C.c_double(0); ng = C.c_int64(0); nu = C.c_int64(0)
        outs = None
        if per_group:
            outs = dict(group=np.empty(p.size, np.int64), n=np.empty(p.size, np.int32), pos=np.empty(p.size, np.int32),
                        auc=np.empty(p.size, np.float64))
        ptr = (lambda k, ty: outs[k].ctypes.data_as(C.POINTER(ty))) if outs else (lambda k, ty: None)
        self._ck(self.L.ctr_group_auc(self.h, pp, tp, gr.ctypes.data_as(_lp), C.c_int64(p.size), C.byref(gauc), C.byref(ng),
                                      C.byref(nu), ptr("group", C.c_int64), ptr("n", C.c_int32), ptr("pos", C.c_int32),
                                      ptr("auc", C.c_double)))
        if outs is None:
            return gauc.value, ng.value, nu.value
        return gauc.value, ng.value, nu.value, {k: v[:ng.value].copy() for k, v in outs.items()}

    def roc_auc_dist(self, pred, y):
        """ROC AUC over every rank's samples (ctr_roc_auc_dist): collective on a multi-GPU handle, each rank passing its
        own samples (possibly none); every rank gets roc_auc of all ranks' samples concatenated in rank order."""
        p, pp = _f(pred); t, tp = _f(y)
        if p.size != t.size:
            raise ValueError("pred and y differ in length: %d, %d" % (p.size, t.size))
        auc = C.c_double(0)
        self._ck(self.L.ctr_roc_auc_dist(self.h, pp, tp, C.c_int64(p.size), C.byref(auc)))
        return auc.value

    def group_auc_dist(self, pred, y, group, per_group=False):
        """group_auc over every rank's samples (ctr_group_auc_dist): collective on a multi-GPU handle, each rank passing
        its own samples (possibly none).  Returns what group_auc returns on all ranks' samples concatenated in rank
        order, on every rank.  With per_group=True the call runs twice: once for the group count, once for the arrays."""
        p, pp = _f(pred); t, tp = _f(y)
        gr = np.ascontiguousarray(group, np.int64)
        if not p.size == t.size == gr.size:
            raise ValueError("pred, y and group differ in length: %d, %d, %d" % (p.size, t.size, gr.size))
        gauc = C.c_double(0); ng = C.c_int64(0); nu = C.c_int64(0)

        def call(outs):
            ptr = (lambda k, ty: outs[k].ctypes.data_as(C.POINTER(ty))) if outs else (lambda k, ty: None)
            cap = outs["group"].size if outs else 0
            self._ck(self.L.ctr_group_auc_dist(self.h, pp, tp, gr.ctypes.data_as(_lp), C.c_int64(p.size), C.byref(gauc), C.byref(ng),
                                               C.byref(nu), C.c_int64(cap), ptr("group", C.c_int64), ptr("n", C.c_int32),
                                               ptr("pos", C.c_int32), ptr("auc", C.c_double)))
        call(None)
        if not per_group:
            return gauc.value, ng.value, nu.value
        k = ng.value
        outs = dict(group=np.empty(k, np.int64), n=np.empty(k, np.int32), pos=np.empty(k, np.int32), auc=np.empty(k, np.float64))
        call(outs)
        return gauc.value, ng.value, nu.value, outs

    def _curve(self, fn, pred, y, pos_label):
        p, pp = _f(pred); t, tp = _f(y)
        if p.size != t.size:
            raise ValueError("pred and y differ in length: %d, %d" % (p.size, t.size))
        cap = p.size + 1
        a, b, th = np.empty(cap), np.empty(cap), np.empty(cap)
        npts = C.c_int64(0)
        dp = lambda x: x.ctypes.data_as(C.POINTER(C.c_double))
        self._ck(fn(self.h, pp, tp, C.c_int64(p.size), C.c_double(pos_label), dp(a), dp(b), dp(th), C.c_int64(cap),
                    C.byref(npts)))
        return a, b, th, npts.value

    def roc_curve(self, pred, y, pos_label=1.0):
        """ROCCurve (ctr_roc_curve): (fpr, tpr, thresholds) as float64 arrays, one point per distinct score from the
        highest down, (0, 0) first when the top score holds a negative.  A sample is positive when y == pos_label."""
        fpr, tpr, th, m = self._curve(self.L.ctr_roc_curve, pred, y, pos_label)
        return fpr[:m].copy(), tpr[:m].copy(), th[:m].copy()

    def precision_recall_curve(self, pred, y, pos_label=1.0):
        """PrecisionRecallCurve (ctr_pr_curve): (precision, recall, thresholds), recall decreasing to the final
        (precision 1, recall 0), which has no threshold.  A sample is positive when y == pos_label."""
        prec, rec, th, m = self._curve(self.L.ctr_pr_curve, pred, y, pos_label)
        return prec[:m].copy(), rec[:m].copy(), th[:m - 1].copy()

    def average_precision(self, pred, y):
        """AveragePrecisionScore of a binary target (ctr_average_precision): the area under the precision-recall
        curve as the reference sums it, positives y == 1; NaN with no positives, CtrError (EINVAL) for non-binary labels."""
        p, pp = _f(pred); t, tp = _f(y)
        if p.size != t.size:
            raise ValueError("pred and y differ in length: %d, %d" % (p.size, t.size))
        ap = C.c_double(0)
        self._ck(self.L.ctr_average_precision(self.h, pp, tp, C.c_int64(p.size), C.byref(ap)))
        return ap.value

    def group_average_precision(self, pred, y, group, per_group=False):
        """Mean average precision over groups (ctr_group_average_precision): AP within each group (normally the user
        id), averaged without weights over the groups that hold a positive.  Returns (map, n_groups, n_used); with
        per_group=True also a dict of the ascending group ids and their n, positives and AP (NaN with no positive)."""
        p, pp = _f(pred); t, tp = _f(y)
        gr = np.ascontiguousarray(group, np.int64)
        if not p.size == t.size == gr.size:
            raise ValueError("pred, y and group differ in length: %d, %d, %d" % (p.size, t.size, gr.size))
        m = C.c_double(0); ng = C.c_int64(0); nu = C.c_int64(0)
        outs = None
        if per_group:
            outs = dict(group=np.empty(p.size, np.int64), n=np.empty(p.size, np.int32), pos=np.empty(p.size, np.int32),
                        ap=np.empty(p.size, np.float64))
        ptr = (lambda k, ty: outs[k].ctypes.data_as(C.POINTER(ty))) if outs else (lambda k, ty: None)
        self._ck(self.L.ctr_group_average_precision(self.h, pp, tp, gr.ctypes.data_as(_lp), C.c_int64(p.size), C.byref(m),
                                                    C.byref(ng), C.byref(nu), ptr("group", C.c_int64), ptr("n", C.c_int32),
                                                    ptr("pos", C.c_int32), ptr("ap", C.c_double)))
        if outs is None:
            return m.value, ng.value, nu.value
        return m.value, ng.value, nu.value, {k: v[:ng.value].copy() for k, v in outs.items()}

    def accuracy_score(self, y_true, y_pred, normalize=True, weight=None):
        """AccuracyScore (ctr_accuracy_score): the weight of the rows whose every column is equal (==) over all the
        weight, or that weight itself with normalize=False.  y_true / y_pred: [n] or [n, n_out]; weight: [n] or None."""
        t, p = _targets(y_true, y_pred)
        w, wp = _weights(weight, t.shape[0])
        out = C.c_double(0)
        self._ck(self.L.ctr_accuracy_score(self.h, t.ctypes.data_as(_dp), p.ctypes.data_as(_dp), C.c_int64(t.shape[0]),
                                           C.c_int32(t.shape[1]), wp, C.c_int32(int(bool(normalize))), C.byref(out)))
        return out.value

    def _class_labels(self, y_true, y_pred):
        t = np.ascontiguousarray(y_true, np.float64).reshape(-1); p = np.ascontiguousarray(y_pred, np.float64).reshape(-1)
        if t.size != p.size:
            raise ValueError("y_true and y_pred differ in length: %d, %d" % (t.size, p.size))
        return t, p

    def confusion_matrix(self, y_true, y_pred, weight=None):
        """ConfusionMatrix (ctr_confusion_matrix) of 1-D labels: (classes [C] float64 ascending, cm [C, C] float64),
        cm[r, c] the weight (or count) of true class r predicted as c; a prediction between two classes counts as the
        higher one.  Runs the pipeline twice: once for C, once for the matrix."""
        t, p = self._class_labels(y_true, y_pred)
        w, wp = _weights(weight, t.size)
        nc = C.c_int32(0)
        classes = np.empty(t.size, np.float64)
        args = (self.h, t.ctypes.data_as(_dp), p.ctypes.data_as(_dp), C.c_int64(t.size), wp)
        self._ck(self.L.ctr_confusion_matrix(*args, classes.ctypes.data_as(_dp), None, C.c_int64(t.size * t.size), C.byref(nc)))
        cm = np.empty((nc.value, nc.value), np.float64)
        self._ck(self.L.ctr_confusion_matrix(*args, None, cm.ctypes.data_as(_dp), C.c_int64(cm.size), C.byref(nc)))
        return classes[:nc.value].copy(), cm

    def precision_recall_fscore(self, y_true, y_pred, beta=1.0, average="macro", pos_label=-1, weight=None, per_class=False):
        """PrecisionRecallFScoreSupport (ctr_precision_recall_fscore): (precision, recall, fscore, support) of the class
        index pos_label, or with pos_label < 0 their average ("macro", "micro" or "weighted", which equals "macro" as in
        the reference; support 0).  per_class=True also returns the [C, 4] rows (p, r, f, support) of every class."""
        t, p = self._class_labels(y_true, y_pred)
        w, wp = _weights(weight, t.size)
        avg = _mode(AVERAGE, average, "average")
        nc = C.c_int32(0)
        o = [C.c_double(0) for _ in range(4)]
        pc = np.empty((t.size, 4), np.float64) if per_class else None
        self._ck(self.L.ctr_precision_recall_fscore(self.h, t.ctypes.data_as(_dp), p.ctypes.data_as(_dp), C.c_int64(t.size), wp,
                                                    C.c_double(beta), C.c_int32(avg), C.c_int32(pos_label),
                                                    *[C.byref(x) for x in o], pc.ctypes.data_as(_dp) if per_class else None,
                                                    C.c_int64(t.size), C.byref(nc)))
        res = tuple(x.value for x in o)
        return res + (pc[:nc.value].copy(),) if per_class else res

    def r2_score(self, y_true, y_pred, weight=None, multioutput="uniform_average"):
        """R2Score (ctr_r2_score): "raw_values" gives the [n_out] scores, "uniform_average" (or "") their mean,
        "variance_weighted" their mean weighted by each column's weighted variance.  weight: [n] or None."""
        t, p = _targets(y_true, y_pred)
        w, wp = _weights(weight, t.shape[0])
        mode = _mode(MULTIOUTPUT, "uniform_average" if multioutput == "" else multioutput, "multioutput")
        out = np.empty(t.shape[1], np.float64)
        self._ck(self.L.ctr_r2_score(self.h, t.ctypes.data_as(_dp), p.ctypes.data_as(_dp), C.c_int64(t.shape[0]), C.c_int32(t.shape[1]),
                                     wp, C.c_int32(mode), out.ctypes.data_as(_dp)))
        return out if mode == MULTIOUTPUT["raw_values"] else float(out[0])

    def mean_error(self, y_true, y_pred, kind="squared", multioutput="uniform_average"):
        """MeanSquaredError (kind "squared") or MeanAbsoluteError ("absolute") (ctr_mean_error): "raw_values" gives the
        [n_out] column means, "uniform_average" (or "") their mean.  "variance_weighted" raises CtrError (EINVAL)."""
        t, p = _targets(y_true, y_pred)
        k = _mode(ERROR_KIND, kind, "kind")
        mode = _mode(MULTIOUTPUT, "uniform_average" if multioutput == "" else multioutput, "multioutput")
        out = np.empty(t.shape[1], np.float64)
        self._ck(self.L.ctr_mean_error(self.h, t.ctypes.data_as(_dp), p.ctypes.data_as(_dp), C.c_int64(t.shape[0]), C.c_int32(t.shape[1]),
                                       C.c_int32(k), C.c_int32(mode), out.ctypes.data_as(_dp)))
        return out if mode == MULTIOUTPUT["raw_values"] else float(out[0])

    def knn_search(self, k, queries=None, rows=None):
        """search.Searcher on ITEM_EMB (ctr_knn_search): queries [nq, D] float64 vectors (rows: optional row to exclude
        per query, -1 = none), or queries=None and rows = the query rows.  Returns (rows [nq, k] int32, sims [nq, k]
        float64, counts [nq] int32); positions past a query's count hold row -1 and similarity 0.
        On a row-sharded ITEM_EMB (world > 1, large table) the call is collective: every rank calls it with the same
        arguments and receives the same complete result, bit-identical to one GPU holding the whole table; arguments
        that differ between the ranks raise CTR_EINVAL on every rank.  No sync is needed after training."""
        qp = rp = None
        if queries is not None:
            q = np.ascontiguousarray(queries, np.float64)
            q = q.reshape(1, -1) if q.ndim == 1 else q
            nq, qp = q.shape[0], q.ctypes.data_as(C.POINTER(C.c_double))
        if rows is not None:
            r, rp = _i(np.atleast_1d(rows))
            nq = r.size if queries is None else nq
            assert r.size == nq
        if qp is None and rp is None:
            raise ValueError("knn_search needs queries or rows")
        out_r = np.empty((nq, k), np.int32); out_s = np.empty((nq, k), np.float64); cnt = np.empty(nq, np.int32)
        self._ck(self.L.ctr_knn_search(self.h, qp, rp, C.c_int64(nq), C.c_int32(k), out_r.ctypes.data_as(_ip),
                                       out_s.ctypes.data_as(C.POINTER(C.c_double)), cnt.ctypes.data_as(_ip)))
        return out_r, out_s, cnt

    def recommend_topk(self, user_rows, hist, k, exclude_history=True, max_ts=None, exclude_seen=False):
        """Top-k recommendation over every ITEM_EMB row (ctr_recommend_topk_ex): user_rows [nu], hist [nu, S] (-1 padded).
        Returns (rows [nu, k] int32, scores [nu, k] float32, logits [nu, k] float32, counts [nu] int32), best first
        (logit descending, then row ascending); positions past a user's count hold row -1, score 0 and logit 0.
        exclude_seen (implies exclude_history) also drops every item of the user's ubcache events with ts <= max_ts
        (a scalar or [nu]; None or 0: every event).
        On a row-sharded ITEM_EMB the call is collective, under the same rule as knn_search; max_ts must agree too.
        There exclude_seen follows the owner rule: row g is dropped when it is in the window, or when the ubcache of
        rank g % world holds an event of the user with ts <= max_ts whose item is g.  With the same cache on every rank
        (every ubcache upload, append and set applied on every rank) the lists equal one GPU's with that cache."""
        u, up = _i(np.atleast_1d(user_rows))
        hs, hp = _i(np.asarray(hist).reshape(u.size, self.cfg.S))
        mode, t = _exclusion(u.size, max_ts, exclude_history, exclude_seen)
        out_r = np.empty((u.size, k), np.int32); out_s = np.empty((u.size, k), np.float32)
        out_l = np.empty((u.size, k), np.float32); cnt = np.empty(u.size, np.int32)
        self._ck(self.L.ctr_recommend_topk_ex(self.h, up, hp, None if t is None else t.ctypes.data_as(_lp), C.c_int64(u.size), C.c_int32(k),
                                              C.c_int32(mode), out_r.ctypes.data_as(_ip), out_s.ctypes.data_as(_fp), out_l.ctypes.data_as(_fp),
                                              cnt.ctypes.data_as(_ip)))
        return out_r, out_s, out_l, cnt

    def rank_items(self, user_rows, hist, item_rows, exclude_history=True, max_ts=None, exclude_seen=False):
        """Full-catalogue rank of held-out items (ctr_rank_items): key i is (user_rows[i], hist[i] [S], item_rows[i]).
        Returns (ranks [n] int64, logits [n] float32): rank r means recommend_topk(user, hist, k) lists the item at
        position r - 1 for every k >= r; -1 when it can never be listed (outside the table, in an excluded history, or a
        NaN logit).  Each logit is bit for bit the one the list reports for that row (NaN outside the table).
        On a row-sharded ITEM_EMB the call is collective, under the same rule as knn_search: every rank calls it with
        the same user, history and item rows and receives the same ranks and logits, bit-identical to one GPU holding the
        whole table; rows that differ between the ranks raise CTR_EINVAL on every rank.  No sync is needed after
        training.  exclude_seen and max_ts (a scalar or [n], key i's cut) as for recommend_topk: a target the user has
        seen by the cut ranks -1 and still reports its logit; on a row-sharded ITEM_EMB whether a row is seen is decided
        by the rank that owns it, from its own ubcache (the owner rule of recommend_topk)."""
        u, up = _i(np.atleast_1d(user_rows))
        it, ip = _i(np.atleast_1d(item_rows))
        hs, hp = _i(np.asarray(hist).reshape(u.size, self.cfg.S))
        if it.size != u.size:
            raise ValueError("user_rows and item_rows differ in length: %d, %d" % (u.size, it.size))
        mode, t = _exclusion(u.size, max_ts, exclude_history, exclude_seen)
        ranks = np.empty(u.size, np.int64); logits = np.empty(u.size, np.float32)
        self._ck(self.L.ctr_rank_items_ex(self.h, up, hp, None if t is None else t.ctypes.data_as(_lp), ip, C.c_int64(u.size), C.c_int32(mode),
                                          ranks.ctypes.data_as(_lp), logits.ctypes.data_as(_fp)))
        return ranks, logits


def rank_metrics(ranks, groups, ks):
    """HR@k, Recall@k and NDCG@k for every k in ks, and MRR, of ranks from rank_items (ctr_rank_metrics); groups[i] is
    key i's group (normally its user).  Returns (hit [len(ks)], recall [len(ks)], ndcg [len(ks)], mrr)."""
    r = np.ascontiguousarray(ranks, np.int64).ravel(); g = np.ascontiguousarray(groups, np.int64).ravel()
    k = np.ascontiguousarray(np.atleast_1d(ks), np.int32)
    if r.size != g.size:
        raise ValueError("ranks and groups differ in length: %d, %d" % (r.size, g.size))
    hit = np.empty(k.size, np.float64); rec = np.empty(k.size, np.float64); ndcg = np.empty(k.size, np.float64)
    mrr = C.c_double(0)
    dp = C.POINTER(C.c_double)
    L = load_library()
    rc = L.ctr_rank_metrics(r.ctypes.data_as(_lp), g.ctypes.data_as(_lp), C.c_int64(r.size), k.ctypes.data_as(_ip), C.c_int32(k.size),
                            hit.ctypes.data_as(dp), rec.ctypes.data_as(dp), ndcg.ctypes.data_as(dp), C.byref(mrr))
    if rc != 0:
        raise CtrError(rc, L.ctr_last_error(None).decode())
    return hit, rec, ndcg, mrr.value


MLP_ACT = {"relu": 0, "logistic": 1, "identity": 2, "tanh": 3}
MLP_SOLVER = {"adam": 0, "sgd": 1}
MLP_LR = {"constant": 0, "invscaling": 1, "adaptive": 2}


class _Mlp64:
    """What MLPClassifier and MLPRegressor share: BaseMultilayerPerceptron64 on the device (float64), its
    constructor, fits and the key-fed calls."""
    n_outputs = 1
    _CREATE = "ctr_mlp_create_ex"

    def __init__(self, n_features, hidden=(100,), activation="relu", alpha=1e-4, batch=200, max_iter=200, lr_init=1e-3,
                 adaptive=False, shuffle=True, seed=0, tol=1e-4, n_iter_no_change=10, warm_start=False, device=0,
                 solver="adam", learning_rate=None, power_t=0.5, momentum=0.9, nesterovs_momentum=True, weight_decay=0.0,
                 early_stopping=False, batch_normalize=False):
        if solver == "lbfgs":
            raise ValueError("solver 'lbfgs' is not built: the reference runs gonum's optimize.Minimize (basemlp64.go:675-727), "
                             "which is not part of the reference tree and cannot be restated or checked")
        if early_stopping:
            raise ValueError("early_stopping is not built: the reference scores raw probabilities by exact-equality accuracy "
                             "(basemlp64.go:933-938, 1143-1155) and then restores a best-parameter copy it never wrote (:850-853)")
        if batch_normalize:
            raise ValueError("batch_normalize is not built: the reference normalises activations in training only (:347-351), never in predict (:897-915)")
        if solver not in MLP_SOLVER:
            raise ValueError("solver must be one of %s, got %r" % (sorted(MLP_SOLVER), solver))
        if activation not in MLP_ACT:
            raise ValueError("activation must be one of %s, got %r" % (sorted(MLP_ACT), activation))
        if learning_rate is None:
            learning_rate = "adaptive" if adaptive else "constant"
        elif adaptive and learning_rate != "adaptive":
            raise ValueError("adaptive=True contradicts learning_rate=%r" % (learning_rate,))
        if learning_rate not in MLP_LR:
            raise ValueError("learning_rate must be one of %s, got %r" % (sorted(MLP_LR), learning_rate))
        self.L = load_library()
        opts = MlpOptions()
        self.L.ctr_mlp_options_default(C.byref(opts))
        opts.solver = MLP_SOLVER[solver]; opts.lr_schedule = MLP_LR[learning_rate]; opts.nesterov = int(bool(nesterovs_momentum))
        opts.power_t = power_t; opts.momentum = momentum; opts.weight_decay = weight_decay
        self.opts = opts
        cfg = MlpConfig()
        self.L.ctr_mlp_config_default(C.byref(cfg), C.c_int32(n_features))
        units = [n_features, *hidden, self.n_outputs]
        cfg.n_layers = len(units)
        for i, u in enumerate(units):
            cfg.units[i] = u
        cfg.hidden_act = MLP_ACT[activation]; cfg.alpha = alpha; cfg.batch = batch; cfg.max_iter = max_iter; cfg.lr_init = lr_init
        cfg.adaptive = int(learning_rate == "adaptive"); cfg.shuffle = int(shuffle); cfg.seed = seed; cfg.tol = tol; cfg.n_iter_no_change = n_iter_no_change
        cfg.warm_start = int(warm_start); cfg.device = device
        self.cfg = cfg
        self.h = C.c_void_p()
        rc = getattr(self.L, self._CREATE)(C.byref(cfg), C.byref(opts), C.byref(self.h))
        if rc != 0:
            raise CtrError(rc, self.L.ctr_mlp_last_error(None).decode())
        self.n_iter = 0; self.loss_curve = np.zeros(0); self.rows_used = 0

    def _ck(self, rc):
        if rc != 0:
            raise CtrError(rc, self.L.ctr_mlp_last_error(self.h).decode())

    def close(self):
        if getattr(self, "h", None) and self.h.value:
            self.L.ctr_mlp_destroy(self.h); self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def fit(self, X, Y):
        Xa, Xp = _f(X); Ya, Yp = _f(Y)
        it = C.c_int32(0); curve = np.zeros(self.cfg.max_iter, np.float64)
        self._ck(self.L.ctr_mlp_fit(self.h, Xp, Yp, C.c_int64(Xa.shape[0]), C.c_int32(Xa.shape[1]), C.byref(it), curve.ctypes.data_as(C.POINTER(C.c_double))))
        self.n_iter = it.value; self.loss_curve = curve[:it.value]
        return self

    @staticmethod
    def _keys(user_ids, item_ids, ts):
        u = np.ascontiguousarray(user_ids, np.int64); i = np.ascontiguousarray(item_ids, np.int64); t = np.ascontiguousarray(ts, np.int64)
        if not u.size == i.size == t.size:
            raise ValueError("user_ids, item_ids and ts differ in length: %d, %d, %d" % (u.size, i.size, t.size))
        return u, i, t

    def fit_keys(self, engine, user_ids, item_ids, ts, label):
        """recommend.Train with SimpleMlpFitWrap over sample keys (ctr_mlp_fit_keys): `engine` is the feature store (id
        maps, tables, optional ubcache).  Keys with an unknown user or item are dropped; sets n_iter, loss_curve and
        rows_used (the surviving samples).  Bit-identical to fit() on the rows engine.gather_rows builds for the survivors."""
        u, i, t = self._keys(user_ids, item_ids, ts)
        y, yp = _f(label)
        if y.size != u.size:
            raise ValueError("label has %d entries for %d keys" % (y.size, u.size))
        it = C.c_int32(0); used = C.c_int64(0); curve = np.zeros(self.cfg.max_iter, np.float64)
        self._ck(self.L.ctr_mlp_fit_keys(self.h, engine.h, u.ctypes.data_as(_lp), i.ctypes.data_as(_lp), t.ctypes.data_as(_lp), yp,
                                         C.c_int64(u.size), C.byref(it), curve.ctypes.data_as(C.POINTER(C.c_double)), C.byref(used)))
        self.n_iter = it.value; self.loss_curve = curve[:it.value]; self.rows_used = used.value
        return self

    def fit_keys_dist(self, engine, user_ids, item_ids, ts, label):
        """fit_keys on a multi-GPU feature store (ctr_mlp_fit_keys_dist), a row-sharded ITEM_EMB included.  Collective
        when engine's world > 1: every rank calls it with its own keys (possibly none) and ends with the model, n_iter,
        loss_curve and rows_used (the survivors of all ranks) that fit_keys on one GPU would give over all ranks' keys
        concatenated in rank order, bit for bit.  Each key is windowed by the ubcache of the rank that passed it.  A
        configuration, options or warm-start model that differs across ranks raises CtrError (EINVAL) everywhere; any
        other refusal raises the lowest failing rank's error on every rank.  No sync() is needed after training.  On
        world == 1 this is fit_keys."""
        u, i, t = self._keys(user_ids, item_ids, ts)
        y, yp = _f(label)
        if y.size != u.size:
            raise ValueError("label has %d entries for %d keys" % (y.size, u.size))
        it = C.c_int32(0); used = C.c_int64(0); curve = np.zeros(self.cfg.max_iter, np.float64)
        self._ck(self.L.ctr_mlp_fit_keys_dist(self.h, engine.h, u.ctypes.data_as(_lp), i.ctypes.data_as(_lp), t.ctypes.data_as(_lp), yp,
                                              C.c_int64(u.size), C.byref(it), curve.ctypes.data_as(C.POINTER(C.c_double)), C.byref(used)))
        self.n_iter = it.value; self.loss_curve = curve[:it.value]; self.rows_used = used.value
        return self

    def predict_keys(self, engine, user_ids, item_ids, ts):
        """recommend.BatchPredict for the MLP over sample keys (ctr_mlp_predict_keys) → float32 [n].  An unknown key
        scores as an all-zero row, except key 0, which raises CtrError with code ENOTFOUND.  On a row-sharded ITEM_EMB
        (world > 1) each rank scores its own keys and reads the rows from their owners, as Engine.batch_predict_keys
        does: the first call after a table change publishes the shard mappings and must run on every rank, and a
        prediction after training needs sync() on every rank and a barrier between the processes first."""
        u, i, t = self._keys(user_ids, item_ids, ts)
        out = np.empty(u.size, np.float32)
        self._ck(self.L.ctr_mlp_predict_keys(self.h, engine.h, u.ctypes.data_as(_lp), i.ctypes.data_as(_lp), t.ctypes.data_as(_lp),
                                             C.c_int64(u.size), out.ctypes.data_as(_fp)))
        return out

    def recommend_topk(self, engine, user_ids, ts, k, exclude_history=True, exclude_seen=False):
        """Top-k recommendation over every ITEM_EMB row of the feature store `engine` (ctr_mlp_recommend_topk): users
        are external ids, each windowed at its ts (empty history without a ubcache).  Returns (rows [nu, k] int32, scores
        [nu, k] float32, logits [nu, k] float64, counts [nu] int32), best first (logit descending, then row ascending);
        positions past a user's count hold row -1, score 0 and logit 0.  Each score is bit for bit what predict_keys
        returns for (user, the row's item id, ts).  An unknown user raises CtrError with code ENOTFOUND.  exclude_seen
        (implies exclude_history) also drops every item of the user's ubcache events with ts <= the user's ts (0: every
        event).  On a row-sharded ITEM_EMB (world > 1) the call is collective: every rank calls it with the same
        arguments and gets the same complete result, bit-identical to one GPU holding the whole table; arguments or id
        maps that differ across ranks raise CtrError (EINVAL) everywhere, else every rank raises the lowest failing rank's
        error.  Each user's window is the one rank 0's ubcache cuts; under exclude_seen the owner of a row decides from
        its own ubcache.  No sync() is needed after training."""
        u = np.atleast_1d(np.ascontiguousarray(user_ids, np.int64)); t = np.atleast_1d(np.ascontiguousarray(ts, np.int64))
        if u.size != t.size:
            raise ValueError("user_ids and ts differ in length: %d, %d" % (u.size, t.size))
        out_r = np.empty((u.size, k), np.int32); out_s = np.empty((u.size, k), np.float32)
        out_l = np.empty((u.size, k), np.float64); cnt = np.empty(u.size, np.int32)
        mode = _exclusion(u.size, None, exclude_history, exclude_seen)[0]
        self._ck(self.L.ctr_mlp_recommend_topk_ex(self.h, engine.h, u.ctypes.data_as(_lp), t.ctypes.data_as(_lp), C.c_int64(u.size),
                                                  C.c_int32(k), C.c_int32(mode), out_r.ctypes.data_as(_ip),
                                                  out_s.ctypes.data_as(_fp), out_l.ctypes.data_as(C.POINTER(C.c_double)),
                                                  cnt.ctypes.data_as(_ip)))
        return out_r, out_s, out_l, cnt

    def rank_items(self, engine, user_ids, item_ids, ts, exclude_history=True, exclude_seen=False):
        """Full-catalogue rank of held-out items over the feature store `engine` (ctr_mlp_rank_items): key i is (user,
        item, ts) in external ids, windowed at ts as recommend_topk windows it.  Returns (ranks [n] int64, logits [n]
        float64) under Engine.rank_items' rules; an unknown item id ranks -1 (logit NaN), an unknown user raises CtrError
        with code ENOTFOUND.  exclude_seen as for recommend_topk, each key cut at its ts.  On a row-sharded ITEM_EMB the
        call is collective under recommend_topk's rule."""
        u, i, t = self._keys(np.atleast_1d(user_ids), np.atleast_1d(item_ids), np.atleast_1d(ts))
        mode = _exclusion(u.size, None, exclude_history, exclude_seen)[0]
        ranks = np.empty(u.size, np.int64); logits = np.empty(u.size, np.float64)
        self._ck(self.L.ctr_mlp_rank_items_ex(self.h, engine.h, u.ctypes.data_as(_lp), i.ctypes.data_as(_lp), t.ctypes.data_as(_lp),
                                              C.c_int64(u.size), C.c_int32(mode), ranks.ctypes.data_as(_lp),
                                              logits.ctypes.data_as(C.POINTER(C.c_double))))
        return ranks, logits

    def get_params(self):
        """The packed parameter vector (its length follows classes_ on a classifier)."""
        n = C.c_int64(0)
        self._ck(self.L.ctr_mlp_get_params(self.h, None, C.c_int64(0), C.byref(n)))
        p = np.empty(n.value, np.float64)
        self._ck(self.L.ctr_mlp_get_params(self.h, p.ctypes.data_as(C.POINTER(C.c_double)), C.c_int64(n.value), C.byref(n)))
        return p


class MLPClassifier(_Mlp64):
    """nn.MLPClassifier on the device (float64): NewMLPClassifier(hidden, activation, solver, alpha) with
    NewBaseMultilayerPerceptron64's defaults (multilayer_perceptron.go:81-90, basemlp64.go:227-256).

    `adaptive=True` is `learning_rate="adaptive"`; naming another schedule beside it raises.  solver "lbfgs",
    early_stopping and batch_normalize are not built and raise instead of being ignored.

    Labels all 0 or 1 train one logistic output and predict returns probabilities.  Other labels are classes (the
    reference's LabelBinarizer64): after a cold fit, classes_ holds their distinct values ascending, the network has a
    softmax output per class (one logistic output for a single class), and predict / predict_keys return the predicted
    class label of each row.  A warm start keeps the classes and refuses labels with a different class set."""

    def predict(self, X):
        Xa, Xp = _f(X)
        out = np.empty(Xa.shape[0], np.float32)
        self._ck(self.L.ctr_mlp_predict(self.h, Xp, C.c_int64(Xa.shape[0]), C.c_int32(Xa.shape[1]), out.ctypes.data_as(_fp)))
        return out

    def score(self, X, Y):
        """MLPClassifier.Score (ctr_mlp_accuracy): the share of rows whose prediction equals the label.  With classes the
        prediction is the class label; a binary model compares the float64 probability itself, as the reference does,
        so only probabilities of exactly 0.0 or 1.0 can count."""
        Xa, Xp = _f(X); Ya, Yp = _f(Y)
        if Ya.size != Xa.shape[0]:
            raise ValueError("Y has %d labels for %d rows" % (Ya.size, Xa.shape[0]))
        acc = C.c_double(0)
        self._ck(self.L.ctr_mlp_accuracy(self.h, Xp, Yp, C.c_int64(Xa.shape[0]), C.c_int32(Xa.shape[1]), C.byref(acc)))
        return acc.value

    @property
    def classes_(self):
        """The installed classes, float64 ascending; empty for labels all 0 or 1 (ctr_mlp_get_classes)."""
        n = C.c_int32(0)
        self._ck(self.L.ctr_mlp_get_classes(self.h, None, C.c_int32(0), C.byref(n)))
        c = np.empty(n.value, np.float64)
        self._ck(self.L.ctr_mlp_get_classes(self.h, c.ctypes.data_as(C.POINTER(C.c_double)), C.c_int32(n.value), C.byref(n)))
        return c

    def set_params(self, p, classes=None):
        """Installs the packed parameters and marks the model fitted.  classes (ascending, at most 1024; empty for a
        binary model) first installs those classes and sizes the output layer for them (ctr_mlp_set_classes); None
        keeps the current ones."""
        p = np.ascontiguousarray(p, np.float64)
        if classes is not None:
            c = np.ascontiguousarray(classes, np.float64).reshape(-1)
            self._ck(self.L.ctr_mlp_set_classes(self.h, c.ctypes.data_as(C.POINTER(C.c_double)), C.c_int32(c.size)))
        self._ck(self.L.ctr_mlp_set_params(self.h, p.ctypes.data_as(C.POINTER(C.c_double)), C.c_int64(p.size)))


MLP_OUT = {"identity": 0, "logistic": 1, "softmax": 2}


class MLPRegressor(_Mlp64):
    """nn.MLPRegressor on the device (float64): NewMLPRegressor(hidden, activation, solver, alpha) with
    NewBaseMultilayerPerceptron64's defaults (multilayer_perceptron.go:19-28), and the same constructor as
    MLPClassifier plus n_outputs, the number of target columns (1 to 1024).

    Targets are float32 [n, n_outputs] ([n] for one).  A cold fit decides the output from all of them: some target not
    0 or 1 gives an identity output on square_loss; 0/1 targets give a logistic output (one column, the binary
    classifier) or a softmax (more).  out_activation_ names it.  A NaN or infinite target raises CtrError (EINVAL) and
    changes nothing.  predict returns [n, n_outputs]; score is R², the mean of the columns' (MLPRegressor.Score)."""
    _CREATE = "ctr_mlp_regressor_create"

    def __init__(self, n_features, *args, n_outputs=1, **kw):
        if kw.get("early_stopping"):
            raise ValueError("early_stopping is not built: the reference's validation split, best score and best-parameter copy "
                             "(basemlp64.go:826-853) are a change of their own, on top of score")
        self.n_outputs = int(n_outputs)
        super().__init__(n_features, *args, **kw)

    def _targets(self, X, Y):
        Xa, Xp = _f(X); Ya, Yp = _f(Y)
        if Ya.size != Xa.shape[0] * self.n_outputs:
            raise ValueError("Y has %d values for %d rows of %d targets" % (Ya.size, Xa.shape[0], self.n_outputs))
        return Xa, Xp, Ya, Yp

    def fit(self, X, Y):
        self._targets(X, Y)
        return super().fit(X, Y)

    def predict(self, X):
        """MLPRegressor.Predict → float32 [n, n_outputs], float32 of predict_f64 bit for bit"""
        Xa, Xp = _f(X)
        out = np.empty((Xa.shape[0], self.n_outputs), np.float32)
        self._ck(self.L.ctr_mlp_predict(self.h, Xp, C.c_int64(Xa.shape[0]), C.c_int32(Xa.shape[1]), out.ctypes.data_as(_fp)))
        return out

    def predict_f64(self, X):
        """the float64 output layer [n, n_outputs] (ctr_mlp_predict_f64)"""
        Xa, Xp = _f(X)
        out = np.empty((Xa.shape[0], self.n_outputs), np.float64)
        self._ck(self.L.ctr_mlp_predict_f64(self.h, Xp, C.c_int64(Xa.shape[0]), C.c_int32(Xa.shape[1]),
                                            out.ctypes.data_as(C.POINTER(C.c_double))))
        return out

    def score(self, X, Y):
        """MLPRegressor.Score: R² per target column, averaged.  A constant column raises CtrError (EINVAL)."""
        Xa, Xp, Ya, Yp = self._targets(X, Y)
        r2 = C.c_double(0)
        self._ck(self.L.ctr_mlp_score(self.h, Xp, Yp, C.c_int64(Xa.shape[0]), C.c_int32(Xa.shape[1]), C.byref(r2)))
        return r2.value

    @property
    def out_activation_(self):
        """"identity", "logistic" or "softmax" (ctr_mlp_get_output)"""
        k = C.c_int32(0)
        self._ck(self.L.ctr_mlp_get_output(self.h, C.byref(k)))
        return {v: n for n, v in MLP_OUT.items()}[k.value]

    def set_params(self, p, out_activation=None):
        """Installs the packed parameters and marks the model fitted.  out_activation ("identity", "logistic" or
        "softmax") first sets the output kind (ctr_mlp_set_output); None keeps the current one."""
        p = np.ascontiguousarray(p, np.float64)
        if out_activation is not None:
            if out_activation not in MLP_OUT:
                raise ValueError("out_activation must be one of %s, got %r" % (sorted(MLP_OUT), out_activation))
            self._ck(self.L.ctr_mlp_set_output(self.h, C.c_int32(MLP_OUT[out_activation])))
        self._ck(self.L.ctr_mlp_set_params(self.h, p.ctypes.data_as(C.POINTER(C.c_double)), C.c_int64(p.size)))
