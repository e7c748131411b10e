"""ctypes binding of tests/mlp64_class_oracle.c: the float64 MLP classifier on labels that are not all 0 or 1 (classes,
softmax, log_loss, class-label predictions) restated on the CPU.  Test infrastructure only.

Compiled on first use into the system temporary directory, keyed by a hash of its sources, like
tests/mlp64_solver_oracle.py.  Configs are oracle.Mlp64Cfg; options are mlp64_solver_oracle.Opts."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from tests import mlp64_solver_oracle as so

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "mlp64_class_oracle.c")
_HDR = os.path.join(os.path.dirname(_HERE), "oracle", "ctr_oracle.h")
_dp = C.POINTER(C.c_double)
_fp = C.POINTER(C.c_float)
_lib = None
opts = so.opts


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256()
        for p in (_SRC, _HDR):
            with open(p, "rb") as f:
                h.update(f.read())
        so_path = os.path.join(tempfile.gettempdir(), "mlp64_class_oracle_%s_%d.so" % (h.hexdigest()[:16], os.getuid()))
        if not os.path.exists(so_path):
            tmp = "%s.tmp.%d" % (so_path, os.getpid())
            subprocess.check_call(["gcc", "-O2", "-std=c99", "-fPIC", "-shared", "-ffp-contract=off",
                                   "-Wall", "-Wextra", "-o", tmp, _SRC, "-lm"])
            os.replace(tmp, so_path)
        L = C.CDLL(so_path)
        L.cls_classes.restype = C.c_long
        L.cls_classes.argtypes = [_fp, C.c_long, _dp]
        L.cls_transform.argtypes = [_fp, C.c_long, _dp, C.c_long, _dp]
        L.cls_labels.argtypes = [_dp, C.c_long, C.c_long, _dp, _fp]
        L.cls_nparams.restype = C.c_long
        L.cls_loss_grad.restype = C.c_double
        _lib = L
    return _lib


def _f32(a):
    a = np.ascontiguousarray(a, dtype=np.float32).reshape(-1)
    return a, a.ctypes.data_as(_fp)


def _d(a):
    a = np.ascontiguousarray(a, dtype=np.float64)
    return a, a.ctypes.data_as(_dp)


def classes(labels):
    """isBinarized64 + LabelBinarizer64.Fit: None for a NaN label, an empty array for binary labels, else the classes."""
    y, yp = _f32(labels)
    out = np.empty(max(y.size, 1), np.float64)
    c = lib().cls_classes(yp, y.size, out.ctypes.data_as(_dp))
    return None if c < 0 else out[:c].copy()


def transform(labels, cls):
    """LabelBinarizer64.Transform → float64 [n, max(1, C)] (C = 0: the labels as a column)"""
    y, yp = _f32(labels); c, cp = _d(cls)
    out = np.empty((y.size, max(1, c.size)), np.float64)
    lib().cls_transform(yp, y.size, cp, c.size, out.ctypes.data_as(_dp))
    return out


def labels_of(h, cls):
    """InverseTransform over MaxIdx64: float32 [n]"""
    h, hp = _d(h); c, cp = _d(cls)
    out = np.empty(h.shape[0], np.float32)
    lib().cls_labels(hp, h.shape[0], h.shape[1], cp, out.ctypes.data_as(_fp))
    return out


def widen(cfg, cls):
    """the config with the output width max(1, C) that the classes give (the caller's cfg is left as it is)"""
    c = type(cfg).from_buffer_copy(cfg)
    c.units[c.n_layers - 1] = max(1, len(cls))
    return c


def nparams(cfg):
    return int(lib().cls_nparams(C.byref(cfg)))


def init(cfg):
    p = np.empty(nparams(cfg), np.float64)
    lib().cls_init(C.byref(cfg), p.ctypes.data_as(_dp))
    return p


def loss_grad(cfg, params, X, Y):
    X, xp = _d(X); Y, yp = _d(Y); params, pp = _d(params)
    g = np.empty_like(params)
    loss = lib().cls_loss_grad(C.byref(cfg), pp, xp, yp, C.c_long(X.shape[0]), g.ctypes.data_as(_dp))
    return float(loss), g


def predict_proba(cfg, params, X):
    X, xp = _d(X); params, pp = _d(params)
    out = np.empty((X.shape[0], cfg.units[cfg.n_layers - 1]), np.float64)
    lib().cls_predict(C.byref(cfg), pp, xp, C.c_long(X.shape[0]), out.ctypes.data_as(_dp))
    return out


def fit(cfg, o, params, X, Y, t=0.0):
    """fitStochastic on binarized targets Y [n, units[-1]], in place on params → (n_iter, loss_curve, t)"""
    X, xp = _d(X); Y, yp = _d(Y)
    assert params.dtype == np.float64 and params.flags.c_contiguous
    curve = np.zeros(cfg.max_iter, np.float64); tt = C.c_double(t)
    it = lib().cls_fit(C.byref(cfg), C.byref(o), params.ctypes.data_as(_dp), xp, yp, C.c_long(X.shape[0]),
                       curve.ctypes.data_as(_dp), C.byref(tt))
    return it, curve[:it], tt.value


def cold_fit(cfg, o, X, labels):
    """BaseMultilayerPerceptron64.Fit at a cold initialise on float32 labels: → (classes, wide cfg, params, n_iter,
    loss_curve)"""
    cls = classes(labels)
    assert cls is not None, "NaN label"
    wc = widen(cfg, cls)
    p = init(wc)
    it, curve, _ = fit(wc, o, p, X, transform(labels, cls))
    return cls, wc, p, it, curve


def predict(wc, params, cls, X):
    """float32 [n]: probabilities (no classes) or class labels"""
    h = predict_proba(wc, params, X)
    return h[:, 0].astype(np.float32) if len(cls) == 0 else labels_of(h, cls)
