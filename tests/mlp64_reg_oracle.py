"""ctypes binding of tests/mlp64_reg_oracle.c: the float64 MLP regressor (identity output on square_loss, or the
logistic / softmax output 0/1 targets give; R² score) restated on the CPU.  Test infrastructure only.

Compiled on first use into the system temporary directory, keyed by a hash of its sources, like
tests/mlp64_solver_oracle.py.  Configs are oracle.Mlp64Cfg with units[-1] = the target count; options are
mlp64_solver_oracle.Opts."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from tests import mlp64_solver_oracle as so

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "mlp64_reg_oracle.c")
_HDR = os.path.join(os.path.dirname(_HERE), "oracle", "ctr_oracle.h")
_dp = C.POINTER(C.c_double)
_fp = C.POINTER(C.c_float)
_lib = None
opts = so.opts
OUT = {"identity": 0, "logistic": 1, "softmax": 2}


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256()
        for p in (_SRC, _HDR):
            with open(p, "rb") as f:
                h.update(f.read())
        so_path = os.path.join(tempfile.gettempdir(), "mlp64_reg_oracle_%s_%d.so" % (h.hexdigest()[:16], os.getuid()))
        if not os.path.exists(so_path):
            tmp = "%s.tmp.%d" % (so_path, os.getpid())
            subprocess.check_call(["gcc", "-O2", "-std=c99", "-fPIC", "-shared", "-ffp-contract=off",
                                   "-Wall", "-Wextra", "-o", tmp, _SRC, "-lm"])
            os.replace(tmp, so_path)
        L = C.CDLL(so_path)
        L.reg_out_kind.argtypes = [_fp, C.c_long, C.c_int]
        L.reg_nparams.restype = C.c_long
        L.reg_loss_grad.restype = C.c_double
        L.reg_r2.restype = C.c_double
        L.reg_r2.argtypes = [_dp, _dp, C.c_long, C.c_int, C.POINTER(C.c_long)]
        _lib = L
    return _lib


def _d(a):
    a = np.ascontiguousarray(a, dtype=np.float64)
    return a, a.ctypes.data_as(_dp)


def out_kind(Y):
    """the output kind ("identity", "logistic", "softmax") a cold fit takes from float32 targets [n, no]"""
    y = np.ascontiguousarray(Y, np.float32)
    y2 = y.reshape(y.shape[0], -1)
    k = lib().reg_out_kind(y2.ctypes.data_as(_fp), y2.shape[0], y2.shape[1])
    return {v: n for n, v in OUT.items()}[k]


def nparams(cfg):
    return int(lib().reg_nparams(C.byref(cfg)))


def init(cfg):
    p = np.empty(nparams(cfg), np.float64)
    lib().reg_init(C.byref(cfg), p.ctypes.data_as(_dp))
    return p


def loss_grad(cfg, kind, params, X, Y):
    X, xp = _d(X); Y, yp = _d(Y); params, pp = _d(params)
    g = np.empty_like(params)
    loss = lib().reg_loss_grad(C.byref(cfg), OUT[kind], pp, xp, yp, C.c_long(X.shape[0]), g.ctypes.data_as(_dp))
    return float(loss), g


def predict(cfg, kind, params, X):
    """the float64 output layer [n, units[-1]]"""
    X, xp = _d(X); params, pp = _d(params)
    out = np.empty((X.shape[0], cfg.units[cfg.n_layers - 1]), np.float64)
    lib().reg_predict(C.byref(cfg), OUT[kind], pp, xp, C.c_long(X.shape[0]), out.ctypes.data_as(_dp))
    return out


def r2(y_true, y_pred):
    """r2Score64 → (score, first constant column or -1)"""
    yt, tp = _d(y_true); yp, pp = _d(y_pred)
    n = yt.shape[0]; no = yt.size // n
    bad = C.c_long(0)
    s = lib().reg_r2(tp, pp, C.c_long(n), C.c_int(no), C.byref(bad))
    return s, bad.value


def fit(cfg, kind, o, params, X, Y, t=0.0):
    """fitStochastic on targets Y [n, units[-1]], in place on params → (n_iter, loss_curve, t)"""
    X, xp = _d(X); Y, yp = _d(Y)
    assert params.dtype == np.float64 and params.flags.c_contiguous
    curve = np.zeros(cfg.max_iter, np.float64); tt = C.c_double(t)
    it = lib().reg_fit(C.byref(cfg), OUT[kind], C.byref(o), params.ctypes.data_as(_dp), xp, yp, C.c_long(X.shape[0]),
                       curve.ctypes.data_as(_dp), C.byref(tt))
    return it, curve[:it], tt.value


def cold_fit(cfg, o, X, Y):
    """MLPRegressor.Fit at a cold initialise on float32 targets [n, no] → (kind, params, n_iter, loss_curve)"""
    Y32 = np.asarray(Y, np.float32).reshape(X.shape[0], -1)
    kind = out_kind(Y32)
    p = init(cfg)
    it, curve, _ = fit(cfg, kind, o, p, X, Y32.astype(np.float64))
    return kind, p, it, curve
