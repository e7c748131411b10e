"""ctypes binding of tests/mlp64_solver_oracle.c: the float64 MLP classifier's solver surface (adam / sgd, lr schedules,
tanh, weight decay) restated on the CPU.  Test infrastructure only.

The library is compiled on first use into the system temporary directory, keyed by a hash of its sources, so the
repository tree is never written to.  Configs are oracle.Mlp64Cfg (oracle.mlp64_cfg builds them)."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "mlp64_solver_oracle.c")
_HDR = os.path.join(os.path.dirname(_HERE), "oracle", "ctr_oracle.h")
_dp = C.POINTER(C.c_double)
_lib = None

SOLVER = {"adam": 0, "sgd": 1}
LR = {"constant": 0, "invscaling": 1, "adaptive": 2}
ACT_TANH = 3


class Opts(C.Structure):
    """ctr_mlp_options' layout (include/ctr_b200.h)."""
    _fields_ = [("solver", C.c_int32), ("lr_schedule", C.c_int32), ("nesterov", C.c_int32), ("reserved0", C.c_int32),
                ("power_t", C.c_double), ("momentum", C.c_double), ("weight_decay", C.c_double), ("reserved", C.c_double * 5)]


def opts(solver="adam", learning_rate="constant", power_t=0.5, momentum=0.9, nesterov=True, weight_decay=0.0):
    """BaseMultilayerPerceptron64's defaults (basemlp64.go:227-256)."""
    o = Opts()
    o.solver = SOLVER[solver]; o.lr_schedule = LR[learning_rate]; o.nesterov = int(bool(nesterov))
    o.power_t = power_t; o.momentum = momentum; o.weight_decay = weight_decay
    return o


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256()
        for p in (_SRC, _HDR):
            with open(p, "rb") as f:
                h.update(f.read())
        so = os.path.join(tempfile.gettempdir(), "mlp64_solver_oracle_%s_%d.so" % (h.hexdigest()[:16], os.getuid()))
        if not os.path.exists(so):
            tmp = "%s.tmp.%d" % (so, os.getpid())
            subprocess.check_call(["gcc", "-O2", "-std=c99", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off",
                                   "-Wall", "-Wextra", "-o", tmp, _SRC, "-lm"])
            os.replace(tmp, so)
        L = C.CDLL(so)
        L.sol_nparams.restype = C.c_long
        L.sol_loss_grad.restype = C.c_double
        L.sol_sgd.argtypes = [C.c_void_p, C.c_double, _dp, _dp, _dp, C.c_long]
        L.sol_decay.argtypes = [C.c_double, _dp, C.c_long]
        _lib = L
    return _lib


def _d(a):
    a = np.ascontiguousarray(a, dtype=np.float64)
    return a, a.ctypes.data_as(_dp)


def nparams(cfg):
    return int(lib().sol_nparams(C.byref(cfg)))


def init(cfg):
    p = np.empty(nparams(cfg), np.float64)
    lib().sol_init(C.byref(cfg), p.ctypes.data_as(_dp))
    return p


def loss_grad(cfg, params, X, y):
    X, xp = _d(X); y, yp = _d(y); params, pp = _d(params)
    g = np.empty_like(params)
    loss = lib().sol_loss_grad(C.byref(cfg), pp, xp, yp, C.c_long(X.shape[0]), g.ctypes.data_as(_dp))
    return float(loss), g


def predict(cfg, params, X):
    X, xp = _d(X); params, pp = _d(params)
    out = np.empty((X.shape[0], cfg.units[cfg.n_layers - 1]), np.float64)
    lib().sol_predict(C.byref(cfg), pp, xp, C.c_long(X.shape[0]), out.ctypes.data_as(_dp))
    return out


def sgd(o, lr, params, grads, vel):
    """one SGDOptimizer64.updateParams, in place on params and vel"""
    assert params.dtype == vel.dtype == np.float64 and params.flags.c_contiguous and vel.flags.c_contiguous
    grads, gp = _d(grads)
    lib().sol_sgd(C.byref(o), lr, params.ctypes.data_as(_dp), gp, vel.ctypes.data_as(_dp), params.size)


def decay(weight_decay, params):
    assert params.dtype == np.float64 and params.flags.c_contiguous
    lib().sol_decay(weight_decay, params.ctypes.data_as(_dp), params.size)


def fit(cfg, o, params, X, y, t=0.0):
    """In place on params; returns (n_iter, loss_curve, lr_curve, t) — t = samples seen since the cold initialise,
    carried in and out (pass the previous fit's t for a warm start)."""
    X, xp = _d(X); y, yp = _d(y)
    assert params.dtype == np.float64 and params.flags.c_contiguous
    curve = np.zeros(cfg.max_iter, np.float64); lrs = np.zeros(cfg.max_iter, np.float64); tt = C.c_double(t)
    it = lib().sol_fit(C.byref(cfg), C.byref(o), params.ctypes.data_as(_dp), xp, yp, C.c_long(X.shape[0]),
                       curve.ctypes.data_as(_dp), lrs.ctypes.data_as(_dp), C.byref(tt))
    return it, curve[:it], lrs[:it], tt.value
