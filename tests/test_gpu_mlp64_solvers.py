"""model/mlp on the device beyond Adam: SGD with momentum / Nesterov, the invscaling and adaptive schedules, tanh and
weight decay, against the CPU restatement tests/mlp64_solver_oracle.c (float64 both sides: FMA contraction and libm
ulps are the only differences, so the bars are those of test_gpu_mlp64.py)."""
import ctypes as C

import numpy as np
import pytest

import go_ctr_b200 as g
from oracle import oracle as orc
from tests import mlp64_solver_oracle as so

pytestmark = pytest.mark.gpu


def _data(n, nf, seed):
    rng = np.random.default_rng(seed)
    X = rng.random((n, nf), np.float32)
    w = rng.standard_normal(nf)
    y = ((X - 0.5) @ w + 0.3 * rng.standard_normal(n) > 0).astype(np.float32)
    return X, y


def _pair(nf, hidden, activation="relu", solver="adam", learning_rate="constant", power_t=0.5, momentum=0.9,
          nesterov=True, weight_decay=0.0, **kw):
    """the device classifier and the oracle's (cfg, opts) for one setting"""
    m = g.MLPClassifier(nf, hidden=hidden, activation=activation, solver=solver, learning_rate=learning_rate,
                        power_t=power_t, momentum=momentum, nesterovs_momentum=nesterov, weight_decay=weight_decay, **kw)
    okw = {k: v for k, v in kw.items() if k != "warm_start"}
    ocfg = orc.mlp64_cfg(nf, hidden=hidden, activation="relu" if activation == "tanh" else activation,
                         adaptive=learning_rate == "adaptive", **okw)
    if activation == "tanh":
        ocfg.hidden_act = so.ACT_TANH
    return m, ocfg, so.opts(solver, learning_rate, power_t, momentum, nesterov, weight_decay)


def _f64(X, y):
    return X.astype(np.float64), y.astype(np.float64).reshape(-1, 1)


@pytest.mark.parametrize("momentum", [0.0, 0.9])
@pytest.mark.parametrize("nesterov", [False, True])
def test_full_batch_sgd_steps_match_the_oracle(momentum, nesterov):
    """Two full-batch SGDOptimizer64.updateParams calls (basemlp64.go:1024-1039) from set parameters, so the
    velocity of the first step feeds the second."""
    nf, n = 281, 200
    X, y = _data(n, nf, 1)
    m, ocfg, o = _pair(nf, (100,), solver="sgd", momentum=momentum, nesterov=nesterov, batch=n, max_iter=2,
                       shuffle=False, seed=5, lr_init=0.05, warm_start=True)
    p0 = so.init(ocfg)
    po = p0.copy()
    it, curve, _, _ = so.fit(ocfg, o, po, *_f64(X, y))
    m.set_params(p0)
    m.fit(X, y)
    assert m.n_iter == it == 2
    np.testing.assert_allclose(m.loss_curve, curve, rtol=1e-12)
    np.testing.assert_allclose(m.get_params(), po, rtol=1e-9, atol=1e-12)


def _five_epochs(m, ocfg, o, X, y, n_iter=None):
    po = so.init(ocfg)
    it, curve, _, _ = so.fit(ocfg, o, po, *_f64(X, y))
    m.fit(X, y)
    assert m.n_iter == it
    if n_iter is not None:
        assert it == n_iter
    np.testing.assert_allclose(m.loss_curve, curve, rtol=1e-7)
    pg = m.predict(X[:500]); pc = so.predict(ocfg, po, X[:500].astype(np.float64)).ravel().astype(np.float32)
    np.testing.assert_allclose(pg, pc, rtol=1e-5, atol=1e-7)
    return curve


@pytest.mark.parametrize("schedule", ["constant", "invscaling"])
def test_sgd_over_shuffled_epochs_follows_the_oracle(schedule):
    """configs[0] shape: 281 -> 100 -> 1, relu, batch 200, five shuffled epochs."""
    X, y = _data(3000, 281, 2)
    m, ocfg, o = _pair(281, (100,), solver="sgd", learning_rate=schedule, max_iter=5, seed=9, lr_init=0.05)
    curve = _five_epochs(m, ocfg, o, X, y, n_iter=5)
    assert curve[-1] < curve[0]


def test_adaptive_sgd_stops_at_the_oracle_epoch():
    """tol so large that no epoch improves: every second epoch triggers (:826-840), the current rate shrinks by .8
    (:1018) from 1.5e-6 to 1.2e-6 and 9.6e-7, and the next trigger stops (:1012-1017) — at epoch 7 of 10."""
    X, y = _data(3000, 281, 3)
    m, ocfg, o = _pair(281, (100,), solver="sgd", learning_rate="adaptive", max_iter=10, seed=4, lr_init=1.5e-6,
                       tol=1e9, n_iter_no_change=1)
    _five_epochs(m, ocfg, o, X, y, n_iter=7)


@pytest.mark.parametrize("solver", ["adam", "sgd"])
def test_tanh_two_hidden_layers_follows_the_oracle(solver):
    """281 -> 64 -> 32 -> 1 tanh: tanh(-z) forward, 1 - a² backward (:88-94, :131-138), layer 0 below two tanh
    layers, layer 1 below one (its data gradient negated, as in the reference)."""
    X, y = _data(3000, 281, 5)
    m, ocfg, o = _pair(281, (64, 32), activation="tanh", solver=solver, max_iter=5, seed=6,
                       lr_init=0.02 if solver == "sgd" else 1e-3)
    _five_epochs(m, ocfg, o, X, y, n_iter=5)


@pytest.mark.parametrize("solver", ["adam", "sgd"])
def test_weight_decay_follows_the_oracle(solver):
    """every packed parameter times (1 - wd) before each minibatch (:342-346); the L2 term sees the decayed values."""
    X, y = _data(3000, 281, 7)
    m, ocfg, o = _pair(281, (100,), solver=solver, weight_decay=1e-3, max_iter=5, seed=8,
                       lr_init=0.05 if solver == "sgd" else 1e-3)
    _five_epochs(m, ocfg, o, X, y, n_iter=5)


def test_warm_start_invscaling_continues_the_sample_count():
    """The second fit of a warm-started classifier keeps its parameters and t (initialize is skipped, :502-512):
    its learning rates continue at lr_init / (t+1)^power_t with t = 3000·epochs so far, from lr_init again (a
    fresh optimizer, :731-752)."""
    X, y = _data(3000, 281, 9)
    m, ocfg, o = _pair(281, (100,), solver="sgd", learning_rate="invscaling", power_t=0.4, max_iter=3, seed=10,
                       lr_init=0.05, warm_start=True)
    po = so.init(ocfg)
    Xd, yd = _f64(X, y)
    _, c1, _, t = so.fit(ocfg, o, po, Xd, yd)
    _, c2, _, t = so.fit(ocfg, o, po, Xd, yd, t=t)
    assert t == 6 * 3000
    m.fit(X, y)
    np.testing.assert_allclose(m.loss_curve, c1, rtol=1e-7)
    m.fit(X, y)
    np.testing.assert_allclose(m.loss_curve, c2, rtol=1e-7)
    pc = so.init(ocfg)                                 # had t restarted at 0, the second curve would sit well outside 1e-7
    so.fit(ocfg, o, pc, Xd, yd)
    _, c2_cold, _, _ = so.fit(ocfg, o, pc, Xd, yd, t=0.0)
    assert np.max(np.abs(c2_cold - c2) / np.abs(c2)) > 20 * 1e-7
    pg = m.predict(X[:500]); pc = so.predict(ocfg, po, Xd[:500]).ravel().astype(np.float32)
    np.testing.assert_allclose(pg, pc, rtol=1e-5, atol=1e-7)


def test_create_and_create_ex_with_default_options_train_identically():
    """ctr_mlp_create(cfg) is ctr_mlp_create_ex(cfg, NULL) is ctr_mlp_create_ex(cfg, defaults): same parameters to
    the bit after a shuffled multi-epoch fit."""
    L = g.load_library()
    X, y = _data(1000, 50, 11)
    cfg = g.MlpConfig()
    L.ctr_mlp_config_default(C.byref(cfg), C.c_int32(50))
    cfg.max_iter = 3; cfg.seed = 12
    o = g.MlpOptions()
    L.ctr_mlp_options_default(C.byref(o))
    Xa = np.ascontiguousarray(X); ya = np.ascontiguousarray(y)
    out = []
    for create in (lambda h: L.ctr_mlp_create(C.byref(cfg), C.byref(h)),
                   lambda h: L.ctr_mlp_create_ex(C.byref(cfg), None, C.byref(h)),
                   lambda h: L.ctr_mlp_create_ex(C.byref(cfg), C.byref(o), C.byref(h))):
        h = C.c_void_p()
        assert create(h) == 0
        it = C.c_int32(0)
        assert L.ctr_mlp_fit(h, Xa.ctypes.data_as(C.POINTER(C.c_float)), ya.ctypes.data_as(C.POINTER(C.c_float)),
                             C.c_int64(1000), C.c_int32(50), C.byref(it), None) == 0
        n = C.c_int64(0)
        assert L.ctr_mlp_get_params(h, None, C.c_int64(0), C.byref(n)) == 0
        p = np.empty(n.value, np.float64)
        assert L.ctr_mlp_get_params(h, p.ctypes.data_as(C.POINTER(C.c_double)), n, C.byref(n)) == 0
        L.ctr_mlp_destroy(h)
        out.append((it.value, p.tobytes()))
    assert out[0] == out[1] == out[2] and out[0][0] == 3
    m = g.MLPClassifier(50, max_iter=3, seed=12)            # the wrapper's default path is the same classifier
    m.fit(X, y)
    assert m.get_params().tobytes() == out[0][1]
