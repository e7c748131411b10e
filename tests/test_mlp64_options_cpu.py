"""The MLP classifier's solver options at the API boundary: ctr_mlp_create_ex validates them before it looks for a
device, so every refusal is checked here without a GPU; the Python wrapper refuses what the engine does not build."""
import ctypes as C

import pytest

import go_ctr_b200 as g


def _cfg(L, adaptive=0):
    cfg = g.MlpConfig()
    L.ctr_mlp_config_default(C.byref(cfg), C.c_int32(20))
    cfg.adaptive = adaptive
    return cfg


def _opts(L, **kw):
    o = g.MlpOptions()
    L.ctr_mlp_options_default(C.byref(o))
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def test_options_default_are_the_reference_defaults():
    """NewBaseMultilayerPerceptron64 (basemlp64.go:227-256): adam, constant, power_t .5, momentum .9, Nesterov, 0."""
    L = g.load_library()
    o = _opts(L)
    assert (o.solver, o.lr_schedule, o.nesterov, o.reserved0) == (0, 0, 1, 0)
    assert (o.power_t, o.momentum, o.weight_decay) == (0.5, 0.9, 0.0) and list(o.reserved) == [0.0] * 5
    assert C.sizeof(g.MlpOptions) == 80


@pytest.mark.parametrize("kw,adaptive,msg", [
    ({"momentum": 1.5}, 0, b"momentum"),
    ({"momentum": -0.1}, 0, b"momentum"),
    ({"momentum": float("nan")}, 0, b"momentum"),
    ({"weight_decay": 1.0}, 0, b"weight_decay"),
    ({"weight_decay": -1e-3}, 0, b"weight_decay"),
    ({"solver": 2}, 0, b"lbfgs is not built"),
    ({"solver": -1}, 0, b"solver"),
    ({"lr_schedule": 3}, 0, b"lr_schedule"),
    ({"lr_schedule": -1}, 0, b"lr_schedule"),
    ({"lr_schedule": 0}, 1, b"adaptive"),
    ({"lr_schedule": 1}, 1, b"adaptive"),
    ({"nesterov": 2}, 0, b"nesterov"),
    ({"power_t": float("inf")}, 0, b"power_t"),
    ({"reserved0": 1}, 0, b"reserved"),
])
def test_invalid_options_are_einval_with_a_reason(kw, adaptive, msg):
    L = g.load_library()
    cfg = _cfg(L, adaptive)
    o = _opts(L, **kw)
    h = C.c_void_p()
    assert L.ctr_mlp_create_ex(C.byref(cfg), C.byref(o), C.byref(h)) == g.EINVAL
    assert msg in L.ctr_mlp_last_error(None) and not h.value


def test_reserved_tail_must_be_zero():
    L = g.load_library()
    o = _opts(L)
    o.reserved[4] = 1.0
    h = C.c_void_p()
    assert L.ctr_mlp_create_ex(C.byref(_cfg(L)), C.byref(o), C.byref(h)) == g.EINVAL
    assert b"reserved" in L.ctr_mlp_last_error(None)


@pytest.mark.parametrize("kw,match", [
    ({"solver": "lbfgs"}, "lbfgs"),
    ({"early_stopping": True}, "early_stopping"),
    ({"batch_normalize": True}, "batch_normalize"),
    ({"adaptive": True, "learning_rate": "invscaling"}, "contradicts"),
    ({"adaptive": True, "learning_rate": "constant"}, "contradicts"),
    ({"solver": "lbgfs"}, "solver"),
    ({"learning_rate": "optimal"}, "learning_rate"),
    ({"activation": "softmax"}, "activation"),
])
def test_wrapper_refuses_what_is_not_built(kw, match):
    with pytest.raises(ValueError, match=match):
        g.MLPClassifier(20, **kw)
