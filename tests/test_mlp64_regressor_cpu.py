"""The MLP regressor at the API boundary: ctr_mlp_regressor_create validates its arguments before it looks for a device,
so every refusal is checked here without a GPU; the Python wrapper refuses what the engine does not build."""
import ctypes as C

import pytest

import go_ctr_b200 as g


def _cfg(L, no):
    cfg = g.MlpConfig()
    L.ctr_mlp_config_default(C.byref(cfg), C.c_int32(20))
    cfg.units[cfg.n_layers - 1] = no
    return cfg


def _opts(L, **kw):
    o = g.MlpOptions()
    L.ctr_mlp_options_default(C.byref(o))
    for k, v in kw.items():
        setattr(o, k, v)
    return o


@pytest.mark.parametrize("no", [0, -1, 1025])
def test_output_width_outside_1_to_1024_is_einval(no):
    L = g.load_library()
    h = C.c_void_p()
    assert L.ctr_mlp_regressor_create(C.byref(_cfg(L, no)), None, C.byref(h)) == g.EINVAL and not h.value


@pytest.mark.parametrize("kw,msg", [
    ({"momentum": 1.5}, b"momentum"),
    ({"weight_decay": 1.0}, b"weight_decay"),
    ({"solver": 2}, b"lbfgs is not built"),
    ({"lr_schedule": 3}, b"lr_schedule"),
    ({"nesterov": 2}, b"nesterov"),
    ({"power_t": float("nan")}, b"power_t"),
    ({"reserved0": 1}, b"reserved"),
])
def test_options_are_refused_as_for_the_classifier(kw, msg):
    L = g.load_library()
    h = C.c_void_p()
    assert L.ctr_mlp_regressor_create(C.byref(_cfg(L, 3)), C.byref(_opts(L, **kw)), C.byref(h)) == g.EINVAL
    assert msg in L.ctr_mlp_last_error(None) and not h.value


def test_a_classifier_still_needs_one_output_and_widths_up_to_1024_reach_the_device_check():
    L = g.load_library()
    h = C.c_void_p()
    assert L.ctr_mlp_create_ex(C.byref(_cfg(L, 3)), None, C.byref(h)) == g.EINVAL
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    for no in (1, 4, 1024):
        assert L.ctr_mlp_regressor_create(C.byref(_cfg(L, no)), None, C.byref(h)) == 2      # CTR_ENODEV: no CPU fallback
        assert b"no CPU fallback" in L.ctr_mlp_last_error(None)


def test_null_model_calls_are_einval():
    L = g.load_library()
    k = C.c_int32(7)
    assert L.ctr_mlp_get_output(None, C.byref(k)) == g.EINVAL and k.value == 7
    assert L.ctr_mlp_set_output(None, C.c_int32(0)) == g.EINVAL
    r2 = C.c_double(0)
    assert L.ctr_mlp_score(None, None, None, C.c_int64(1), C.c_int32(1), C.byref(r2)) == g.EINVAL
    assert L.ctr_mlp_predict_f64(None, None, C.c_int64(1), C.c_int32(1), None) == g.EINVAL


@pytest.mark.parametrize("kw,match", [
    ({"solver": "lbfgs"}, "lbfgs"),
    ({"early_stopping": True}, "early_stopping"),
    ({"batch_normalize": True}, "batch_normalize"),
    ({"adaptive": True, "learning_rate": "constant"}, "contradicts"),
    ({"activation": "softmax"}, "activation"),
])
def test_wrapper_refuses_what_is_not_built(kw, match):
    with pytest.raises(ValueError, match=match):
        g.MLPRegressor(20, n_outputs=2, **kw)


def test_wrapper_is_exported_beside_the_classifier():
    assert "MLPRegressor" in g.engine.__all__ and g.MLPRegressor is g.engine.MLPRegressor
    assert not issubclass(g.MLPRegressor, g.MLPClassifier)
