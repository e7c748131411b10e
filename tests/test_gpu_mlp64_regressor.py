"""The float64 MLP regressor on the device (MLPRegressor, multilayer_perceptron.go:9-71): dense fits against the CPU
restatement tests/mlp64_reg_oracle.c, 0/1 targets against the classifier, predict / predict_f64 / score, the key-fed
calls against the dense path, recommendation against a full sort, warm starts, restore and the refusals."""
import ctypes as C
import zlib

import numpy as np
import pytest

import go_ctr_b200 as g
from oracle import oracle as orc
from tests import mlp64_reg_oracle as ro
from tests import mlp64_solver_oracle as so
from tests.test_gpu_mlp64_keys import Store, assert_same_fit

pytestmark = pytest.mark.gpu


def _data(n, nf, no, seed):
    """X float32 [n, nf], Y float32 [n, no]: a noisy smooth function of X, one column per target"""
    rng = np.random.default_rng(seed)
    X = rng.random((n, nf), np.float32)
    W = rng.standard_normal((nf, no))
    Y = np.tanh((X - 0.5) @ W) * 2 + 0.1 * rng.standard_normal((n, no)) + 3.0
    return X, Y.astype(np.float32)


def _pair(nf, hidden, no, activation="relu", solver="adam", nesterov=True, learning_rate="constant", **kw):
    m = g.MLPRegressor(nf, hidden=hidden, activation=activation, solver=solver, nesterovs_momentum=nesterov,
                       learning_rate=learning_rate, n_outputs=no, **kw)
    ocfg = orc.mlp64_cfg(nf, hidden=hidden, activation="relu" if activation == "tanh" else activation, n_outputs=no,
                         adaptive=learning_rate == "adaptive", **{k: v for k, v in kw.items() if k != "warm_start"})
    if activation == "tanh":
        ocfg.hidden_act = so.ACT_TANH
    return m, ocfg, so.opts(solver, learning_rate, nesterov=nesterov)


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint64 if a.dtype == np.float64 else np.uint32)


# ---- dense fit against the restatement ----------------------------------------------------------------------------------
DENSE = {
    "adam_relu_1": dict(hidden=(32, 16), no=1),
    "adam_tanh_3": dict(hidden=(32, 16), no=3, activation="tanh"),
    "adam_logistic_3_noshuffle": dict(hidden=(16,), no=3, activation="logistic", shuffle=False),
    "adam_identity_nohidden_1": dict(hidden=(), no=1, activation="identity"),
    "sgd_nesterov_relu_3": dict(hidden=(32, 16), no=3, solver="sgd", lr_init=0.01),
    "sgd_invscaling_tanh_1": dict(hidden=(16,), no=1, solver="sgd", learning_rate="invscaling", lr_init=0.05, activation="tanh"),
    "sgd_adaptive_relu_1": dict(hidden=(), no=1, solver="sgd", learning_rate="adaptive", lr_init=0.01, tol=1e-2, n_iter_no_change=1),
}


@pytest.mark.parametrize("case", sorted(DENSE))
def test_dense_fit_follows_the_restatement(case):
    spec = dict(DENSE[case])
    hidden, no = spec.pop("hidden"), spec.pop("no")
    nf = 24
    X, Y = _data(1130, nf, no, zlib.crc32(case.encode()))        # 1130 rows: a ragged last minibatch of 130
    X64 = X.astype(np.float64)
    spec.setdefault("tol", 0.0)
    # one full-batch step, no shuffle: the device's only differences are FMA contraction and the loss's tree sum
    one = {k: v for k, v in spec.items() if k not in ("shuffle", "tol", "n_iter_no_change")}
    m, ocfg, o = _pair(nf, hidden, no, batch=1130, max_iter=1, shuffle=False, seed=3, **one)
    m.fit(X, Y)
    kind, po, it, curve = ro.cold_fit(ocfg, o, X64, Y)
    assert kind == "identity" and m.out_activation_ == "identity"
    assert m.get_params().size == ro.nparams(ocfg) and m.n_iter == it == 1
    np.testing.assert_allclose(m.loss_curve, curve, rtol=1e-9)
    np.testing.assert_allclose(m.get_params(), po, rtol=1e-9, atol=1e-12)
    # six epochs in minibatches of 200, the last ragged; those differences compound, as in the classifier's tests
    m, ocfg, o = _pair(nf, hidden, no, max_iter=6, seed=3, **spec)
    m.fit(X, Y)
    kind, po, it, curve = ro.cold_fit(ocfg, o, X64, Y)
    assert m.n_iter == it
    np.testing.assert_allclose(m.loss_curve, curve, rtol=1e-7)
    np.testing.assert_allclose(m.get_params(), po, rtol=1e-5, atol=1e-7)
    f64 = m.predict_f64(X)
    np.testing.assert_allclose(f64, ro.predict(ocfg, kind, m.get_params(), X64), rtol=1e-12, atol=1e-13)
    assert np.array_equal(_bits(m.predict(X)), _bits(f64.astype(np.float32)))
    s = m.score(X, Y)
    want, bad = ro.r2(Y.astype(np.float64), f64)
    assert bad == -1 and abs(s - want) <= 1e-12
    assert _bits(np.float64(m.score(X, Y))) == _bits(np.float64(s))


# ---- 0/1 targets -----------------------------------------------------------------------------------------------------------
def test_one_zero_one_column_is_the_binary_classifier_bit_for_bit():
    X, _ = _data(900, 20, 1, 1)
    y = (np.random.default_rng(1).random(900) < 0.4).astype(np.float32)
    y[::11] = -0.0
    kw = dict(hidden=(16,), max_iter=4, seed=7, tol=0.0)
    r = g.MLPRegressor(20, **kw).fit(X, y)
    c = g.MLPClassifier(20, **kw).fit(X, y)
    assert r.out_activation_ == "logistic" and r.n_iter == c.n_iter
    assert _bits(r.loss_curve).tobytes() == _bits(c.loss_curve).tobytes()
    assert r.get_params().tobytes() == c.get_params().tobytes()
    assert np.array_equal(_bits(r.predict(X).ravel()), _bits(c.predict(X)))


def test_three_zero_one_columns_train_a_softmax_on_dense_log_loss():
    X, _ = _data(700, 16, 3, 2)
    Y = (np.random.default_rng(2).random((700, 3)) < 0.4).astype(np.float32)     # not one-hot: rows of 0, 1, 2 or 3 ones
    m, ocfg, o = _pair(16, (12,), 3, max_iter=4, seed=5, tol=0.0)
    m.fit(X, Y)
    kind, po, it, curve = ro.cold_fit(ocfg, o, X.astype(np.float64), Y)
    assert kind == "softmax" and m.out_activation_ == "softmax" and m.n_iter == it
    np.testing.assert_allclose(m.loss_curve, curve, rtol=1e-7)
    np.testing.assert_allclose(m.get_params(), po, rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(m.predict_f64(X).sum(axis=1), 1.0, rtol=1e-14)


# ---- score --------------------------------------------------------------------------------------------------------------------
def test_score_matches_the_restatement_and_refuses_a_constant_column():
    X, Y = _data(50_000, 10, 3, 3)
    m = g.MLPRegressor(10, hidden=(8,), max_iter=2, seed=1, n_outputs=3).fit(X, Y)
    want, _ = ro.r2(Y.astype(np.float64), m.predict_f64(X))
    s = [m.score(X, Y) for _ in range(3)]
    assert abs(s[0] - want) <= 1e-12 and len({_bits(np.float64(v)).tobytes() for v in s}) == 1
    Yc = Y.copy(); Yc[:, 1] = 3.0
    with pytest.raises(g.CtrError) as e:
        m.score(X, Yc)
    assert e.value.code == g.EINVAL and "column 1" in str(e.value)


# ---- key-fed fit, predict and recommend -----------------------------------------------------------------------------------
def _ratings(rng, n):
    return rng.choice(np.float32([0.5, 1.0, 1.5, 2.0, 2.5, 3.0, 3.5, 4.0, 4.5, 5.0]), n)


@pytest.mark.parametrize("mlp", [dict(), dict(solver="sgd", lr_init=0.02, activation="tanh")])
def test_fit_keys_and_predict_keys_are_bit_identical_to_the_dense_path(mlp):
    rng = np.random.default_rng(8)
    st = Store(rng, pred_batch=64)
    u, i, t, _ = st.keys(rng, 1500)
    y = _ratings(rng, u.size)
    X, Y = st.dense(u, i, t, y)
    kw = dict(hidden=(16,), max_iter=4, seed=3, tol=0.0, **mlp)
    mk = g.MLPRegressor(st.nin, **kw).fit_keys(st.eng, u, i, t, y)
    mr = g.MLPRegressor(st.nin, **kw).fit(X, Y)
    assert mk.out_activation_ == mr.out_activation_ == "identity"
    assert_same_fit(mk, mr, X.shape[0])
    q = st.keys(rng, 231)
    qu, qi, qt = q[0].copy(), q[1].copy(), q[2]
    qu[0], qi[0] = st.uid[3], st.iid[5]                       # key 0 known; later unknown keys score as a zero row
    ur, ir, hist, ok = st.rows(qu, qi, qt, drop=False)
    want = mk.predict(st.eng.gather_rows(ur, ir, hist)).ravel()
    got = mk.predict_keys(st.eng, qu, qi, qt)
    assert np.array_equal(_bits(got), _bits(want)) and (~ok).any()
    with pytest.raises(g.CtrError) as e:
        mk.predict_keys(st.eng, q[0], q[1], q[2])               # key 0 unknown
    assert e.value.code == g.ENOTFOUND


def test_fit_keys_with_zero_one_labels_is_the_binary_classifier():
    rng = np.random.default_rng(9)
    st = Store(rng)
    u, i, t, y = st.keys(rng, 1200)
    kw = dict(hidden=(16,), max_iter=3, seed=3, tol=0.0)
    r = g.MLPRegressor(st.nin, **kw).fit_keys(st.eng, u, i, t, y)
    c = g.MLPClassifier(st.nin, **kw).fit_keys(st.eng, u, i, t, y)
    assert r.out_activation_ == "logistic"
    assert_same_fit(r, c, c.rows_used)
    uid = np.array([st.uid[2]], np.int64); ts = np.array([4_990_000], np.int64)
    a, b = r.recommend_topk(st.eng, uid, ts, 20), c.recommend_topk(st.eng, uid, ts, 20)
    assert all(np.array_equal(_bits(x) if x.dtype.kind == "f" else x, _bits(z) if z.dtype.kind == "f" else z) for x, z in zip(a, b))


@pytest.mark.parametrize("exclude", [False, True])
def test_recommend_is_a_full_sort_of_predict_f64(exclude):
    rng = np.random.default_rng(10)
    st = Store(rng, pred_batch=256)
    u, i, t, _ = st.keys(rng, 1500)
    m = g.MLPRegressor(st.nin, hidden=(16, 8), max_iter=3, seed=1).fit_keys(st.eng, u, i, t, _ratings(rng, u.size))
    I = st.iid.size
    for uk, ts in ((st.uid[2], 4_990_000), (st.uid[7], 0)):
        urow = st.umap[int(uk)]
        hist = st.eng.ubcache_window(np.array([urow], np.int32), np.array([ts], np.int64))
        X = st.eng.gather_rows(np.full(I, urow, np.int32), np.arange(I, dtype=np.int32), np.repeat(hist, I, axis=0))
        v = m.predict_f64(X).ravel()
        keep = np.ones(I, bool)
        if exclude:
            keep[hist[0][(hist[0] >= 0) & (hist[0] < I)]] = False
        rows = np.arange(I)[keep]
        order = rows[np.lexsort((rows, -v[keep]))]
        k = 50
        r, s, lg, cnt = m.recommend_topk(st.eng, np.array([uk], np.int64), np.array([ts], np.int64), k, exclude_history=exclude)
        assert cnt[0] == k and np.array_equal(r[0], order[:k])
        assert np.array_equal(_bits(lg[0]), _bits(v[order[:k]]))
        assert np.array_equal(_bits(s[0]), _bits(v[order[:k]].astype(np.float32)))


def test_recommend_with_three_targets_is_refused_and_key_fed_calls_are_einval():
    rng = np.random.default_rng(11)
    st = Store(rng)
    u, i, t, _ = st.keys(rng, 600)
    X, Y = _data(300, st.nin, 3, 11)
    m = g.MLPRegressor(st.nin, hidden=(8,), max_iter=2, seed=1, n_outputs=3).fit(X, Y)
    with pytest.raises(g.CtrError) as e:
        m.recommend_topk(st.eng, np.array([st.uid[1]], np.int64), np.array([0], np.int64), 5)
    assert e.value.code == g.ESTATE
    before = m.get_params().tobytes()
    with pytest.raises(g.CtrError) as e:
        m.fit_keys(st.eng, u, i, t, _ratings(rng, u.size))
    assert e.value.code == g.EINVAL and m.get_params().tobytes() == before
    with pytest.raises(g.CtrError) as e:
        m.predict_keys(st.eng, u[1:5], i[1:5], t[1:5])
    assert e.value.code == g.EINVAL


# ---- warm start, restore, refusals ---------------------------------------------------------------------------------------
def test_warm_start_keeps_parameters_and_output_kind():
    X, Y = _data(800, 12, 2, 12)
    kw = dict(hidden=(8,), max_iter=2, seed=5, tol=0.0, n_outputs=2)
    m = g.MLPRegressor(12, warm_start=True, **kw).fit(X, Y)
    p1 = m.get_params()
    Yb = (Y > 3.0).astype(np.float32)                        # 0/1 targets would make a cold fit softmax
    m.fit(X, Yb)
    assert m.out_activation_ == "identity" and not np.array_equal(m.get_params(), p1)
    ocfg = orc.mlp64_cfg(12, hidden=(8,), n_outputs=2, max_iter=2, seed=5, tol=0.0)
    p = p1.copy()
    ro.fit(ocfg, "identity", so.opts(), p, X.astype(np.float64), Yb.astype(np.float64))
    np.testing.assert_allclose(m.get_params(), p, rtol=1e-5, atol=1e-7)
    assert g.MLPRegressor(12, **kw).fit(X, Yb).out_activation_ == "softmax"


def test_restore_through_output_kind_and_params_predicts_bit_identically():
    X, Y = _data(500, 10, 1, 13)
    m = g.MLPRegressor(10, hidden=(6,), max_iter=3, seed=2).fit(X, Y)
    r = g.MLPRegressor(10, hidden=(6,))
    r.set_params(np.zeros_like(m.get_params()), out_activation="logistic")
    assert r.out_activation_ == "logistic"
    r.L.ctr_mlp_set_output(r.h, C.c_int32(0))
    with pytest.raises(g.CtrError) as e:
        r.predict(X)                                           # set_output leaves it unfitted until set_params
    assert e.value.code == g.ESTATE
    r.set_params(m.get_params(), out_activation=m.out_activation_)
    assert np.array_equal(_bits(r.predict_f64(X)), _bits(m.predict_f64(X)))
    with pytest.raises(g.CtrError) as e:
        r.set_params(m.get_params(), out_activation="softmax")  # one target: never softmax
    assert e.value.code == g.EINVAL
    c = np.array([1.0, 2.0]); n = C.c_int32(9)
    assert r.L.ctr_mlp_set_classes(r.h, c.ctypes.data_as(C.POINTER(C.c_double)), C.c_int32(2)) == g.ESTATE
    assert r.L.ctr_mlp_get_classes(r.h, None, C.c_int32(0), C.byref(n)) == 0 and n.value == 0
    # a classifier: its output follows its classes, and its accuracy score is not built
    cl = g.MLPClassifier(10, hidden=(6,), max_iter=2).fit(X, (Y[:, 0] > 3).astype(np.float32))
    assert cl.L.ctr_mlp_set_output(cl.h, C.c_int32(0)) == g.ESTATE
    r2 = C.c_double(0)
    assert cl.L.ctr_mlp_score(cl.h, X.ctypes.data_as(C.POINTER(C.c_float)), Y.ctypes.data_as(C.POINTER(C.c_float)),
                              C.c_int64(500), C.c_int32(10), C.byref(r2)) == g.ESTATE


def test_non_finite_targets_are_refused_and_change_nothing():
    X, Y = _data(600, 10, 2, 14)
    m = g.MLPRegressor(10, hidden=(6,), max_iter=2, seed=1, n_outputs=2).fit(X, Y)
    before = m.get_params().tobytes()
    for v in (np.nan, np.inf, -np.inf):
        bad = Y.copy(); bad[123, 1] = v
        with pytest.raises(g.CtrError) as e:
            m.fit(X, bad)
        assert e.value.code == g.EINVAL and m.get_params().tobytes() == before and m.out_activation_ == "identity"
