"""The float64 MLP classifier on labels that are not all 0 or 1: classes, a softmax output on log_loss, class-label
predictions (BaseMultilayerPerceptron64.Fit, basemlp64.go:578-598), against the CPU restatement
tests/mlp64_class_oracle.c, the dense path against the key-fed one, and every refusal."""
import ctypes as C
import zlib

import numpy as np
import pytest

import go_ctr_b200 as g
from go_ctr_b200 import model as gm
from go_ctr_b200 import serving as sv
from oracle import oracle as orc
from tests import mlp64_class_oracle as co
from tests import mlp64_solver_oracle as so
from tests.test_gpu_mlp64_keys import Store, assert_same_fit

pytestmark = pytest.mark.gpu

RATINGS = [0.5, 1.0, 1.5, 2.0, 2.5, 3.0, 3.5, 4.0, 4.5, 5.0]


def _data(n, nf, seed, values):
    """X float32 [n, nf] and labels from `values`, by quantile of a noisy linear score (every value present)"""
    rng = np.random.default_rng(seed)
    X = rng.random((n, nf), np.float32)
    score = (X - 0.5) @ rng.standard_normal(nf) + 0.3 * rng.standard_normal(n)
    q = np.quantile(score, np.linspace(0, 1, len(values) + 1)[1:-1])
    return X, np.asarray(values, np.float32)[np.searchsorted(q, score)]


def _pair(nf, hidden, activation="relu", solver="adam", nesterov=True, weight_decay=0.0, **kw):
    m = g.MLPClassifier(nf, hidden=hidden, activation=activation, solver=solver, nesterovs_momentum=nesterov,
                        weight_decay=weight_decay, **kw)
    ocfg = orc.mlp64_cfg(nf, hidden=hidden, activation="relu" if activation == "tanh" else activation,
                         **{k: v for k, v in kw.items() if k != "warm_start"})
    if activation == "tanh":
        ocfg.hidden_act = so.ACT_TANH
    return m, ocfg, so.opts(solver, nesterov=nesterov, weight_decay=weight_decay)


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64 if np.asarray(a).dtype == np.float64 else np.uint32)


def _snapshot(m):
    return m.get_params().tobytes(), m.classes_.tobytes()


# ---- dense fit against the restatement ------------------------------------------------------------------------------
DENSE = {
    "c2_not01_adam_relu": dict(values=[1.0, 5.0], hidden=(16,)),
    "c3_adam_relu": dict(values=[0.0, 1.0, 2.0], hidden=(16,)),
    "c10_adam_relu": dict(values=RATINGS, hidden=(32,)),
    "c10_sgd_nesterov": dict(values=RATINGS, hidden=(32,), solver="sgd", lr_init=0.05),
    "c3_tanh_two_layers": dict(values=[-1.0, 0.0, 3.0], hidden=(12, 8), activation="tanh"),
    "c3_weight_decay": dict(values=[2.0, 4.0, 8.0], hidden=(16,), weight_decay=0.01),
    "c10_no_hidden": dict(values=RATINGS, hidden=()),
}


@pytest.mark.parametrize("case", sorted(DENSE))
def test_dense_fit_follows_the_restatement(case):
    spec = dict(DENSE[case])
    values, hidden = spec.pop("values"), spec.pop("hidden")
    nf = 40
    X, y = _data(1200, nf, zlib.crc32(case.encode()), values)
    X64 = X.astype(np.float64)
    # one full-batch step, no shuffle
    m, ocfg, o = _pair(nf, hidden, batch=1200, max_iter=1, shuffle=False, seed=3, **spec)
    m.fit(X, y)
    cls, wc, po, it, curve = co.cold_fit(ocfg, o, X64, y)
    assert m.classes_.tobytes() == cls.tobytes() and cls.tolist() == sorted(values)
    assert m.get_params().size == co.nparams(wc) and m.n_iter == it == 1
    np.testing.assert_allclose(m.loss_curve, curve, rtol=1e-9)
    np.testing.assert_allclose(m.get_params(), po, rtol=1e-9, atol=1e-12)
    # five shuffled epochs in minibatches of 200
    m, ocfg, o = _pair(nf, hidden, max_iter=5, seed=9, tol=0.0, **spec)
    m.fit(X, y)
    cls, wc, po, it, curve = co.cold_fit(ocfg, o, X64, y)
    assert m.n_iter == it == 5
    np.testing.assert_allclose(m.loss_curve, curve, rtol=1e-7)
    got = m.predict(X)
    assert set(np.unique(got)) <= set(np.float32(values))
    # the device's own parameters through the restatement's predict: equal labels except near-ties
    h = co.predict_proba(wc, m.get_params(), X64)
    top2 = np.sort(h, axis=1)[:, -2:] if h.shape[1] > 1 else np.zeros((h.shape[0], 2))
    tie = (top2[:, 1] - top2[:, 0]) < 1e-9 if h.shape[1] > 1 else np.zeros(h.shape[0], bool)
    assert tie.sum() <= 3
    want = co.labels_of(h, cls)
    assert np.array_equal(got[~tie], want[~tie])
    # the restatement's own fit predicts the same labels but for a few rows near a boundary
    assert np.mean(co.predict(wc, po, cls, X64) != got) < 0.01


# ---- label edge cases -------------------------------------------------------------------------------------------------
def test_single_class_trains_a_logistic_unit_on_ones_and_predicts_it():
    X, _ = _data(600, 20, 1, [0.0, 1.0])
    y = np.full(600, 3.0, np.float32)
    m, ocfg, o = _pair(20, (16,), max_iter=3, seed=2, tol=0.0)
    m.fit(X, y)
    po = so.init(ocfg)
    it, curve, _, _ = so.fit(ocfg, o, po, X.astype(np.float64), np.ones((600, 1)))
    assert m.classes_.tolist() == [3.0] and m.get_params().size == so.nparams(ocfg) and m.n_iter == it
    np.testing.assert_allclose(m.loss_curve, curve, rtol=1e-7)
    assert np.all(m.predict(X) == 3.0)


def test_signed_zero_is_one_class_with_the_sign_of_its_first_occurrence():
    X, y = _data(500, 10, 3, [0.0, 1.0, 2.0])
    y[y == 0] = np.where(np.arange((y == 0).sum()) % 2 == 0, np.float32(-0.0), np.float32(0.0))
    first_zero = np.flatnonzero(y == 0)[0]
    m = g.MLPClassifier(10, hidden=(8,), max_iter=2, seed=1)
    m.fit(X, y)
    c = m.classes_
    assert c.tolist() == [0.0, 1.0, 2.0] and c.tobytes() == co.classes(y).tobytes()
    assert np.signbit(c[0]) == np.signbit(y[first_zero])
    y[first_zero] = np.float32(-0.0) if not np.signbit(y[first_zero]) else np.float32(0.0)
    m.fit(X, y)
    assert np.signbit(m.classes_[0]) == np.signbit(y[first_zero])
    assert m.get_params().size == co.nparams(co.widen(orc.mlp64_cfg(10, hidden=(8,)), c))


def test_infinite_labels_are_classes():
    X, y = _data(400, 10, 4, [-np.inf, 0.0, 1.0, np.inf])
    m = g.MLPClassifier(10, hidden=(8,), max_iter=3, seed=1).fit(X, y)
    assert m.classes_.tolist() == [-np.inf, 0.0, 1.0, np.inf]
    assert np.isfinite(m.loss_curve).all()
    assert set(np.unique(m.predict(X)).tolist()) <= {-np.inf, 0.0, 1.0, np.inf}


def test_softmax_overflow_gives_nan_and_max_idx_picks_as_the_reference():
    """No max subtraction: exp overflows to inf and inf / inf is NaN.  MaxIdx64 keeps a NaN in column 0 and never
    moves to a NaN elsewhere."""
    cls = np.array([1.0, 2.0, 3.0])
    m = g.MLPClassifier(2, hidden=(), max_iter=1)
    ocfg = co.widen(orc.mlp64_cfg(2, hidden=()), cls)
    rng = np.random.default_rng(5)
    p = rng.standard_normal(co.nparams(ocfg))
    p[:3] = [0.0, 0.0, 0.0]
    p[3:] = [900.0, -5.0, 0.3, -900.0, 900.0, 0.1]        # W [2, 3] row-major
    m.set_params(p, classes=cls)
    X = np.array([[1, 0], [0, 1], [0.5, 0.5], [0.001, 0.002], [0.3, 0.0], [0.0, 0.2]], np.float32)
    h = co.predict_proba(ocfg, p, X.astype(np.float64))
    assert np.isnan(h[0, 0]) and np.isnan(h[1, 1])
    got = m.predict(X)
    assert got.tobytes() == co.labels_of(h, cls).tobytes()
    assert got[0] == 1.0 and got[1] != 3.0


# ---- binary labels keep today's results ------------------------------------------------------------------------------
def test_binary_dense_fit_has_no_classes_and_follows_the_binary_restatement():
    X, y = _data(1500, 30, 6, [0.0, 1.0])
    y[::7] = -0.0
    m, ocfg, o = _pair(30, (16,), max_iter=5, seed=4, tol=0.0)
    m.fit(X, y)
    po = so.init(ocfg)
    it, curve, _, _ = so.fit(ocfg, o, po, X.astype(np.float64), y.astype(np.float64).reshape(-1, 1))
    assert m.classes_.size == 0 and m.get_params().size == so.nparams(ocfg) and m.n_iter == it
    np.testing.assert_allclose(m.loss_curve, curve, rtol=1e-7)
    np.testing.assert_allclose(m.predict(X[:300]), so.predict(ocfg, po, X[:300].astype(np.float64)).ravel().astype(np.float32),
                               rtol=1e-5, atol=1e-7)


def test_binary_fit_keys_has_no_classes_and_matches_the_dense_fit():
    rng = np.random.default_rng(7)
    st = Store(rng)
    u, i, t, y = st.keys(rng, 1500)
    X, Y = st.dense(u, i, t, y)
    kw = dict(hidden=(16,), max_iter=4, seed=3, tol=0.0)
    mk = g.MLPClassifier(st.nin, **kw).fit_keys(st.eng, u, i, t, y)
    mr = g.MLPClassifier(st.nin, **kw).fit(X, Y)
    assert mk.classes_.size == 0 and mr.classes_.size == 0
    assert_same_fit(mk, mr, X.shape[0])


# ---- key-fed fit and predict -------------------------------------------------------------------------------------------
def _ratings(rng, n):
    return rng.choice(np.float32(RATINGS), n)


@pytest.mark.parametrize("mlp", [dict(), dict(solver="sgd", lr_init=0.02, activation="tanh")])
def test_fit_keys_with_ratings_is_bit_identical_to_dense_fit(mlp):
    rng = np.random.default_rng(8)
    st = Store(rng)
    u, i, t, _ = st.keys(rng, 1500)
    y = _ratings(rng, u.size)
    X, Y = st.dense(u, i, t, y)
    kw = dict(hidden=(16,), max_iter=4, seed=3, tol=0.0, **mlp)
    mk = g.MLPClassifier(st.nin, **kw).fit_keys(st.eng, u, i, t, y)
    mr = g.MLPClassifier(st.nin, **kw).fit(X, Y)
    assert mk.classes_.tobytes() == mr.classes_.tobytes() == co.classes(Y).tobytes()
    assert_same_fit(mk, mr, X.shape[0])


def test_labels_only_on_dropped_keys_leave_a_binary_model():
    rng = np.random.default_rng(9)
    st = Store(rng)
    u, i, t, y = st.keys(rng, 1200)
    ok = st.rows(u, i, t)[3]
    y = y.copy(); y[~ok] = 3.0
    X, Y = st.dense(u, i, t, y)
    kw = dict(hidden=(16,), max_iter=3, seed=3, tol=0.0)
    mk = g.MLPClassifier(st.nin, **kw).fit_keys(st.eng, u, i, t, y)
    mr = g.MLPClassifier(st.nin, **kw).fit(X, Y)
    assert mk.classes_.size == 0
    assert_same_fit(mk, mr, X.shape[0])


def test_predict_keys_returns_the_dense_labels_bit_for_bit():
    rng = np.random.default_rng(10)
    st = Store(rng, pred_batch=64)
    u, i, t, _ = st.keys(rng, 1000)
    m = g.MLPClassifier(st.nin, hidden=(16, 8), max_iter=3, seed=1).fit_keys(st.eng, u, i, t, _ratings(rng, u.size))
    q = st.keys(rng, 231)                                   # four pred_batch chunks, the last ragged
    qu, qi, qt = q[0].copy(), q[1].copy(), q[2]
    qu[0], qi[0] = st.uid[3], st.iid[5]
    ur, ir, hist, ok = st.rows(qu, qi, qt, drop=False)
    want = m.predict(st.eng.gather_rows(ur, ir, hist))
    got = m.predict_keys(st.eng, qu, qi, qt)
    assert np.array_equal(_bits(got), _bits(want))
    assert set(np.unique(got).tolist()) <= set(m.classes_.tolist())


# ---- warm starts, restore -----------------------------------------------------------------------------------------------
def test_warm_starts_keep_the_head_and_refuse_other_classes():
    X, y = _data(800, 20, 11, [1.0, 2.0, 3.0])
    kw = dict(hidden=(8,), max_iter=2, seed=5, tol=0.0, warm_start=True)
    m = g.MLPClassifier(20, **kw).fit(X, y)
    twin = g.MLPClassifier(20, **kw).fit(X, y)
    p1 = m.get_params()
    m.fit(X[:400], y[:400])                                 # same classes: continues from the fitted parameters
    twin_p = twin.get_params()
    assert m.classes_.tolist() == [1.0, 2.0, 3.0] and p1.size == m.get_params().size and not np.array_equal(m.get_params(), p1)
    assert np.array_equal(twin_p, p1)
    before = _snapshot(m)
    for bad in (np.where(y == 3.0, np.float32(4.0), y), (y > 1.5).astype(np.float32), np.full(800, 2.0, np.float32)):
        with pytest.raises(g.CtrError) as e:
            m.fit(X, bad)
        assert e.value.code == g.EINVAL and _snapshot(m) == before
    # binary first, classes after
    mb = g.MLPClassifier(20, **kw).fit(X, (y > 1.5).astype(np.float32))
    before = _snapshot(mb)
    with pytest.raises(g.CtrError) as e:
        mb.fit(X, y)
    assert e.value.code == g.EINVAL and _snapshot(mb) == before
    # a cold refit re-decides the head
    mc = g.MLPClassifier(20, **dict(kw, warm_start=False)).fit(X, y)
    n3 = mc.get_params().size
    mc.fit(X, (y > 1.5).astype(np.float32))
    assert mc.classes_.size == 0 and mc.get_params().size < n3
    mc.fit(X, y)
    assert mc.classes_.tolist() == [1.0, 2.0, 3.0] and mc.get_params().size == n3


def test_restore_through_get_and_set_classes_predicts_bit_identically():
    X, y = _data(700, 15, 12, RATINGS)
    m = g.MLPClassifier(15, hidden=(10,), max_iter=3, seed=6).fit(X, y)
    p, c = m.get_params(), m.classes_
    r = g.MLPClassifier(15, hidden=(10,))
    assert r.get_params().size != p.size
    with pytest.raises(g.CtrError) as e:
        r.set_params(p)                                      # np follows the classes: they go first
    assert e.value.code == g.EINVAL
    r.L.ctr_mlp_set_classes(r.h, c.ctypes.data_as(C.POINTER(C.c_double)), C.c_int32(c.size))
    assert r.get_params().size == p.size
    with pytest.raises(g.CtrError) as e:
        r.predict(X)                                         # not fitted until set_params
    assert e.value.code == g.ESTATE
    r.set_params(p)
    assert np.array_equal(_bits(r.predict(X)), _bits(m.predict(X)))
    r2 = g.MLPClassifier(15, hidden=(10,))
    r2.set_params(p, classes=c)
    assert np.array_equal(_bits(r2.predict(X)), _bits(m.predict(X))) and r2.classes_.tobytes() == c.tobytes()
    r2.set_params(r2.get_params()[:(1 + 15) * 10 + 11], classes=[])   # back to binary
    assert r2.classes_.size == 0 and np.all((r2.predict(X) >= 0) & (r2.predict(X) <= 1))


# ---- refusals -------------------------------------------------------------------------------------------------------------
def test_nan_labels_and_too_many_classes_are_refused_and_change_nothing():
    X, y = _data(2000, 12, 13, [1.0, 2.0, 3.0])
    m = g.MLPClassifier(12, hidden=(8,), max_iter=2, seed=1).fit(X, y)
    before = _snapshot(m)
    bad = y.copy(); bad[100] = np.nan
    with pytest.raises(g.CtrError) as e:
        m.fit(X, bad)
    assert e.value.code == g.EINVAL and b"NaN" in str(e.value).encode() and _snapshot(m) == before
    many = np.arange(2000, dtype=np.float32) % 1025
    with pytest.raises(g.CtrError) as e:
        m.fit(X, many)
    assert e.value.code == g.EINVAL and "1025" in str(e.value) and _snapshot(m) == before
    exact = np.arange(2000, dtype=np.float32) % 1024                # 1024 classes are allowed
    m.fit(X, exact)
    assert m.classes_.size == 1024


def test_recommend_on_a_multiclass_model_is_refused_and_writes_nothing():
    rng = np.random.default_rng(14)
    st = Store(rng)
    u, i, t, _ = st.keys(rng, 800)
    m = g.MLPClassifier(st.nin, hidden=(8,), max_iter=2, seed=1).fit_keys(st.eng, u, i, t, _ratings(rng, u.size))
    k = 5
    rows = np.full(k, 77, np.int32); scores = np.full(k, 7.0, np.float32); logits = np.full(k, 7.0); cnt = np.full(1, 9, np.int32)
    uid = np.array([st.uid[1]], np.int64); ts = np.array([4_990_000], np.int64)
    rc = m.L.ctr_mlp_recommend_topk(m.h, st.eng.h, uid.ctypes.data_as(C.POINTER(C.c_int64)), ts.ctypes.data_as(C.POINTER(C.c_int64)),
                                    C.c_int64(1), C.c_int32(k), C.c_int32(1), rows.ctypes.data_as(C.POINTER(C.c_int32)),
                                    scores.ctypes.data_as(C.POINTER(C.c_float)), logits.ctypes.data_as(C.POINTER(C.c_double)),
                                    cnt.ctypes.data_as(C.POINTER(C.c_int32)))
    assert rc == g.ESTATE and b"class" in m.L.ctr_mlp_last_error(m.h)
    assert (rows == 77).all() and (scores == 7).all() and (logits == 7).all() and cnt[0] == 9


# ---- serving ----------------------------------------------------------------------------------------------------------------
def test_serving_returns_predicted_ratings_and_recommend_is_refused():
    rng = np.random.default_rng(15)
    st = Store(rng, pred_batch=50)
    u, i, t, _ = st.keys(rng, 900)
    pred = gm.SimpleMlpFitWrap(hidden=(32,), max_iter=3).FitKeys(st.eng, u, i, t, _ratings(rng, u.size))
    assert pred.pred.classes_.tolist() == RATINGS
    samples = [sv.Sample(int(st.uid[k % 40]), int(st.iid[(7 * k) % 300]), 4_990_000 + k) for k in range(120)]
    got = sv.BatchPredict(pred, samples)
    want = pred.pred.predict_keys(st.eng, [s.UserId for s in samples], [s.ItemId for s in samples], [s.Timestamp for s in samples])
    assert got.shape == (120, 1) and np.array_equal(got.ravel(), want) and set(np.unique(want).tolist()) <= set(RATINGS)
    items = [int(v) for v in st.iid[:75]]
    ranked = sv.Rank(pred, int(st.uid[2]), items, now=4_995_000)
    want = pred.pred.predict_keys(st.eng, [st.uid[2]] * 75, items, [4_995_000] * 75)
    assert [r.ItemId for r in ranked] == items and np.array_equal(np.array([r.Score for r in ranked], np.float32), want)
    with pytest.raises(g.CtrError) as e:
        sv.Recommend(pred, int(st.uid[2]), 10, now=4_995_000)
    assert e.value.code == g.ESTATE
