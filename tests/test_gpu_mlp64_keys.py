"""The float64 MLP fed by sample keys (ctr_mlp_fit_keys / ctr_mlp_predict_keys) against the dense path it replaces.

Every reference run is built independently of the key path: survivors from host dicts, windows from
Engine.ubcache_window, X from Engine.gather_rows, and a second MLPClassifier fitted on (X, Y) with the same config.
The key path gathers the same float32 values widened to float64 into a staging buffer and runs the same kernels in the
same order, so parameters, loss curves and probabilities must agree bit for bit."""
import ctypes as C
import zlib

import numpy as np
import pytest

import go_ctr_b200 as g
from go_ctr_b200 import model as gm
from go_ctr_b200 import serving as sv
from oracle import oracle as orc

pytestmark = pytest.mark.gpu


# ---- fixtures ---------------------------------------------------------------------------------------------------
def histories(rng, U, I, max_len):
    """Behaviour CSR, timestamps descending, in long runs of one timestamp (MovieLens users rate many items in the same
    second); a few users are empty."""
    lens = rng.integers(0, max_len + 1, U)
    lens[:: 7] = 0
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    ts = []
    for L in lens:
        runs = rng.choice([1, 2, 5, 30, 80], size=max(L, 1))
        run_of = np.repeat(np.arange(runs.size), runs)[:L]
        ts.append(5_000_000 - 10 * np.cumsum(rng.integers(1, 3, max(L, 1)))[run_of])
    return off, np.concatenate(ts).astype(np.int64), rng.integers(0, I, off[-1]).astype(np.int32)


class Store:
    """A feature store: tables, sparse id maps, optionally a ubcache."""

    def __init__(self, rng, U=400, I=700, uP=5, S=10, D=16, cF=7, with_ub=True, pred_batch=256, max_len=120):
        self.uid = rng.choice(10**12, U, replace=False).astype(np.int64) - 5 * 10**11
        self.iid = rng.choice(10**12, I, replace=False).astype(np.int64)
        self.eng = g.Engine(g.engine.default_config(g.MODEL_DIN_COS, uP=uP, S=S, D=D, cF=cF, batch=128, pred_batch=pred_batch))
        uf = rng.random((U, uP), np.float32) if uP else np.zeros((U, 0), np.float32)
        itf = rng.random((I, cF), np.float32) if cF else np.zeros((I, 0), np.float32)
        emb = (rng.standard_normal((I, D)) / np.sqrt(D)).astype(np.float32)
        if uP:
            self.eng.table_upload(g.TABLE_USER_FEAT, uf)
        if cF:
            self.eng.table_upload(g.TABLE_ITEM_FEAT, itf)
        self.eng.table_upload(g.TABLE_ITEM_EMB, emb)
        sv.load_id_maps(self.eng, self.uid, self.iid)
        self.umap = {int(v): r for r, v in enumerate(self.uid)}
        self.imap = {int(v): r for r, v in enumerate(self.iid)}
        self.ub = None
        if with_ub:
            self.ub = histories(rng, U, I, max_len)
            self.eng.ubcache_upload(*self.ub)
        self.nin = uP + S * D + D + cF

    def keys(self, rng, n, unknown=0.15):
        """n keys; about `unknown` of the users and of the items are ids the maps do not hold (so ~30 % of the keys drop),
        among them the first and the last key.  Timestamps fall on the user's events (tied-run boundaries), one either
        side, or 0 ("from the newest")."""
        ur = rng.integers(0, self.uid.size, n); ir = rng.integers(0, self.iid.size, n)
        u = self.uid[ur].copy(); i = self.iid[ir].copy()
        bad_u = rng.random(n) < unknown; bad_i = rng.random(n) < unknown
        u[bad_u] = 10**15 + np.arange(bad_u.sum()); i[bad_i] = -10**15 - np.arange(bad_i.sum())
        u[0] = 10**16; i[-1] = 10**16
        t = rng.integers(1, 6_000_000, n).astype(np.int64)
        if self.ub is not None:
            off, ts, _ = self.ub
            L = off[ur + 1] - off[ur]
            e = off[ur] + (rng.random(n) * np.maximum(L, 1)).astype(np.int64)
            on = L > 0
            t[on] = ts[np.minimum(e[on], ts.size - 1)] + rng.integers(-1, 2, on.sum())
        t[rng.random(n) < 0.05] = 0
        y = (rng.random(n) < 0.4).astype(np.float32)
        return u, i, t, y

    def rows(self, u, i, t, drop=True):
        """GetSample with dicts: (user row, item row, history) per key; unknown keys dropped (drop) or all -1."""
        ur = np.array([self.umap.get(int(x), -1) for x in u], np.int32)
        ir = np.array([self.imap.get(int(x), -1) for x in i], np.int32)
        ok = (ur >= 0) & (ir >= 0)
        S = self.eng.cfg.S
        hist = np.full((u.size, S), -1, np.int32)
        if self.ub is not None and ok.any():
            hist[ok] = self.eng.ubcache_window(ur[ok], t[ok])
        if drop:
            return ur[ok], ir[ok], hist[ok], ok
        ur[~ok] = -1; ir[~ok] = -1
        return ur, ir, hist, ok

    def dense(self, u, i, t, y):
        ur, ir, hist, ok = self.rows(u, i, t)
        return self.eng.gather_rows(ur, ir, hist), y[ok]


def assert_same_fit(mk, mr, n_used):
    assert mk.rows_used == n_used
    assert mk.n_iter == mr.n_iter
    assert np.array_equal(mk.loss_curve.view(np.uint64), mr.loss_curve.view(np.uint64))
    assert np.array_equal(mk.get_params().view(np.uint64), mr.get_params().view(np.uint64))


# ---- 1. fit is bit-identical to the dense path ------------------------------------------------------------------
FIT_CASES = {
    "relu_adam": dict(mlp=dict(activation="relu")),
    "logistic": dict(mlp=dict(activation="logistic")),
    "tanh": dict(mlp=dict(activation="tanh")),
    "identity": dict(mlp=dict(activation="identity")),
    "sgd_nesterov": dict(mlp=dict(solver="sgd", lr_init=0.01)),
    "sgd_invscaling": dict(mlp=dict(solver="sgd", learning_rate="invscaling", nesterovs_momentum=False, lr_init=0.05)),
    "weight_decay": dict(mlp=dict(weight_decay=0.01)),
    "no_shuffle": dict(mlp=dict(shuffle=False)),
    "ragged_batch": dict(mlp=dict(batch=97)),
    "batch_over_survivors": dict(mlp=dict(batch=5000)),
    "S1_odd_cF0": dict(store=dict(uP=3, S=1, D=16, cF=0)),
    "S50_D64": dict(store=dict(uP=5, S=50, D=64, cF=7), n=900),
    "S10_D64_odd": dict(store=dict(uP=9, S=10, D=64, cF=13)),
    "no_ubcache": dict(store=dict(with_ub=False)),
}


@pytest.mark.parametrize("case", sorted(FIT_CASES))
def test_fit_keys_is_bit_identical_to_dense_fit(case):
    spec = FIT_CASES[case]
    rng = np.random.default_rng(zlib.crc32(case.encode()))
    st = Store(rng, **spec.get("store", {}))
    u, i, t, y = st.keys(rng, spec.get("n", 1500))
    X, Y = st.dense(u, i, t, y)
    kw = dict(hidden=(16,), max_iter=4, seed=3, tol=0.0)
    kw.update(spec.get("mlp", {}))
    mk = g.MLPClassifier(st.nin, **kw).fit_keys(st.eng, u, i, t, y)
    mr = g.MLPClassifier(st.nin, **kw).fit(X, Y)
    assert 0.55 * u.size < X.shape[0] < 0.85 * u.size
    assert_same_fit(mk, mr, X.shape[0])
    assert np.isfinite(mk.loss_curve).all()


# ---- 2. warm start ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("solver", [dict(), dict(solver="sgd", learning_rate="invscaling", lr_init=0.05)])
def test_warm_start_sequences_match_the_dense_sequence(solver):
    rng = np.random.default_rng(11)
    st = Store(rng)
    k1 = st.keys(rng, 1200); k2 = st.keys(rng, 700)
    (X1, Y1), (X2, Y2) = st.dense(*k1), st.dense(*k2)
    kw = dict(hidden=(12,), max_iter=3, seed=4, tol=0.0, warm_start=True, **solver)
    # fit_keys, then fit_keys again from the fitted parameters (the invscaling t carries over)
    mk = g.MLPClassifier(st.nin, **kw); mr = g.MLPClassifier(st.nin, **kw)
    mk.fit_keys(st.eng, *k1); mr.fit(X1, Y1)
    assert_same_fit(mk, mr, X1.shape[0])
    mk.fit_keys(st.eng, *k2); mr.fit(X2, Y2)
    assert_same_fit(mk, mr, X2.shape[0])
    # dense fit, then a key-fed warm start
    ma = g.MLPClassifier(st.nin, **kw); mb = g.MLPClassifier(st.nin, **kw)
    ma.fit(X1, Y1); mb.fit(X1, Y1)
    ma.fit_keys(st.eng, *k2); mb.fit(X2, Y2)
    assert_same_fit(ma, mb, X2.shape[0])


# ---- 3. against the oracle, configs[0] shape --------------------------------------------------------------------
def test_configs0_shape_follows_the_oracle():
    """uP 52, S 10, D 16, cF 53 (nin 281), hidden 100, relu + Adam, as main.go sets it: the CPU restatement on the
    host-gathered X, loss curve at rtol 1e-7 and probabilities at test_gpu_mlp64.py's bars."""
    rng = np.random.default_rng(5)
    st = Store(rng, U=300, I=500, uP=52, S=10, D=16, cF=53)
    assert st.nin == 281
    u, i, t, y = st.keys(rng, 2500)
    X, Y = st.dense(u, i, t, y)
    m = g.MLPClassifier(281, hidden=(100,), max_iter=5, seed=9).fit_keys(st.eng, u, i, t, y)
    ocfg = orc.mlp64_cfg(281, hidden=(100,), max_iter=5, seed=9)
    po = orc.mlp64_init(ocfg)
    it, curve, _ = orc.mlp64_fit(ocfg, po, X.astype(np.float64), Y.astype(np.float64).reshape(-1, 1))
    assert m.n_iter == it and m.rows_used == X.shape[0]
    np.testing.assert_allclose(m.loss_curve, curve[:it], rtol=1e-7)
    ur, ir, _, ok = st.rows(u, i, t)
    sel = np.flatnonzero(ok)[:500]
    pg = m.predict_keys(st.eng, u[sel], i[sel], t[sel])
    pc = orc.mlp64_predict(ocfg, po, X[:500].astype(np.float64)).ravel().astype(np.float32)
    np.testing.assert_allclose(pg, pc, rtol=1e-5, atol=1e-7)


# ---- 4. predict -------------------------------------------------------------------------------------------------
def test_predict_keys_is_bit_identical_to_dense_predict():
    rng = np.random.default_rng(21)
    st = Store(rng, pred_batch=64)
    u, i, t, y = st.keys(rng, 1000)
    m = g.MLPClassifier(st.nin, hidden=(16, 8), max_iter=2, seed=1).fit_keys(st.eng, u, i, t, y)
    q = st.keys(rng, 231)                                   # four pred_batch chunks, the last ragged
    qu, qi, qt = q[0].copy(), q[1].copy(), q[2]
    qu[0], qi[0] = st.uid[3], st.iid[5]                    # key 0 must resolve
    qu[64] = 10**17                                          # an unknown key opening a chunk
    ur, ir, hist, ok = st.rows(qu, qi, qt, drop=False)
    assert ok[0] and not ok.all()
    want = m.predict(st.eng.gather_rows(ur, ir, hist))
    got = m.predict_keys(st.eng, qu, qi, qt)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    zero = m.predict(np.zeros((1, st.nin), np.float32))[0]
    assert (got[~ok] == zero).all()
    # an unknown key 0 fails the call (rcmd.go:300-303)
    with pytest.raises(g.CtrError) as e:
        m.predict_keys(st.eng, [10**17], [st.iid[0]], [0])
    assert e.value.code == g.ENOTFOUND
    # the live cache: an append between two calls is seen by the second
    row = 3
    before = m.predict_keys(st.eng, [st.uid[row]], [st.iid[1]], [7_000_000])
    st.eng.ubcache_append([row] * 4, [6_900_000] * 4, [10, 11, 12, 13])
    after = m.predict_keys(st.eng, [st.uid[row]], [st.iid[1]], [7_000_000])
    hist = st.eng.ubcache_window([row], [7_000_000])
    assert list(hist[0, :4]) == [13, 12, 11, 10]
    assert after[0] == m.predict(st.eng.gather_rows([row], [1], hist))[0] and after[0] != before[0]


def test_serving_through_the_fitkeys_predictor():
    rng = np.random.default_rng(31)
    st = Store(rng, pred_batch=50)
    u, i, t, y = st.keys(rng, 900)
    pred = gm.SimpleMlpFitWrap(hidden=(100,), activation="relu", solver="adam", alpha=1e-4, max_iter=3).FitKeys(st.eng, u, i, t, y)
    assert pred.pred.rows_used == st.rows(u, i, t)[0].size
    samples = [sv.Sample(int(st.uid[k % 40]), int(st.iid[(7 * k) % 300]), 4_990_000 + k) for k in range(120)]
    got = sv.BatchPredict(pred, samples)
    want = pred.pred.predict_keys(st.eng, [s.UserId for s in samples], [s.ItemId for s in samples], [s.Timestamp for s in samples])
    assert got.shape == (120, 1) and np.array_equal(got.ravel(), want)
    items = [int(v) for v in st.iid[:75]]
    ranked = sv.Rank(pred, int(st.uid[2]), items, now=4_995_000)
    want = pred.pred.predict_keys(st.eng, [st.uid[2]] * 75, items, [4_995_000] * 75)
    assert [r.ItemId for r in ranked] == items and np.array_equal(np.array([r.Score for r in ranked], np.float32), want)


# ---- 5. beyond a dense X that fits in HBM -----------------------------------------------------------------------
def test_fit_keys_where_dense_float64_x_exceeds_hbm():
    """S = 100, D = 128 (nin = 12 951), 800 000 samples: the dense float64 X would take 83 GB."""
    rng = np.random.default_rng(41)
    U, I, uP, S, D, cF, n = 20_000, 50_000, 7, 100, 128, 16, 800_000
    st = Store(rng, U=U, I=I, uP=uP, S=S, D=D, cF=cF, pred_batch=512, max_len=160)
    assert n * st.nin * 8 > 80e9
    u = st.uid[rng.integers(0, U, n)]; i = st.iid[rng.integers(0, I, n)]
    t = rng.integers(4_000_000, 5_000_000, n).astype(np.int64); y = (rng.random(n) < 0.3).astype(np.float32)
    m = g.MLPClassifier(st.nin, hidden=(8,), max_iter=1, seed=2).fit_keys(st.eng, u, i, t, y)
    assert m.rows_used == n and m.n_iter == 1 and np.isfinite(m.loss_curve).all()
    sel = rng.choice(n, 1000, replace=False)
    ur, ir, hist, ok = st.rows(u[sel], i[sel], t[sel], drop=False)
    assert ok.all()
    want = m.predict(st.eng.gather_rows(ur, ir, hist))
    got = m.predict_keys(st.eng, u[sel], i[sel], t[sel])
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


# ---- 6. refusals leave the parameters as they were ----------------------------------------------------------------
def test_refusals_change_nothing():
    rng = np.random.default_rng(51)
    st = Store(rng)
    u, i, t, y = st.keys(rng, 400)
    m = g.MLPClassifier(st.nin, hidden=(8,), max_iter=2, seed=6, warm_start=True)
    fresh = m.get_params().copy()
    with pytest.raises(g.CtrError) as e:                      # predict before any fit
        m.predict_keys(st.eng, u, i, t)
    assert e.value.code == g.ESTATE and "before fit" in str(e.value)
    m.fit_keys(st.eng, u, i, t, y)
    p0 = m.get_params().copy()
    assert not np.array_equal(p0, fresh)

    def unchanged():
        assert np.array_equal(m.get_params().view(np.uint64), p0.view(np.uint64))

    wide = g.MLPClassifier(st.nin + 1, hidden=(8,))
    with pytest.raises(g.CtrError) as e:
        wide.fit_keys(st.eng, u, i, t, y)
    assert e.value.code == g.EINVAL and "inputs" in str(e.value)
    L = m.L
    n = C.c_int64(u.size); it = C.c_int32(0); used = C.c_int64(0)
    lp = u.ctypes.data_as(C.POINTER(C.c_int64)); yp = y.ctypes.data_as(C.POINTER(C.c_float))
    assert L.ctr_mlp_fit_keys(m.h, st.eng.h, None, lp, lp, yp, n, C.byref(it), None, C.byref(used)) == g.EINVAL
    assert L.ctr_mlp_fit_keys(m.h, None, lp, lp, lp, yp, n, C.byref(it), None, C.byref(used)) == g.EINVAL
    assert L.ctr_mlp_fit_keys(m.h, st.eng.h, lp, lp, lp, yp, C.c_int64(0), C.byref(it), None, C.byref(used)) == g.EINVAL
    assert L.ctr_mlp_predict_keys(m.h, st.eng.h, lp, lp, lp, n, None) == g.EINVAL
    unchanged()
    bare = g.Engine(st.eng.cfg)                                # tables but no id maps
    bare.table_upload(g.TABLE_USER_FEAT, np.zeros((4, st.eng.cfg.uP), np.float32))
    bare.table_upload(g.TABLE_ITEM_FEAT, np.zeros((4, st.eng.cfg.cF), np.float32))
    bare.table_upload(g.TABLE_ITEM_EMB, np.zeros((4, st.eng.cfg.D), np.float32))
    for call in (lambda: m.fit_keys(bare, u, i, t, y), lambda: m.predict_keys(bare, u, i, t)):
        with pytest.raises(g.CtrError) as e:
            call()
        assert e.value.code == g.ESTATE and "id map" in str(e.value)
    unchanged()
    with pytest.raises(g.CtrError) as e:                      # no survivors
        m.fit_keys(st.eng, np.full(5, 10**17), i[:5], t[:5], y[:5])
    assert e.value.code == g.ENOTFOUND
    unchanged()
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("different devices need two GPUs")
    other = g.MLPClassifier(st.nin, hidden=(8,), device=1)
    with pytest.raises(g.CtrError) as e:
        other.fit_keys(st.eng, u, i, t, y)
    assert e.value.code == g.EINVAL and "device" in str(e.value)


# ---- 7. which path ran ------------------------------------------------------------------------------------------
def test_profile_shows_the_device_path():
    rng = np.random.default_rng(61)
    st = Store(rng)
    u, i, t, y = st.keys(rng, 600)
    m = g.MLPClassifier(st.nin, hidden=(8,), max_iter=2, batch=100)
    st.eng.profile(True); st.eng.profile_reset()
    m.fit_keys(st.eng, u, i, t, y)
    prof = st.eng.profile_dump()
    for key in ("keys_rows", "keys_compact", "ubcache_window", "mlp_gather"):
        assert prof.get(key, (0, 0))[1] > 0, (key, prof)
    assert prof["ubcache_window"][1] == 1                              # one window cut per fit
    assert prof["mlp_gather"][1] == m.n_iter * int(np.ceil(m.rows_used / 100))   # one gather per minibatch
    assert "gather_rows" not in prof
    st.eng.profile_reset()
    m.predict_keys(st.eng, u[1:300], i[1:300], t[1:300])
    prof = st.eng.profile_dump()
    assert prof["keys_resolve"][1] == prof["mlp_gather"][1] == int(np.ceil(299 / st.eng.cfg.pred_batch))
    st.eng.profile(False)
