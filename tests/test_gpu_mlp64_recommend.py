"""Top-k recommendation over the whole item table with the float64 MLP (ctr_mlp_recommend_topk).

The call computes the user's part of layer 0 once and continues each item's float64 chain from it, so every score must
equal, bit for bit, what ctr_mlp_predict_keys returns for (user, the row's item id, ts).  Logits are also checked against
tests/mlp_rec_restatement.c, which walks the same chain with C99 fma(): bit for bit where the chain has no libm call
(relu / identity hidden layers), within 1e-12 relative otherwise."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile
import zlib

import numpy as np
import pytest

import go_ctr_b200 as g
from go_ctr_b200 import model as gm
from go_ctr_b200 import serving as sv

pytestmark = pytest.mark.gpu

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "mlp_rec_restatement.c")
_lib = None
ACT = {"relu": 0, "logistic": 1, "identity": 2, "tanh": 3}


def restatement():
    """tests/mlp_rec_restatement.c, compiled on first use into the temporary directory (keyed by its source hash)."""
    global _lib
    if _lib is None:
        with open(_SRC, "rb") as f:
            tag = hashlib.sha256(f.read()).hexdigest()[:16]
        so = os.path.join(tempfile.gettempdir(), "mlp_rec_restatement_%s_%d.so" % (tag, os.getuid()))
        if not os.path.exists(so):
            tmp = "%s.tmp.%d" % (so, os.getpid())
            subprocess.check_call(["gcc", "-O2", "-std=c99", "-fPIC", "-shared", "-ffp-contract=off", "-Wall", "-Wextra",
                                   "-o", tmp, _SRC, "-lm"])
            os.replace(tmp, so)
        _lib = C.CDLL(so)
    return _lib


def ref_logits(m, X):
    units = np.array([m.cfg.units[i] for i in range(m.cfg.n_layers)], np.int32)
    p = m.get_params()
    X = np.ascontiguousarray(X, np.float64)
    out = np.empty(X.shape[0], np.float64)
    dp = C.POINTER(C.c_double)
    restatement().rec_logits(p.ctypes.data_as(dp), C.c_int(units.size), units.ctypes.data_as(C.POINTER(C.c_int)),
                             C.c_int(m.cfg.hidden_act), X.ctypes.data_as(dp), C.c_long(X.shape[0]), out.ctypes.data_as(dp))
    return out


# ---- fixtures ---------------------------------------------------------------------------------------------------
def histories(rng, U, I, max_len):
    """Behaviour CSR, timestamps descending, in runs of one timestamp (tied windows); every 7th user is empty."""
    lens = rng.integers(0, max_len + 1, U)
    lens[:: 7] = 0
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    ts = []
    for L in lens:
        runs = rng.choice([1, 2, 5, 30], size=max(L, 1))
        run_of = np.repeat(np.arange(runs.size), runs)[:L]
        ts.append(5_000_000 - 10 * np.cumsum(rng.integers(1, 3, max(L, 1)))[run_of])
    return off, np.concatenate(ts).astype(np.int64), rng.integers(0, I, off[-1]).astype(np.int32)


class Store:
    """A feature store: tables, sparse id maps, optionally a ubcache.  dup: pairs (a, b), item row b copies row a."""

    def __init__(self, seed, U=40, I=300, uP=5, S=10, D=16, cF=7, with_ub=True, pred_batch=256, max_len=60, dup=()):
        rng = np.random.default_rng(seed)
        self.uid = rng.choice(10**12, U, replace=False).astype(np.int64) - 5 * 10**11
        self.iid = rng.choice(10**12, I, replace=False).astype(np.int64)
        self.eng = g.Engine(g.engine.default_config(g.MODEL_DIN_COS, uP=uP, S=S, D=D, cF=cF, batch=128, pred_batch=pred_batch))
        self.uf = rng.random((U, uP), np.float32)
        self.itf = rng.random((I, cF), np.float32)
        self.emb = (rng.standard_normal((I, D)) / np.sqrt(D)).astype(np.float32)
        for a, b in dup:
            self.itf[b] = self.itf[a]; self.emb[b] = self.emb[a]
        if uP:
            self.eng.table_upload(g.TABLE_USER_FEAT, self.uf)
        if cF:
            self.eng.table_upload(g.TABLE_ITEM_FEAT, self.itf)
        self.eng.table_upload(g.TABLE_ITEM_EMB, self.emb)
        sv.load_id_maps(self.eng, self.uid, self.iid)
        self.ub = None
        if with_ub:
            self.ub = histories(rng, U, I, max_len)
            self.eng.ubcache_upload(*self.ub)
        self.nin = uP + S * D + D + cF

    @property
    def N(self):
        return int(np.asarray(self.eng.item_ids).size)

    def user_ts(self, r, which):
        """A timestamp for user row r: on an event inside a tied run (which=0), one past it (1), or 0 (newest)."""
        if self.ub is None or which == 2:
            return 0
        off, ts, _ = self.ub
        L = off[r + 1] - off[r]
        return int(ts[off[r] + L // 2]) + (which == 1) if L else 4_000_000

    def window(self, r, t):
        if self.ub is None:
            return np.full(self.eng.cfg.S, -1, np.int32)
        return self.eng.ubcache_window([r], [t])[0]

    def X(self, r, t):
        """GetSampleVector for user row r against every item row, float32 as the gather builds it."""
        N = self.N
        hist = np.tile(self.window(r, t), (N, 1))
        return self.eng.gather_rows(np.full(N, r, np.int32), np.arange(N, dtype=np.int32), hist)


def classifier(st, hidden=(100,), activation="relu", seed=0, scale=1.0):
    """A classifier with random parameters (set_params marks it fitted): ~N(0, 1/fan_in) weights, so that the hidden
    activations sit in their interesting range."""
    m = g.MLPClassifier(st.nin, hidden=hidden, activation=activation, max_iter=3, seed=seed)
    rng = np.random.default_rng(seed + 1)
    units = [st.nin, *hidden, 1]
    p = []
    for fi, fo in zip(units[:-1], units[1:]):
        p.append(rng.standard_normal(fo) * 0.1)
        p.append(rng.standard_normal(fi * fo) * scale / np.sqrt(fi))
    m.set_params(np.concatenate(p))
    return m


def predict_all(m, st, uid, t):
    N = st.N
    return m.predict_keys(st.eng, np.full(N, uid, np.int64), np.asarray(st.eng.item_ids)[:N], np.full(N, t, np.int64))


def assert_order(rows, logits):
    """(logit descending, row ascending)"""
    for a in range(rows.size - 1):
        assert logits[a] > logits[a + 1] or (logits[a] == logits[a + 1] and rows[a] < rows[a + 1]), a


def check_user(m, st, r, t, exact, exclude=False):
    """One user's full list (k = N) against predict_keys (bitwise) and the restatement; returns (rows, logits)."""
    N = st.N
    uid = int(st.uid[r])
    rows, sc, lg, cnt = m.recommend_topk(st.eng, [uid], [t], N, exclude_history=exclude)
    rows, sc, lg, n = rows[0], sc[0], lg[0], int(cnt[0])
    win = st.window(r, t)
    excl = set(int(x) for x in win if 0 <= x < N) if exclude else set()
    assert n == N - len(excl)
    assert np.all(rows[n:] == -1) and np.all(sc[n:] == 0) and np.all(lg[n:] == 0)
    rows, sc, lg = rows[:n], sc[:n], lg[:n]
    assert sorted(rows.tolist()) == sorted(set(range(N)) - excl)
    p = predict_all(m, st, uid, t)
    assert np.array_equal(sc.view(np.uint32), p[rows].view(np.uint32)), "scores differ from ctr_mlp_predict_keys"
    assert_order(rows, lg)
    ref = ref_logits(m, st.X(r, t).astype(np.float64))
    if exact:
        assert np.array_equal(lg.view(np.uint64), ref[rows].view(np.uint64)), "logits differ from the fma restatement"
        order = sorted((i for i in range(N) if i not in excl), key=lambda i: (-ref[i], i))
        assert rows.tolist() == order
    else:
        np.testing.assert_allclose(lg, ref[rows], rtol=1e-12, atol=1e-300)
        # the restatement's logits in the device's order descend, up to near-ties
        d = np.diff(ref[rows])
        assert np.all(d <= 1e-12 * np.maximum(np.abs(ref[rows][:-1]), 1e-300)), d.max()
    return rows, lg


# ---- 1. bit-identity with the predict route ----------------------------------------------------------------------
CASES = {
    "relu_100": dict(mlp=dict(activation="relu")),
    "logistic_100": dict(mlp=dict(activation="logistic")),
    "tanh_100": dict(mlp=dict(activation="tanh")),
    "identity_100": dict(mlp=dict(activation="identity")),
    "relu_64_32": dict(mlp=dict(activation="relu", hidden=(64, 32))),
    "tanh_64_32": dict(mlp=dict(activation="tanh", hidden=(64, 32))),
    "S1_cF0_odd_uP": dict(store=dict(uP=3, S=1, D=16, cF=0)),
    "S50_D64": dict(store=dict(uP=7, S=50, D=64, cF=9, I=500)),
    "S10_D64_logistic": dict(store=dict(uP=9, S=10, D=64, cF=13), mlp=dict(activation="logistic", hidden=(64, 32))),
    "no_ubcache": dict(store=dict(with_ub=False)),
    "no_hidden_layer": dict(mlp=dict(hidden=())),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_scores_match_predict_keys_bit_for_bit(case):
    spec = CASES[case]
    st = Store(zlib.crc32(case.encode()), **spec.get("store", {}))
    kw = dict(spec.get("mlp", {}))
    act = kw.get("activation", "relu")
    m = classifier(st, seed=zlib.crc32(case.encode()) % 1000, **kw)
    exact = act in ("relu", "identity") or kw.get("hidden") == ()
    for r, which in ((1, 0), (3, 1), (5, 2)):
        check_user(m, st, r, st.user_ts(r, which), exact)
    check_user(m, st, 3, st.user_ts(3, 0), exact, exclude=True)


# ---- 2. consistency: prefixes, chunking, duplicates --------------------------------------------------------------
def lists(m, st, uids, ts, k, exclude=True):
    rows, sc, lg, cnt = m.recommend_topk(st.eng, uids, ts, k, exclude_history=exclude)
    return rows, sc, lg, cnt


@pytest.mark.parametrize("I", [1, 300, 1000])
def test_lists_do_not_depend_on_k_or_the_chunk(I):
    dup = ((2, 7), (2, 150), (40, 41)) if I >= 300 else ()
    ref = None
    for pb in (128, 300, 100_000):          # >= 3 chunks, N not a multiple of the chunk, one chunk
        st = Store(11, I=I, pred_batch=pb, dup=dup)
        m = classifier(st, seed=5)
        uids = st.uid[[1, 2, 9]]; ts = [st.user_ts(r, 0) for r in (1, 2, 9)]
        full = lists(m, st, uids, ts, st.N)
        if ref is None:
            ref = full
        for a, b in zip(full, ref):
            assert np.array_equal(a, b), pb
        for k in (1, 7, 100):
            part = lists(m, st, uids, ts, k)
            kk = min(k, st.N)
            for j in range(3):
                n = min(k, int(full[3][j]))
                assert int(part[3][j]) == n
                assert np.array_equal(part[0][j, :n], full[0][j, :n])
                assert np.array_equal(part[1][j, :n].view(np.uint32), full[1][j, :n].view(np.uint32))
                assert np.array_equal(part[2][j, :n].view(np.uint64), full[2][j, :n].view(np.uint64))
                assert np.all(part[0][j, n:kk] == -1)
    if dup:                                  # duplicate rows: equal logits, the lower row first
        rows, lg, n = ref[0][0], ref[2][0], int(ref[3][0])
        pos = {int(r): i for i, r in enumerate(rows[:n])}
        for a, b in dup:
            if a in pos and b in pos:
                assert lg[pos[a]] == lg[pos[b]] and pos[a] < pos[b]


# ---- 3. edges ----------------------------------------------------------------------------------------------------
def test_short_lists_and_exclusion():
    st = Store(21, I=40, S=10, max_len=60)
    m = classifier(st, seed=2)
    off = st.ub[0]
    r = int(np.argmax(np.diff(off)))                 # a user with a full window
    assert off[r + 1] - off[r] >= 10
    t = 0
    win = set(int(x) for x in st.window(r, t) if x >= 0)
    for ex in (False, True):
        rows, sc, lg, cnt = m.recommend_topk(st.eng, [st.uid[r]], [t], 100, exclude_history=ex)
        n = int(cnt[0])
        assert n == (40 - len(win) if ex else 40)
        assert np.all(rows[0, n:] == -1) and np.all(sc[0, n:] == 0) and np.all(lg[0, n:] == 0)
        assert (set(rows[0, :n].tolist()) & win) == (set() if ex else win)


def test_several_users_and_one_user_twice():
    st = Store(22, I=500)
    m = classifier(st, seed=3, hidden=(64, 32))
    rs = [1, 2, 1, 8, 13]
    ts = [st.user_ts(1, 0), st.user_ts(2, 1), st.user_ts(1, 2), st.user_ts(8, 0), st.user_ts(13, 1)]
    assert ts[0] != ts[2]
    rows, sc, lg, cnt = m.recommend_topk(st.eng, st.uid[rs], ts, 50)
    for j, (r, t) in enumerate(zip(rs, ts)):
        r1, s1, l1, c1 = m.recommend_topk(st.eng, [st.uid[r]], [t], 50)
        assert np.array_equal(rows[j], r1[0]) and np.array_equal(sc[j].view(np.uint32), s1[0].view(np.uint32))
        assert np.array_equal(lg[j].view(np.uint64), l1[0].view(np.uint64)) and cnt[j] == c1[0]


def test_nan_parameters_give_empty_lists():
    st = Store(23, I=200)
    m = classifier(st, seed=4)
    p = m.get_params()
    p[-1] = np.nan                                   # the output layer's last coefficient
    m.set_params(p)
    rows, sc, lg, cnt = m.recommend_topk(st.eng, st.uid[[1, 2]], [0, 0], 10)
    assert np.all(cnt == 0) and np.all(rows == -1) and np.all(sc == 0) and np.all(lg == 0)


def test_wide_hidden_layer_runs_the_global_path():
    """A W0 item slice of 23 x 1300 float64 (239 KB) does not fit in shared memory: W0 is read through L1."""
    st = Store(24, I=260, D=16, cF=7)
    m = classifier(st, seed=6, hidden=(1300,))
    check_user(m, st, 1, st.user_ts(1, 0), exact=True)
    check_user(m, st, 3, st.user_ts(3, 1), exact=True, exclude=True)


# ---- 4. live state -----------------------------------------------------------------------------------------------
def test_next_call_sees_live_updates():
    st = Store(25, I=300)
    m = classifier(st, seed=7)
    r = 2
    uid = int(st.uid[r])
    t = 0
    top = m.recommend_topk(st.eng, [uid], [t], 300)[0][0]
    best = int(top[0])
    # an appended event of the user's current best item: the window changes and the item is excluded
    st.eng.ubcache_append([r], [6_000_000], [best])
    assert st.window(r, t)[0] == best
    rows, _, _, cnt = m.recommend_topk(st.eng, [uid], [t], 300)
    assert best not in rows[0, :cnt[0]].tolist()
    check_user(m, st, r, t, exact=True, exclude=True)
    # a new item: id map insert and table rows, then it is scored
    new_id = 10**13 + 5
    row = int(st.eng.idmap_insert(g.IDMAP_ITEM, [new_id])[0])
    assert row == 300
    rng = np.random.default_rng(3)
    st.eng.table_write_rows(g.TABLE_ITEM_EMB, [row], rng.standard_normal((1, 16)).astype(np.float32))
    st.eng.table_write_rows(g.TABLE_ITEM_FEAT, [row], rng.random((1, 7), np.float32))
    rows, sc, lg, cnt = m.recommend_topk(st.eng, [uid], [t], 301, exclude_history=False)
    assert int(cnt[0]) == 301 and row in rows[0].tolist()
    check_user(m, st, r, t, exact=True)
    # a later fit_keys: the new parameters are used
    n = 600
    rng = np.random.default_rng(4)
    u = st.uid[rng.integers(0, st.uid.size, n)]; i = np.asarray(st.eng.item_ids)[rng.integers(0, 301, n)]
    before = m.recommend_topk(st.eng, [uid], [t], 301, exclude_history=False)
    m.fit_keys(st.eng, u, i, np.zeros(n, np.int64), (rng.random(n) < 0.4).astype(np.float32))
    after = check_user(m, st, r, t, exact=True)
    assert not np.array_equal(before[2][0], after[1])


# ---- 5. refusals leave the outputs untouched ---------------------------------------------------------------------
def raw_call(m, eng, uids, ts, k, nu=None, null=None):
    uids = np.ascontiguousarray(uids, np.int64); ts = np.ascontiguousarray(ts, np.int64)
    nu = uids.size if nu is None else nu
    kk = max(k, 1)
    rows = np.full((max(uids.size, 1), kk), 1234, np.int32); sc = np.full((max(uids.size, 1), kk), 7.5, np.float32)
    lg = np.full((max(uids.size, 1), kk), 9.25, np.float64); cnt = np.full(max(uids.size, 1), 77, np.int32)
    ptr = {"user_ids": uids.ctypes.data_as(C.POINTER(C.c_int64)), "ts": ts.ctypes.data_as(C.POINTER(C.c_int64)),
           "rows": rows.ctypes.data_as(C.POINTER(C.c_int32)), "scores": sc.ctypes.data_as(C.POINTER(C.c_float)),
           "count": cnt.ctypes.data_as(C.POINTER(C.c_int32))}
    if null:
        ptr[null] = None
    rc = m.L.ctr_mlp_recommend_topk(m.h, eng.h if eng is not None else None, ptr["user_ids"], ptr["ts"], C.c_int64(nu),
                                    C.c_int32(k), C.c_int32(1), ptr["rows"], ptr["scores"],
                                    lg.ctypes.data_as(C.POINTER(C.c_double)), ptr["count"])
    untouched = np.all(rows == 1234) and np.all(sc == 7.5) and np.all(lg == 9.25) and np.all(cnt == 77)
    return rc, untouched


def test_refusals_write_nothing():
    st = Store(26, I=100)
    m = classifier(st, seed=8)
    uids = st.uid[[1, 2]]
    rc, ok = raw_call(m, st.eng, uids, [0, 0], 5)
    assert rc == 0 and not ok
    for k in (0, 1025):
        rc, ok = raw_call(m, st.eng, uids, [0, 0], k)
        assert rc == g.engine.EINVAL and ok
    rc, ok = raw_call(m, st.eng, uids, [0, 0], 5, nu=0)
    assert rc == g.engine.EINVAL and ok
    for null in ("user_ids", "ts", "rows", "scores", "count"):
        rc, ok = raw_call(m, st.eng, uids, [0, 0], 5, null=null)
        assert rc == g.engine.EINVAL and ok, null
    rc, ok = raw_call(m, None, uids, [0, 0], 5)
    assert rc == g.engine.EINVAL and ok
    # an unknown user anywhere in the request: nothing is written, the first one is named
    rc, ok = raw_call(m, st.eng, [uids[0], 10**15 + 3, 10**15 + 4], [0, 0, 0], 5)
    assert rc == g.engine.ENOTFOUND and ok
    assert str(10**15 + 3) in m.L.ctr_mlp_last_error(m.h).decode()
    # not fitted
    fresh = g.MLPClassifier(st.nin, hidden=(100,))
    rc, ok = raw_call(fresh, st.eng, uids, [0, 0], 5)
    assert rc == g.engine.ESTATE and ok
    # a width mismatch
    other = classifier(Store(27, I=50, uP=6), seed=1)
    rc, ok = raw_call(other, st.eng, uids, [0, 0], 5)
    assert rc == g.engine.EINVAL and ok
    # no id maps
    bare = g.Engine(g.engine.default_config(g.MODEL_DIN_COS, uP=5, S=10, D=16, cF=7, batch=128, pred_batch=256))
    bare.table_upload(g.TABLE_USER_FEAT, st.uf); bare.table_upload(g.TABLE_ITEM_FEAT, st.itf); bare.table_upload(g.TABLE_ITEM_EMB, st.emb)
    rc, ok = raw_call(m, bare, uids, [0, 0], 5)
    assert rc == g.engine.ESTATE and ok
    # a missing table
    bare2 = g.Engine(g.engine.default_config(g.MODEL_DIN_COS, uP=5, S=10, D=16, cF=7, batch=128, pred_batch=256))
    sv.load_id_maps(bare2, st.uid, st.iid)
    bare2.table_upload(g.TABLE_ITEM_EMB, st.emb)
    rc, ok = raw_call(m, bare2, uids, [0, 0], 5)
    assert rc == g.engine.ESTATE and ok
    with pytest.raises(g.engine.CtrError) as e:
        m.recommend_topk(st.eng, [10**15 + 9], [0], 5)
    assert e.value.code == g.engine.ENOTFOUND


# ---- 6. profile and wrappers ---------------------------------------------------------------------------------------
def test_profile_keys():
    st = Store(28, I=700, pred_batch=256)
    m = classifier(st, seed=9, hidden=(64, 32))
    st.eng.profile(True)
    st.eng.profile_reset()
    m.recommend_topk(st.eng, st.uid[[1, 2, 3]], [0, 0, 0], 20)
    prof = st.eng.profile_dump()
    st.eng.profile(False)
    assert "mlp_gather" not in prof
    assert prof["mlp_rec_prefix"][1] == 3
    assert prof["mlp_rec_resolve"][1] == 1
    chunks = 3 * 3                                   # 700 items in chunks of 256, three users
    assert prof["mlp_rec_layer0"][1] == chunks
    assert prof["mlp_rec_layers"][1] == 2 * chunks   # layers 1 and 2 of [nin, 64, 32, 1]
    assert prof["mlp_rec_topk"][1] == chunks and prof["mlp_rec_merge"][1] == chunks
    assert prof["mlp_rec_finish"][1] == 1


def test_serving_recommend_over_fit_keys_predictor():
    st = Store(29, I=400)
    rng = np.random.default_rng(5)
    n = 800
    u = st.uid[rng.integers(0, st.uid.size, n)]; i = st.iid[rng.integers(0, st.iid.size, n)]
    y = (rng.random(n) < 0.4).astype(np.float32)
    pred = gm.SimpleMlpFitWrap(max_iter=3, seed=1).FitKeys(st.eng, u, i, np.zeros(n, np.int64), y)
    for r in (1, 2, 7):
        now = st.user_ts(r, 0)
        out = sv.Recommend(pred, int(st.uid[r]), 25, now=now)
        rows, sc, lg, cnt = pred.pred.recommend_topk(st.eng, [st.uid[r]], [now], 25)
        assert [(x.ItemId, x.Score) for x in out] == [(int(st.iid[rows[0, j]]), float(sc[0, j])) for j in range(int(cnt[0]))]
        rows2, sc2, _ = pred.recommend(int(st.uid[r]), 25, now=now, exclude_history=True)
        assert np.array_equal(rows2, rows[0, :cnt[0]])
        # Rank over the same items gives the same scores
        ranked = sv.Rank(pred, int(st.uid[r]), [x.ItemId for x in out], now=now)
        assert [x.Score for x in ranked] == [x.Score for x in out]
    with pytest.raises(g.engine.CtrError) as e:
        sv.Recommend(pred, 10**15 + 1, 5, now=0)
    assert e.value.code == g.engine.ENOTFOUND
