"""The live behaviour cache: ctr_ubcache_append / ctr_ubcache_set (ubcache.cuh's update kernels) against a plain-Python
model of UserBehaviorCache (cache.go:27-55) plus the online append, and through its consumers.

  * UbModel restates append / set / delete over a dict of (ts, items) lists; a CPU test holds it against naive
    one-event-at-a-time insertion and plain dict assignment;
  * after every call the device CSR (ctr_ubcache_download) must EQUAL the model's, and ctr_ubcache_window must equal
    orc.ub_filter over the model's sequences at S in {1, 32, 50, 100} and maxTs at 0, tied-run boundaries +-1 and the
    int64 extremes;
  * every rejected call leaves the cache exactly as it was;
  * a handle brought to a state by appends and sets must predict, train and recommend exactly like a handle that
    uploaded the same CSR."""
import ctypes as C

import numpy as np
import pytest

import go_ctr_b200 as g
from go_ctr_b200 import serving
from oracle import oracle as orc
from tests.util import INT64_MAX, INT64_MIN, make_tables, scaled_init

INT32_MAX = 2**31 - 1


# ---- the model ---------------------------------------------------------------------------------------------------
class UbModel:
    """seq[row] = (ts list, item list), time-descending.  append: a new event goes after the stored events with a
    strictly greater ts and before those with an equal one; among one call's events of a user with equal ts the later
    one comes first.  set: dict assignment (an empty sequence is Delete).  The user count grows to the largest row + 1."""

    def __init__(self, csr=None):
        self.seq, self.n_users = {}, 0
        if csr is not None:
            off, ts, items = csr
            self.n_users = off.size - 1
            for u in range(self.n_users):
                if off[u + 1] > off[u]:
                    self.seq[u] = (ts[off[u]:off[u + 1]].tolist(), items[off[u]:off[u + 1]].tolist())

    def append(self, rows, ts, items):
        by_user = {}
        for i, (u, t, it) in enumerate(zip(np.asarray(rows).tolist(), np.asarray(ts).tolist(), np.asarray(items).tolist())):
            by_user.setdefault(u, []).append((t, i, it))
        for u, ev in by_user.items():
            ev.sort(key=lambda e: (-e[0], -e[1]))                   # ts descending, later arrival first
            ots, oit = self.seq.get(u, ([], []))
            nts, nit, a = [], [], 0
            for t, _, it in ev:
                while a < len(ots) and ots[a] > t:
                    nts.append(ots[a]); nit.append(oit[a]); a += 1
                nts.append(t); nit.append(it)
            self.seq[u] = (nts + ots[a:], nit + oit[a:])
        if by_user:
            self.n_users = max(self.n_users, max(by_user) + 1)

    def set(self, entries):
        for u, (t, it) in entries.items():
            self.seq[u] = (list(t), list(it))
        if entries:
            self.n_users = max(self.n_users, max(entries) + 1)

    def csr(self):
        lens = np.array([len(self.seq.get(u, ((),))[0]) for u in range(self.n_users)], np.int64)
        off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        ts = np.fromiter((t for u in range(self.n_users) for t in self.seq.get(u, ([], []))[0]), np.int64, int(off[-1]))
        items = np.fromiter((i for u in range(self.n_users) for i in self.seq.get(u, ([], []))[1]), np.int32, int(off[-1]))
        return off, ts, items


def set_args(entries):
    """{row: (ts, items)} → ctr_ubcache_set's (user_rows, offsets, ts, item_rows)."""
    rows = list(entries)
    off = np.concatenate([[0], np.cumsum([len(entries[u][0]) for u in rows])]).astype(np.int64)
    ts = np.concatenate([np.asarray(entries[u][0], np.int64) for u in rows]) if rows else np.zeros(0, np.int64)
    it = np.concatenate([np.asarray(entries[u][1], np.int32) for u in rows]) if rows else np.zeros(0, np.int32)
    return np.array(rows, np.int32), off, ts.astype(np.int64), it.astype(np.int32)


def tied_histories(rng, U, max_len, n_items):
    """Per-user CSR, timestamps descending, in runs of one timestamp up to 150 long; some users empty."""
    lens = np.where(rng.random(U) < 0.3, rng.integers(0, 40, U), rng.integers(0, max_len + 1, U))
    lens[1], lens[2], lens[3] = max_len, 33, 1
    lens[U // 2:U // 2 + 4] = 0
    segs = []
    for L in lens:
        runs = rng.choice([1, 1, 2, 3, 8, 40, 150], size=L)
        run_of = np.repeat(np.arange(L), runs)[:L]
        segs.append(2_000_000 - np.cumsum(rng.integers(1, 4, L)).astype(np.int64)[run_of])
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    return off, np.concatenate(segs).astype(np.int64), rng.integers(0, n_items, off[-1]).astype(np.int32)


def naive_append(seq, rows, ts, items):
    """One event at a time, in arrival order: before the first stored event with ts <= its own."""
    for u, t, it in zip(np.asarray(rows).tolist(), np.asarray(ts).tolist(), np.asarray(items).tolist()):
        s = seq.setdefault(u, ([], []))
        p = next((k for k, x in enumerate(s[0]) if x <= t), len(s[0]))
        s[0].insert(p, t); s[1].insert(p, it)


@pytest.mark.parametrize("seed", range(6))
def test_model_is_one_at_a_time_insertion_and_dict_assignment(seed):
    rng = np.random.default_rng(seed)
    off, ts, items = tied_histories(rng, 40, 60, 30)
    model = UbModel((off, ts, items))
    naive = {u: (list(v[0]), list(v[1])) for u, v in model.seq.items()}
    for _ in range(5):
        m = int(rng.integers(1, 300))
        rows = rng.integers(0, 45, m)
        t = rng.choice(np.concatenate([ts[:50], [0, 1_999_990, 2_100_000, -5]]), m) + rng.integers(-1, 2, m) * (rng.random(m) < 0.3)
        it = rng.integers(-1, 40, m)
        model.append(rows, t, it)
        naive_append(naive, rows, t, it)
        assert {u: v for u, v in model.seq.items() if v[0]} == {u: v for u, v in naive.items() if v[0]}
        assert all(all(a >= b for a, b in zip(v[0], v[0][1:])) for v in model.seq.values())
        assert model.n_users == max(40, max(naive) + 1)
    entries = {3: ([9, 9, 4], [1, 2, 3]), 7: ([], []), 44: ([5], [-1]), 60: ([], [])}
    want = {**{u: v for u, v in model.seq.items()}, **{u: (list(t), list(i)) for u, (t, i) in entries.items()}}
    model.set(entries)
    assert model.seq == want and model.n_users == 61
    o2, t2, i2 = model.csr()
    assert o2[61] - o2[60] == 0 and o2[8] - o2[7] == 0 and t2[o2[3]:o2[4]].tolist() == [9, 9, 4]


# ---- device against the model ------------------------------------------------------------------------------------
S_LIST = (1, 32, 50, 100)


def windows(csr, rows, max_ts, S):
    """TimeSeq.Filter(max_ts, S) per probe through the oracle, -1 padded; rows outside [0, n_users) are empty."""
    off, ts, items = csr
    out = np.full((len(rows), S), -1, np.int32)
    for b, (u, t) in enumerate(zip(rows, max_ts)):
        if 0 <= u < off.size - 1 and off[u + 1] > off[u]:
            start, cnt = orc.ub_filter(ts[off[u]:off[u + 1]], int(t), S)
            out[b, :cnt] = items[off[u] + start: off[u] + start + cnt]
    return out


def probes(rng, csr, touched=()):
    """(row, maxTs) pairs: for every user a few of its tied-run timestamps +-1, 0 and the int64 extremes; the
    (row, ts) of events just written +-1; rows past the cache."""
    off, ts, _ = csr
    rows, mts = [], []
    for u in range(off.size - 1):
        seg = np.unique(ts[off[u]:off[u + 1]])
        pick = rng.choice(seg, min(4, seg.size), replace=False).tolist() if seg.size else [5]
        for t in pick:
            for d in (-1, 0, 1):
                rows.append(u); mts.append(max(INT64_MIN, min(INT64_MAX, t + d)))
        rows += [u, u, u]; mts += [0, INT64_MIN, INT64_MAX]
    touched = list(touched)
    for k in (rng.choice(len(touched), min(len(touched), 1500), replace=False) if touched else []):
        u, t = touched[k]
        for d in (-1, 0, 1):
            if INT64_MIN < t + d < INT64_MAX:
                rows.append(u); mts.append(t + d)
    rows += [off.size - 1, off.size + 3]; mts += [0, 0]
    return np.array(rows, np.int32), np.array(mts, np.int64)


def assert_state(engs, model, rng, touched=()):
    csr = model.csr()
    rows, mts = probes(rng, csr, touched)
    for eng in engs:
        got = eng.ubcache_download()
        for a, b, name in zip(got, csr, ("offsets", "ts", "item_rows")):
            assert a.dtype == b.dtype and a.shape == b.shape and (a == b).all(), (eng.cfg.S, name, a.shape, b.shape)
        want = windows(csr, rows, mts, eng.cfg.S)
        gw = eng.ubcache_window(rows, mts)
        bad = np.flatnonzero((gw != want).any(1))
        assert bad.size == 0, (eng.cfg.S, [(int(rows[b]), int(mts[b])) for b in bad[:5]])


def ub_engine(S, feat_rows):
    eng = g.Engine(g.engine.default_config(g.MODEL_DIN_COS, uP=4, S=S, batch=8, pred_batch=8))
    eng.table_upload(g.TABLE_USER_FEAT, np.zeros((feat_rows, 4), np.float32))
    return eng


def random_events(rng, model, m, rows_from, n_items, wide_ts=False):
    """m events over rows_from: ts tied with a stored event of the user, one either side of it, newer than the user's
    newest, older than its oldest, or anywhere between; a fifth repeat the (user, ts) of an earlier event of the call;
    item rows include -1 and rows past the table.  wide_ts: a tenth at or near the int64 extremes."""
    off, ts_all, _ = model.csr()
    rows = rng.choice(rows_from, m).astype(np.int32)
    r = np.minimum(rows, off.size - 2) if off.size > 1 else np.zeros(m, np.int64)
    L = np.where(rows < off.size - 1, off[r + 1] - off[r], 0) if off.size > 1 else np.zeros(m, np.int64)
    has = L > 0
    pick = lambda: ts_all[np.where(has, off[r] + (rng.random(m) * np.maximum(L, 1)).astype(np.int64), 0)] if ts_all.size else np.zeros(m, np.int64)
    newest = np.where(has, ts_all[np.where(has, off[r], 0)] if ts_all.size else 0, 0)
    oldest = np.where(has, ts_all[np.where(has, off[r] + L - 1, 0)] if ts_all.size else 0, 0)
    kind = rng.integers(0, 5, m)
    ts = np.select([kind == 0, kind == 1, kind == 2, kind == 3],
                   [pick(), pick() + rng.choice([-1, 1], m), newest + rng.integers(1, 4, m), oldest - rng.integers(1, 4, m)],
                   oldest + ((newest - oldest + 1) * rng.random(m)).astype(np.int64))
    ts = np.where(has, ts, 1_000_000 + rng.integers(0, 3, m)).astype(np.int64)
    dup = np.flatnonzero(rng.random(m) < 0.2)
    dup = dup[dup > 0]
    src = (rng.random(dup.size) * dup).astype(np.int64)
    rows[dup], ts[dup] = rows[src], ts[src]
    if wide_ts:
        ext = np.flatnonzero(rng.random(m) < 0.1)
        ts[ext] = rng.choice(np.array([INT64_MIN, INT64_MIN + 1, INT64_MAX, INT64_MAX - 1, -(2**62)], np.int64), ext.size)
    items = rng.integers(0, n_items, m).astype(np.int32)
    odd = rng.random(m)
    items[odd < 0.05] = -1
    past = (odd >= 0.05) & (odd < 0.08)
    items[past] = rng.choice(np.array([n_items, n_items + 7, INT32_MAX], np.int32), int(past.sum()))
    return rows, ts, items


@pytest.mark.gpu
def test_append_and_set_match_the_model_after_every_call():
    """One sequence of calls on four handles (S = 1, 32, 50, 100), checked against UbModel after each: m = 1 tied inside
    a long run, m = 1 for an empty user, a mixed append, a set with replacements / deletes / growth, m = 10^6, an append
    whose timestamps span the int64 range (the two-pass sort), and a last set."""
    rng = np.random.default_rng(2024)
    U, I, FEAT = 300, 1000, 360                        # USER_FEAT rows 300..359 let the cache grow
    base = tied_histories(rng, U, 5000, I)
    engs = [ub_engine(S, FEAT) for S in S_LIST]
    for e in engs:
        e.ubcache_upload(*base)
    model = UbModel(base)
    assert_state(engs, model, rng)
    long_u = 1
    empty_u = U // 2
    all_rows = np.arange(FEAT)

    def append(rows, ts, items):
        for e in engs:
            e.ubcache_append(rows, ts, items)
        model.append(rows, ts, items)
        assert_state(engs, model, rng, list(zip(rows.tolist(), ts.tolist())))

    def set_(entries):
        for e in engs:
            e.ubcache_set(*set_args(entries))
        model.set(entries)
        assert_state(engs, model, rng, [(u, t) for u, (ts, _) in entries.items() for t in ts])

    mid = model.seq[long_u][0][2500]
    append(np.array([long_u], np.int32), np.array([mid], np.int64), np.array([7], np.int32))
    append(np.array([empty_u], np.int32), np.array([123], np.int64), np.array([-1], np.int32))
    append(*random_events(rng, model, 2000, all_rows[:U], I))
    s0 = model.seq[2][0]
    set_({2: ([s0[0] + 5] + [s0[3]] * 40 + [s0[-1] - 9], list(range(42))),   # replace, a long tied run inside
          long_u: ([], []),                                                  # delete a long history
          empty_u + 1: ([], []),                                             # delete an empty one
          U + 10: ([50, 50, 49], [3, -1, I + 2]),                            # past the user count: grows it
          4: (list(range(10, 0, -1)), [I] * 10)})                           # item rows past the table
    append(*random_events(rng, model, 1_000_000, all_rows, I))
    append(*random_events(rng, model, 5000, all_rows, I, wide_ts=True))
    set_({FEAT - 1: ([9], [1])})
    assert model.n_users == FEAT and max(len(v[0]) for v in model.seq.values()) > 5000


@pytest.mark.gpu
def test_append_without_a_cache_creates_it():
    rng = np.random.default_rng(5)
    eng = ub_engine(32, 50)
    with pytest.raises(g.CtrError) as e:
        eng.ubcache_download()
    assert e.value.code == g.ESTATE
    model = UbModel()
    rows, ts, items = random_events(rng, model, 700, np.arange(0, 40), 100)
    eng.ubcache_append(rows, ts, items)
    model.append(rows, ts, items)
    assert_state([eng], model, rng, list(zip(rows.tolist(), ts.tolist())))
    eng2 = ub_engine(32, 50)                          # and a set on a handle with no cache
    eng2.ubcache_set(*set_args({7: ([3, 3], [1, 2])}))
    assert [a.tolist() for a in eng2.ubcache_download()] == [[0] * 8 + [2], [3, 3], [1, 2]]


@pytest.mark.gpu
def test_errors_leave_the_cache_unchanged():
    rng = np.random.default_rng(9)
    eng = ub_engine(32, 100)
    eng.ubcache_upload(*tied_histories(rng, 80, 300, 50))
    before = eng.ubcache_download()
    ok_rows = np.arange(0, 99, dtype=np.int32)

    def expect(code, f, *a):
        with pytest.raises(g.CtrError) as e:
            f(*a)
        assert e.value.code == code, str(e.value)
        got = eng.ubcache_download()
        assert all((x == y).all() and x.shape == y.shape for x, y in zip(got, before))

    for bad in (-1, 100, INT32_MAX, -(2**31)):              # the bound is USER_FEAT's 100 rows
        rows = np.concatenate([ok_rows, [bad]]).astype(np.int32)
        expect(g.EINVAL, eng.ubcache_append, rows, np.arange(rows.size), np.zeros(rows.size, np.int32))
        expect(g.EINVAL, eng.ubcache_set, [5, bad], [0, 1, 2], [7, 6], [1, 2])
    expect(g.EINVAL, eng.ubcache_set, [5, 9, 5], [0, 1, 2, 3], [7, 6, 5], [1, 2, 3])          # user twice
    expect(g.EINVAL, eng.ubcache_set, [5, 9], [0, 1, 4], [7, 6, 6, 8], [1, 2, 3, 4])           # increasing
    expect(g.EINVAL, eng.ubcache_set, [5, 9, 11], [0, 2, 1, 3], [7, 6, 6], [1, 2, 3])          # offsets decrease
    expect(g.EINVAL, eng.ubcache_set, [5, 9], [0, 5, 3], [7, 6, 6], [1, 2, 3])                 # offsets past n
    expect(g.EINVAL, eng.ubcache_set, [5, 9], [0, 1, 3], [7, 6], [1, 2])                       # offsets end past n
    L = eng.L
    nu, n = C.c_int64(0), C.c_int64(0)
    off = np.empty(before[0].size, np.int64); ts = np.empty(before[1].size, np.int64); it = np.empty(before[1].size, np.int32)
    lp, ip = C.POINTER(C.c_int64), C.POINTER(C.c_int32)
    for cu, ce in ((off.size - 2, ts.size), (off.size - 1, ts.size - 1)):
        rc = L.ctr_ubcache_download(eng.h, off.ctypes.data_as(lp), ts.ctypes.data_as(lp), it.ctypes.data_as(ip), C.c_int64(cu), C.c_int64(ce),
                                    C.byref(nu), C.byref(n))
        assert rc == g.EINVAL and (nu.value, n.value) == (off.size - 1, ts.size)
    expect(g.EINVAL, lambda: eng._ck(L.ctr_ubcache_download(eng.h, None, ts.ctypes.data_as(lp), None, C.c_int64(0), C.c_int64(ts.size - 1),
                                                             C.byref(nu), C.byref(n))))
    eng2 = ub_engine(32, 100)
    with pytest.raises(g.CtrError) as e:
        eng2.ubcache_download()
    assert e.value.code == g.ESTATE
    with pytest.raises(g.CtrError) as e:
        ub_engine(32, 1).ubcache_append([1], [5], [0])                       # no cache, 1 USER_FEAT row
    assert e.value.code == g.EINVAL


# ---- through the consumers ---------------------------------------------------------------------------------------
DIMS = (8, 50, 16, 5)
U_C, I_C, TB = 120, 400, 64


def world(seed, model_kind, dense_lr=0.0):
    """Two handles with the same tables, weights and id maps.  Dense lr 0: the dense gradients sum with float atomics,
    so only with the dense weights fixed is training bit-reproducible across handles; the deterministic table path is
    (and it reads every history row)."""
    rng = np.random.default_rng(seed)
    uP, S, D, cF = DIMS
    tabs = make_tables(rng, U_C, I_C, uP, cF, D)
    ocfg = orc.make_cfg(model_kind, uP, S, D, cF, 200, 80)
    W = scaled_init(orc, ocfg, seed)
    uid = rng.choice(10**9, U_C, replace=False).astype(np.int64) + 1
    iid = rng.choice(10**9, I_C, replace=False).astype(np.int64) + 1

    def make():
        eng = g.Engine(g.engine.default_config(model_kind, uP=uP, S=S, D=D, cF=cF, batch=TB, pred_batch=TB, lr=dense_lr,
                                               table_opt=g.TABLE_SGD_DETERMINISTIC, table_lr=0.3, dropout0=0.0, dropout1=0.0, seed=3))
        for w, t in zip((g.TABLE_USER_FEAT, g.TABLE_ITEM_FEAT, g.TABLE_ITEM_EMB), tabs):
            eng.table_upload(w, t)
        eng.set_weights(*W)
        serving.load_id_maps(eng, uid, iid)
        return eng
    return rng, tabs, uid, iid, make


def updated_pair(rng, make):
    """A: upload, append, set, append (rows past the upload included).  B: upload of the model's CSR."""
    base = tied_histories(rng, U_C - 20, 600, I_C)
    A, B = make(), make()
    A.ubcache_upload(*base)
    model = UbModel(base)
    for step in range(3):
        if step == 1:
            entries = {3: ([1_999_999, 1_999_999, 10], [5, 6, -1]), 7: ([], []), U_C - 5: ([1_500_000], [9])}
            A.ubcache_set(*set_args(entries)); model.set(entries)
        else:
            ev = random_events(rng, model, 3000, np.arange(U_C), I_C)
            A.ubcache_append(*ev); model.append(*ev)
    B.ubcache_upload(*model.csr())
    for a, b in zip(A.ubcache_download(), B.ubcache_download()):
        assert (a == b).all()
    return A, B, model


def sample_keys(rng, model, uid, iid, n):
    """Sample keys whose ts is a stored timestamp of the user +-1 (or 0, "from the newest")."""
    off, ts, _ = model.csr()
    su = rng.integers(0, U_C, n)
    r = np.minimum(su, off.size - 2)
    L = np.where(su < off.size - 1, off[r + 1] - off[r], 0)
    kt = np.where(L > 0, ts[np.where(L > 0, off[r] + (rng.random(n) * np.maximum(L, 1)).astype(np.int64), 0)], 5) + rng.integers(-1, 2, n)
    kt[rng.random(n) < 0.1] = 0
    return uid[su], iid[rng.integers(0, I_C, n)], kt.astype(np.int64)


@pytest.mark.gpu
@pytest.mark.parametrize("model_kind", [g.MODEL_DIN_COS, g.MODEL_DIN_EUC, g.MODEL_YOUTUBE], ids=["din_cos", "din_euc", "youtube"])
def test_updated_cache_predicts_and_trains_like_an_uploaded_one(model_kind):
    rng, tabs, uid, iid, make = world(31 + model_kind, model_kind)
    A, B, model = updated_pair(rng, make)
    ku, ki, kt = sample_keys(rng, model, uid, iid, 1000)
    pa, pb = A.batch_predict_keys(ku, ki, kt), B.batch_predict_keys(ku, ki, kt)
    assert pa.tobytes() == pb.tobytes()
    y = (rng.random(ku.size) > 0.5).astype(np.float32)
    ra, rb = A.train_keys(ku, ki, kt, y, epochs=2), B.train_keys(ku, ki, kt, y, epochs=2)
    assert ra == rb, (ra, rb)
    for wa, wb in zip(A.get_weights(), B.get_weights()):
        assert wa.tobytes() == wb.tobytes()
    ea, eb = A.table_download(g.TABLE_ITEM_EMB, I_C, DIMS[2]), B.table_download(g.TABLE_ITEM_EMB, I_C, DIMS[2])
    assert ea.tobytes() == eb.tobytes() and not np.array_equal(ea, tabs[2])


@pytest.mark.gpu
def test_append_between_train_calls_is_used_by_the_second():
    rng, tabs, uid, iid, make = world(77, g.MODEL_DIN_COS)
    base = tied_histories(rng, U_C, 300, I_C)
    A, B, Cn = make(), make(), make()
    for e in (A, B, Cn):
        e.ubcache_upload(*base)
    model = UbModel(base)
    k1 = sample_keys(rng, model, uid, iid, 300)
    y1 = (rng.random(300) > 0.5).astype(np.float32)
    for e in (A, B, Cn):
        e.train_keys(*k1, y1)
    ev = random_events(rng, model, 2000, np.arange(U_C), I_C)
    ev[1][:] = 2_500_000 + np.arange(ev[1].size)                    # newer than every stored event
    cache = serving.UserBehaviorCache(A)
    unknown = 10**12 + 1
    dropped = cache.Append(np.concatenate([uid[ev[0]], [unknown]]), np.concatenate([iid[np.clip(ev[2], 0, I_C - 1)], [iid[0]]]),
                           np.concatenate([ev[1], [5]]))
    assert dropped == 1
    model.append(ev[0], ev[1], np.clip(ev[2], 0, I_C - 1).astype(np.int32))
    B.ubcache_upload(*model.csr())
    for a, b in zip(A.ubcache_download(), B.ubcache_download()):
        assert (a == b).all()
    su = rng.integers(0, U_C, 300)
    k2 = (uid[su], iid[rng.integers(0, I_C, 300)], np.full(300, 3_000_000, np.int64))
    y2 = (rng.random(300) > 0.5).astype(np.float32)
    out = [e.train_keys(*k2, y2) for e in (A, B, Cn)]
    emb = [e.table_download(g.TABLE_ITEM_EMB, I_C, DIMS[2]) for e in (A, B, Cn)]
    assert out[0] == out[1] and emb[0].tobytes() == emb[1].tobytes()
    assert out[0][1] != out[2][1] and not np.array_equal(emb[0], emb[2])           # the append changed what trained


@pytest.mark.gpu
def test_user_behavior_cache_through_serving():
    """Recommend with exclude_history stops returning an item as soon as it is appended to the user's history;
    Set / BatchSet / Delete / Clear over external ids."""
    rng, tabs, uid, iid, make = world(5, g.MODEL_DIN_COS, dense_lr=0.01)
    eng = make()
    eng.ubcache_upload(*tied_histories(rng, U_C, 200, I_C))
    cache = serving.UserBehaviorCache(eng)
    now = 3_000_000
    user = int(uid[9])
    row = 9
    first = serving.Recommend(eng, user, 10, now=now)
    assert len(first) == 10
    for rnd in range(3):
        top = first[0].ItemId
        assert cache.Append([user], [top], [now - 1 - rnd]) == 0
        after = serving.Recommend(eng, user, 10, now=now)
        assert top not in [r.ItemId for r in after] and len(after) == 10
        first = after
    imap = {int(v): r for r, v in enumerate(iid)}
    before = eng.ubcache_download()
    with pytest.raises(g.CtrError) as e:
        cache.BatchSet({user: ([5], [iid[1]]), 10**12 + 7: ([4], [iid[2]])})
    assert e.value.code == g.ENOTFOUND
    assert all((a == b).all() for a, b in zip(eng.ubcache_download(), before))
    cache.Set(user, [now - 1, now - 5, now - 5], [iid[3], -424_242, iid[4]])       # no item id is negative
    off, ts, items = eng.ubcache_download()
    assert ts[off[row]:off[row + 1]].tolist() == [now - 1, now - 5, now - 5]
    assert items[off[row]:off[row + 1]].tolist() == [imap[int(iid[3])], -1, imap[int(iid[4])]]
    cache.BatchSet({int(uid[1]): ([8, 7], [iid[5], iid[6]]), int(uid[2]): ([], [])})
    off, ts, items = eng.ubcache_download()
    assert items[off[1]:off[2]].tolist() == [5, 6] and off[3] == off[2]
    cache.Delete(user)
    cache.Delete(10**12 + 9)                                                         # unknown: nothing to delete
    assert (eng.ubcache_window([row], [now]) == -1).all()
    assert len(serving.Recommend(eng, user, 10, now=now)) == 10
    cache.Clear()
    off, ts, items = eng.ubcache_download()
    assert off.tolist() == [0, 0] and ts.size == 0
    assert cache.Append([user, user], [iid[1], iid[2]], [4, 4]) == 0
    off, ts, items = eng.ubcache_download()
    assert off.size == row + 2 and items[off[row]:].tolist() == [2, 1]           # equal ts: the later event first
