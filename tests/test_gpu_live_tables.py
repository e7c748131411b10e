"""Live id maps and tables: ctr_idmap_insert / ctr_idmap_download / ctr_table_write_rows against plain models.

  * id maps against a Python dict (row of every id, misses, download) after every call, through creation, repeats,
    present ids, the int64 extremes, one-at-a-time growth across capacity doublings, one call across many doublings and
    probe chains that wrap past the last slot and are then rehashed; refusals change nothing;
  * row writes against a numpy table at D in {16, 64, 128} with widths that are not multiples of 4: overwrites,
    appends (one row, far past the end, thousands of one-row appends across chunk and reservation boundaries), writes
    without a table, refusals;
  * a handle grown live predicts, recommends, searches, gathers and trains bit for bit like one built from scratch out
    of its downloads;
  * the row-Adam moments, the hot-row accumulators, tables past 2^31 / 2^32 elements and the profile keys."""
import ctypes as C

import numpy as np
import pytest

import go_ctr_b200 as g
from go_ctr_b200 import serving
from oracle import oracle as orc
from tests.util import INT64_MAX, INT64_MIN, idmap_capacity, ids_probing_from, make_tables, scaled_init

INT32_MAX = 2**31 - 1
USER, ITEM = g.IDMAP_USER, g.IDMAP_ITEM
WIDTH = {g.TABLE_USER_FEAT: "uP", g.TABLE_ITEM_FEAT: "cF", g.TABLE_ITEM_EMB: "D"}


def engine(uP=5, S=4, D=16, cF=7, batch=32, **kw):
    return g.Engine(g.engine.default_config(g.MODEL_DIN_COS, uP=uP, S=S, D=D, cF=cF, batch=batch, pred_batch=batch, **kw))


def expect(code, f, *a):
    with pytest.raises(g.CtrError) as e:
        f(*a)
    assert e.value.code == code, str(e.value)


# ---- id maps ---------------------------------------------------------------------------------------------------------
class MapModel:
    def __init__(self):
        self.row = {}

    def insert(self, ids):
        for v in np.asarray(ids, np.int64).tolist():
            self.row.setdefault(v, len(self.row))
        return np.array([self.row[v] for v in np.asarray(ids, np.int64).tolist()], np.int32)

    def ids(self):
        out = np.empty(len(self.row), np.int64)
        for v, r in self.row.items():
            out[r] = v
        return out


def assert_map(e, which, model, rng, extra=()):
    ids = model.ids()
    assert e.idmap_download(which).tobytes() == ids.tobytes()
    if ids.size:
        assert (e.idmap_lookup(which, ids) == np.arange(ids.size)).all()
    miss = np.array([v for v in list(rng.integers(INT64_MIN + 1, INT64_MAX, 64)) + list(extra) if int(v) not in model.row], np.int64)
    if miss.size:
        assert (e.idmap_lookup(which, miss) == -1).all()


@pytest.mark.gpu
def test_insert_creates_a_map_and_equals_build_on_distinct_ids():
    rng = np.random.default_rng(1)
    ids = rng.choice(10**12, 5000, replace=False).astype(np.int64) - 10**11
    a, b = engine(), engine()
    rows = a.idmap_insert(USER, ids)
    b.idmap_build(USER, ids)
    assert (rows == np.arange(ids.size)).all()
    assert a.idmap_download(USER).tobytes() == b.idmap_download(USER).tobytes() == ids.tobytes()
    probe = np.concatenate([ids, rng.integers(-2**62, 2**62, 500)])
    assert a.idmap_lookup(USER, probe).tobytes() == b.idmap_lookup(USER, probe).tobytes()


@pytest.mark.gpu
def test_insert_matches_a_dict():
    rng = np.random.default_rng(2)
    e, model = engine(), MapModel()
    extremes = np.array([INT64_MAX, INT64_MIN + 1, -1, 0], np.int64)
    calls = [np.array([5, 5, 7, 5, 9], np.int64),                          # creation, repeats
             np.array([7, 11, 5, 11, 12], np.int64),                       # present and new, mixed
             extremes, extremes[::-1].copy(),                              # the extremes, then all present
             rng.integers(-50, 50, 300),                                   # heavy repeats
             rng.integers(INT64_MIN + 1, INT64_MAX, 2000)]
    for ids in calls:
        ids = np.asarray(ids, np.int64)
        assert e.idmap_insert(USER, ids).tobytes() == model.insert(ids).tobytes()
        assert_map(e, USER, model, rng, extra=extremes)


@pytest.mark.gpu
def test_one_id_at_a_time_across_capacity_doublings():
    rng = np.random.default_rng(3)
    e, model = engine(), MapModel()
    ids = rng.choice(2**40, 300, replace=False).astype(np.int64)
    for k, v in enumerate(ids):
        assert e.idmap_insert(ITEM, [v])[0] == model.insert([v])[0] == k
        n = k + 1
        # check right after every doubling (the 33rd id at capacity 64, the 65th at 128, ...) and at a few other counts
        if idmap_capacity(n) != idmap_capacity(n - 1) or n in (1, 2, 32, 299):
            assert_map(e, ITEM, model, rng)
    assert_map(e, ITEM, model, rng)


@pytest.mark.gpu
def test_one_call_across_many_doublings():
    rng = np.random.default_rng(4)
    e, model = engine(), MapModel()
    first = rng.choice(2**50, 10, replace=False).astype(np.int64)
    e.idmap_insert(USER, first); model.insert(first)
    big = np.concatenate([rng.integers(INT64_MIN + 1, INT64_MAX, 100_000), first[:3], rng.integers(0, 1000, 1000)]).astype(np.int64)
    rng.shuffle(big)
    assert e.idmap_insert(USER, big).tobytes() == model.insert(big).tobytes()
    assert_map(e, USER, model, rng)


@pytest.mark.gpu
def test_wrapped_probe_chains_are_rehashed():
    rng = np.random.default_rng(5)
    e, model = engine(), MapModel()
    cap = idmap_capacity(1)
    # chains that start in the last slots and wrap past slot cap-1 to the front
    wrap = ids_probing_from(rng, [cap - 2, cap - 1, cap - 1, cap - 2, cap - 1, 0, cap - 1], cap)
    e.idmap_insert(ITEM, wrap); model.insert(wrap)
    assert_map(e, ITEM, model, rng)
    # grows the table twice: the wrapped chains are rehashed into larger tables
    more = ids_probing_from(rng, rng.integers(0, 4 * cap, 100), 4 * cap, avoid=wrap)
    for chunk in (more[:30], more[30:]):
        assert e.idmap_insert(ITEM, chunk).tobytes() == model.insert(chunk).tobytes()
        assert_map(e, ITEM, model, rng, extra=more)


@pytest.mark.gpu
def test_insert_refusals_change_nothing():
    rng = np.random.default_rng(6)
    e, model = engine(), MapModel()
    base = rng.choice(10**9, 40, replace=False).astype(np.int64)
    e.idmap_insert(USER, base); model.insert(base)
    L = e.L
    expect(g.EINVAL, e.idmap_insert, USER, np.array([1, 2, INT64_MIN, 3], np.int64))     # INT64_MIN among new ids
    expect(g.EINVAL, e.idmap_insert, USER, np.array([base[0], INT64_MIN], np.int64))
    assert L.ctr_idmap_insert(e.h, C.c_int(USER), None, C.c_int64(3), None) == g.EINVAL
    a = np.array([1, 2], np.int64)
    assert L.ctr_idmap_insert(e.h, C.c_int(USER), a.ctypes.data_as(C.POINTER(C.c_int64)), C.c_int64(0), None) == g.EINVAL
    assert L.ctr_idmap_insert(e.h, C.c_int(2), a.ctypes.data_as(C.POINTER(C.c_int64)), C.c_int64(2), None) == g.EINVAL
    assert_map(e, USER, model, rng, extra=[1, 2, 3])
    # rows may be NULL
    assert L.ctr_idmap_insert(e.h, C.c_int(USER), a.ctypes.data_as(C.POINTER(C.c_int64)), C.c_int64(2), None) == 0
    model.insert(a)
    assert_map(e, USER, model, rng)
    # download rules: no map is ESTATE, a short array EINVAL
    expect(g.ESTATE, e.idmap_download, ITEM)
    n = C.c_int64(0); out = np.empty(3, np.int64)
    assert L.ctr_idmap_download(e.h, C.c_int(USER), out.ctypes.data_as(C.POINTER(C.c_int64)), C.c_int64(3), C.byref(n)) == g.EINVAL


# ---- row writes ------------------------------------------------------------------------------------------------------
def dims_for(D):
    return dict(uP=5, D=D, cF=7)


@pytest.mark.gpu
@pytest.mark.parametrize("D", [16, 64, 128])
def test_row_writes_match_numpy(D):
    rng = np.random.default_rng(10 + D)
    e = engine(**dims_for(D))
    for which in (g.TABLE_USER_FEAT, g.TABLE_ITEM_FEAT, g.TABLE_ITEM_EMB):
        w = getattr(e.cfg, WIDTH[which])
        # no table yet: the write creates one, rows before the written one are zero
        model = np.zeros((4, w), np.float32)
        d = rng.standard_normal((1, w)).astype(np.float32)
        e.table_write_rows(which, [3], d); model[3] = d
        assert e.table_download(which, *model.shape).tobytes() == model.tobytes()
        up = rng.standard_normal((50, w)).astype(np.float32)
        e.table_upload(which, up); model = up.copy()

        def write(rows, data):
            nonlocal model
            rows = np.asarray(rows, np.int32)
            top = int(rows.max()) + 1
            if top > model.shape[0]:
                model = np.concatenate([model, np.zeros((top - model.shape[0], w), np.float32)])
            model[rows] = data
            e.table_write_rows(which, rows, data)
            assert e.table_download(which, *model.shape).tobytes() == model.tobytes()

        write(rng.permutation(50)[:17], rng.standard_normal((17, w)).astype(np.float32))          # overwrites
        write([50], rng.standard_normal((1, w)).astype(np.float32))                              # one-row append
        write([20, 3000, 7], rng.standard_normal((3, w)).astype(np.float32))                     # far past the end
        bad = np.array([np.nan, -0.0, np.inf], np.float32)                                       # bits, not values
        write([1], np.resize(bad, (1, w)))
        # refusals leave the table bitwise unchanged
        snap = model.tobytes()
        one = rng.standard_normal((2, w)).astype(np.float32)
        for rows in ([4, 4], [-1, 3], [INT32_MAX, 0]):
            expect(g.EINVAL, e.table_write_rows, which, rows, one)
        expect(g.EINVAL, e.table_write_rows, which, [1], rng.standard_normal((1, w + 1)).astype(np.float32))
        assert e.L.ctr_table_write_rows(e.h, C.c_int(which), None, None, C.c_int64(1), C.c_int32(w)) == g.EINVAL
        assert e.table_download(which, *model.shape).tobytes() == snap


@pytest.mark.gpu
def test_thousands_of_one_row_appends():
    """2000 one-row appends, each 2048 rows past the last (128 KiB at D = 16): the table grows from one 2 MiB granule to
    256 MiB, through about forty mapped chunks (1/8 of the mapped size each) and several larger reservations."""
    rng = np.random.default_rng(11)
    D, step, n = 16, 2048, 2000
    e = engine(D=D)
    rows = np.arange(n, dtype=np.int64) * step + 5
    data = rng.standard_normal((n, D)).astype(np.float32)
    for k in range(n):
        e.table_write_rows(g.TABLE_ITEM_EMB, rows[k:k + 1].astype(np.int32), data[k:k + 1])
        if k in (0, 1, 15, 16, 17, 500, n - 1):
            got = e.table_download(g.TABLE_ITEM_EMB, int(rows[k]) + 1, D)
            want = np.zeros_like(got); want[rows[:k + 1]] = data[:k + 1]
            assert got.tobytes() == want.tobytes(), k
    # one call whose staging takes several 32 MiB chunks, overwrites and appends mixed
    N = int(rows[-1]) + 1
    big_rows = rng.permutation(N + 600_000)[:700_000].astype(np.int32)
    big = rng.standard_normal((big_rows.size, D)).astype(np.float32)
    want = np.zeros((max(N, int(big_rows.max()) + 1), D), np.float32); want[rows] = data; want[big_rows] = big
    e.table_write_rows(g.TABLE_ITEM_EMB, big_rows, big)
    assert e.table_download(g.TABLE_ITEM_EMB, *want.shape).tobytes() == want.tobytes()


# ---- a live handle equals one built from scratch ---------------------------------------------------------------------
DIMS = (5, 6, 16, 7)
U0, I0, TB = 60, 150, 64


def twin_world(seed, model_kind, table_opt=g.TABLE_SGD_DETERMINISTIC):
    rng = np.random.default_rng(seed)
    uP, S, D, cF = DIMS
    tabs = make_tables(rng, U0, I0, uP, cF, D)
    W = scaled_init(orc, orc.make_cfg(model_kind, uP, S, D, cF, 200, 80), seed)
    uid = rng.choice(10**9, U0, replace=False).astype(np.int64) + 1
    iid = rng.choice(10**9, I0, replace=False).astype(np.int64) + 1

    def make():
        e = g.Engine(g.engine.default_config(model_kind, uP=uP, S=S, D=D, cF=cF, batch=TB, pred_batch=TB, lr=0.0,
                                             table_opt=table_opt, table_lr=0.3, dropout0=0.0, dropout1=0.0, seed=3))
        e.set_weights(*W)
        return e
    return rng, tabs, uid, iid, make


def grow_live(rng, e, tabs, uid, iid):
    """Applies a mixed sequence to e; returns the new user / item ids."""
    uP, S, D, cF = DIMS
    for w, t in zip((g.TABLE_USER_FEAT, g.TABLE_ITEM_FEAT, g.TABLE_ITEM_EMB), tabs):
        e.table_upload(w, t)
    serving.load_id_maps(e, uid, iid)
    new_u = rng.choice(10**9, 25, replace=False).astype(np.int64) + 2 * 10**9
    new_i = rng.choice(10**9, 60, replace=False).astype(np.int64) + 2 * 10**9
    fc = serving.FeatureCache(e)
    for k, u in enumerate(new_u[:10]):
        assert fc.SetUser(u, rng.random(uP)) == U0 + k
    ur = e.idmap_insert(USER, np.concatenate([new_u[5:], uid[:3]]))
    e.table_write_rows(g.TABLE_USER_FEAT, ur[5:-3], rng.random((ur.size - 8, uP)).astype(np.float32))
    for k, it in enumerate(new_i[:20]):
        assert fc.SetItem(it, rng.random(cF), rng.standard_normal(D) / 4 if k % 2 else None) == I0 + k
    ir = e.idmap_insert(ITEM, np.concatenate([new_i[20:], new_i[20:30], iid[:4]]))
    e.table_write_rows(g.TABLE_ITEM_FEAT, ir[:40], rng.random((40, cF)).astype(np.float32))
    e.table_write_rows(g.TABLE_ITEM_EMB, ir[:40:3], (rng.standard_normal((14, D)) / 4).astype(np.float32))
    e.table_write_rows(g.TABLE_ITEM_EMB, rng.permutation(I0)[:30].astype(np.int32), (rng.standard_normal((30, D)) / 4).astype(np.float32))
    n_u, n_i = U0 + 25, I0 + 60
    urows = rng.integers(0, n_u, 2000).astype(np.int32)
    e.ubcache_append(urows, rng.integers(1, 10**6, 2000), rng.integers(-1, n_i, 2000).astype(np.int32))
    return new_u, new_i


def twin_of(e, make):
    uP, S, D, cF = DIMS
    b = make()
    for which in (USER, ITEM):
        b.idmap_build(which, e.idmap_download(which))
    b.item_ids = e.idmap_download(ITEM)
    n = {USER: e.idmap_download(USER).size, ITEM: e.idmap_download(ITEM).size}
    for w, width, rows in ((g.TABLE_USER_FEAT, uP, n[USER]), (g.TABLE_ITEM_FEAT, cF, n[ITEM]), (g.TABLE_ITEM_EMB, D, n[ITEM])):
        b.table_upload(w, e.table_download(w, rows, width))
    b.ubcache_upload(*e.ubcache_download())
    return b


@pytest.mark.gpu
@pytest.mark.parametrize("model_kind", [g.MODEL_DIN_COS, g.MODEL_DIN_EUC, g.MODEL_YOUTUBE], ids=["din_cos", "din_euc", "youtube"])
def test_live_handle_equals_one_built_from_scratch(model_kind):
    rng, tabs, uid, iid, make = twin_world(40 + model_kind, model_kind)
    A = make()
    new_u, new_i = grow_live(rng, A, tabs, uid, iid)
    B = twin_of(A, make)
    all_u, all_i = np.concatenate([uid, new_u]), np.concatenate([iid, new_i])
    n = 1500
    ku, ki = all_u[rng.integers(0, all_u.size, n)], all_i[rng.integers(0, all_i.size, n)]
    kt = rng.integers(0, 10**6, n).astype(np.int64)
    ku[0], ki[0] = uid[0], iid[0]
    assert A.batch_predict_keys(ku, ki, kt).tobytes() == B.batch_predict_keys(ku, ki, kt).tobytes()
    S = DIMS[1]
    ur = A.idmap_lookup(USER, all_u[:40:3]); hist = A.ubcache_window(ur, np.zeros(ur.size, np.int64))
    for x, y in zip(A.recommend_topk(ur, hist, 12), B.recommend_topk(ur, hist, 12)):
        assert x.tobytes() == y.tobytes()
    assert serving.Recommend(A, new_u[3], 5, now=10**7) == serving.Recommend(B, new_u[3], 5, now=10**7)
    qr = np.arange(0, I0 + 60, 7).astype(np.int32)
    for x, y in zip(A.knn_search(10, rows=qr), B.knn_search(10, rows=qr)):
        assert x.tobytes() == y.tobytes()
    ir = rng.integers(-1, I0 + 60, 300).astype(np.int32)
    h = rng.integers(-1, I0 + 60, (300, S)).astype(np.int32)
    ugr = rng.integers(0, U0 + 25, 300).astype(np.int32)
    assert A.gather_rows(ugr, ir, h).tobytes() == B.gather_rows(ugr, ir, h).tobytes()
    y = (rng.random(n) > 0.5).astype(np.float32)
    assert A.train_keys(ku, ki, kt, y, epochs=2) == B.train_keys(ku, ki, kt, y, epochs=2)
    for wa, wb in zip(A.get_weights(), B.get_weights()):
        assert wa.tobytes() == wb.tobytes()
    for w, width, rows in ((g.TABLE_ITEM_EMB, DIMS[2], I0 + 60), (g.TABLE_USER_FEAT, DIMS[0], U0 + 25)):
        assert A.table_download(w, rows, width).tobytes() == B.table_download(w, rows, width).tobytes()


@pytest.mark.gpu
def test_new_item_scores_as_zero_row_then_with_its_features():
    rng, tabs, uid, iid, make = twin_world(50, g.MODEL_DIN_COS)
    uP, S, D, cF = DIMS
    A = make()
    for w, t in zip((g.TABLE_USER_FEAT, g.TABLE_ITEM_FEAT, g.TABLE_ITEM_EMB), tabs):
        A.table_upload(w, t)
    serving.load_id_maps(A, uid, iid)
    new = 77_000_000_000
    ku, ki, kt = np.array([uid[0], uid[1], uid[2]]), np.array([iid[0], new, iid[3]]), np.zeros(3, np.int64)
    before = A.batch_predict_keys(ku, ki, kt)
    zero = A.batch_predict_keys(ku, np.array([iid[0], -5, iid[3]]), kt)           # -5: another unknown item
    assert before.tobytes() == zero.tobytes()
    feat = rng.random(cF).astype(np.float32)
    row = serving.FeatureCache(A).SetItem(new, feat)
    assert row == I0 and A.item_ids[row] == new
    X = A.gather_rows(np.array([A.idmap_lookup(USER, [uid[1]])[0]], np.int32), np.array([row], np.int32), np.full((1, S), -1, np.int32))
    assert (X[0, uP + S * D:uP + S * D + D] == 0).all() and X[0, -cF:].tobytes() == feat.tobytes()
    after = A.batch_predict_keys(ku, ki, kt)
    assert after[0] == before[0] and after[2] == before[2] and after[1] != before[1]


# ---- solver state ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_row_adam_moments_survive_a_write(tmp_path):
    rng, tabs, uid, iid, make = twin_world(60, g.MODEL_DIN_COS, table_opt=g.TABLE_ADAM)
    uP, S, D, cF = DIMS
    A = make()
    for w, t in zip((g.TABLE_USER_FEAT, g.TABLE_ITEM_FEAT, g.TABLE_ITEM_EMB), tabs):
        A.table_upload(w, t)
    serving.load_id_maps(A, uid, iid)
    n = 600
    ku, ki, kt = uid[rng.integers(0, U0, n)], iid[rng.integers(0, I0, n)], np.zeros(n, np.int64)
    A.train_keys(ku, ki, kt, (rng.random(n) > 0.5).astype(np.float32), epochs=2)
    p0, p1, p2 = (str(tmp_path / ("c%d" % k)) for k in range(3))
    A.checkpoint_save(p0)
    rows = np.array([3, 40, 41, 149], np.int32)
    data = rng.standard_normal((4, D)).astype(np.float32)
    A.table_write_rows(g.TABLE_ITEM_EMB, rows, data)
    A.checkpoint_save(p1)
    grow = np.array([160], np.int32)
    A.table_write_rows(g.TABLE_ITEM_EMB, grow, data[:1])
    A.checkpoint_save(p2)
    # the file: header, dense W/M/V, tables (USER_FEAT, ITEM_FEAT, ITEM_EMB), then ITEM_EMB's m and v
    b0, b1, b2 = (open(p, "rb").read() for p in (p0, p1, p2))
    tail = lambda b, rows_: np.frombuffer(b[len(b) - 3 * rows_ * D * 4:], np.float32).reshape(3, rows_, D)
    head = lambda b, rows_: b[:len(b) - 3 * rows_ * D * 4]
    assert head(b0, I0) == head(b1, I0)                      # header (step counter), dense tensors, feature tables
    t0, t1 = tail(b0, I0), tail(b1, I0)
    keep = np.setdiff1d(np.arange(I0), rows)
    assert t1[:, keep].tobytes() == t0[:, keep].tobytes()
    assert t1[0, rows].tobytes() == data.tobytes() and not t1[1:, rows].any()
    assert t0[1:, rows].any()                                 # the written rows had moments to lose
    t2 = tail(b2, 161)
    assert t2[:, :I0].tobytes() == t1.tobytes()
    assert not t2[:, I0:160].any() and t2[0, 160].tobytes() == data[0].tobytes() and not t2[1:, 160].any()


@pytest.mark.gpu
def test_hot_rows_read_the_written_values():
    """Fused SGD with automatic hot rows (every row of a small table is hot): a write between two steps is what the next
    step's gradients see, and growing the table leaves no stale accumulator."""
    rng, tabs, uid, iid, make = twin_world(70, g.MODEL_DIN_COS, table_opt=g.TABLE_SGD)
    uP, S, D, cF = DIMS
    A, B = make(), make()
    for e in (A, B):
        for w, t in zip((g.TABLE_USER_FEAT, g.TABLE_ITEM_FEAT, g.TABLE_ITEM_EMB), tabs):
            e.table_upload(w, t)
    ur = rng.integers(0, U0, TB).astype(np.int32); ir = rng.integers(0, I0, TB).astype(np.int32)
    hist = rng.integers(-1, I0, (TB, S)).astype(np.int32); y = (rng.random(TB) > 0.5).astype(np.float32)
    A.train_step_idx(ur, ir, hist, y)
    rows = np.unique(np.concatenate([ir[:5], hist[:3].ravel()]))
    rows = rows[rows >= 0].astype(np.int32)
    data = rng.standard_normal((rows.size, D)).astype(np.float32)
    A.table_write_rows(g.TABLE_ITEM_EMB, rows, data)
    B.table_upload(g.TABLE_ITEM_EMB, A.table_download(g.TABLE_ITEM_EMB, I0, D))
    ga, gb = A.debug_grads_idx(ur, ir, hist, y, training=False), B.debug_grads_idx(ur, ir, hist, y, training=False)
    for k in ga:
        if k == "datt":      # summed with float atomics: equal up to the order of the adds, on one handle as on two
            assert np.allclose(ga[k], gb[k], rtol=1e-5, atol=1e-7)
        else:
            assert np.asarray(ga[k]).tobytes() == np.asarray(gb[k]).tobytes(), k
    # growth of a small (all-hot) table, then training on: A and B stay equal step for step
    more = rng.standard_normal((40, D)).astype(np.float32)
    A.table_write_rows(g.TABLE_ITEM_EMB, np.arange(I0, I0 + 40, dtype=np.int32), more)
    B.table_upload(g.TABLE_ITEM_EMB, A.table_download(g.TABLE_ITEM_EMB, I0 + 40, D))
    ir2 = rng.integers(0, I0 + 40, TB).astype(np.int32)
    for _ in range(3):
        A.train_step_idx(ur, ir2, hist, y); B.train_step_idx(ur, ir2, hist, y)
    ea, eb = A.table_download(g.TABLE_ITEM_EMB, I0 + 40, D), B.table_download(g.TABLE_ITEM_EMB, I0 + 40, D)
    assert np.allclose(ea, eb, rtol=1e-5, atol=1e-6)


# ---- big tables and profile keys -------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_growth_across_2_31_and_2_32_elements():
    D = 64
    e = engine(uP=4, S=8, D=D, cF=4, batch=512)
    I = (1 << 31) // D - 3
    e.table_fill(g.TABLE_ITEM_EMB, I, D, seed=5, dist=1, scale=0.125)
    e.table_fill(g.TABLE_USER_FEAT, 1, 4); e.table_fill(g.TABLE_ITEM_FEAT, 1, 4)
    rng = np.random.default_rng(80)
    r31 = np.array([I - 1 + 5], np.int32)                                   # past 2^31 elements
    r32 = np.array([(1 << 32) // D + 2], np.int32)                          # past 2^32 elements
    d = rng.standard_normal((2, D)).astype(np.float32)
    before = e.gather_rows(np.zeros(3, np.int32), np.array([0, I - 2, I - 1], np.int32), np.full((3, 8), -1, np.int32))
    e.table_write_rows(g.TABLE_ITEM_EMB, r31, d[:1])
    e.table_write_rows(g.TABLE_ITEM_EMB, r32, d[1:])
    look = np.array([0, I - 2, I - 1, I, r31[0] - 1, r31[0], r31[0] + 1, r32[0] - 1, r32[0]], np.int32)
    X = e.gather_rows(np.zeros(look.size, np.int32), look, np.full((look.size, 8), -1, np.int32))
    emb = X[:, 4 + 8 * D:4 + 9 * D]
    assert emb[:3].tobytes() == before[:, 4 + 8 * D:4 + 9 * D].tobytes()     # filled rows untouched
    assert not emb[3].any() and not emb[4].any() and not emb[6].any() and not emb[7].any()
    assert emb[5].tobytes() == d[0].tobytes() and emb[8].tobytes() == d[1].tobytes()


@pytest.mark.gpu
def test_profile_keys():
    rng = np.random.default_rng(90)
    e = engine()
    ids = rng.choice(10**9, 100, replace=False).astype(np.int64)
    e.idmap_insert(ITEM, ids)
    e.table_write_rows(g.TABLE_ITEM_FEAT, np.arange(100, dtype=np.int32), rng.random((100, 7)).astype(np.float32))
    e.profile(True)
    e.profile_reset()
    e.idmap_insert(ITEM, ids[::-3])
    assert set(e.profile_dump()) == {"idmap_probe"}
    e.profile_reset()
    e.table_write_rows(g.TABLE_ITEM_FEAT, np.array([4, 99, 0], np.int32), rng.random((3, 7)).astype(np.float32))
    assert "table_grow" not in e.profile_dump() and "table_write_rows" in e.profile_dump()
    e.profile_reset()
    e.table_write_rows(g.TABLE_ITEM_FEAT, np.array([100], np.int32), rng.random((1, 7)).astype(np.float32))
    assert e.profile_dump()["table_grow"][1] == 1
    e.profile_reset()
    e.idmap_insert(ITEM, rng.choice(10**9, 200, replace=False).astype(np.int64) + 10**10)
    assert {"idmap_probe", "idmap_number", "idmap_rehash", "idmap_insert", "idmap_lookup"} <= set(e.profile_dump())
    e.profile(False)
