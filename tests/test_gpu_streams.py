"""When the engine's kernels run, not what they compute: the stream-ordering promises of include/ctr_b200.h.

  * the *_dev entry points queue their work on the engine stream and return without waiting for it;
  * ctr_set_stream adopts a caller's stream (and first drains the stream it leaves);
  * live updates and serving calls run on the engine stream: work queued before a call sees the old state, work queued
    after it the new one, whatever other streams the call uses inside (the copy stream of ctr_train_idx, the window
    stream of ctr_train_keys, the classifier's stream of the key-fed MLP calls).

The technique is a HELD stream: torch.cuda._sleep spins on the stream, then torch writes the engine's device inputs on
the same stream, then the engine calls under test are queued.  A consumer that skips a dependency then reads the
inputs' earlier contents (their bitwise complement) or a stale table every time instead of by luck of timing.  Each
case checks that its hold was still in force when the last asynchronous engine call returned, which is also the
header's promise that the *_dev calls do not block.

The reference is a twin handle of the same config and seed that makes the same calls with a ctr_sync after each one.
Windows, id lookups, search and recommendation lists and predictions from one state are compared bit for bit; anything
that went through training at the bars the suite uses for training twins (split-K weight gradients add in arbitrary
order), with the tables trained by CTR_TABLE_SGD_DETERMINISTIC.  The kernels themselves are checked against the oracle
elsewhere."""
import ctypes as C

import numpy as np
import pytest

import go_ctr_b200 as g
from oracle import oracle as orc
from tests.test_gpu_ubcache_update import windows
from tests.util import INT64_MAX, INT64_MIN, assert_mostly_close, make_batch, make_tables, scaled_init

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

NS = dict(uP=8, S=10, D=16, cF=8)
S, D = NS["S"], NS["D"]
U, I, B = 300, 2000, 128
TRAIN = dict(table_opt=g.TABLE_SGD_DETERMINISTIC, table_lr=2.0, seed=3, dropout0=0.0, dropout1=0.0)
# ~0.1 s at the H100's SM clock (not measured): far longer than queueing a handful of engine calls from Python
HOLD_CYCLES = 200_000_000


# ---- the hold ----------------------------------------------------------------------------------------------------
class Held:
    """Device buffers that hold the bitwise complement of `arrays` (1 - y for float labels) until a hold queued on
    `stream` ends; then torch, on the same stream, overwrites them with `arrays`.  `bufs` are the engine's inputs;
    `event` is recorded right after the hold."""

    def __init__(self, stream, arrays):
        dev = torch.device("cuda", 0)
        self.good = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in arrays]
        self.bufs = [(1 - x) if x.is_floating_point() else torch.bitwise_not(x) for x in self.good]
        torch.cuda._sleep(1)                                 # the sleep and copy kernels are loaded before the hold
        torch.cuda.synchronize()
        with torch.cuda.stream(stream):
            torch.cuda._sleep(HOLD_CYCLES)
            self.event = torch.cuda.Event()
            self.event.record(stream)
            for b, x in zip(self.bufs, self.good):
                b.copy_(x)

    def ptrs(self):
        return [b.data_ptr() for b in self.bufs]

    def assert_held(self):
        assert not self.event.query(), "the hold ended before the last asynchronous engine call returned: raise HOLD_CYCLES"


def out_buffer(shape, dtype):
    return torch.full(shape, -7, dtype=dtype, device="cuda")


# ---- a small world: tables, id maps, behaviour cache, batches ------------------------------------------------------
class World:
    def __init__(self, seed):
        rng = np.random.default_rng(seed)
        self.uf, self.itf, self.emb = make_tables(rng, U, I, NS["uP"], NS["cF"], D)
        self.user_ids = rng.choice(10**9, U, replace=False).astype(np.int64) + 1
        self.item_ids = rng.choice(10**9, I, replace=False).astype(np.int64) + 1
        lens = rng.integers(0, 3 * S, U)
        lens[:4] = (0, 1, S, 3 * S)
        self.off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        # time-descending, with tied runs
        self.ts = np.concatenate([np.sort(rng.integers(1, 50, l) * 1000)[::-1] for l in lens]).astype(np.int64)
        self.items = rng.integers(0, I, self.off[-1]).astype(np.int32)
        self.batches = [make_batch(rng, U, I, B, S, zipf=True) for _ in range(3)]
        ocfg = orc.make_cfg(orc.DIN_COS, NS["uP"], S, D, NS["cF"], 200, 80)
        self.W = scaled_init(orc, ocfg, seed)
        self.rng = rng

    def engine(self):
        cfg = g.engine.default_config(g.MODEL_DIN_COS, batch=B, pred_batch=B, **NS, **TRAIN)
        e = g.Engine(cfg)
        e.table_upload(g.TABLE_USER_FEAT, self.uf); e.table_upload(g.TABLE_ITEM_FEAT, self.itf); e.table_upload(g.TABLE_ITEM_EMB, self.emb)
        e.idmap_build(g.IDMAP_USER, self.user_ids); e.idmap_build(g.IDMAP_ITEM, self.item_ids)
        e.ubcache_upload(self.off, self.ts, self.items)
        e.set_weights(*self.W)
        return e

    def csr(self):
        return self.off, self.ts, self.items

    def keys(self, n, seed):
        """n sample keys: external ids of the batches' users and items, timestamps inside the cache's range"""
        ur, ir, y = (np.concatenate([b[k] for b in self.batches]) for k in (0, 1, 3))
        return self.user_ids[ur[:n]], self.item_ids[ir[:n]], np.random.default_rng(seed).integers(0, 60_000, n).astype(np.int64), y[:n]


def table(e):
    return e.table_download(g.TABLE_ITEM_EMB, I, D)


def assert_trained_close(got, want, what):
    """the bars of the suite's training twins: dense weights mostly close, ITEM_EMB at rtol 1e-4"""
    if what == "table":
        np.testing.assert_allclose(got, want, rtol=1e-4, atol=1e-6)
    else:
        for a, b in zip(got, want):
            assert_mostly_close(a, b, 1e-3, 1e-5, 0.999, what)


def assert_far(a, b, what, rtol=1e-3, atol=1e-5):
    """a stale read would land here: some element differs from b by more than ten times the bar (by default ITEM_EMB's)"""
    assert not np.allclose(np.asarray(a, np.float64), np.asarray(b, np.float64), rtol=rtol, atol=atol), what + " did not move"


def window_probes(w, rng, n):
    """(user row, maxTs) pairs: cached users at tied-run timestamps +-1, maxTs 0 and the int64 extremes; users past the
    cache"""
    rows, mts = [], []
    while len(rows) < n:
        u = int(rng.integers(0, U + 8))
        seg = w.ts[w.off[u]:w.off[u + 1]] if u < U else np.zeros(0, np.int64)
        t = int(rng.choice(seg)) + int(rng.integers(-1, 2)) if seg.size and rng.random() < 0.6 else \
            int(rng.choice([0, INT64_MIN, INT64_MAX, 5]))
        rows.append(u); mts.append(t)
    return np.array(rows, np.int32), np.array(mts, np.int64)


def lookup_probes(w, rng, n):
    """known ids, unknown ones, 0, -1 and the int64 extremes (INT64_MIN is the empty-slot marker)"""
    known = set(w.user_ids.tolist())
    odd = [v for v in (0, -1, INT64_MIN, INT64_MAX, INT64_MAX - 1) if v not in known]
    ids = np.where(rng.random(n) < 0.7, rng.choice(w.user_ids, n), rng.integers(-10**12, 10**12, n)).astype(np.int64)
    ids[:len(odd)] = odd
    return ids


def lookup_dict(ids, table_ids):
    row = {int(v): r for r, v in enumerate(table_ids)}
    return np.array([row.get(int(v), -1) for v in ids], np.int32)


# ---- adoption ----------------------------------------------------------------------------------------------------
def test_an_adopted_caller_stream_orders_the_engine_after_the_caller():
    """ctr_set_stream adopts a torch stream: the engine's work follows torch's on it, ctr_get_stream returns it, leaving
    a held stream for another waits for the held work (nothing is lost), ctr_destroy leaves the caller's stream usable,
    and the legacy default stream (0) can be adopted too."""
    w = World(11)
    eng, ref = w.engine(), w.engine()
    bs = w.batches
    ref_costs = [ref.train_step_idx(*b).cost for b in bs[:2]]

    s1 = torch.cuda.Stream()
    eng.set_stream(s1.cuda_stream)
    assert eng.stream == s1.cuda_stream
    held = Held(s1, [a for b in bs[:2] for a in b])
    p = held.ptrs()
    eng.train_step_idx_dev(*p[0:4], B)
    eng.train_step_idx_dev(*p[4:8], B)
    held.assert_held()
    s2 = torch.cuda.Stream()
    eng.set_stream(s2.cuda_stream)                       # drains s1 first
    assert held.event.query() and s1.query()
    assert eng.stream == s2.cuda_stream
    assert abs(eng.last_cost() - ref_costs[1]) <= 1e-5 * max(1.0, abs(ref_costs[1]))

    want = ref.predict_idx(*bs[2][:3])          # (every kernel the held calls launch is loaded before a hold)
    out = out_buffer((B,), torch.float32)
    held2 = Held(s2, bs[2][:3])
    eng.predict_idx_dev(*held2.ptrs(), B, out.data_ptr())
    held2.assert_held()
    eng.sync()
    got = out.cpu().numpy()
    assert got.tobytes() == eng.predict_idx(*bs[2][:3]).tobytes()      # the same state
    assert_mostly_close(got, want, 2e-3, 1e-5, 0.99, "predictions")
    assert_trained_close(table(eng), table(ref), "table")
    assert_trained_close(eng.get_weights(), ref.get_weights(), "dense weights")
    assert_far(table(ref), w.emb, "ITEM_EMB")

    eng.close()
    with torch.cuda.stream(s2):                         # the caller's stream outlives the handle
        x = torch.arange(1000, device="cuda", dtype=torch.int64).sum()
    s2.synchronize()
    assert int(x) == 999 * 1000 // 2

    e0 = w.engine()
    e0.set_stream(0)
    assert e0.stream is None                             # ctr_get_stream returns the adopted NULL stream
    c0 = [e0.train_step_idx(*b).cost for b in bs[:2]]
    np.testing.assert_allclose(c0, ref_costs, rtol=1e-5)
    assert_mostly_close(e0.predict_idx(*bs[2][:3]), ref.predict_idx(*bs[2][:3]), 2e-3, 1e-5, 0.99, "predictions")
    assert_trained_close(table(e0), table(ref), "table")


# ---- *_dev inputs torch wrote behind the hold ---------------------------------------------------------------------
def test_dev_entry_points_read_what_torch_wrote_behind_a_hold():
    """On the engine's own stream (torch.cuda.ExternalStream): three train steps, a predict, a behaviour window and an
    id lookup whose inputs torch writes behind a hold equal the host entry points on the twin, and the two wrappers of
    device pointers equal orc.ub_filter and a dict at B past Bmax and not a multiple of 8 warps, users past the cache,
    unknown ids and maxTs at 0 and the int64 extremes."""
    w = World(12)
    eng, ref = w.engine(), w.engine()
    rng = np.random.default_rng(5)
    bs = w.batches
    NW, NL = B + 13, 1001
    wr, wt = window_probes(w, rng, NW)
    ids = lookup_probes(w, rng, NL)

    # the twin first, so every kernel the held calls launch is loaded before the hold
    ref_costs = [ref.train_step_idx(*b).cost for b in bs]
    ref_pred, ref_hist, ref_rows = ref.predict_idx(*bs[0][:3]), ref.ubcache_window(wr, wt), ref.idmap_lookup(g.IDMAP_USER, ids)

    es = torch.cuda.ExternalStream(eng.stream)
    out = out_buffer((B,), torch.float32)
    hist = out_buffer((NW, S), torch.int32)
    rows = out_buffer((NL,), torch.int32)
    held = Held(es, [a for b in bs for a in b] + list(bs[0][:3]) + [wr, wt, ids])
    p = held.ptrs()
    for k in range(3):
        eng.train_step_idx_dev(*p[4 * k:4 * k + 4], B)
    eng.predict_idx_dev(*p[12:15], B, out.data_ptr())
    eng.ubcache_window_dev(p[15], p[16], NW, hist.data_ptr())
    eng.idmap_lookup_dev(g.IDMAP_USER, p[17], NL, rows.data_ptr())
    held.assert_held()
    eng.sync()

    assert abs(eng.last_cost() - ref_costs[2]) <= 1e-5 * max(1.0, abs(ref_costs[2]))
    assert_trained_close(table(eng), table(ref), "table")
    assert_trained_close(eng.get_weights(), ref.get_weights(), "dense weights")
    assert_far(table(ref), w.emb, "ITEM_EMB")
    got = out.cpu().numpy()
    assert got.tobytes() == eng.predict_idx(*bs[0][:3]).tobytes()      # the same state
    assert_mostly_close(got, ref_pred, 2e-3, 1e-5, 0.99, "predictions")

    want_hist = windows(w.csr(), wr, wt, S)
    assert (want_hist >= 0).any() and (want_hist < 0).any()
    np.testing.assert_array_equal(hist.cpu().numpy(), want_hist)
    np.testing.assert_array_equal(ref_hist, want_hist)
    want_rows = lookup_dict(ids, w.user_ids)
    assert (want_rows >= 0).any() and (want_rows < 0).any()
    np.testing.assert_array_equal(rows.cpu().numpy(), want_rows)
    np.testing.assert_array_equal(ref_rows, want_rows)


# ---- host calls after held asynchronous work --------------------------------------------------------------------
def _mlp(w):
    """a key-fed classifier with random parameters over the world's feature store"""
    m = g.MLPClassifier(NS["uP"] + S * D + D + NS["cF"], hidden=(16,), max_iter=3, seed=0)
    n = m.get_params().size
    m.set_params(np.random.default_rng(9).standard_normal(n) * 0.2)
    return m


def _pure_calls(w):
    """calls that change nothing: name → f(engine) returning arrays"""
    bs = w.batches
    q = np.unique(bs[0][1])[:16]                             # ITEM_EMB rows the steps train
    users, hist = bs[0][0][:8], bs[0][2][:8]
    ku, ki, kt, _ = w.keys(300, 2)
    m = _mlp(w)
    return {
        "table_download": lambda e: [table(e)],
        "get_weights": lambda e: list(e.get_weights()),
        "knn_search": lambda e: list(e.knn_search(10, rows=q)),
        "recommend_topk": lambda e: list(e.recommend_topk(users, hist, 10)),
        "batch_predict_keys": lambda e: [e.batch_predict_keys(ku, ki, kt)],
        "predict_idx": lambda e: [e.predict_idx(*bs[2][:3])],
        "mlp_predict_keys": lambda e: [m.predict_keys(e, ku, ki, kt)],
        "mlp_recommend_topk": lambda e: list(m.recommend_topk(e, ku[:4], kt[:4], 10)),
    }


# which outputs of a pure call are lists (compared as sorted values against the twin) and which are values
_LISTS = {"knn_search": (1,), "recommend_topk": (1, 2), "mlp_recommend_topk": (1, 2)}

CALLS = ["table_download", "get_weights", "knn_search", "recommend_topk", "batch_predict_keys", "predict_idx",
         "mlp_predict_keys", "mlp_recommend_topk", "table_write_rows", "checkpoint_save", "train_idx", "train_keys",
         "ubcache_append", "idmap_insert"]


def _held_steps(w, eng, extra=()):
    """two train steps with table SGD on the engine stream, their inputs written by torch behind a hold"""
    es = torch.cuda.ExternalStream(eng.stream)
    held = Held(es, [a for b in w.batches[:2] for a in b] + list(extra))
    p = held.ptrs()
    eng.train_step_idx_dev(*p[0:4], B)
    eng.train_step_idx_dev(*p[4:8], B)
    return held, p[8:]


@pytest.mark.parametrize("call", CALLS)
def test_a_host_call_after_held_dev_steps_sees_them(call, tmp_path):
    """Train steps queued by *_dev calls behind a hold change ITEM_EMB rows and the dense weights; the host call made
    right after them (before the hold ends) must see the trained state, as the twin that synchronised after every call
    does.  A call that changes nothing also equals itself repeated once the handle is idle, bit for bit, and differs
    from its answer before the steps.  A window or id lookup queued before an append / insert returns the old state, one
    queued after it the new state."""
    w = World(13)
    eng, ref = w.engine(), w.engine()
    rng = np.random.default_rng(17)
    pure = _pure_calls(w) if call in CALLS[:8] else {}
    stale = pure[call](ref) if pure else None
    for b in w.batches[:2]:
        ref.train_step_idx(*b)
    ref_table, ref_w = table(ref), ref.get_weights()
    assert_far(ref_table, w.emb, "ITEM_EMB")                  # what a call that missed the steps would see
    assert_far(ref_w[0], w.W[0], "mlp0", 1e-2, 1e-4)

    if pure:
        held, _ = _held_steps(w, eng)
        held.assert_held()
        got = pure[call](eng)
        eng.sync()
        again = pure[call](eng)
        want = pure[call](ref)
        for k, (a, b) in enumerate(zip(got, again)):
            assert a.tobytes() == b.tobytes(), "%s output %d differs from the idle repeat" % (call, k)
        if call == "table_download":
            assert_trained_close(got[0], want[0], "table")
        elif call == "get_weights":
            assert_trained_close(got, want, "dense weights")
        else:
            for k in _LISTS.get(call, (0,)):
                a, b = (np.sort(x, axis=-1) for x in (got[k], want[k])) if call in _LISTS else (got[k], want[k])
                assert_mostly_close(a, b, 2e-3, 1e-5, 0.99, call)
        # the twin's answer before its steps is, bit for bit, what a call that missed the held steps would return
        assert any(a.tobytes() != b.tobytes() for a, b in zip(again, stale)), "%s does not see the steps" % call
        return

    if call == "table_write_rows":
        rows = np.unique(w.batches[0][1])[:8]
        data = rng.standard_normal((rows.size, D)).astype(np.float32)
        held, _ = _held_steps(w, eng)
        held.assert_held()
        eng.table_write_rows(g.TABLE_ITEM_EMB, rows, data)
        ref.table_write_rows(g.TABLE_ITEM_EMB, rows, data)
        got = table(eng)
        assert got[rows].tobytes() == data.tobytes()          # written after the steps' updates, not under them
        assert_far(ref_table[rows], w.emb[rows], "the written rows")
        assert_trained_close(got, table(ref), "table")
    elif call == "checkpoint_save":
        held, _ = _held_steps(w, eng)
        held.assert_held()
        path = str(tmp_path / "held.ckpt")
        eng.checkpoint_save(path)
        eng.sync()
        back = w.engine()
        back.checkpoint_load(path)
        assert table(back).tobytes() == table(eng).tobytes()
        for a, b in zip(back.get_weights(), eng.get_weights()):
            assert a.tobytes() == b.tobytes()
        assert_trained_close(table(back), ref_table, "table")
        assert_trained_close(back.get_weights(), ref_w, "dense weights")
    elif call in ("train_idx", "train_keys"):
        ur, ir, hist, y = w.batches[2]
        n = B + 37
        held, _ = _held_steps(w, eng)
        held.assert_held()
        if call == "train_idx":
            got, want = eng.train_idx(ur[:n], ir[:n], hist[:n], y[:n]), ref.train_idx(ur[:n], ir[:n], hist[:n], y[:n])
        else:
            keys = w.keys(n, 3)
            got, want = eng.train_keys(*keys)[1], ref.train_keys(*keys)[1]
        np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-6)
        assert_trained_close(table(eng), table(ref), "table")
        assert_trained_close(eng.get_weights(), ref.get_weights(), "dense weights")
    elif call == "ubcache_append":
        urows = np.array([0, 1, 2, 3, 3, 7, U - 1], np.int32)              # an empty user, a tie with a stored event
        ats = np.array([10**6, w.ts[w.off[1]], 5, 10**6, 10**6, 1, 3], np.int64)
        aitems = np.array([1, 2, 3, 4, 5, 6, 7], np.int32)
        pu = np.concatenate([urows, [U + 4]]).astype(np.int32)               # and a user past the cache
        pr = np.repeat(pu, 4); pt = np.tile(np.array([0, INT64_MAX, 10**6 - 1, 5], np.int64), pu.size)
        want_before = windows(w.csr(), pr, pt, S)
        np.testing.assert_array_equal(ref.ubcache_window(pr, pt), want_before)
        before, after = out_buffer((pr.size, S), torch.int32), out_buffer((pr.size, S), torch.int32)
        held, (d_u, d_t) = _held_steps(w, eng, [pr, pt])
        eng.ubcache_window_dev(d_u, d_t, pr.size, before.data_ptr())
        held.assert_held()
        eng.ubcache_append(urows, ats, aitems)
        eng.ubcache_window_dev(d_u, d_t, pr.size, after.data_ptr())
        eng.sync()
        ref.ubcache_append(urows, ats, aitems)
        ref.sync()
        new_csr = ref.ubcache_download()
        want_after = windows(new_csr, pr, pt, S)
        assert not np.array_equal(want_before, want_after)
        np.testing.assert_array_equal(before.cpu().numpy(), want_before)
        np.testing.assert_array_equal(after.cpu().numpy(), want_after)
        np.testing.assert_array_equal(ref.ubcache_window(pr, pt), want_after)
        for a, b in zip(eng.ubcache_download(), new_csr):
            np.testing.assert_array_equal(a, b)
        assert_trained_close(table(eng), ref_table, "table")
    elif call == "idmap_insert":
        # 300 ids in a map of 1024 slots; 300 more (some twice, some known) outgrow it: the insert rehashes into 2048
        fresh = rng.choice(10**9, 400, replace=False).astype(np.int64) + 2 * 10**9
        new = np.concatenate([fresh[:300], fresh[:20], w.user_ids[:10]])
        rng.shuffle(new)
        probe = np.concatenate([w.user_ids[:50], fresh, [0, INT64_MIN, INT64_MAX]]).astype(np.int64)
        np.testing.assert_array_equal(ref.idmap_lookup(g.IDMAP_USER, probe), lookup_dict(probe, w.user_ids))
        before, after = out_buffer((probe.size,), torch.int32), out_buffer((probe.size,), torch.int32)
        held, (d_ids,) = _held_steps(w, eng, [probe])
        eng.idmap_lookup_dev(g.IDMAP_USER, d_ids, probe.size, before.data_ptr())
        held.assert_held()
        got_rows = eng.idmap_insert(g.IDMAP_USER, new)
        eng.idmap_lookup_dev(g.IDMAP_USER, d_ids, probe.size, after.data_ptr())
        eng.sync()
        _, first = np.unique(new[~np.isin(new, w.user_ids)], return_index=True)
        order = new[~np.isin(new, w.user_ids)][np.sort(first)]
        grown = np.concatenate([w.user_ids, order])
        assert grown.size == U + 300
        np.testing.assert_array_equal(got_rows, lookup_dict(new, grown))
        np.testing.assert_array_equal(ref.idmap_insert(g.IDMAP_USER, new), got_rows)
        np.testing.assert_array_equal(before.cpu().numpy(), lookup_dict(probe, w.user_ids))
        np.testing.assert_array_equal(after.cpu().numpy(), lookup_dict(probe, grown))
        np.testing.assert_array_equal(eng.idmap_download(g.IDMAP_USER), grown)
        assert_trained_close(table(eng), ref_table, "table")
    else:
        raise AssertionError(call)


# ---- a live cache rewrite still running when ctr_train_keys starts --------------------------------------------------
RU, RL, RI = 100_000, 3000, 256          # 3·10^8 cached events: the rewrite's stored-event move takes milliseconds
RN = RU * RL
LAST = np.arange(RU - 8, RU, dtype=np.int32)      # the users whose events go in at the end of the CSR
FRESH = np.arange(RI - 8, RI, dtype=np.int32)     # ITEM_EMB rows named only by the timed append


def _cache_counts(e):
    nu, n = C.c_int64(0), C.c_int64(0)
    e._ck(e.L.ctr_ubcache_download(e.h, None, None, None, C.c_int64(0), C.c_int64(0), C.byref(nu), C.byref(n)))
    return nu.value, n.value


def test_train_keys_windows_follow_a_pending_cache_rewrite():
    """ctr_ubcache_append returns with its rewrite of the CSR still queued on the engine stream.  ctr_train_keys cuts its
    history windows on a stream of its own, so its first windows must wait for that rewrite.

    The cache holds 3·10^8 events (even timestamps, items among rows [0, 64)).  Two warm-up appends of the same shape
    (one event for each of the last 8 users, odd timestamps) make the spare CSR a complete earlier cache whose capacity
    (the rewrite keeps 1/8 slack) already covers the timed append, so the timed append reallocates nothing and a window
    that ran too early would read a stale but in-bounds CSR.  The timed append gives each of those users its newest
    event, on an ITEM_EMB row no other event or sample names.  train_keys is called on samples of those users while the
    rewrite is still pending, with CTR_TABLE_SGD_DETERMINISTIC: the fresh rows change if and only if the first batches'
    windows held the new events."""
    rng = np.random.default_rng(23)
    off = np.arange(RU + 1, dtype=np.int64) * RL
    ts = np.tile(2 * np.arange(RL, 0, -1, dtype=np.int64), RU)
    items = np.tile((np.arange(RL) % 64).astype(np.int32), RU)
    uf, itf, emb = make_tables(rng, RU, RI, NS["uP"], NS["cF"], D)
    user_ids = np.arange(RU, dtype=np.int64) * 7 + 11
    item_ids = np.arange(RI, dtype=np.int64) * 5 + 3
    ocfg = orc.make_cfg(orc.DIN_COS, NS["uP"], S, D, NS["cF"], 200, 80)
    W = scaled_init(orc, ocfg, 4)
    warm = [(LAST, np.full(8, 2 * (RL // 2) + 1 + 2 * k, np.int64), rng.integers(0, 64, 8).astype(np.int32)) for k in range(2)]
    timed = (LAST, np.full(8, 2 * RL + 11, np.int64), FRESH)
    n = 2 * B + 40
    su = rng.choice(LAST, n).astype(np.int32)
    k_user, k_item = user_ids[su], item_ids[rng.integers(64, 128, n)]
    k_ts = np.full(n, 10**7, np.int64)
    y = (rng.random(n) < 0.5).astype(np.float32)
    # the spare after the warm-ups is the first warm-up's output, allocated for RN + 8 events with 1/8 slack
    assert RN + 24 <= (RN + 8) + (RN + 8) // 8

    engs = []
    for synced in (False, True):
        cfg = g.engine.default_config(g.MODEL_DIN_COS, batch=B, pred_batch=B, **NS, **TRAIN)
        e = g.Engine(cfg)
        e.table_upload(g.TABLE_USER_FEAT, uf); e.table_upload(g.TABLE_ITEM_FEAT, itf); e.table_upload(g.TABLE_ITEM_EMB, emb)
        e.idmap_build(g.IDMAP_USER, user_ids); e.idmap_build(g.IDMAP_ITEM, item_ids)
        e.set_weights(*W)
        e.ubcache_upload(off, ts, items)
        assert _cache_counts(e) == (RU, RN)
        for k, a in enumerate(warm):
            e.ubcache_append(*a)
            e.sync()
            assert _cache_counts(e) == (RU, RN + 8 * (k + 1))
        engs.append(e)
    eng, ref = engs
    del ts, items

    eng.ubcache_append(*timed)
    pending = torch.cuda.Event()
    pending.record(torch.cuda.ExternalStream(eng.stream))
    still_running = not pending.query()
    _, cost, used = eng.train_keys(k_user, k_item, k_ts, y)
    assert still_running, "the rewrite had finished before ctr_train_keys started: raise the cache size"
    ref.ubcache_append(*timed)
    ref.sync()
    _, ref_cost, ref_used = ref.train_keys(k_user, k_item, k_ts, y)
    assert used == ref_used == n
    assert _cache_counts(eng) == (RU, RN + 24)

    got, want = eng.table_download(g.TABLE_ITEM_EMB, RI, D), ref.table_download(g.TABLE_ITEM_EMB, RI, D)
    assert (got[FRESH] != emb[FRESH]).any(axis=1).all(), "a fresh row did not train: its event was missing from the windows"
    np.testing.assert_allclose(got, want, rtol=1e-4, atol=1e-6)
    assert abs(cost - ref_cost) <= 1e-5 * max(1.0, abs(ref_cost))
    assert_trained_close(eng.get_weights(), ref.get_weights(), "dense weights")

    # the windows of those samples, against the oracle over the users' whole sequences
    seqs = {}
    for j, u in enumerate(LAST):                        # no timestamp ties: stored ones are even, appended ones odd
        seq_ts = np.concatenate([2 * np.arange(RL, 0, -1, dtype=np.int64), [a[1][j] for a in warm + [timed]]])
        seq_it = np.concatenate([(np.arange(RL) % 64).astype(np.int32), [a[2][j] for a in warm + [timed]]]).astype(np.int32)
        order = np.argsort(-seq_ts, kind="stable")
        seqs[int(u)] = (seq_ts[order], seq_it[order])
    want_hist = np.full((n, S), -1, np.int32)
    for b, u in enumerate(su):
        sts, sit = seqs[int(u)]
        start, cnt = orc.ub_filter(sts, int(k_ts[b]), S)
        want_hist[b, :cnt] = sit[start:start + cnt]
    assert (want_hist[:, 0] == FRESH[su - (RU - 8)]).all()
    np.testing.assert_array_equal(eng.ubcache_window(su, k_ts), want_hist)
