"""The key-fed sample path and the device AUC at their edges, against plain restatements: dicts, numpy, orc.ub_filter
and orc.IdxTrainer — never another engine entry point that shares the kernel under test.

  * id maps (idmap.cuh): ids built to collide — a cluster whose chain wraps past the last slot, ids that run into it,
    misses whose probe starts inside it — at the smallest capacities and at 1e5 ids, and a rebuild; each through
    ctr_idmap_lookup (k_idmap_lookup), ctr_batch_predict_keys (k_keys_resolve) and ctr_train_keys (k_keys_rows,
    k_keys_compact), the last three probing with their own copy of the loop (idmap_find);
  * behaviour windows (ubcache.cuh): histories up to 5000 events with long runs of one timestamp across the
    binary-search midpoints of ub_first_leq, every S around the 32-lane ballot, grid-capped batches;
  * serving over keys at S = 50: several pred_batch chunks, unknown keys opening a later chunk, rows past the ubcache;
  * key-fed training against the oracle: the streaming first epoch's chunk boundaries, empty chunks, epochs 0,
    early stop, a failed call and a second call on one handle;
  * the AUC exactly: integer trapezoid sums, so the engine's one division must give the same double."""
import numpy as np
import pytest

import go_ctr_b200 as g
from oracle import oracle as orc
from tests.util import (INT64_MAX, INT64_MIN, assert_mostly_close, idmap_capacity, ids_probing_from, make_tables,
                        scaled_init)

pytestmark = pytest.mark.gpu

INT32_MAX, INT32_MIN = 2**31 - 1, -2**31


# ---- shared restatements ---------------------------------------------------------------------------------------
def tied_histories(rng, U, max_len, n_items):
    """Per-user behaviour CSR, timestamps descending (TimeSeq).  Events come in runs of one timestamp, as MovieLens
    users rate many items in the same second; runs are laid over the first binary-search midpoints (L/2, L/4, 3L/4,
    ...).  Lengths reach max_len, users in the middle of the CSR are empty (repeated offsets), one user's events all
    share one timestamp and one user's timestamps are negative."""
    lens = np.where(rng.random(U) < 0.3, rng.integers(0, 40, U), rng.integers(0, max_len + 1, U))
    lens[1], lens[2], lens[3], lens[4], lens[5] = max_len, 33, 32, 1, max_len // 2
    lens[U // 2:U // 2 + 4] = 0
    segs = []
    for u, L in enumerate(lens):
        runs = rng.choice([1, 1, 1, 2, 3, 8, 40, 150], size=L)
        run_of = np.repeat(np.arange(L), runs)[:L]
        t = 2_000_000 - np.cumsum(rng.integers(1, 4, L)).astype(np.int64)[run_of]
        for q in (2, 4, 8):
            for c in range(1, q, 2):
                a = max(0, c * L // q - L // 32 - 2)
                t[a:c * L // q + L // 32 + 2] = t[a:a + 1]
        if u == 5:
            t[:] = 777
        if u == 6:
            t -= 3_000_000
        assert (np.diff(t) <= 0).all()
        segs.append(t)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    return off, np.concatenate(segs).astype(np.int64), rng.integers(0, n_items, off[-1]).astype(np.int32)


def probe_times(rng, ub, rows):
    """max_ts per sample: an event's timestamp (so a run boundary) or one either side of it, 0 ("from the newest"),
    negative, and the int64 extremes."""
    off, ts, _ = ub
    r = np.clip(rows, 0, off.size - 2)
    L = off[r + 1] - off[r]
    e = np.minimum(off[r] + (rng.random(r.size) * np.maximum(L, 1)).astype(np.int64), ts.size - 1)
    t = np.where(L > 0, ts[e], 5) + rng.integers(-1, 2, r.size)
    kind = rng.random(r.size)
    t[kind < 0.08] = 0
    t[(kind >= 0.08) & (kind < 0.12)] = -3
    t[(kind >= 0.12) & (kind < 0.14)] = INT64_MAX
    t[(kind >= 0.14) & (kind < 0.16)] = INT64_MIN
    return t.astype(np.int64)


def windows(ub, user_row, max_ts, S):
    """TimeSeq.Filter(max_ts, S) per sample through the oracle, -1 padded; a row outside [0, n_users) is empty."""
    off, ts, items = ub
    out = np.full((len(user_row), S), -1, np.int32)
    for b, (u, t) in enumerate(zip(user_row, max_ts)):
        if 0 <= u < off.size - 1 and off[u + 1] > off[u]:
            start, cnt = orc.ub_filter(ts[off[u]:off[u + 1]], int(t), S)
            out[b, :cnt] = items[off[u] + start: off[u] + start + cnt]
    return out


def _expected_scores(ocfg, W, tabs, ids, ub, keys, with_ub=True):
    """rcmd.go:277-337 + 462-536 restated with dicts: rows (or a zero row), history window, oracle forward.
    A user whose row is at or past the uploaded ubcache's user count has an empty history."""
    uf, itf, emb = tabs; uid, iid = ids
    umap = {int(v): r for r, v in enumerate(uid)}; imap = {int(v): r for r, v in enumerate(iid)}
    S = ocfg.S
    n = len(keys)
    ur = np.full(n, -1, np.int32); ir = np.full(n, -1, np.int32); hist = np.full((n, S), -1, np.int32)
    for k, (u, i, t) in enumerate(keys):
        r, c = umap.get(int(u), -1), imap.get(int(i), -1)
        if r < 0 or c < 0:
            continue                                         # GetSampleVector error → zero X row (rcmd.go:299-307)
        ur[k], ir[k] = r, c
        if with_ub:
            hist[k] = windows(ub, [r], [t], S)[0]
    X = orc.gather_rows(uf, itf, emb, ur, ir, hist)
    p, _ = orc.forward(ocfg, W, X, orc.make_ranges(ocfg.uP, ocfg.S, ocfg.D, ocfg.cF))
    return p, X


def _engine(model, dims, B, tabs, W, **kw):
    uP, S, D, cF = dims
    eng = g.Engine(g.engine.default_config(model, uP=uP, S=S, D=D, cF=cF, batch=B, pred_batch=kw.pop("pred_batch", B), **kw))
    for w, t in zip((g.TABLE_USER_FEAT, g.TABLE_ITEM_FEAT, g.TABLE_ITEM_EMB), tabs):
        eng.table_upload(w, t)
    eng.set_weights(*W)
    return eng


# ---- 1. id maps with constructed collisions --------------------------------------------------------------------
def collision_ids(rng, n, cap, at):
    """n distinct ids for a map of cap slots and misses that probe through them.  Up to a third (at most 2000) start at
    slot `at` — with at = cap - 1 their chain wraps through slot 0 — as many start at the slots right after it and run
    into that chain; 0, -1 and INT64_MAX are members when n allows, the rest are random.  Misses start inside the
    cluster, at its first and last slot, and just past it."""
    k = min(n // 3, 2000)
    after = (at + 1 + np.arange(k)) % cap
    special = [0, -1, INT64_MAX] if n >= 8 else []
    built = ids_probing_from(rng, np.concatenate([np.full(max(k, 1), at), after]), cap, avoid=special)[:max(k, 1) + k]
    n_rand = n - built.size - len(special)
    rand = rng.integers(INT64_MIN + 1, INT64_MAX, n_rand + 64, dtype=np.int64)
    rand = rng.permutation(np.setdiff1d(rand, np.concatenate([built, special])))[:n_rand]
    ids = np.concatenate([built, np.array(special, np.int64), rand])       # row r is ids[r]: the colliding ids first
    assert ids.size == n and np.unique(ids).size == n
    miss_slots = np.concatenate([[at, at, (at + 1) % cap], after[k // 2:k // 2 + 3], (at + 2 * k + np.arange(3)) % cap])
    miss = ids_probing_from(rng, miss_slots, cap, avoid=np.concatenate([ids, [0, -1, INT64_MAX]]))
    return ids, miss


@pytest.mark.parametrize("n", [1, 32, 33, 64, 100_000])
def test_idmap_collision_chains_through_every_probe(n):
    """Every case against a dict, three ways: ctr_idmap_lookup, ctr_batch_predict_keys (unknown → zero row) and
    ctr_train_keys (rows_used); then a rebuild of the user map with other ids, after which the old ids are unknown."""
    rng = np.random.default_rng(n)
    cap = idmap_capacity(n)
    uid, umiss = collision_ids(rng, n, cap, cap - 1)
    iid, imiss = collision_ids(rng, n, cap, cap - 1)
    dims = uP, S, D, cF = 4, 3, 16, 4
    tabs = make_tables(rng, n, n, uP, cF, D)
    ocfg = orc.make_cfg(g.MODEL_DIN_COS, uP, S, D, cF, 200, 80)
    W = scaled_init(orc, ocfg, 3)
    eng = _engine(g.MODEL_DIN_COS, dims, 256, tabs, W)
    eng.idmap_build(g.IDMAP_USER, uid); eng.idmap_build(g.IDMAP_ITEM, iid)

    edge = [0, -1, INT64_MAX, INT64_MIN, 1, INT64_MIN + 1]
    for which, ids, miss in ((g.IDMAP_USER, uid, umiss), (g.IDMAP_ITEM, iid, imiss)):
        want = {int(v): r for r, v in enumerate(ids)}
        q = rng.permutation(np.concatenate([ids, ids[rng.integers(0, n, 200)], miss, edge]))
        assert eng.idmap_lookup(which, q).tolist() == [want.get(int(v), -1) for v in q]

    def pool(ids, miss):                 # every colliding id and every miss, a sample of the rest, the edge ids
        return np.concatenate([ids[:4100], ids[rng.integers(0, n, 500)], miss, edge])

    # the call's first key must resolve; the rest mix members, misses and the edge ids on both sides
    m = max(pool(uid, umiss).size, pool(iid, imiss).size)
    ku = np.concatenate([uid[:1], rng.permutation(np.resize(pool(uid, umiss), m))])
    ki = np.concatenate([iid[:1], rng.permutation(np.resize(pool(iid, imiss), m))])
    kt = np.zeros(ku.size, np.int64)
    want, X = _expected_scores(ocfg, W, tabs, (uid, iid), None, list(zip(ku, ki, kt)), with_ub=False)
    got = eng.batch_predict_keys(ku, ki, kt)
    np.testing.assert_allclose(got, want, rtol=1e-4, atol=1e-7)
    umap = {int(v) for v in uid}; imap = {int(v) for v in iid}
    known = np.array([int(u) in umap and int(i) in imap for u, i in zip(ku, ki)])
    assert not known.all() and not X[~known].any()
    y = (rng.random(ku.size) > 0.5).astype(np.float32)
    assert eng.train_keys(ku, ki, kt, y, epochs=1)[2] == int(known.sum())
    # rebuild the user map with new ids whose cluster sits elsewhere: the old ids must all be gone
    uid2, _ = collision_ids(np.random.default_rng(n + 1), n, cap, cap // 2)
    eng.idmap_build(g.IDMAP_USER, uid2)
    want2 = {int(v): r for r, v in enumerate(uid2)}
    q = rng.permutation(np.concatenate([uid, uid2, umiss]))
    assert eng.idmap_lookup(g.IDMAP_USER, q).tolist() == [want2.get(int(v), -1) for v in q]
    ku2 = np.where(rng.random(ku.size) < 0.5, ku, uid2[rng.integers(0, n, ku.size)])
    known2 = np.array([int(u) in want2 and int(i) in imap for u, i in zip(ku2, ki)])
    if known2.any():
        assert eng.train_keys(ku2, ki, kt, y, epochs=1)[2] == int(known2.sum())
    else:
        with pytest.raises(g.CtrError) as e:
            eng.train_keys(ku2, ki, kt, y, epochs=1)
        assert e.value.code == g.ENOTFOUND


# ---- 2. behaviour windows ---------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def long_ub():
    rng = np.random.default_rng(77)
    return tied_histories(rng, 300, 5000, 1 << 30)


@pytest.mark.parametrize("S", [1, 31, 32, 33, 50, 100])
def test_ubcache_window_over_long_tied_histories(long_ub, S):
    """ctr_ubcache_window == orc.ub_filter row for row.  B = 30 000 samples is more than the capped grid has warps
    (num_sms * 64), so each warp windows several samples."""
    off, ts, items = long_ub
    n_users = off.size - 1
    eng = g.Engine(g.engine.default_config(g.MODEL_DIN_COS, S=S, batch=8, pred_batch=8))
    eng.ubcache_upload(off, ts, items)
    rng = np.random.default_rng(S)
    B = 30_000
    rows = rng.integers(0, n_users, B).astype(np.int64)
    rows[:n_users] = np.arange(n_users)                                     # every user, the empty ones included
    bad = rng.random(B) < 0.02
    rows[bad] = rng.choice([-1, -7, n_users, n_users + 5, INT32_MAX, INT32_MIN], int(bad.sum()))
    max_ts = probe_times(rng, long_ub, rows)
    got = eng.ubcache_window(rows.astype(np.int32), max_ts)
    want = windows(long_ub, rows, max_ts, S)
    bad_rows = np.flatnonzero((got != want).any(1))
    assert bad_rows.size == 0, [(int(b), int(rows[b]), int(max_ts[b])) for b in bad_rows[:5]]
    assert np.diff(off).max() >= 4000 and (want >= 0).sum(1).max() == S   # long searches ran, full windows were cut


# ---- 3. serving over keys ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", [g.MODEL_DIN_COS, g.MODEL_DIN_EUC, g.MODEL_YOUTUBE], ids=["din_cos", "din_euc", "youtube"])
def test_batch_predict_keys_over_chunks_and_long_histories(model):
    """S = 50 over long tied histories; n spans four pred_batch chunks and a ragged one.  Users whose row is in the id
    map but at or past the ubcache's user count get an empty history.  An unknown key opening a later chunk scores as
    a zero row; an unknown first key of the call fails it with CTR_ENOTFOUND."""
    rng = np.random.default_rng(11 + model)
    U, I, PB = 200, 300, 64
    dims = uP, S, D, cF = 9, 50, 16, 7
    tabs = make_tables(rng, U, I, uP, cF, D)
    ocfg = orc.make_cfg(model, uP, S, D, cF, 200, 80)
    W = scaled_init(orc, ocfg, 5)
    eng = _engine(model, dims, PB, tabs, W)
    uid = rng.choice(10_000_000, U, replace=False).astype(np.int64) + 1
    iid = rng.choice(10_000_000, I, replace=False).astype(np.int64) + 1
    eng.idmap_build(g.IDMAP_USER, uid); eng.idmap_build(g.IDMAP_ITEM, iid)
    ub = tied_histories(rng, U - 20, 2000, I)                               # rows U-20 .. U-1 have no ubcache entry
    eng.ubcache_upload(*ub)
    n = 4 * PB + 17
    su = rng.integers(0, U, n); ku = uid[su]; ki = iid[rng.integers(0, I, n)]
    kt = probe_times(rng, ub, su)
    ku[PB] = 987_654_321_012                                                # opens chunk 2: unknown user
    ki[2 * PB] = -4                                                         # opens chunk 3: unknown item
    ku[3 * PB] = INT64_MIN; ku[7] = 0; ki[70] = INT64_MAX                   # more unknowns, one opening chunk 4
    assert (su >= U - 20).sum() > 3
    keys = list(zip(ku, ki, kt))
    want, X = _expected_scores(ocfg, W, tabs, (uid, iid), ub, keys)
    got = eng.batch_predict_keys(ku, ki, kt)
    np.testing.assert_allclose(got, want, rtol=1e-4, atol=1e-7)
    zero = [7, 70, PB, 2 * PB, 3 * PB]
    assert not X[zero].any() and len({float(got[z]) for z in zero}) == 1
    for bad in ((123_456_789_012, ki[1]), (ku[1], -55)):                    # unknown user / unknown item as key 0
        u0, i0 = ku.copy(), ki.copy()
        u0[0], i0[0] = bad
        with pytest.raises(g.CtrError) as e:
            eng.batch_predict_keys(u0, i0, kt)
        assert e.value.code == g.ENOTFOUND and "get sample vector error" in str(e.value)
    assert eng.batch_predict_keys(ku, ki, kt).tobytes() == got.tobytes()     # the failed calls left nothing behind


# ---- 4. key-fed training against the oracle ---------------------------------------------------------------------
TB = 64                   # training batch; at S = 50 one streaming chunk of the first epoch is min(n, 2 * TB) keys
CHUNK = 2 * TB
TDIMS = (8, 50, 16, 5)
TABLE_LR = 0.4


def _unknown_keys(rng, ku, ki, mask):
    """Replace the user, the item or both of the masked keys by ids no map holds (INT64_MIN among them)."""
    idx = np.flatnonzero(mask)
    kind = np.arange(idx.size) % 4
    ku[idx[kind == 0]] = 10**15 + idx[kind == 0]
    ki[idx[kind == 1]] = -(10**15) - idx[kind == 1]
    ku[idx[kind == 2]] = INT64_MIN
    ki[idx[kind == 2]] = 10**15
    ku[idx[kind == 3]] = -5
    ki[idx[kind == 3]] = INT64_MIN


def _drop(n, how, rng):
    if how is None:
        return np.zeros(n, bool)
    if how == "all":
        return np.ones(n, bool)
    if isinstance(how, tuple):                     # a [start, stop) range of keys
        m = np.zeros(n, bool); m[how[0]:how[1]] = True
        return m
    m = np.zeros(n, bool); m[rng.choice(n, how, replace=False)] = True   # this many random keys
    return m


TRAIN_CASES = {
    "n_below_batch": [dict(n=40, drop=5, epochs=1)],
    "first_chunk_empty": [dict(n=5 * CHUNK + 30, drop=(0, CHUNK), epochs=1)],
    "first_chunks_empty": [dict(n=4 * CHUNK + 7, drop=(0, 3 * CHUNK), epochs=1)],
    "last_chunk_empty": [dict(n=4 * CHUNK + 50, drop=(4 * CHUNK, None), epochs=1)],
    "survivors_k_batches": [dict(n=250, drop=250 - 3 * TB, epochs=2)],
    "survivors_k_batches_plus_one": [dict(n=250, drop=250 - 3 * TB - 1, epochs=2)],
    "long_histories_many_chunks": [dict(n=1000, drop=90, epochs=2)],
    "no_ubcache": [dict(n=300, drop=30, epochs=1, ub=False)],
    "no_epochs": [dict(n=300, drop=30, epochs=0)],
    # lr 3e-4: the last batch's cost rises by ~0.2 an epoch, so the stop after epoch 3 of 6 is far from a tie
    "early_stop": [dict(n=4 * TB, drop=None, epochs=6, early_stop=2, flip_last=True, lr=3e-4)],
    "all_unknown_then_valid": [dict(n=200, drop="all", epochs=1), dict(n=150, drop=20, epochs=1)],
    "second_call_regrows": [dict(n=100, drop=10, epochs=1), dict(n=700, drop=60, epochs=2)],
}


def _oracle_train_keys(tr, maps, ub, keys, epochs, early_stop):
    """recommend.Train over keys restated: drop keys with an unknown user or item (order kept), window each survivor
    at its timestamp, then model.Train's loop over batches of TB with the tail padded by -1 ids and label 0."""
    umap, imap = maps
    ku, ki, kt, y = keys
    keep = [k for k in range(ku.size) if int(ku[k]) in umap and int(ki[k]) in imap]
    used = len(keep)
    if used == 0:
        return 0, None, None, []
    ur = np.array([umap[int(ku[k])] for k in keep], np.int32); ir = np.array([imap[int(ki[k])] for k in keep], np.int32)
    S = tr.cfg.S
    hist = windows(ub, ur, kt[keep], S) if ub is not None else np.full((used, S), -1, np.int32)
    yy = y[keep]
    best, no_improve, ran, cost, epoch_costs = np.inf, 0, 0, 0.0, []
    for _ in range(epochs):
        for s in range(0, used, TB):
            e = min(used, s + TB); pad = TB - (e - s)
            cost, _ = tr.step(np.concatenate([ur[s:e], np.full(pad, -1, np.int32)]), np.concatenate([ir[s:e], np.full(pad, -1, np.int32)]),
                              np.concatenate([hist[s:e], np.full((pad, S), -1, np.int32)]), np.concatenate([yy[s:e], np.zeros(pad, np.float32)]),
                              table_lr=TABLE_LR)
        ran += 1; epoch_costs.append(cost)
        if cost < best:
            best, no_improve = cost, 0
        else:
            no_improve += 1
        if early_stop and no_improve >= early_stop:
            break
    return used, ran, cost, epoch_costs


@pytest.fixture(scope="module")
def train_world():
    rng = np.random.default_rng(404)
    U, I = 150, 400
    uP, S, D, cF = TDIMS
    tabs = make_tables(rng, U, I, uP, cF, D)
    uid = rng.choice(10**9, U, replace=False).astype(np.int64) + 1
    iid = rng.choice(10**9, I, replace=False).astype(np.int64) + 1
    ub = tied_histories(rng, U - 6, 2000, I)                                # rows U-6 .. U-1: empty histories
    return tabs, uid, iid, ub


@pytest.mark.parametrize("case", list(TRAIN_CASES))
def test_train_keys_against_the_oracle(train_world, case):
    """ctr_train_keys on the deterministic table path, dropout 0, against _oracle_train_keys: each call's last cost,
    rows_used and epochs_run, then the dense weights and ITEM_EMB."""
    tabs, uid, iid, ub = train_world
    uP, S, D, cF = TDIMS
    rng = np.random.default_rng(sum(map(ord, case)))
    ocfg = orc.make_cfg(orc.DIN_COS, uP, S, D, cF, 200, 80, 0.0, 0.0)
    W = scaled_init(orc, ocfg, 9)
    calls = TRAIN_CASES[case]
    with_ub = calls[0].get("ub", True)
    solver = orc.default_solver(seed=6)
    solver.lr = calls[0].get("lr", solver.lr)
    eng = _engine(g.MODEL_DIN_COS, TDIMS, TB, tabs, W, table_opt=g.TABLE_SGD_DETERMINISTIC, table_lr=TABLE_LR, seed=6,
                  dropout0=0.0, dropout1=0.0, lr=solver.lr)
    eng.idmap_build(g.IDMAP_USER, uid); eng.idmap_build(g.IDMAP_ITEM, iid)
    if with_ub:
        eng.ubcache_upload(*ub)
    tr = orc.IdxTrainer(ocfg, solver, W, *tabs)
    maps = ({int(v): r for r, v in enumerate(uid)}, {int(v): r for r, v in enumerate(iid)})
    for c in calls:
        n = c["n"]
        su = rng.integers(0, uid.size, n)
        ku, ki = uid[su].copy(), iid[rng.integers(0, iid.size, n)].copy()
        kt = probe_times(rng, ub, su)
        y = (rng.random(n) > 0.5).astype(np.float32)
        if c.get("flip_last"):
            # the same TB samples four times, labelled 1, 1, 1 and then 0: every epoch pushes the last batch's cost up
            ku, ki, kt = (np.tile(a[:TB], 4) for a in (ku, ki, kt))
            y = np.repeat(np.array([1, 1, 1, 0], np.float32), TB)
        _unknown_keys(rng, ku, ki, _drop(n, c["drop"], rng))
        keys = (ku, ki, kt, y)
        used, ran, cost, epoch_costs = _oracle_train_keys(tr, maps, ub if with_ub else None, keys, c["epochs"], c.get("early_stop", 0))
        if used == 0:
            with pytest.raises(g.CtrError) as e:
                eng.train_keys(ku, ki, kt, y, epochs=c["epochs"])
            assert e.value.code == g.ENOTFOUND
            continue
        ep, got_cost, got_used = eng.train_keys(ku, ki, kt, y, epochs=c["epochs"], early_stop=c.get("early_stop", 0))
        assert (got_used, ep) == (used, ran), (case, got_used, used, ep, ran)
        assert abs(got_cost - cost) <= 1e-6 + 2e-4 * abs(cost), (case, got_cost, cost)
        if c.get("early_stop"):
            assert ran < c["epochs"]                                        # it did stop early ...
            assert min(abs(x - epoch_costs[0]) for x in epoch_costs[1:]) > 1e-3   # ... on costs far apart
    if all(c["epochs"] == 0 for c in calls):
        assert got_cost == 0.0
        for a, b in zip(eng.get_weights(), W):
            assert a.tobytes() == np.asarray(b, np.float32).reshape(a.shape).tobytes()
        assert eng.table_download(g.TABLE_ITEM_EMB, *tabs[2].shape).tobytes() == tabs[2].tobytes()
    for a, b, name in zip(eng.get_weights(), tr.W, ("mlp0", "mlp1", "mlp2", "att0")):
        assert_mostly_close(a, b, 2e-3, 2e-4, 0.995, case + ": " + name)
    np.testing.assert_allclose(eng.table_download(g.TABLE_ITEM_EMB, *tabs[2].shape), tr.emb, rtol=2e-3, atol=2e-5, err_msg=case)


# ---- 5. the AUC, exactly ----------------------------------------------------------------------------------------
def auc_exact(pred, y):
    """RocAuc32 with integer counts: -0 read as +0, scores descending, equal scores one threshold group, cumulative tp
    and fp at each group's end, area2 = sum (fp_i - fp_{i-1}) (tp_i + tp_{i-1}) in int64, AUC = area2 / (2 P N)
    (Python's int division rounds once, correctly).  NaN when one class is absent."""
    p = np.asarray(pred, np.float32).astype(np.float64)
    p[p == 0] = 0.0
    pos = np.asarray(y, np.float32) > np.float32(0.5)
    order = np.argsort(-p, kind="stable")
    ps = p[order]
    tp = np.cumsum(pos[order], dtype=np.int64); fp = np.arange(1, p.size + 1, dtype=np.int64) - tp
    end = np.r_[ps[1:] != ps[:-1], True]
    tpg = np.r_[0, tp[end]]; fpg = np.r_[0, fp[end]]
    P = int(tp[-1]); N = p.size - P
    if P == 0 or N == 0:
        return float("nan")
    area2 = int(np.sum((fpg[1:] - fpg[:-1]) * (tpg[1:] + tpg[:-1])))
    return area2 / (2 * P * N)


def auc_scores(kind, n, rng):
    f = np.float32
    if kind == "all_equal":
        return np.full(n, 0.37, f)
    if kind == "distinct":
        return (rng.permutation(n) - n // 2).astype(f)                     # exact integers, n < 2^24
    if kind == "two_decimal_ties":
        return np.round(rng.random(n), 2).astype(f)
    if kind == "signed_zero_inf":
        return rng.choice(np.array([-0.0, 0.0, np.inf, -np.inf, 1.0, -1.0, 0.5], f), n)
    # float32 denormals around 0 (a sigmoid of a logit below about -87 is one) and the smallest normal
    tiny = np.array([0.0, -0.0, 1e-45, -1e-45, 3e-45, 1e-40, -1e-40, 6e-39, np.finfo(f).tiny, 1e-3], f)
    return rng.choice(tiny, n)


AUC_KINDS = ["all_equal", "distinct", "two_decimal_ties", "signed_zero_inf", "denormals"]


@pytest.fixture(scope="module")
def auc_engine():
    return g.Engine(g.engine.default_config(g.MODEL_YOUTUBE, batch=1, pred_batch=1))


@pytest.mark.parametrize("n", [1, 2, 31, 32, 33, 256, 257, 300_001, 5_000_003])
@pytest.mark.parametrize("kind", AUC_KINDS)
def test_auc_equals_the_integer_restatement(auc_engine, kind, n):
    """ctr_roc_auc sums half-integer trapezoids below 2^53 (exact in any order) and divides once, so it must EQUAL
    auc_exact.  Labels in {0, 1, 0.5, 0.5000001, 2, -1}, binarised at > 0.5.  The two largest n make the capped grid
    (1056 blocks of 256 threads) stride over the keys and the areas more than once."""
    rng = np.random.default_rng(n * 7 + AUC_KINDS.index(kind))
    s = auc_scores(kind, n, rng)
    y = rng.choice(np.array([0, 1, 0.5, 0.5000001, 2, -1], np.float32), n)
    want = auc_exact(s, y)
    got = auc_engine.roc_auc(s, y)
    if np.isnan(want):
        assert np.isnan(got), (kind, n, got)
    else:
        assert got == want, (kind, n, got, want)


def test_auc_is_nan_when_one_class_is_absent(auc_engine):
    rng = np.random.default_rng(3)
    s = auc_scores("two_decimal_ties", 333, rng)
    for labels in ([0, 0.5, -1], [1, 2, 0.5000001]):
        assert np.isnan(auc_engine.roc_auc(s, rng.choice(np.array(labels, np.float32), s.size)))
    assert np.isnan(auc_engine.roc_auc([0.3], [1]))
