"""CTR_EXCLUDE_SEEN on ctr_mlp_recommend_topk_ex / ctr_mlp_rank_items_ex: each key's ts is both its window cut and its
seen cut, so no item of the user's cached events with ts <= the key's ts is listed, and such a target ranks -1.

As for DIN, the reference is the full order of the unexcluded scoring pass of the same (user, ts): every item ranked
under CTR_EXCLUDE_NONE; the seen set is computed in plain Python from the sequences the test uploads."""
import ctypes as C

import numpy as np
import pytest

import go_ctr_b200 as g
from go_ctr_b200 import model as gm
from go_ctr_b200 import serving as sv
from tests.test_gpu_mlp64_rank_items import regressor
from tests.test_gpu_mlp64_recommend import Store, classifier
from tests.test_gpu_recommend_seen import INT64_MIN, INT64_MAX, long_sequence, seen_rows

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

I = 200_003
LONG = 3                                                  # rows 0, 7, 14, ... of Store's cache are empty
_lp = C.POINTER(C.c_int64)
_ip = C.POINTER(C.c_int32)
_dp = C.POINTER(C.c_double)
_fp = C.POINTER(C.c_float)


def _filled(shape, dtype, byte):
    """An output buffer whose every byte is `byte`, so that a write of any value shows."""
    a = np.empty(shape, dtype)
    a.view(np.uint8)[...] = byte
    return a


def full_order(m, st, uid, t):
    N = st.N
    ranks, logits = m.rank_items(st.eng, np.full(N, uid), np.asarray(st.eng.item_ids)[:N], np.full(N, t), exclude_history=False)
    ok = ranks > 0
    order = np.full(int(ok.sum()), -1, np.int64)
    order[ranks[ok] - 1] = np.flatnonzero(ok)
    assert (order >= 0).all()
    return order, logits


def sequence(st, r):
    off, ts, items = st.eng.ubcache_download()
    return ts[off[r]:off[r + 1]], items[off[r]:off[r + 1]]


def check_scores(kind, scores, logits):
    if kind == "regressor":
        assert scores.tobytes() == logits.astype(np.float32).tobytes()
    else:
        np.testing.assert_allclose(scores, 1.0 / (1.0 + np.exp(-logits)), rtol=1e-6, atol=1e-30)


def setup(kind, S, D, seed):
    st = Store(seed, I=I, S=S, D=D, uP=5, cF=7, pred_batch=16384)
    ts, items = long_sequence(np.random.default_rng(seed), I)
    st.eng.ubcache_set([LONG], [0, ts.size], ts, items)
    m = (classifier if kind == "classifier" else regressor)(st, hidden=(64, 32) if kind == "classifier" else (100,), seed=seed)
    return st, m, (ts, items)


CASES = [(kind, S, D) for kind in ("classifier", "regressor") for S, D in ((1, 16), (50, 64))]


@pytest.mark.parametrize("kind,S,D", CASES)
def test_seen_lists_and_ranks(kind, S, D):
    st, m, seq = setup(kind, S, D, 11 + S + D)
    uid = int(st.uid[LONG])
    ts = seq[0]
    L = ts.size
    inside = int(ts[L - 1000])
    cuts = [inside, inside + 1, int(ts[L - 100_000]), 0, INT64_MIN, INT64_MAX]
    rng = np.random.default_rng(S)
    tg, tt, want_r, want_l = [], [], [], []
    orders = {}
    for t in cuts:
        order, zl = orders[t] = full_order(m, st, uid, t)
        seen = seen_rows(seq, [], t, I)
        keep = order[~np.isin(order, seen)]
        for k in (1, 100, 1024):
            r, s, l, n = m.recommend_topk(st.eng, [uid], [t], k, exclude_seen=True)
            want = keep[:k]
            assert n[0] == want.size
            np.testing.assert_array_equal(r[0, :want.size], want)
            assert l[0, :want.size].tobytes() == zl[want].tobytes()
            assert (r[0, want.size:] == -1).all() and (s[0, want.size:] == 0).all() and (l[0, want.size:] == 0).all()
            check_scores(kind, s[0, :want.size], l[0, :want.size])
        place = np.full(I, -1, np.int64)
        place[keep] = np.arange(1, keep.size + 1)
        unseen = np.setdiff1d(np.arange(I), seen)
        rows = np.concatenate([rng.choice(seen, 10) if seen.size else [], rng.choice(unseen, 20) if unseen.size else [], keep[:3]]).astype(np.int64)
        tg.append(rows); tt.append(np.full(rows.size, t, np.int64)); want_r.append(place[rows]); want_l.append(zl[rows])
    # every cut's keys in one call: keys share a pass only with the same (user, ts)
    rows = np.concatenate(tg); t_all = np.concatenate(tt)
    perm = rng.permutation(rows.size)
    ids = np.asarray(st.eng.item_ids)[rows[perm]]
    ranks, logits = m.rank_items(st.eng, np.full(rows.size, uid), ids, t_all[perm], exclude_seen=True)
    np.testing.assert_array_equal(ranks, np.concatenate(want_r)[perm])
    assert logits.tobytes() == np.concatenate(want_l)[perm].tobytes()
    # the invariant at k = rank and rank - 1, for every mode
    for ex_hist, ex_seen in ((True, True), (True, False), (False, False)):
        t = cuts[0]
        order = orders[t][0]
        cand = np.asarray(st.eng.item_ids)[order[:1500:61]]
        r, _ = m.rank_items(st.eng, np.full(cand.size, uid), cand, np.full(cand.size, t), exclude_history=ex_hist, exclude_seen=ex_seen)
        done = 0
        for c, rr in zip(order[:1500:61], r):
            if 1 < rr <= 1024 and done < 2:
                for k, present in ((int(rr), True), (int(rr) - 1, False)):
                    rk, _, _, ck = m.recommend_topk(st.eng, [uid], [t], k, exclude_history=ex_hist, exclude_seen=ex_seen)
                    assert (int(c) in rk[0, :ck[0]].tolist()) == present, (c, rr, k)
                    if present:
                        assert rk[0, k - 1] == c
                done += 1
        assert done == 2


def test_several_users_live_updates_and_no_cache():
    st = Store(60, I=3000, S=10, D=16, pred_batch=1024)
    m = classifier(st, seed=3)
    users = st.uid[[1, 2, 7, 14]]                        # 7 and 14: no events
    ts = [st.user_ts(1, 0), st.user_ts(2, 1), 0, st.user_ts(14, 0)]
    base = m.recommend_topk(st.eng, users, ts, 1024, exclude_history=False)
    for k in (1, 100):
        got = m.recommend_topk(st.eng, users, ts, k, exclude_seen=True)
        for j, r in enumerate((1, 2, 7, 14)):
            one = m.recommend_topk(st.eng, users[j:j + 1], ts[j:j + 1], k, exclude_seen=True)
            assert all(a.tobytes() == b[j:j + 1].tobytes() for a, b in zip(one, got))
            seen = seen_rows(sequence(st, r), [], ts[j], st.N)
            keep = ~np.isin(base[0][j], seen)
            assert got[0][j].tobytes() == base[0][j][keep][:k].tobytes() and got[2][j].tobytes() == base[2][j][keep][:k].tobytes()
            assert got[1][j].tobytes() == base[1][j][keep][:k].tobytes() and got[3][j] == k
        w = m.recommend_topk(st.eng, users[2:], ts[2:], k, exclude_history=True)
        assert all(a.tobytes() == b[2:].tobytes() for a, b in zip(w, got))
    # an append, then a set, seen by the next call
    top = base[0][0][:5]
    before = m.recommend_topk(st.eng, users[:1], ts[:1], 100, exclude_seen=True)
    st.eng.ubcache_append(np.full(5, 1, np.int32), np.full(5, 7_000_000, np.int64), top)
    r, _, _, _ = m.recommend_topk(st.eng, users[:1], [0], 100, exclude_seen=True)
    assert not np.isin(top, r[0]).any()
    after = m.recommend_topk(st.eng, users[:1], ts[:1], 100, exclude_seen=True)      # the cut is before the new events
    assert all(a.tobytes() == b.tobytes() for a, b in zip(before, after))
    st.eng.ubcache_set([1], [0, 2], [20, 10], top[:2])
    r, _, _, _ = m.recommend_topk(st.eng, users[:1], [0], 100, exclude_seen=True)
    assert not np.isin(top[:2], r[0]).any()
    ranks, _ = m.rank_items(st.eng, users[[0, 0, 0]], np.asarray(st.eng.item_ids)[top[:3]], [0, 0, 15], exclude_seen=True)
    assert ranks[0] == -1 and ranks[1] == -1 and ranks[2] > 0
    # no cache: the window (empty) alone
    st2 = Store(61, I=2000, S=10, D=16, pred_batch=1024, with_ub=False)
    m2 = classifier(st2, seed=4)
    a = m2.recommend_topk(st2.eng, st2.uid[:3], [0, 5, INT64_MAX], 100, exclude_history=True)
    b = m2.recommend_topk(st2.eng, st2.uid[:3], [0, 5, INT64_MAX], 100, exclude_seen=True)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


def test_plain_calls_are_the_ex_calls_and_refusals_write_nothing():
    st = Store(62, I=2000, S=10, D=16, pred_batch=1024)
    m = classifier(st, seed=5)
    u = np.ascontiguousarray(st.uid[[1, 2, 3]], np.int64); t = np.array([st.user_ts(1, 0), 0, st.user_ts(3, 1)], np.int64)
    it = np.ascontiguousarray(st.iid[[5, 6, 7]], np.int64)
    k = 40

    def rec(fn, ex, fill=0x7F):
        o = [_filled((3, k), np.int32, fill), _filled((3, k), np.float32, fill), _filled((3, k), np.float64, fill), _filled(3, np.int32, fill)]
        rc = fn(m.h, st.eng.h, u.ctypes.data_as(_lp), t.ctypes.data_as(_lp), C.c_int64(3), C.c_int32(k), C.c_int32(ex),
                o[0].ctypes.data_as(_ip), o[1].ctypes.data_as(_fp), o[2].ctypes.data_as(_dp), o[3].ctypes.data_as(_ip))
        return rc, o

    def rank(fn, ex, fill=0x7F):
        o = [_filled(3, np.int64, fill), _filled(3, np.float64, fill)]
        rc = fn(m.h, st.eng.h, u.ctypes.data_as(_lp), it.ctypes.data_as(_lp), t.ctypes.data_as(_lp), C.c_int64(3), C.c_int32(ex),
                o[0].ctypes.data_as(_lp), o[1].ctypes.data_as(_dp))
        return rc, o

    for flag in (0, 1):
        for call, plain, ex in ((rec, m.L.ctr_mlp_recommend_topk, m.L.ctr_mlp_recommend_topk_ex), (rank, m.L.ctr_mlp_rank_items, m.L.ctr_mlp_rank_items_ex)):
            rc0, a = call(plain, flag)
            rc1, b = call(ex, flag)
            assert rc0 == rc1 == 0 and all(x.tobytes() == y.tobytes() for x, y in zip(a, b))
    for bad in (3, -1, 1000):
        for call, fn in ((rec, m.L.ctr_mlp_recommend_topk_ex), (rank, m.L.ctr_mlp_rank_items_ex)):
            rc, o = call(fn, bad, fill=0x55)
            assert rc == g.EINVAL and all((x.view(np.uint8) == 0x55).all() for x in o)
    st.eng.profile(True)
    m.recommend_topk(st.eng, u, t, 5, exclude_seen=True)
    m.rank_items(st.eng, u, it, t, exclude_seen=True)
    prof = st.eng.profile_dump()
    assert prof["mlp_rec_seen"][1] == 3 and prof["mlp_rank_seen"][1] == 3, sorted(prof)


@pytest.mark.parametrize("kind", ["classifier", "regressor"])
def test_evaluate_exclude_seen(kind):
    st = Store(63, I=400)
    rng = np.random.default_rng(6)
    if kind == "classifier":
        n = 600
        u = st.uid[rng.integers(0, st.uid.size, n)]; i = st.iid[rng.integers(0, st.iid.size, n)]
        pred = gm.SimpleMlpFitWrap(max_iter=3, seed=1).FitKeys(st.eng, u, i, np.zeros(n, np.int64), (rng.random(n) < 0.4).astype(np.float32))
    else:
        pred = gm.SimpleMlpPredWrap(regressor(st, seed=2), st.eng)
    held = []
    for r in range(1, 30):
        t = st.user_ts(r, r % 3)
        seq = sequence(st, r)
        for it in [*rng.integers(0, st.N, 3), *(seq[1][-1:] if seq[1].size else [])]:
            held.append(sv.Sample(int(st.uid[r]), int(np.asarray(st.eng.item_ids)[it]), int(t)))
    got = sv.Evaluate(pred, held, ks=(1, 10, 100), exclude_seen=True)
    hu = np.array([s.UserId for s in held]); hi = np.array([s.ItemId for s in held]); ht = np.array([s.Timestamp for s in held], np.int64)
    ranks, _ = pred.pred.rank_items(st.eng, hu, hi, ht, exclude_seen=True)
    key = {}
    groups = [key.setdefault((int(a), int(c)), len(key)) for a, c in zip(hu, ht)]
    hit, rec, ndcg, mrr = g.rank_metrics(ranks, groups, [1, 10, 100])
    for a, k in enumerate((1, 10, 100)):
        assert got["HR@%d" % k] == hit[a] and got["Recall@%d" % k] == rec[a] and got["NDCG@%d" % k] == ndcg[a]
    assert got["MRR"] == mrr
    # a target among the user's events up to the cut is a miss
    rows = st.eng.idmap_lookup(g.IDMAP_USER, hu); irows = st.eng.idmap_lookup(g.IDMAP_ITEM, hi)
    for j in range(len(held)):
        seen = seen_rows(sequence(st, int(rows[j])), [], int(ht[j]), st.N)
        assert (ranks[j] == -1) == (irows[j] < 0 or irows[j] in seen), j
