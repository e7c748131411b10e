"""CTR_EXCLUDE_SEEN on ctr_recommend_topk_ex / ctr_rank_items_ex (DIN / YouTube): no item the user has seen by the cut
is listed, and a seen target ranks -1.

The reference for every list is the full order of the unexcluded scoring pass itself: every item ranked as a target
under CTR_EXCLUDE_NONE (ctr_rank_items_ex), so the ranks are the (logit descending, row ascending) order and the logits
are the lists' bits.  The seen set is computed in plain Python from the uploaded and appended sequences."""
import ctypes as C

import numpy as np
import pytest

import go_ctr_b200 as g
from go_ctr_b200 import serving
from tests.test_gpu_recommend import make, user_hist
from tests.test_gpu_serving import _serving_engine

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

MODELS = [g.MODEL_YOUTUBE, g.MODEL_DIN_COS, g.MODEL_DIN_EUC]
I = 200_003                      # 13 chunks of pred_batch; a seen set of 10^5 rows leaves 10^5 to list
PB = 16384
INT64_MIN, INT64_MAX = -2 ** 63, 2 ** 63 - 1
LONG, SMALL, EMPTY, PAST = 3, 5, 7, 90          # user rows; the cache holds users [0, 60)
_lp = C.POINTER(C.c_int64)
_ip = C.POINTER(C.c_int32)
_fp = C.POINTER(C.c_float)


def _filled(shape, dtype, byte):
    """An output buffer whose every byte is `byte`, so that a write of any value shows."""
    a = np.empty(shape, dtype)
    a.view(np.uint8)[...] = byte
    return a


def long_sequence(rng, n_items):
    """A time-descending sequence over I - 3 distinct rows, in tied runs of 3 (ts apart by 2 between runs), with repeated
    rows and rows -1, I and I + 5 mixed in."""
    items = rng.permutation(n_items)[: n_items - 3].astype(np.int32)
    extra = np.concatenate([items[rng.integers(0, items.size, 500)], [-1, n_items, n_items + 5, -1]]).astype(np.int32)
    items = np.insert(items, np.sort(rng.integers(0, items.size, extra.size)), extra)
    ts = 10 ** 6 - (np.arange(items.size) // 3) * 2
    return ts.astype(np.int64), items


def small_sequence(rng, n_items, L=60):
    items = rng.integers(0, n_items, L).astype(np.int32)
    items[5:10] = items[0]
    items[11] = -1
    return (2 * 10 ** 6 - np.arange(L) // 2 * 7).astype(np.int64), items


def upload(eng, seqs, n_users=60):
    """seqs: {user row: (ts, items)}; the others are empty."""
    lens = np.array([seqs[u][0].size if u in seqs else 0 for u in range(n_users)])
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    ts = np.concatenate([seqs[u][0] for u in range(n_users) if u in seqs]).astype(np.int64)
    it = np.concatenate([seqs[u][1] for u in range(n_users) if u in seqs]).astype(np.int32)
    eng.ubcache_upload(off, ts, it)


def seen_rows(seq, hist, mt, n_items):
    """The seen set, sorted: the window's valid rows and the rows of the events with ts <= mt (mt == 0: every event)."""
    parts = [np.asarray(hist, np.int64)]
    if seq is not None:
        ts, items = seq
        parts.append(items if mt == 0 else items[ts <= mt])
    s = np.unique(np.concatenate(parts).astype(np.int64))
    return s[(s >= 0) & (s < n_items)]


def full_order(eng, user, hist, n_items):
    """(rows in list order, logits [n_items]) of the unexcluded pass for (user, hist)."""
    ranks, logits = eng.rank_items(np.full(n_items, user, np.int32), np.tile(hist, (n_items, 1)), np.arange(n_items, dtype=np.int32),
                                   exclude_history=False)
    ok = ranks > 0
    order = np.full(int(ok.sum()), -1, np.int64)
    order[ranks[ok] - 1] = np.flatnonzero(ok)
    assert (order >= 0).all(), "the unexcluded ranks are not a permutation"
    return order, logits


def check_list(rows, scores, logits, cnt, want, zl, k, known_scores):
    """One user's list against the expected rows (logits from the full pass zl); score bits where the unexcluded list
    holds the same logit, else within the sigmoid's error."""
    n = want.size
    assert cnt == n, (cnt, n)
    np.testing.assert_array_equal(rows[:n], want)
    assert (rows[n:] == -1).all() and (scores[n:] == 0).all() and (logits[n:] == 0).all()
    assert logits[:n].tobytes() == zl[want].tobytes(), "logits differ from the scoring pass"
    for s, l in zip(scores[:n], logits[:n]):
        ref = known_scores.get(l.tobytes())
        if ref is not None:
            assert s.tobytes() == ref
    ref = 1.0 / (1.0 + np.exp(-logits[:n].astype(np.float64)))
    np.testing.assert_allclose(scores[:n], ref, rtol=1e-5, atol=1e-30)


class Case:
    """One engine at I items, the long user's full order for its window, and a small user's unexcluded top 1024."""

    def __init__(self, model, D, S, seed=0, **kw):
        self.eng, self.cfg, _, _, _, self.rng = make(model, D=D, S=S, I=I, seed=seed, pred_batch=PB, **kw)
        rng = self.rng
        self.seq = {LONG: long_sequence(rng, I), SMALL: small_sequence(rng, I)}
        upload(self.eng, self.seq)
        self.hist = user_hist(rng, S, I)
        self.order, self.zl = full_order(self.eng, LONG, self.hist, I)
        r, s, l, c = self.eng.recommend_topk([LONG], self.hist[None], 1024, exclude_history=False)
        self.known = {a.tobytes(): b.tobytes() for a, b in zip(l[0, :c[0]], s[0, :c[0]])}
        assert np.array_equal(r[0, :c[0]], self.order[:c[0]])

    def expect(self, seen, k):
        keep = self.order[~np.isin(self.order, seen)]
        return keep[:k]

    def cuts(self):
        ts = self.seq[LONG][0]
        L = ts.size
        inside = int(ts[L - 1000])                      # runs of 3: L - 1000 sits inside one or at its start
        return [INT64_MIN, int(ts[-1]) - 1, int(ts[-1]), inside, inside + 1, inside - 1, int(ts[L - 100_000]), 0, INT64_MAX,
                int(ts[0])]

    def seen(self, user, hist, mt):
        return seen_rows(self.seq.get(user), hist, mt, I)


def check_long_user(c, ks=(1, 100, 1024)):
    eng = c.eng
    sizes = []
    for mt in c.cuts():
        seen = c.seen(LONG, c.hist, mt)
        sizes.append(seen.size)
        for k in ks:
            r, s, l, n = eng.recommend_topk([LONG], c.hist[None], k, max_ts=mt, exclude_seen=True)
            check_list(r[0], s[0], l[0], int(n[0]), c.expect(seen, k), c.zl, k, c.known)
    assert min(sizes) <= c.hist.size and max(sizes) >= I - 3 and any(9e4 < x < 1.1e5 for x in sizes), sizes
    return sizes


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("S,D", [(1, 16), (1, 64), (50, 16), (50, 64)])
def test_seen_lists(model, S, D):
    c = Case(model, D, S, seed=S + D)
    check_long_user(c)
    check_ranks(c)


@pytest.mark.parametrize("model", MODELS)
def test_seen_lists_generic_fallback(model):
    """D = 7 takes the ordinary _gen attention kernel through index buffers."""
    c = Case(model, 7, 10, uP=5, cF=3)
    check_long_user(c, ks=(100,))
    check_ranks(c, modes=False)


def check_ranks(c, modes=True):
    eng, rng = c.eng, c.rng
    cuts = [c.cuts()[i] for i in (3, 6, 8)]
    tg, users, mts = [], [], []
    for mt in cuts:
        seen = c.seen(LONG, c.hist, mt)
        unseen = np.setdiff1d(np.arange(I), seen)
        t = np.concatenate([rng.choice(seen, 20), rng.choice(unseen, 40), c.expect(seen, 5), [-1, I]]).astype(np.int32)
        tg.append(t); mts.append(np.full(t.size, mt, np.int64))
    t = np.concatenate(tg); mt = np.concatenate(mts)
    ranks, logits = eng.rank_items(np.full(t.size, LONG, np.int32), np.tile(c.hist, (t.size, 1)), t, max_ts=mt, exclude_seen=True)
    inside = (t >= 0) & (t < I)
    assert (ranks[~inside] == -1).all() and np.isnan(logits[~inside]).all()
    assert logits[inside].tobytes() == c.zl[t[inside]].tobytes()
    for m in cuts:                                   # the numpy count: 1 + the unseen items before the target
        seen = c.seen(LONG, c.hist, m)
        keep = c.order[~np.isin(c.order, seen)]
        place = np.full(I, -1, np.int64)
        place[keep] = np.arange(1, keep.size + 1)
        sel = inside & (mt == m)
        np.testing.assert_array_equal(ranks[sel], place[t[sel]])
        assert (ranks[sel][np.isin(t[sel], seen)] == -1).all() and (ranks[sel] == -1).sum() >= 20
    # the invariant at k = rank and rank - 1, for every mode
    for mode_seen, mode_hist in ((True, True), (False, True), (False, False)) if modes else ((True, True),):
        m = int(cuts[0])
        cand = np.concatenate([c.order[:3000:97], c.order[:40]]).astype(np.int32)
        r, _ = eng.rank_items(np.full(cand.size, LONG, np.int32), np.tile(c.hist, (cand.size, 1)), cand, exclude_history=mode_hist,
                              max_ts=m, exclude_seen=mode_seen)
        done = 0
        for tt, rr in zip(cand, r):
            if 1 < rr <= 1024 and done < 2:
                for k, present in ((int(rr), True), (int(rr) - 1, False)):
                    rk, _, _, ck = eng.recommend_topk([LONG], c.hist[None], k, exclude_history=mode_hist, max_ts=m, exclude_seen=mode_seen)
                    assert (int(tt) in rk[0, :ck[0]].tolist()) == present, (tt, rr, k)
                    if present:
                        assert rk[0, k - 1] == tt
                done += 1
        assert done == 2


def test_several_users_in_one_call_and_live_updates():
    """Users with a long, a short, no and no cached sequence, each at its own cut, against the single-user lists; then
    an append and a set, seen by the next call."""
    c = Case(g.MODEL_DIN_COS, 32, 20, seed=7)
    eng = c.eng
    S = c.cfg.S
    hs = np.stack([c.hist, user_hist(c.rng, S, I), user_hist(c.rng, S, I), np.full(S, -1, np.int32)])
    users = np.array([LONG, SMALL, EMPTY, PAST], np.int32)
    cut = [c.cuts()[6], int(c.seq[SMALL][0][30]), 0, 0]
    for k in (1, 100, 1024):
        r, s, l, n = eng.recommend_topk(users, hs, k, max_ts=cut, exclude_seen=True)
        for j in range(4):
            r1, s1, l1, n1 = eng.recommend_topk(users[j:j + 1], hs[j:j + 1], k, max_ts=cut[j], exclude_seen=True)
            assert r1.tobytes() == r[j:j + 1].tobytes() and s1.tobytes() == s[j:j + 1].tobytes() and l1.tobytes() == l[j:j + 1].tobytes()
            assert n1[0] == n[j]
        check_list(r[0], s[0], l[0], int(n[0]), c.expect(c.seen(LONG, c.hist, cut[0]), k), c.zl, k, c.known)
        # no events, or past the cache: the window alone
        w = eng.recommend_topk(users[2:], hs[2:], k, exclude_history=True)
        assert all(a.tobytes() == b[2:].tobytes() for a, b in zip(w, (r, s, l, n)))
    # the short user: its unexcluded top 1024 with the seen rows removed
    base = eng.recommend_topk([SMALL], hs[1:2], 1024, exclude_history=False)

    def check_small(seq, mt):
        seen = seen_rows(seq, hs[1], mt, I)
        r, s, l, n = eng.recommend_topk([SMALL], hs[1:2], 100, max_ts=mt, exclude_seen=True)
        keep = ~np.isin(base[0][0], seen)
        want = base[0][0][keep][:100]
        np.testing.assert_array_equal(r[0], want)
        assert l[0].tobytes() == base[2][0][keep][:100].tobytes() and s[0].tobytes() == base[1][0][keep][:100].tobytes()
        assert n[0] == 100

    check_small(c.seq[SMALL], cut[1])
    check_small(c.seq[SMALL], 0)
    top = base[0][0][:10]
    t_new = np.full(10, 3 * 10 ** 6, np.int64)
    eng.ubcache_append(np.full(10, SMALL, np.int32), t_new, top)
    seq2 = (np.concatenate([t_new, c.seq[SMALL][0]]), np.concatenate([top, c.seq[SMALL][1]]))
    check_small(seq2, 0)
    check_small(seq2, cut[1])                      # the appended events are after the cut
    top2 = base[0][0][20:25]
    seq3 = (np.array([9, 8, 8, 7, 1], np.int64), top2.astype(np.int32))
    eng.ubcache_set([SMALL], [0, 5], *seq3)
    check_small(seq3, 0)
    check_small(seq3, 8)


def test_no_cache_is_the_window():
    eng, cfg, _, _, _, rng = make(g.MODEL_DIN_EUC, D=16, S=10, I=5000, pred_batch=1024)
    hs = np.stack([user_hist(rng, 10, 5000) for _ in range(3)])
    for k in (1, 100, 1024):
        w = eng.recommend_topk([1, 2, 96], hs, k, exclude_history=True)
        for cut in (0, INT64_MIN, INT64_MAX, 12345):
            sn = eng.recommend_topk([1, 2, 96], hs, k, max_ts=cut, exclude_seen=True)
            assert all(a.tobytes() == b.tobytes() for a, b in zip(w, sn))
    t = rng.integers(-2, 5002, 300).astype(np.int32)
    u = np.full(300, 2, np.int32)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(eng.rank_items(u, np.tile(hs[1], (300, 1)), t),
                                                          eng.rank_items(u, np.tile(hs[1], (300, 1)), t, max_ts=0, exclude_seen=True)))


def test_a_user_who_has_seen_everything():
    eng, cfg, _, _, _, rng = make(g.MODEL_YOUTUBE, D=16, S=5, I=3000, pred_batch=1024)
    items = np.concatenate([rng.permutation(3000), [-1, 3000]]).astype(np.int32)
    upload(eng, {4: (np.arange(items.size, 0, -1).astype(np.int64), items)}, n_users=10)
    r, s, l, n = eng.recommend_topk([4, 5], np.full((2, 5), -1, np.int32), 64, max_ts=[0, 0], exclude_seen=True)
    assert n[0] == 0 and (r[0] == -1).all() and (s[0] == 0).all() and (l[0] == 0).all() and n[1] == 64
    ranks, _ = eng.rank_items(np.full(3000, 4, np.int32), np.full((3000, 5), -1, np.int32), np.arange(3000, dtype=np.int32),
                              max_ts=0, exclude_seen=True)
    assert (ranks == -1).all()


def _call_recommend(eng, ex_fn, users, hist, k, exclude, max_ts=None, fill=0x7F):
    nu = len(users)
    u = np.ascontiguousarray(users, np.int32); h = np.ascontiguousarray(hist, np.int32)
    outs = [_filled((nu, k), np.int32, fill), _filled((nu, k), np.float32, fill), _filled((nu, k), np.float32, fill), _filled(nu, np.int32, fill)]
    ptrs = [outs[0].ctypes.data_as(_ip), outs[1].ctypes.data_as(_fp), outs[2].ctypes.data_as(_fp), outs[3].ctypes.data_as(_ip)]
    if ex_fn:
        mt = None if max_ts is None else np.ascontiguousarray(max_ts, np.int64).ctypes.data_as(_lp)
        rc = eng.L.ctr_recommend_topk_ex(eng.h, u.ctypes.data_as(_ip), h.ctypes.data_as(_ip), mt, C.c_int64(nu), C.c_int32(k),
                                         C.c_int32(exclude), *ptrs)
    else:
        rc = eng.L.ctr_recommend_topk(eng.h, u.ctypes.data_as(_ip), h.ctypes.data_as(_ip), C.c_int64(nu), C.c_int32(k), C.c_int32(exclude), *ptrs)
    return rc, outs


def _call_rank(eng, ex_fn, users, hist, items, exclude, max_ts=None, fill=0x7F):
    n = len(users)
    u = np.ascontiguousarray(users, np.int32); h = np.ascontiguousarray(hist, np.int32); it = np.ascontiguousarray(items, np.int32)
    ranks = _filled(n, np.int64, fill); logits = _filled(n, np.float32, fill)
    if ex_fn:
        mt = None if max_ts is None else np.ascontiguousarray(max_ts, np.int64).ctypes.data_as(_lp)
        rc = eng.L.ctr_rank_items_ex(eng.h, u.ctypes.data_as(_ip), h.ctypes.data_as(_ip), mt, it.ctypes.data_as(_ip), C.c_int64(n),
                                     C.c_int32(exclude), ranks.ctypes.data_as(_lp), logits.ctypes.data_as(_fp))
    else:
        rc = eng.L.ctr_rank_items(eng.h, u.ctypes.data_as(_ip), h.ctypes.data_as(_ip), it.ctypes.data_as(_ip), C.c_int64(n),
                                  C.c_int32(exclude), ranks.ctypes.data_as(_lp), logits.ctypes.data_as(_fp))
    return rc, [ranks, logits]


def test_plain_calls_are_the_ex_calls_and_refusals_write_nothing():
    eng, cfg, _, _, _, rng = make(g.MODEL_DIN_COS, D=32, S=8, I=4000, pred_batch=512)
    upload(eng, {2: small_sequence(rng, 4000)}, n_users=10)
    hs = np.stack([user_hist(rng, 8, 4000) for _ in range(3)])
    users = [2, 3, 40]
    items = rng.integers(-1, 4001, 3).astype(np.int32)
    for flag in (0, 1):
        rc0, a = _call_recommend(eng, False, users, hs, 50, flag)
        rc1, b = _call_recommend(eng, True, users, hs, 50, flag)
        assert rc0 == rc1 == 0 and all(x.tobytes() == y.tobytes() for x, y in zip(a, b))
        rc0, a = _call_rank(eng, False, users, hs, items, flag)
        rc1, b = _call_rank(eng, True, users, hs, items, flag, max_ts=[5, 6, 7])      # max_ts is not read
        assert rc0 == rc1 == 0 and all(x.tobytes() == y.tobytes() for x, y in zip(a, b))
    for ex, mt in ((3, [0, 0, 0]), (-1, [0, 0, 0]), (g.EXCLUDE_SEEN, None)):
        rc, outs = _call_recommend(eng, True, users, hs, 50, ex, max_ts=mt, fill=0x55)
        assert rc == g.EINVAL
        assert all((o.view(np.uint8) == 0x55).all() for o in outs), "a refusal wrote"
        rc, outs = _call_rank(eng, True, users, hs, items, ex, max_ts=mt, fill=0x55)
        assert rc == g.EINVAL
        assert all((o.view(np.uint8) == 0x55).all() for o in outs), "a refusal wrote"
    with pytest.raises(ValueError):
        eng.recommend_topk(users, hs, 5, max_ts=[1, 2], exclude_seen=True)
    # the profile keys of the seen list
    eng.profile(True)
    eng.recommend_topk(users, hs, 5, max_ts=0, exclude_seen=True)
    eng.rank_items(users, hs, items, max_ts=0, exclude_seen=True)
    prof = eng.profile_dump()
    assert "rec_seen" in prof and "rank_seen" in prof, sorted(prof)


def test_evaluate_exclude_seen():
    """serving.Evaluate(exclude_seen=True) is rank_metrics of rank_items under SEEN at each sample's timestamp, and
    those ranks are the numpy count over the full order of the same window."""
    eng, ocfg, W, tabs, (uid, iid), (off, ts, items, lens), rng = _serving_engine(g.MODEL_DIN_COS, I=150, pred_batch=64)
    eng.ubcache_upload(off, ts, items)
    users = [r for r in range(len(uid)) if lens[r] >= 4][:6]
    held = []
    for r in users:
        t_r = ts[off[r]:off[r + 1]]
        for cut in (int(t_r[0]), int(t_r[len(t_r) // 2]), int(t_r[-1]) - 1):
            for it in [*rng.integers(0, 150, 4), items[off[r + 1] - 1]]:     # the user's oldest item among them
                held.append(serving.Sample(int(uid[r]), int(iid[it]), cut))
    got = serving.Evaluate(eng, held, ks=(1, 5, 20), exclude_seen=True)
    u = np.array([s.UserId for s in held]); t = np.array([s.Timestamp for s in held], np.int64)
    rows = eng.idmap_lookup(g.IDMAP_USER, u); it_rows = eng.idmap_lookup(g.IDMAP_ITEM, [s.ItemId for s in held])
    hist = eng.ubcache_window(rows, t)
    ranks, _ = eng.rank_items(rows, hist, it_rows, max_ts=t, exclude_seen=True)
    _, groups = np.unique(np.stack([u, t], axis=1), axis=0, return_inverse=True)
    hit, rec, ndcg, mrr = g.rank_metrics(ranks, groups.ravel(), [1, 5, 20])
    assert got["MRR"] == mrr and got["HR@5"] == hit[1] and got["Recall@20"] == rec[2] and got["NDCG@1"] == ndcg[0]
    for i in range(len(held)):
        order, _ = full_order(eng, int(rows[i]), hist[i], 150)
        r = int(rows[i])
        seen = seen_rows((ts[off[r]:off[r + 1]], items[off[r]:off[r + 1]]), hist[i], int(t[i]), 150)
        keep = order[~np.isin(order, seen)]
        want = int(np.flatnonzero(keep == it_rows[i])[0]) + 1 if it_rows[i] in keep else -1
        assert ranks[i] == want, (i, ranks[i], want)
