"""ctr_mlp_rank_items: the full-catalogue rank of held-out items under the float64 MLP.

With I <= 1024 a full ctr_mlp_recommend_topk list gives every item's place: each item's rank must be its position + 1
and its logit the list's, bit for bit; excluded items rank -1."""
import ctypes as C

import numpy as np
import pytest

import go_ctr_b200 as g
from go_ctr_b200 import model as gm
from go_ctr_b200 import serving as sv
from tests.test_gpu_mlp64_recommend import Store, classifier

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]


def regressor(st, hidden=(100,), seed=0):
    """An identity-output regressor with random parameters: it ranks by its predicted value."""
    m = g.MLPRegressor(st.nin, hidden=hidden, max_iter=3, seed=seed)
    rng = np.random.default_rng(seed + 1)
    units = [st.nin, *hidden, 1]
    p = []
    for fi, fo in zip(units[:-1], units[1:]):
        p.append(rng.standard_normal(fo) * 0.1)
        p.append(rng.standard_normal(fi * fo) / np.sqrt(fi))
    m.set_params(np.concatenate(p), out_activation="identity")
    return m


def check_full(m, st, r, t, exclude):
    """Every item of the table as a target of one user: ranks and logits against the full list."""
    N = st.N
    uid = int(st.uid[r])
    items = np.asarray(st.eng.item_ids)[:N]
    ranks, logits = m.rank_items(st.eng, np.full(N, uid), items, np.full(N, t), exclude_history=exclude)
    rows, sc, lg, cnt = m.recommend_topk(st.eng, [uid], [t], N, exclude_history=exclude)
    n = int(cnt[0])
    want = np.full(N, -1, np.int64)
    want[rows[0, :n]] = np.arange(1, n + 1)
    np.testing.assert_array_equal(ranks, want)
    assert logits[rows[0, :n]].view(np.uint64).tobytes() == lg[0, :n].view(np.uint64).tobytes()
    if exclude:
        win = set(int(x) for x in st.window(r, t) if 0 <= x < N)
        assert set(np.flatnonzero(ranks == -1).tolist()) == win
    return ranks, logits


CASES = [(kind, hidden, S, D) for kind in ("classifier", "regressor") for hidden in ((100,), (64, 32)) for S, D in ((1, 16), (10, 64))]


@pytest.mark.parametrize("kind,hidden,S,D", CASES)
def test_ranks_are_the_full_lists_places(kind, hidden, S, D):
    st = Store(31 + S + D + len(hidden), I=700, S=S, D=D, uP=5, cF=7, pred_batch=256)
    m = (classifier if kind == "classifier" else regressor)(st, hidden=hidden, seed=3)
    for r, which, ex in ((1, 0, True), (3, 1, False), (5, 2, True)):
        check_full(m, st, r, st.user_ts(r, which), ex)


def test_keys_of_several_users_and_windows_in_one_call():
    st = Store(40, I=500, pred_batch=128)
    m = classifier(st, seed=4, hidden=(64, 32))
    rng = np.random.default_rng(2)
    n = 200
    rs = rng.integers(0, st.uid.size, n)
    ts = np.array([st.user_ts(int(r), int(w)) for r, w in zip(rs, rng.integers(0, 3, n))], np.int64)
    items = st.iid[rng.integers(0, st.iid.size, n)]
    ranks, logits = m.rank_items(st.eng, st.uid[rs], items, ts)
    perm = rng.permutation(n)
    r2, l2 = m.rank_items(st.eng, st.uid[rs][perm], items[perm], ts[perm])
    assert r2.tobytes() == ranks[perm].tobytes() and l2.tobytes() == logits[perm].tobytes()
    for i in range(0, n, 17):
        r1, l1 = m.rank_items(st.eng, st.uid[rs[i:i + 1]], items[i:i + 1], ts[i:i + 1])
        assert r1[0] == ranks[i] and l1.tobytes() == logits[i:i + 1].tobytes()
        rows, _, lg, cnt = m.recommend_topk(st.eng, st.uid[rs[i:i + 1]], ts[i:i + 1], 1024)
        row = int(st.eng.idmap_lookup(g.IDMAP_ITEM, items[i:i + 1])[0])
        if ranks[i] > 0:
            assert rows[0, ranks[i] - 1] == row and lg[0, ranks[i] - 1].tobytes() == logits[i:i + 1].tobytes()
        else:
            assert row not in rows[0, :cnt[0]].tolist()


def test_unknown_items_and_users():
    st = Store(41, I=300)
    m = classifier(st, seed=5)
    uid = st.uid[[1, 1, 2]]
    ranks, logits = m.rank_items(st.eng, uid, [st.iid[0], 10**15 + 1, st.iid[5]], [0, 0, 0])
    assert ranks[1] == -1 and np.isnan(logits[1]) and ranks[0] != 0 and ranks[2] != 0
    with pytest.raises(g.CtrError) as e:
        m.rank_items(st.eng, [st.uid[0], 10**15 + 7, 10**15 + 8], st.iid[:3], [0, 0, 0])
    assert e.value.code == g.ENOTFOUND and str(10**15 + 7) in str(e.value)


def test_live_ubcache_append_is_seen():
    st = Store(42, I=300)
    m = classifier(st, seed=7)
    r, t = 2, 0
    uid = int(st.uid[r])
    ranks, _ = check_full(m, st, r, t, True)
    best = int(np.flatnonzero(ranks == 1)[0])
    st.eng.ubcache_append([r], [6_000_000], [best])
    ranks2, _ = check_full(m, st, r, t, True)
    assert ranks2[best] == -1
    assert m.rank_items(st.eng, [uid], [st.iid[best]], [t], exclude_history=False)[0][0] > 0


def _raw(m, eng, uid, iid, n=1, null=None):
    u = np.full(max(n, 1), uid, np.int64); i = np.full(max(n, 1), iid, np.int64); t = np.zeros(max(n, 1), np.int64)
    rk = np.full(max(n, 1), 77, np.int64); lg = np.full(max(n, 1), 9.25)
    lp = C.POINTER(C.c_int64)
    ptr = {"user": u.ctypes.data_as(lp), "item": i.ctypes.data_as(lp), "ts": t.ctypes.data_as(lp), "rank": rk.ctypes.data_as(lp)}
    if null:
        ptr[null] = None
    rc = m.L.ctr_mlp_rank_items(m.h, eng.h if eng is not None else None, ptr["user"], ptr["item"], ptr["ts"], C.c_int64(n), C.c_int32(1),
                                ptr["rank"], lg.ctypes.data_as(C.POINTER(C.c_double)))
    return rc, bool((rk == 77).all() and (lg == 9.25).all())


def test_refusals_write_nothing():
    st = Store(43, I=100)
    m = classifier(st, seed=8)
    ids = (int(st.uid[0]), int(st.iid[0]))
    assert _raw(m, st.eng, *ids) == (0, False)
    assert _raw(m, st.eng, *ids, n=0) == (g.EINVAL, True)
    for null in ("user", "item", "ts", "rank"):
        assert _raw(m, st.eng, *ids, null=null) == (g.EINVAL, True), null
    assert _raw(m, None, *ids) == (g.EINVAL, True)
    # not fitted
    assert _raw(g.MLPClassifier(st.nin, hidden=(100,)), st.eng, *ids) == (g.ESTATE, True)
    # classes: the classifier predicts labels
    c3 = g.MLPClassifier(st.nin, hidden=(8,), max_iter=2, seed=1)
    rng = np.random.default_rng(1)
    c3.fit(rng.random((40, st.nin), np.float32), rng.integers(1, 4, 40).astype(np.float32))
    assert c3.classes_.size == 3
    assert _raw(c3, st.eng, *ids) == (g.ESTATE, True)
    # several outputs
    r3 = g.MLPRegressor(st.nin, hidden=(8,), max_iter=2, seed=1, n_outputs=3).fit(rng.random((40, st.nin), np.float32),
                                                                                  rng.random((40, 3), np.float32) * 5)
    assert _raw(r3, st.eng, *ids) == (g.ESTATE, True)
    # an unknown user
    rc, ok = _raw(m, st.eng, 10**15 + 11, ids[1])
    assert rc == g.ENOTFOUND and ok


def test_profile_keys():
    st = Store(44, I=700, pred_batch=256)
    m = classifier(st, seed=9, hidden=(64, 32))
    st.eng.profile(True)
    st.eng.profile_reset()
    m.rank_items(st.eng, st.uid[[1, 1, 2]], st.iid[[0, 600, 3]], [0, 0, 0])
    prof = st.eng.profile_dump()
    st.eng.profile(False)
    assert not {"mlp_rec_topk", "mlp_rec_merge", "mlp_rec_finish", "mlp_rec_resolve"} & set(prof), sorted(prof)
    assert prof["mlp_rank_resolve"][1] == 1 and prof["ubcache_window"][1] == 1
    assert prof["mlp_rec_prefix"][1] == 2                   # two (user, ts) passes
    assert prof["mlp_rank_target"][1] == (2 + 1) + (1 + 1)  # user 1: chunks 0 and 2; user 2: chunk 0; each then a sort
    assert prof["mlp_rank_count"][1] == 2 * (3 + 1)         # 700 items in chunks of 256, then the ranks
    assert prof["mlp_rec_layer0"][1] == (2 + 3) + (1 + 3)


@pytest.mark.parametrize("kind", ["classifier", "regressor"])
def test_evaluate_equals_rank_metrics(kind):
    st = Store(45, I=400)
    rng = np.random.default_rng(5)
    n = 800
    u = st.uid[rng.integers(0, st.uid.size, n)]; i = st.iid[rng.integers(0, st.iid.size, n)]
    if kind == "classifier":
        pred = gm.SimpleMlpFitWrap(max_iter=3, seed=1).FitKeys(st.eng, u, i, np.zeros(n, np.int64), (rng.random(n) < 0.4).astype(np.float32))
    else:
        pred = gm.SimpleMlpPredWrap(regressor(st, seed=2), st.eng)
    h = 60
    hu, hi = u[:h], i[:h]
    ht = np.array([st.user_ts(int(np.flatnonzero(st.uid == x)[0]), j % 3) for j, x in enumerate(hu)], np.int64)
    hi[0] = 10**15 + 5                                       # an unknown item: a miss
    held = [sv.Sample(int(a), int(b), int(c)) for a, b, c in zip(hu, hi, ht)]
    got = sv.Evaluate(pred, held, ks=(1, 10, 100))
    ranks, _ = pred.pred.rank_items(st.eng, hu, hi, ht)
    assert ranks[0] == -1
    key = {}
    groups = [key.setdefault((int(a), int(c)), len(key)) for a, c in zip(hu, ht)]
    hit, rec, ndcg, mrr = g.rank_metrics(ranks, groups, [1, 10, 100])
    for a, k in enumerate((1, 10, 100)):
        assert got["HR@%d" % k] == hit[a] and got["Recall@%d" % k] == rec[a] and got["NDCG@%d" % k] == ndcg[a]
    assert got["MRR"] == mrr
