"""ctr_rank_items: the full-catalogue rank of held-out items under DIN / YouTube.

The spec is the invariant with the recommendation lists: for every k in [1, 1024], 0 < rank <= k exactly when
ctr_recommend_topk(user, hist, k, exclude_history) lists the target, at position rank - 1, with the same logit bit for
bit.  Ranks are also held to a numpy count over the engine's own per-row logits (ctr_debug_grads_idx), except for the
one instantiation whose logits differ in the last bit from the predict route (euclid, D = 16)."""
import ctypes as C

import numpy as np
import pytest

import go_ctr_b200 as g
from go_ctr_b200 import serving
from tests.test_gpu_recommend import engine_forward, make, user_hist
from tests.test_gpu_serving import _serving_engine

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

MODELS = [g.MODEL_YOUTUBE, g.MODEL_DIN_COS, g.MODEL_DIN_EUC]


def targets_for(I, B, hist, rng):
    """First, middle and last chunk; several in one chunk; the same row twice; a row of the window; rows outside."""
    mid = (I // B) // 2 * B
    t = [0, I - 1, min(mid + 3, I - 1), min(1, I - 1), min(B - 1, I - 1), I - 1, int(rng.integers(0, I))]
    valid = hist[(hist >= 0) & (hist < I)]
    if valid.size:
        t.append(int(valid[0]))
    return np.array(t + [-1, I, I + 100], np.int32)


def numpy_rank(z, hist, t, exclude):
    """1 + the items before target t in (logit descending, row ascending), NaN and excluded rows not counting."""
    I = z.size
    if not 0 <= t < I or np.isnan(z[t]):
        return -1
    ex = set(int(x) for x in hist if 0 <= x < I) if exclude else set()
    if t in ex:
        return -1
    rows = np.arange(I)
    ok = ~np.isnan(z) & ~np.isin(rows, list(ex))
    before = (z > z[t]) | ((z == z[t]) & (rows < t))
    return 1 + int((ok & before).sum())


def check_ranks(eng, cfg, user, hist, targets, I, exclude=True, exact=True, k_checks=2):
    n = targets.size
    ranks, logits = eng.rank_items(np.full(n, user, np.int32), np.tile(hist, (n, 1)), targets, exclude_history=exclude)
    rows, scores, lg, cnt = eng.recommend_topk([user], hist[None, :], 1024, exclude_history=exclude)
    lst = rows[0, :cnt[0]]
    for t, r, l in zip(targets, ranks, logits):
        t = int(t); r = int(r)
        if 0 < r <= 1024:
            assert lst[r - 1] == t, (t, r, lst[max(0, r - 3):r + 2])
            assert np.float32(l).tobytes() == lg[0, r - 1].tobytes(), "the logit differs from the list's"
        else:
            assert r == -1 or r > 1024, r
            assert t not in lst.tolist(), (t, r)
        if not 0 <= t < I:
            assert r == -1 and np.isnan(l)
    # the invariant at k = rank and k = rank - 1
    done = 0
    for t, r in zip(targets, ranks):
        if 1 < r <= 1024 and done < k_checks:
            for k, present in ((int(r), True), (int(r) - 1, False)):
                rk, _, lk, ck = eng.recommend_topk([user], hist[None, :], k, exclude_history=exclude)
                assert (int(t) in rk[0, :ck[0]].tolist()) == present, (t, r, k)
                if present:
                    assert rk[0, k - 1] == t
            done += 1
    if exact:
        z, _ = engine_forward(eng, cfg, user, hist, I)
        want = [numpy_rank(z, hist, int(t), exclude) for t in targets]
        np.testing.assert_array_equal(ranks, want)
        inside = (targets >= 0) & (targets < I)
        assert logits[inside].tobytes() == z[targets[inside]].tobytes()
    return ranks, logits


def run_case(model, D, S, I, seed=0, exclude=True, **kw):
    eng, cfg, ocfg, W, tabs, rng = make(model, D=D, S=S, I=I, seed=seed, **kw)
    user = int(rng.integers(0, 97)); hist = user_hist(rng, S, I)
    B = max(cfg.batch, cfg.pred_batch)
    check_ranks(eng, cfg, user, hist, targets_for(I, B, hist, rng), I, exclude=exclude,
                exact=not (model == g.MODEL_DIN_EUC and D == 16))
    return eng


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("D", [16, 32, 64, 128])
def test_lane_maps(model, D):
    run_case(model, D, 50, 1000)


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("S", [1, 100])
def test_history_lengths(model, S):
    run_case(model, 64, S, 5000, exclude=S == 1)


@pytest.mark.parametrize("I", [1, 37, 1000, 5000])
def test_catalogue_sizes(I):
    run_case(g.MODEL_DIN_COS, 32, 20, I)


@pytest.mark.parametrize("model", MODELS)
def test_generic_fallback(model):
    """D = 7 takes index buffers for the ordinary _gen kernel (rec_fill_idx)."""
    eng = run_case(model, 7, 10, 1000, uP=5, cF=3)
    eng.profile(True)
    eng.rank_items([3], np.full((1, 10), -1, np.int32), [5])
    prof = eng.profile_dump()
    assert "rec_fill_idx" in prof and "attn_fwd_gen" in prof, sorted(prof)


def test_history_beyond_shared_memory():
    run_case(g.MODEL_DIN_EUC, 128, 500, 600, uP=8, cF=4)


@pytest.mark.parametrize("model", [g.MODEL_DIN_COS, g.MODEL_DIN_EUC])
def test_fp32_gemms(model):
    eng = run_case(model, 64, 50, 1000, gemm=g.GEMM_FP32)
    eng.profile(True)
    eng.rank_items([3], np.full((1, 50), -1, np.int32), [5])
    assert "sgemm_fwd0_sigmoid" in eng.profile_dump()


def test_exact_tie_runs_follow_row_order():
    I, D, cF, S = 600, 32, 9, 20
    eng, cfg, ocfg, W, (uf, itf, emb), rng = make(g.MODEL_YOUTUBE, D=D, S=S, I=I, cF=cF)
    emb = emb.copy(); itf = itf.copy()
    run = [40, 41, 300, 301, 302, 599]
    emb[run] = 0.0; itf[run] = 0.0                              # zero rows: one logit, a tie run
    eng.table_upload(g.TABLE_ITEM_EMB, emb); eng.table_upload(g.TABLE_ITEM_FEAT, itf)
    hist = np.full(S, -1, np.int32)
    ranks, logits = check_ranks(eng, cfg, 3, hist, np.array(run, np.int32), I, exclude=False)
    assert len(set(logits.tolist())) == 1
    np.testing.assert_array_equal(np.diff(ranks), 1)            # adjacent, in row order


def test_nan_weights_rank_nothing():
    eng, cfg, ocfg, W, tabs, rng = make(g.MODEL_DIN_COS, D=32, S=10, I=500)
    W = [np.array(w, np.float32) for w in W]
    W[2].ravel()[0] = np.nan
    eng.set_weights(*W)
    hist = user_hist(rng, 10, 500)
    ranks, logits = eng.rank_items(np.full(5, 2, np.int32), np.tile(hist, (5, 1)), [0, 1, 250, 499, 499])
    assert (ranks == -1).all() and np.isnan(logits).all()


def test_target_in_its_own_window():
    I, S = 800, 16
    eng, cfg, ocfg, W, tabs, rng = make(g.MODEL_YOUTUBE, D=32, S=S, I=I)
    hist = user_hist(rng, S, I)
    t = np.array([hist[0], hist[2], hist[0]], np.int32)
    for ex in (True, False):
        ranks, _ = check_ranks(eng, cfg, 5, hist, t, I, exclude=ex)
        assert (ranks == -1).all() if ex else (ranks > 0).all()


def test_rows_outside_their_tables():
    I, S = 500, 16
    eng, cfg, ocfg, W, tabs, rng = make(g.MODEL_DIN_COS, D=32, S=S, I=I)
    hist = user_hist(rng, S, I)
    hist[[2, 5]] = [I + 7, -5]
    for user in (97 + 3, -2):
        ranks, _ = check_ranks(eng, cfg, user, hist, np.array([0, 17, I - 1, -7, I, 2**31 - 1], np.int32), I)
        assert (ranks[3:] == -1).all()


def test_grouping_does_not_change_ranks():
    I, S = 1300, 12
    eng, cfg, ocfg, W, tabs, rng = make(g.MODEL_DIN_EUC, D=64, S=S, I=I)
    users = np.array([1, 50, 96, 50], np.int32)
    hists = np.stack([user_hist(rng, S, I) for _ in users])
    hists[3] = hists[1]; hists[3, 0] = (hists[1, 0] + 1) % I          # user 50 with two windows
    n = 60
    which = rng.integers(0, users.size, n)
    u = users[which]; h = hists[which]; t = rng.integers(-2, I + 2, n).astype(np.int32)
    t[:5] = h[:5, 0]                                                   # some in their own window
    ranks, logits = eng.rank_items(u, h, t)
    perm = rng.permutation(n)
    r2, l2 = eng.rank_items(u[perm], h[perm], t[perm])
    assert r2.tobytes() == ranks[perm].tobytes() and l2.tobytes() == logits[perm].tobytes()
    for i in range(n):
        r1, l1 = eng.rank_items(u[i:i + 1], h[i:i + 1], t[i:i + 1])
        assert r1[0] == ranks[i] and l1.tobytes() == logits[i:i + 1].tobytes(), i


def test_a_group_beyond_1024_targets_takes_several_passes():
    I, S = 1500, 8
    eng, cfg, ocfg, W, tabs, rng = make(g.MODEL_DIN_COS, D=16, S=S, I=I)
    hist = user_hist(rng, S, I)
    t = np.arange(I, dtype=np.int32)
    ranks, logits = eng.rank_items(np.full(I, 4, np.int32), np.tile(hist, (I, 1)), t, exclude_history=False)
    assert sorted(ranks.tolist()) == list(range(1, I + 1))             # every item once, no excluded rows
    order = np.lexsort((t, -logits.astype(np.float64)))                # the ranks follow the call's own logits
    np.testing.assert_array_equal(ranks[order], np.arange(1, I + 1))
    rows, _, lg, cnt = eng.recommend_topk([4], hist[None, :], 1024, exclude_history=False)
    np.testing.assert_array_equal(rows[0], t[order][:1024])
    assert lg[0].tobytes() == logits[order][:1024].tobytes()


def test_live_updates_are_seen_by_the_next_call():
    I, S, D, cF = 900, 20, 32, 9
    eng, cfg, ocfg, W, tabs, rng = make(g.MODEL_DIN_COS, D=D, S=S, I=I, cF=cF)
    hist = user_hist(rng, S, I)
    t = np.array([10, 450, 899], np.int32)
    _, before = check_ranks(eng, cfg, 7, hist, t, I)
    # a written ITEM_EMB row
    eng.table_write_rows(g.TABLE_ITEM_EMB, [450], (rng.standard_normal((1, D)) * 3).astype(np.float32))
    _, after = check_ranks(eng, cfg, 7, hist, t, I)
    assert after[1] != before[1] and after[0] == before[0]
    # new weights
    W2 = [np.array(w, np.float32) * 1.5 for w in W]
    eng.set_weights(*W2)
    check_ranks(eng, cfg, 7, hist, t, I)


def test_ubcache_append_is_seen_by_evaluate():
    eng, ocfg, W, tabs, (uid, iid), (off, ts, items, lens), rng = _serving_engine(g.MODEL_DIN_COS)
    eng.ubcache_upload(off, ts, items)
    u = int(uid[3])
    win = eng.ubcache_window(eng.idmap_lookup(g.IDMAP_USER, [u]), [5000])[0]
    it = int(iid[next(r for r in range(iid.size) if r not in win)])
    held = [serving.Sample(u, it, 5000)]
    assert serving.Evaluate(eng, held, ks=(150,))["HR@150"] == 1.0
    serving.UserBehaviorCache(eng).Append([u], [it], [4000])
    assert serving.Evaluate(eng, held, ks=(150,))["HR@150"] == 0.0       # now in the window: excluded
    assert serving.Evaluate(eng, held, ks=(150,), exclude_history=False)["HR@150"] == 1.0


def test_evaluate_equals_rank_metrics_of_the_ranks():
    eng, ocfg, W, tabs, (uid, iid), (off, ts, items, lens), rng = _serving_engine(g.MODEL_YOUTUBE)
    eng.ubcache_upload(off, ts, items)
    n = 40
    us = uid[rng.integers(0, uid.size, n)]; its = iid[rng.integers(0, iid.size, n)]; tss = rng.integers(0, 1000, n)
    tss[::3] = 500
    its[0] = 10**15                                                      # unknown item: a miss
    held = [serving.Sample(int(a), int(b), int(c)) for a, b, c in zip(us, its, tss)]
    got = serving.Evaluate(eng, held, ks=(1, 10, 50))
    rows = eng.idmap_lookup(g.IDMAP_USER, us)
    ranks, _ = eng.rank_items(rows, eng.ubcache_window(rows, tss), eng.idmap_lookup(g.IDMAP_ITEM, its))
    assert ranks[0] == -1
    key = {}
    groups = [key.setdefault((int(a), int(c)), len(key)) for a, c in zip(us, tss)]
    hit, rec, ndcg, mrr = g.rank_metrics(ranks, groups, [1, 10, 50])
    for a, k in enumerate((1, 10, 50)):
        assert got["HR@%d" % k] == hit[a] and got["Recall@%d" % k] == rec[a] and got["NDCG@%d" % k] == ndcg[a]
    assert got["MRR"] == mrr
    with pytest.raises(g.CtrError) as e:
        serving.Evaluate(eng, [serving.Sample(10**15 + 3, int(iid[0]), 0)])
    assert e.value.code == g.ENOTFOUND


def _raw(eng, n=1, null=None):
    S = eng.cfg.S
    u = np.zeros(max(n, 1), np.int32); h = np.full((max(n, 1), S), -1, np.int32); t = np.zeros(max(n, 1), np.int32)
    rk = np.full(max(n, 1), 77, np.int64); lg = np.full(max(n, 1), 9.25, np.float32)
    ip = C.POINTER(C.c_int32)
    ptr = {"user": u.ctypes.data_as(ip), "hist": h.ctypes.data_as(ip), "item": t.ctypes.data_as(ip), "rank": rk.ctypes.data_as(C.POINTER(C.c_int64))}
    if null:
        ptr[null] = None
    rc = eng.L.ctr_rank_items(eng.h, ptr["user"], ptr["hist"], ptr["item"], C.c_int64(n), C.c_int32(1), ptr["rank"],
                              lg.ctypes.data_as(C.POINTER(C.c_float)))
    return rc, bool((rk == 77).all() and (lg == 9.25).all())


def test_refusals_write_nothing():
    eng, cfg, ocfg, W, tabs, rng = make(g.MODEL_DIN_COS, D=16, S=8, I=50)
    assert _raw(eng) == (0, False)
    assert _raw(eng, n=0) == (g.EINVAL, True)
    for null in ("user", "hist", "item", "rank"):
        assert _raw(eng, null=null) == (g.EINVAL, True), null
    ranks = np.empty(1, np.int64)
    one = np.zeros(1, np.int32); hist = np.full(8, -1, np.int32)
    ip = C.POINTER(C.c_int32)
    assert eng.L.ctr_rank_items(eng.h, one.ctypes.data_as(ip), hist.ctypes.data_as(ip), one.ctypes.data_as(ip), C.c_int64(1), C.c_int32(1),
                                ranks.ctypes.data_as(C.POINTER(C.c_int64)), None) == 0      # out_logit may be NULL
    bare = g.Engine(g.engine.default_config(g.MODEL_DIN_COS, uP=0, S=8, D=16, cF=0, batch=64, pred_batch=64))
    assert _raw(bare) == (g.ESTATE, True)
    with pytest.raises(g.CtrError) as e:
        bare.rank_items([0], hist[None, :], [0])
    assert e.value.code == g.ESTATE


def test_profile_keys():
    I = 1000
    eng, cfg, ocfg, W, tabs, rng = make(g.MODEL_DIN_COS, D=32, S=20, I=I)      # chunks of 256: 4
    hist = user_hist(rng, 20, I)
    eng.profile(True)
    eng.profile_reset()
    eng.rank_items(np.full(4, 3, np.int32), np.tile(hist, (4, 1)), [0, 5, 700, I + 1])
    prof = eng.profile_dump()
    eng.profile(False)
    assert not {"rec_topk", "rec_merge", "rec_finish"} & set(prof), sorted(prof)
    assert prof["rank_target"][1] == 2 + 1          # chunks 0 and 2, then the sort
    assert prof["rank_count"][1] == 4 + 1           # every chunk, then the ranks
    assert prof["attn_fwd_user"][1] == 2 + 4 and prof["head_fwd"][1] == 2 + 4
