"""ctr_recommend_topk: score every ITEM_EMB row for a user with the trained model and return the best k
(recommend/api.go:115-118, "todo: some default recall algorithm").

The list must be exactly the (logit descending, row ascending) order of the logits the engine's own forward computes for
(user, every item, hist) — ctr_debug_grads_idx(training=0) — with those logits and scores bit for bit; the logits must
also agree with the double-accumulating oracle at the parity bar, and the list with the oracle's up to near-ties."""
import ctypes as C

import numpy as np
import pytest

import go_ctr_b200 as g
from go_ctr_b200 import serving
from oracle import oracle as orc
from tests.test_gpu_parity import SCORE_RTOL
from tests.test_gpu_serving import _serving_engine
from tests.util import make_tables, scaled_init

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]

MODELS = [g.MODEL_YOUTUBE, g.MODEL_DIN_COS, g.MODEL_DIN_EUC]


def make(model, D=32, S=50, I=1000, U=97, uP=12, cF=9, H0=200, H1=80, pred_batch=256, seed=0, **kw):
    rng = np.random.default_rng(seed)
    cfg = g.engine.default_config(model, uP=uP, S=S, D=D, cF=cF, H0=H0, H1=H1, batch=pred_batch, pred_batch=pred_batch,
                                  seed=seed + 5, **kw)
    eng = g.Engine(cfg)
    uf, itf, emb = make_tables(rng, U, I, uP, cF, D)
    if uP:
        eng.table_upload(g.TABLE_USER_FEAT, uf)
    if cF:
        eng.table_upload(g.TABLE_ITEM_FEAT, itf)
    eng.table_upload(g.TABLE_ITEM_EMB, emb)
    ocfg = orc.make_cfg(model, uP, S, D, cF, H0, H1)
    W = scaled_init(orc, ocfg, seed + 1)
    eng.set_weights(*W)
    return eng, cfg, ocfg, W, (uf, itf, emb), rng


def user_hist(rng, S, I, n_valid=None):
    """A history with repeated items and a -1 padded tail."""
    n_valid = min(S, max(1, (2 * S) // 3)) if n_valid is None else n_valid
    h = np.full(S, -1, np.int32)
    h[:n_valid] = rng.integers(0, I, n_valid)
    if n_valid >= 4:
        h[1] = h[0]; h[3] = h[2]
    return h


def engine_forward(eng, cfg, user, hist, I):
    """The engine's own forward of (user, item, hist) for every item, in chunks of the handle's batch."""
    B = max(cfg.batch, cfg.pred_batch)
    z = np.empty(I, np.float32); p = np.empty(I, np.float32)
    for s in range(0, I, B):
        n = min(B, I - s)
        out = eng.debug_grads_idx(np.full(n, user, np.int32), np.arange(s, s + n, dtype=np.int32),
                                  np.tile(hist, (n, 1)), np.zeros(n, np.float32), training=False)
        z[s:s + n] = out["logit"]; p[s:s + n] = out["p"]
    return z, p


def expected(z, hist, I, k, exclude):
    """numpy restatement of the order: logit descending, then row ascending; NaN and (optionally) history excluded."""
    rows = np.arange(I)
    ok = ~np.isnan(z)
    if exclude:
        ok &= ~np.isin(rows, hist[(hist >= 0) & (hist < I)])
    rows = rows[ok]
    order = np.lexsort((rows, -z[ok].astype(np.float64)))
    return rows[order][:k].astype(np.int32)


def check_exact(eng, cfg, user, hist, I, k, exclude=True, exact=True):
    """exact=False: the one instantiation whose rows are not bit-identical to the predict route's (euclid, D = 16: the
    last bit of some logits differs); the list is then held to the engine's forward up to near-ties at 1e-6."""
    rows, scores, logits, cnt = eng.recommend_topk([user], hist[None, :], k, exclude_history=exclude)
    z, p = engine_forward(eng, cfg, user, hist, I)
    want = expected(z, hist, I, k, exclude)
    n = want.size
    assert cnt[0] == n
    assert (rows[0, n:] == -1).all() and (scores[0, n:] == 0).all() and (logits[0, n:] == 0).all()
    if not exact:
        got = rows[0, :n]
        np.testing.assert_allclose(logits[0, :n], z[got], rtol=1e-6, atol=1e-7)
        check_near_ties(got, z.astype(np.float64), hist, k, exclude, 1e-6 * np.abs(z).max())
        return got, logits[0, :n], z
    np.testing.assert_array_equal(rows[0, :n], want)
    assert logits[0, :n].tobytes() == z[want].tobytes(), "logits differ from the engine's forward"
    assert scores[0, :n].tobytes() == p[want].tobytes(), "scores differ from the engine's forward"
    if n:
        pi = eng.predict_idx(np.full(n, user, np.int32), want, np.tile(hist, (n, 1)))
        assert scores[0, :n].tobytes() == pi.tobytes(), "scores differ from ctr_predict_idx"
    return rows[0, :n], logits[0, :n], z


def oracle_logits(ocfg, W, tabs, user, hist, I):
    uf, itf, emb = tabs
    X = orc.gather_rows(uf, itf, emb, np.full(I, user, np.int32), np.arange(I, dtype=np.int32), np.tile(hist, (I, 1)))
    _, z = orc.forward(ocfg, W, X, orc.make_ranges(ocfg.uP, ocfg.S, ocfg.D, ocfg.cF))
    return np.asarray(z, np.float64).ravel()


def check_near_ties(rows, zo, hist, k, exclude, tol):
    """Every returned item is within tol of the oracle's k-th best; no unreturned eligible item beats the returned
    k-th by more than tol."""
    I = zo.size
    ok = np.ones(I, bool)
    if exclude:
        ok &= ~np.isin(np.arange(I), hist[(hist >= 0) & (hist < I)])
    elig = np.flatnonzero(ok)
    kk = min(k, elig.size)
    assert rows.size == kk
    if kk == 0:
        return
    kth = np.sort(zo[elig])[::-1][kk - 1]
    assert (zo[rows] >= kth - tol).all(), "a returned item is far below the oracle's k-th best"
    rest = np.setdiff1d(elig, rows)
    if rest.size:
        assert zo[rest].max() <= zo[rows].min() + tol, "an unreturned item beats the returned k-th"


def dispatch(eng, attn):
    prof = eng.profile_dump()
    assert {k for k in prof if k.startswith("attn_")} == {"attn_fwd_" + attn}, sorted(prof)
    mm = {k for k in prof if k.startswith(("umma_", "sgemm_"))}
    assert mm in ({"umma_fwd0_sigmoid", "umma_fwd1_sigmoid"}, {"sgemm_fwd0_sigmoid", "sgemm_fwd1_sigmoid"}), sorted(prof)
    assert {"head_fwd", "rec_topk", "rec_merge", "rec_finish"} <= set(prof), sorted(prof)
    return mm


def run_case(model, D, S, I, k, attn, gemm="umma", seed=0, **kw):
    eng, cfg, ocfg, W, tabs, rng = make(model, D=D, S=S, I=I, seed=seed, **kw)
    user = int(rng.integers(0, 97)); hist = user_hist(rng, S, I)
    eng.profile(True)
    eng.recommend_topk([user], hist[None, :], k)
    mm = dispatch(eng, attn)
    assert next(iter(mm)).startswith(gemm + "_"), sorted(mm)
    eng.profile(False)
    rows, logits, z = check_exact(eng, cfg, user, hist, I, k, exact=not (model == g.MODEL_DIN_EUC and D == 16))
    zo = oracle_logits(ocfg, W, tabs, user, hist, I)
    np.testing.assert_allclose(z, zo, rtol=SCORE_RTOL, atol=2e-5)
    check_near_ties(rows, zo, hist, k, True, SCORE_RTOL * np.abs(zo).max() + 2e-5)


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("D", [16, 32, 64, 128])
def test_lane_maps(model, D):
    run_case(model, D, 50, 1000, 20, "user")


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("S", [1, 100])
def test_history_lengths(model, S):
    """S = 100 is beyond the _idx kernels' two history ids per lane."""
    run_case(model, 64, S, 5000, 50, "user")


@pytest.mark.parametrize("I", [1, 37, 1000, 5000])
def test_catalogue_sizes(I):
    """Several chunks of 256 rows and a ragged last one; a catalogue smaller than one chunk."""
    run_case(g.MODEL_DIN_COS, 32, 20, I, 10, "user")


@pytest.mark.parametrize("model", MODELS)
def test_generic_fallback(model):
    """D = 7 (model_test.go:24-28) has no lane map: index buffers for the ordinary _gen kernel."""
    run_case(model, 7, 10, 1000, 15, "gen", uP=5, cF=3)


def test_history_beyond_shared_memory_falls_back():
    """A history whose rows do not fit the opt-in shared memory takes the _vec kernel over index buffers."""
    run_case(g.MODEL_DIN_EUC, 128, 500, 600, 10, "vec", uP=8, cF=4)


@pytest.mark.parametrize("model", [g.MODEL_DIN_COS, g.MODEL_DIN_EUC])
def test_fp32_gemms(model):
    eng, cfg, ocfg, W, tabs, rng = make(model, D=64, S=50, I=1000, gemm=g.GEMM_FP32)
    user = 3; hist = user_hist(rng, 50, 1000)
    eng.profile(True)
    eng.recommend_topk([user], hist[None, :], 20)
    assert dispatch(eng, "user") == {"sgemm_fwd0_sigmoid", "sgemm_fwd1_sigmoid"}
    eng.profile(False)
    check_exact(eng, cfg, user, hist, 1000, 20)


def test_wide_hidden_layer_fp32_route():
    """H0 = 300 is past the wgmma tile widths: the fp32 GEMMs run."""
    eng, cfg, ocfg, W, tabs, rng = make(g.MODEL_DIN_COS, D=32, S=30, I=1500, H0=300)
    user = 5; hist = user_hist(rng, 30, 1500)
    eng.profile(True)
    eng.recommend_topk([user], hist[None, :], 25)
    assert dispatch(eng, "user") == {"sgemm_fwd0_sigmoid", "sgemm_fwd1_sigmoid"}
    eng.profile(False)
    rows, logits, z = check_exact(eng, cfg, user, hist, 1500, 25)
    zo = oracle_logits(ocfg, W, tabs, user, hist, 1500)
    np.testing.assert_allclose(z, zo, rtol=SCORE_RTOL, atol=2e-5)


def test_k_bounds_short_results_and_exclusion():
    I = 37
    eng, cfg, ocfg, W, tabs, rng = make(g.MODEL_DIN_COS, D=16, S=12, I=I)
    hist = np.array([4, 4, 9, 30, 9, 2, -1, -1, -1, -1, -1, -1], np.int32)
    for k, ex in ((1, True), (1, False), (I, False), (I, True), (50, True), (1024, False)):
        rows, logits, z = check_exact(eng, cfg, 7, hist, I, k, exclude=ex)
        assert rows.size == min(k, I - (4 if ex else 0))
        if ex:
            assert not np.isin(rows, [2, 4, 9, 30]).any()
        else:
            assert np.isin([2, 4, 9, 30], rows).all() or k < I


def test_empty_history():
    eng, cfg, ocfg, W, tabs, rng = make(g.MODEL_DIN_EUC, D=64, S=50, I=700)
    hist = np.full(50, -1, np.int32)
    check_exact(eng, cfg, 11, hist, 700, 30)


def test_exact_ties_come_in_row_order():
    I, D, cF = 400, 32, 9
    eng, cfg, ocfg, W, (uf, itf, emb), rng = make(g.MODEL_DIN_COS, D=D, S=20, I=I, cF=cF)
    emb = emb.copy(); itf = itf.copy()
    dup = [5, 120, 121, 399]
    emb[dup] = emb[dup[0]] * 4.0; itf[dup] = itf[dup[0]]      # large norm: the duplicates rank first
    eng.table_upload(g.TABLE_ITEM_EMB, emb); eng.table_upload(g.TABLE_ITEM_FEAT, itf)
    hist = user_hist(rng, 20, I)
    hist[hist == 5] = 6
    rows, logits, z = check_exact(eng, cfg, 3, hist, I, I, exclude=False)
    pos = [int(np.flatnonzero(rows == d)[0]) for d in dup]
    assert pos == sorted(pos) and np.ptp(pos) == 3, pos            # adjacent, in row order
    assert len(set(logits[pos].tolist())) == 1


def test_several_users_equal_single_calls():
    I, S = 1300, 40
    eng, cfg, ocfg, W, tabs, rng = make(g.MODEL_DIN_EUC, D=64, S=S, I=I)
    users = np.array([1, 50, 96], np.int32)
    hists = np.stack([user_hist(rng, S, I) for _ in users])
    rows, scores, logits, cnt = eng.recommend_topk(users, hists, 33)
    for j, u in enumerate(users):
        r1, s1, l1, c1 = eng.recommend_topk([u], hists[j:j + 1], 33)
        assert c1[0] == cnt[j]
        assert rows[j].tobytes() == r1[0].tobytes() and scores[j].tobytes() == s1[0].tobytes()
        assert logits[j].tobytes() == l1[0].tobytes()


def test_rows_outside_their_tables_read_as_missing():
    I, S = 500, 16
    eng, cfg, ocfg, W, tabs, rng = make(g.MODEL_DIN_COS, D=32, S=S, I=I)
    hist = user_hist(rng, S, I)
    hist[[2, 5]] = [I + 7, -5]
    for user in (97 + 3, -2):
        rows, logits, z = check_exact(eng, cfg, user, hist, I, 40)
        zo = oracle_logits(ocfg, W, tabs, -1, np.where((hist >= 0) & (hist < I), hist, -1), I)
        np.testing.assert_allclose(z, zo, rtol=SCORE_RTOL, atol=2e-5)


def test_argument_errors():
    eng, cfg, ocfg, W, tabs, rng = make(g.MODEL_DIN_COS, D=16, S=8, I=50)
    hist = user_hist(rng, 8, 50)
    for k in (0, 1025):
        with pytest.raises(g.CtrError) as e:
            eng.recommend_topk([1], hist[None, :], k)
        assert e.value.code == g.EINVAL
    out_r = np.empty(4, np.int32); out_s = np.empty(4, np.float32); cnt = np.empty(1, np.int32)
    u = np.array([1], np.int32)
    ip = C.POINTER(C.c_int32); fp = C.POINTER(C.c_float)
    args = [u.ctypes.data_as(ip), hist.ctypes.data_as(ip), C.c_int64(1), C.c_int32(4), C.c_int32(1),
            out_r.ctypes.data_as(ip), out_s.ctypes.data_as(fp), None, cnt.ctypes.data_as(ip)]
    assert eng.L.ctr_recommend_topk(eng.h, *args) == 0                     # out_logits may be NULL
    for i in (5, 6, 8):
        bad = list(args); bad[i] = None
        assert eng.L.ctr_recommend_topk(eng.h, *bad) == g.EINVAL
    bad = list(args); bad[2] = C.c_int64(0)
    assert eng.L.ctr_recommend_topk(eng.h, *bad) == g.EINVAL
    bare = g.Engine(g.engine.default_config(g.MODEL_DIN_COS, uP=0, S=8, D=16, cF=0, batch=64, pred_batch=64))
    with pytest.raises(g.CtrError) as e:
        bare.recommend_topk([0], hist[None, :], 3)
    assert e.value.code == g.ESTATE


def test_sees_table_and_weight_updates():
    """After training steps with the fused row SGD, the call scores with the updated table and weights."""
    I, U, S, D, uP, cF = 900, 97, 30, 64, 12, 9
    eng, cfg, ocfg, W, tabs, rng = make(g.MODEL_DIN_COS, D=D, S=S, I=I, U=U, uP=uP, cF=cF,
                                        table_opt=g.TABLE_SGD, table_lr=0.5)
    uf, itf, _ = tabs
    B = cfg.batch
    for _ in range(3):
        ur = rng.integers(0, U, B).astype(np.int32); ir = rng.integers(0, I, B).astype(np.int32)
        hs = rng.integers(-1, I, (B, S)).astype(np.int32); y = (rng.random(B) > 0.5).astype(np.float32)
        eng.train_step_idx(ur, ir, hs, y)
    hist = user_hist(rng, S, I)
    rows, scores, logits, cnt = eng.recommend_topk([9], hist[None, :], 40)
    emb = eng.table_download(g.TABLE_ITEM_EMB, I, D)
    W2 = [np.asarray(w, np.float32).reshape(np.asarray(w0).shape) for w, w0 in zip(eng.get_weights(), W)]
    zo = oracle_logits(ocfg, W2, (uf, itf, emb), 9, hist, I)
    np.testing.assert_allclose(logits[0], zo[rows[0]], rtol=SCORE_RTOL, atol=2e-5)
    check_near_ties(rows[0, :cnt[0]], zo, hist, 40, True, SCORE_RTOL * np.abs(zo).max() + 2e-5)


def test_serving_recommend_matches_rank_over_every_item():
    eng, ocfg, W, tabs, (uid, iid), (off, ts, items, lens), rng = _serving_engine(g.MODEL_DIN_COS)
    eng.ubcache_upload(off, ts, items)
    now = 700
    for u in (int(uid[int(np.argmax(lens))]), int(uid[0])):
        rec = serving.Recommend(eng, u, 12, now=now, exclude_history=False)
        ranked = serving.Rank(eng, u, iid.tolist(), now=now)
        score_of = {r.ItemId: r.Score for r in ranked}
        assert len(rec) == 12
        assert [r.Score for r in rec] == sorted((r.Score for r in rec), reverse=True)
        for r in rec:
            assert np.float32(r.Score).tobytes() == np.float32(score_of[r.ItemId]).tobytes()
        top = sorted((r.Score for r in ranked), reverse=True)[:12]
        assert sorted(r.Score for r in rec) == sorted(top)
    with pytest.raises(g.CtrError) as e:
        serving.Recommend(eng, 10_000_000 + 77, 5)
    assert e.value.code == g.ENOTFOUND
