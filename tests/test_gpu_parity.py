"""GPU parity tests proper: the CUDA path, called through the C ABI, against the CPU oracle on the
same seeded inputs.  Bars (BASELINE.json north_star): index gather bit-exact; forward scores and
pre-sigmoid logits within 1e-4 relative; AUC within ±0.002."""
import numpy as np
import pytest

import go_ctr_b200 as g
from oracle import oracle as orc
from tests.util import assert_mostly_close, make_batch, make_tables, scaled_init

pytestmark = pytest.mark.gpu

SCORE_RTOL = 1e-4       # north_star: "within 1e-4 relative on forward scores"
# weight gradients: error-compensated 3xTF32 on the wgmma engine (umma_gemm.cuh k_umma_dw), fp32 FFMA otherwise — both
# are float32-grade sums over the batch, compared with the double-accumulating oracle: the absolute part of the bound is
# relative to the largest gradient entry (cancellation in small entries), not to each entry
GRAD_RTOL = 2e-4
GRAD_ATOL = 1e-5

# (uP, S, D, cF): reference movielens dims (rcmd.go:22-24), north-star dims, the reference test's odd
# dims (model_test.go:24-28, generic kernels), and a >64 history (index-prefetch fallback)
SHAPES = {"ref": (52, 10, 16, 53), "ns": (52, 50, 64, 53), "odd": (5, 3, 7, 5), "long": (8, 70, 32, 9), "d128": (4, 6, 128, 4)}
MODELS = [g.MODEL_YOUTUBE, g.MODEL_DIN_COS, g.MODEL_DIN_EUC]


def setup(model, shape, B, seed=0, U=97, I=211, H0=200, H1=80, hot_rows=0, pred_batch=None, **kw):
    """shape: a SHAPES name or a (uP, S, D, cF) tuple.  A zero-width feature table is not uploaded.  hot_rows: the
    replicated hot-row count of the fused SGD scatter (cfg.reserved[0]: 0 = auto, < 0 = off).  pred_batch defaults
    to the training batch B."""
    uP, S, D, cF = SHAPES[shape] if isinstance(shape, str) else shape
    rng = np.random.default_rng(seed)
    cfg = g.engine.default_config(model, uP=uP, S=S, D=D, cF=cF, H0=H0, H1=H1, batch=B, pred_batch=pred_batch or B,
                                  seed=seed + 5, **kw)
    cfg.reserved[0] = hot_rows
    eng = g.Engine(cfg)
    uf, itf, emb = make_tables(rng, U, I, uP, cF, D)
    if uP:
        eng.table_upload(g.TABLE_USER_FEAT, uf)
    if cF:
        eng.table_upload(g.TABLE_ITEM_FEAT, itf)
    eng.table_upload(g.TABLE_ITEM_EMB, emb)
    ocfg = orc.make_cfg(model, uP, S, D, cF, H0, H1, cfg.dropout0, cfg.dropout1)
    W = scaled_init(orc, ocfg, seed + 1)
    eng.set_weights(*W)
    batch = make_batch(rng, U, I, B, S)
    return eng, cfg, ocfg, W, (uf, itf, emb), batch


@pytest.mark.parametrize("shape", list(SHAPES))
def test_gather_is_bit_exact(shape):
    """recommend.GetSampleVector (rcmd.go:462-536) from the HBM tables == the oracle, bit for bit."""
    eng, cfg, ocfg, W, (uf, itf, emb), (ur, ir, hist, y) = setup(g.MODEL_DIN_COS, shape, 333)
    ir = ir.copy(); ir[::17] = -1                     # missing item → zeros (rcmd.go:502-505)
    X = eng.gather_rows(ur, ir, hist)
    # oracle treats item_row<0 as zeros for both the embedding and the feature
    assert X.tobytes() == orc.gather_rows(uf, itf, emb, ur, ir, hist).tobytes()


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("model", MODELS)
def test_forward_scores_and_logits(model, shape):
    eng, cfg, ocfg, W, (uf, itf, emb), (ur, ir, hist, y) = setup(model, shape, 257)
    out = eng.debug_grads_idx(ur, ir, hist, y, training=False)
    X = orc.gather_rows(uf, itf, emb, ur, ir, hist)
    o0 = orc.make_cfg(model, ocfg.uP, ocfg.S, ocfg.D, ocfg.cF, 200, 80)
    p, z = orc.forward(o0, W, X, orc.make_ranges(ocfg.uP, ocfg.S, ocfg.D, ocfg.cF))
    np.testing.assert_allclose(out["logit"], z, rtol=SCORE_RTOL, atol=2e-5)
    np.testing.assert_allclose(out["p"], p, rtol=SCORE_RTOL, atol=1e-7)
    np.testing.assert_allclose(eng.predict_idx(ur, ir, hist), p, rtol=SCORE_RTOL, atol=1e-7)


@pytest.mark.parametrize("shape", ["ref", "ns", "odd"])
@pytest.mark.parametrize("model", MODELS)
def test_gradients(model, shape):
    """What G.Grad(cost, Learnable...) computes (model.go:56) + the engine's row gradients."""
    eng, cfg, ocfg, W, (uf, itf, emb), (ur, ir, hist, y) = setup(model, shape, 192, seed=3)
    out = eng.debug_grads_idx(ur, ir, hist, y, training=False)
    X = orc.gather_rows(uf, itf, emb, ur, ir, hist)
    o0 = orc.make_cfg(model, ocfg.uP, ocfg.S, ocfg.D, ocfg.cF, 200, 80)
    ws = orc.Workspace(o0, len(y))
    orc.forward(o0, W, X, orc.make_ranges(ocfg.uP, ocfg.S, ocfg.D, ocfg.cF), ws=ws)
    ref = orc.backward(o0, W, ws, y)
    assert abs(out["cost"] - ref["cost"]) <= 1e-5 * max(1.0, abs(ref["cost"]))
    for k in ("dW0", "dW1", "dW2"):
        scale = np.abs(ref[k]).max()
        np.testing.assert_allclose(out[k], ref[k], rtol=GRAD_RTOL, atol=GRAD_ATOL * scale + 1e-12, err_msg=k)
    np.testing.assert_allclose(out["dIt"], ref["dIt"], rtol=2e-3, atol=1e-4 * np.abs(ref["dIt"]).max() + 1e-12, err_msg="dIt")
    if model != g.MODEL_YOUTUBE:
        np.testing.assert_allclose(out["datt"], ref["datt"], rtol=2e-3, atol=2e-5 * np.abs(ref["datt"]).max() + 1e-12)
    valid = hist >= 0                                   # gradients of padded slots are never scattered
    scale = np.abs(ref["dUb"]).max()
    np.testing.assert_allclose(out["dUb"][valid], ref["dUb"][valid], rtol=2e-3, atol=2e-5 * scale + 1e-12)


def test_dropout_masks_match_the_shared_counter_rng():
    eng, cfg, ocfg, W, (uf, itf, emb), (ur, ir, hist, y) = setup(g.MODEL_DIN_COS, "ref", 128, dropout0=0.3, dropout1=0.2)
    out = eng.debug_grads_idx(ur, ir, hist, y, training=True)
    X = orc.gather_rows(uf, itf, emb, ur, ir, hist)
    p, z = orc.forward(ocfg, W, X, orc.make_ranges(ocfg.uP, ocfg.S, ocfg.D, ocfg.cF), training=True, seed=cfg.seed, step=0)
    np.testing.assert_allclose(out["logit"], z, rtol=SCORE_RTOL, atol=2e-5)
    p_nodrop, _ = orc.forward(ocfg, W, X, orc.make_ranges(ocfg.uP, ocfg.S, ocfg.D, ocfg.cF))
    assert np.abs(p - p_nodrop).max() > 1e-3            # the masks did something


@pytest.mark.parametrize("model", [g.MODEL_DIN_COS, g.MODEL_YOUTUBE])
def test_train_dense_matches_model_train(model):
    """model.Train (model.go:27-213): batching, zero-padded ragged tail trained as label 0,
    Adam+L2+1/B, epoch cost = last batch, then model.Predict with its own ragged tail."""
    rng = np.random.default_rng(9)
    uP, S, D, cF, N, B = 5, 3, 7, 5, 1090, 200          # 1090 = 5*200 + 90 → ragged tail
    X = rng.random((N, uP + S * D + D + cF), np.float32)
    Y = (rng.random(N) > 0.5).astype(np.float32)
    si = g.SampleInfo((0, uP), (uP, uP + S * D), (uP + S * D, uP + S * D + D), (uP + S * D + D, uP + S * D + D + cF))
    drop = 0.003 if model == g.MODEL_YOUTUBE else 0.005
    ocfg = orc.make_cfg(model, uP, S, D, cF, 200, 80, drop, drop)
    W = scaled_init(orc, ocfg, 4, 0.2, 0.1, 0.3)
    net = (g.NewYoutubeDnn if model == g.MODEL_YOUTUBE else g.NewDinNet)(uP, S, D, D, cF, seed=21)
    net.weights = tuple(w.copy() for w in W)
    ep, cost = g.Train(uP, S, D, D, cF, N, B, 3, 0, si, X, Y, net)
    Wo = [w.copy() for w in W]
    oep, ocost = orc.train_dense(ocfg, orc.default_solver(seed=21), Wo, X, Y, orc.make_ranges(uP, S, D, cF), B, 3, 0)
    assert ep == oep == 3
    assert abs(cost - ocost) <= 2e-4 * max(1.0, abs(ocost)), (cost, ocost)
    for a, b, name in zip(net.weights, Wo, ("mlp0", "mlp1", "mlp2", "att0")):
        assert_mostly_close(a, b, 2e-3, 2e-4, 0.995, name)
    # predict: JSON round trip like dinimpl.go:73-89, 118 rows with batch 20 (model_test.go:33-34)
    pred_net = (g.NewYoutubeDnnFromJson if model == g.MODEL_YOUTUBE else g.NewDinNetFromJson)(net.Marshal())
    g.InitForwardOnlyVm(uP, S, D, D, cF, 20, pred_net)
    got = g.Predict(pred_net, 118, 20, si, X)
    assert got.shape == (118,)
    o0 = orc.make_cfg(model, uP, S, D, cF, 200, 80)
    want = orc.predict_dense(o0, [np.ascontiguousarray(w) for w in net.weights], X[:118], orc.make_ranges(uP, S, D, cF), 20)
    np.testing.assert_allclose(got, want, rtol=SCORE_RTOL, atol=1e-7)


def test_early_stop_follows_last_batch_cost():
    """model.go:198-209: an lr of 0 never improves the cost → stops after earlyStop+... epochs."""
    rng = np.random.default_rng(1)
    uP, S, D, cF, N, B = 4, 2, 4, 4, 300, 100
    X = rng.random((N, uP + S * D + D + cF), np.float32); Y = (rng.random(N) > 0.5).astype(np.float32)
    cfg = g.engine.default_config(g.MODEL_DIN_COS, uP=uP, S=S, D=D, cF=cF, batch=B, pred_batch=B, lr=0.0, dropout0=0.0, dropout1=0.0)
    eng = g.Engine(cfg)
    ep, cost = eng.train_dense(X, Y, [0, uP, uP, uP + S * D, uP + S * D, uP + S * D + D, uP + S * D + D, uP + S * D + D + cF], 50, 3)
    assert ep == 4          # epoch 0 sets best; epochs 1..3 do not improve → break with ep == 4 epochs run


@pytest.mark.parametrize("model", MODELS)
def test_index_train_steps_with_deterministic_row_update(model):
    """gather → attention → MLP → BCE → backward → scatter-add + SGD(rows) + Adam(dense), 4 steps."""
    eng, cfg, ocfg, W, (uf, itf, emb), (ur, ir, hist, y) = setup(model, "ref", 256, seed=6, table_opt=g.TABLE_SGD_DETERMINISTIC, table_lr=0.7)
    tr = orc.IdxTrainer(ocfg, orc.default_solver(seed=cfg.seed), W, uf, itf, emb)
    rng = np.random.default_rng(66)
    for step in range(4):
        ur, ir, hist, y = make_batch(rng, uf.shape[0], itf.shape[0], 256, cfg.S, zipf=True)   # heavy duplicates
        st = eng.train_step_idx(ur, ir, hist, y)
        ocost, _ = tr.step(ur, ir, hist, y, table_lr=0.7)
        assert abs(st.cost - ocost) <= 2e-4 * max(1.0, abs(ocost)), (step, st.cost, ocost)
    for a, b, name in zip(eng.get_weights(), tr.W, ("mlp0", "mlp1", "mlp2", "att0")):
        if name == "att0" and model == g.MODEL_YOUTUBE:
            continue
        assert_mostly_close(a, b, 2e-3, 2e-4, 0.995, name)
    got = eng.table_download(g.TABLE_ITEM_EMB, *emb.shape)
    assert np.abs(tr.emb - emb).max() > 1e-5            # rows did move
    np.testing.assert_allclose(got, tr.emb, rtol=2e-4, atol=2e-6)


def test_fused_atomic_sgd_agrees_with_deterministic_update():
    """CTR_TABLE_SGD (red.global.add.v4.f32 fused into the backward kernel) vs the sorted segment
    reduction, one step from identical state: equal up to fp32 summation order and the Hogwild
    read-after-update window."""
    res = []
    for opt in (g.TABLE_SGD, g.TABLE_SGD_DETERMINISTIC):
        eng, cfg, ocfg, W, (uf, itf, emb), (ur, ir, hist, y) = setup(g.MODEL_DIN_COS, "ns", 512, seed=8, table_opt=opt, table_lr=0.5)
        eng.train_step_idx(ur, ir, hist, y)
        res.append(eng.table_download(g.TABLE_ITEM_EMB, *emb.shape))
    assert np.abs(res[1] - emb).max() > 1e-6
    np.testing.assert_allclose(res[0], res[1], rtol=1e-3, atol=1e-6)


def test_frozen_table_is_the_reference_behaviour():
    """din.go:161-169: embeddings are inputs, not learnables — the default must not touch the table."""
    eng, cfg, ocfg, W, (uf, itf, emb), (ur, ir, hist, y) = setup(g.MODEL_DIN_COS, "ref", 64)
    eng.train_step_idx(ur, ir, hist, y)
    assert eng.table_download(g.TABLE_ITEM_EMB, *emb.shape).tobytes() == emb.tobytes()


def test_auc_on_device_matches_reference_semantics():
    rng = np.random.default_rng(0)
    eng = g.Engine(g.engine.default_config(g.MODEL_YOUTUBE, batch=1, pred_batch=1))
    assert eng.roc_auc([0.1, 0.4, 0.35, 0.8], [0, 0, 1, 1]) == 0.75        # ranking_test.go:33-42
    assert eng.roc_auc([0.1, 0.35, 0.4, 0.8], [0, 1, 0, 1]) == 0.75        # util_test.go:25-32
    y = (rng.random(20600) > 0.6).astype(np.float32)
    s = np.round(rng.random(20600) * 0.5 + y * 0.2, 2).astype(np.float32)   # many ties (ranking.go:27-35)
    assert abs(eng.roc_auc(s, y) - orc.roc_auc(s, y)) < 1e-12
    assert np.isnan(eng.roc_auc([0.3, 0.4], [1, 1]))


def test_errors_are_codes_with_messages():
    eng, cfg, ocfg, W, tabs, (ur, ir, hist, y) = setup(g.MODEL_DIN_COS, "ref", 64)
    with pytest.raises(g.CtrError, match="configured batch"):
        eng.train_step_idx(ur[:32], ir[:32], hist[:32], y[:32])
    with pytest.raises(g.CtrError, match="SampleInfo"):
        eng.predict_dense(np.zeros((4, 300), np.float32), [0, 1, 1, 2, 2, 3, 3, 4])
    fresh = g.Engine(g.engine.default_config(g.MODEL_DIN_COS, batch=8, pred_batch=8))
    with pytest.raises(g.CtrError, match="not uploaded"):
        fresh.predict_idx(np.zeros(8, np.int32), np.zeros(8, np.int32), np.zeros((8, 10), np.int32))


def test_reference_synthetic_end_to_end_auc_parity():
    """model/model_test.go:18-147 at reduced size through the mirrored API: train DIN, marshal →
    json → predict 118 rows with batch 20, AUC > 0.5; and AUC within ±0.002 of the oracle trained
    from the same init on the same split (north_star)."""
    rng = np.random.default_rng(42)
    uP, S, D, cF, N, B = 5, 3, 7, 5, 20000, 200
    xu = rng.random((N, uP), np.float32); cx = rng.random((N, cF), np.float32)
    ub = np.zeros((N, S, D), np.float32); ub[:, 1] = rng.random((N, D), np.float32)
    it = rng.random((N, D), np.float32)
    lab = np.round((np.abs(xu - cx).mean(1) + np.abs(ub[:, 1] - it).mean(1)) * 0.6).astype(np.float32)   # model_test.go:64-77
    X = np.concatenate([xu, ub.reshape(N, -1), it, cx], 1)
    si = g.SampleInfo((0, uP), (uP, uP + S * D), (uP + S * D, uP + S * D + D), (uP + S * D + D, uP + S * D + D + cF))
    ntrain = 16000
    impl = g.DinImpl(S, D, PredBatchSize=20, BatchSize=B, epochs=4, earlyStop=0, seed=7)
    impl.Fit(g.TrainSample(X[:ntrain], lab[:ntrain], ntrain, X.shape[1], si))
    pred = impl.Predict(X[:118])
    assert pred.shape == (118, 1)
    assert g.RocAuc32(pred.ravel(), lab[:118]) > 0.5
    test_pred = impl.Predict(X[ntrain:]).ravel()
    auc_gpu = orc.roc_auc(test_pred, lab[ntrain:])
    ocfg = orc.make_cfg(orc.DIN_COS, uP, S, D, cF, 200, 80, 0.005, 0.005)
    Wo = [w.copy() for w in orc.init_weights(ocfg, 7)]
    orc.train_dense(ocfg, orc.default_solver(seed=7), Wo, X[:ntrain], lab[:ntrain], orc.make_ranges(uP, S, D, cF), B, 4, 0)
    o0 = orc.make_cfg(orc.DIN_COS, uP, S, D, cF, 200, 80)
    auc_cpu = orc.roc_auc(orc.predict_dense(o0, Wo, X[ntrain:], orc.make_ranges(uP, S, D, cF), 20), lab[ntrain:])
    assert auc_gpu > 0.5 and abs(auc_gpu - auc_cpu) <= 0.002, (auc_gpu, auc_cpu)


def test_full_size_properties_at_north_star_batch():
    """B=65536, S=50, D=64 (too big for the oracle): size-independent properties.
      * gather == numpy fancy indexing, bit-exact;
      * scatter-add conserves mass: sum over the table of the SGD delta == -lr * sum of all row
        gradients the backward produced (a checksum of checksums);
      * prediction is per-sample: any 1000-row slice scores the same alone as inside the batch."""
    uP, S, D, cF, B, U, I = 52, 50, 64, 53, 65536, 5000, 40000
    rng = np.random.default_rng(12)
    cfg = g.engine.default_config(g.MODEL_DIN_COS, uP=uP, S=S, D=D, cF=cF, batch=B, pred_batch=B, table_opt=g.TABLE_SGD, table_lr=100.0,
                                  dropout0=0.0, dropout1=0.0)
    eng = g.Engine(cfg)
    uf, itf, emb = make_tables(rng, U, I, uP, cF, D)
    eng.table_upload(g.TABLE_USER_FEAT, uf); eng.table_upload(g.TABLE_ITEM_FEAT, itf); eng.table_upload(g.TABLE_ITEM_EMB, emb)
    ocfg = orc.make_cfg(orc.DIN_COS, uP, S, D, cF)
    eng.set_weights(*scaled_init(orc, ocfg, 2))
    ur, ir, hist, y = make_batch(rng, U, I, B, S, zipf=True)
    X = eng.gather_rows(ur[:4096], ir[:4096], hist[:4096])
    embz = np.concatenate([emb, np.zeros((1, D), np.float32)])
    want = np.concatenate([uf[ur[:4096]], embz[hist[:4096]].reshape(4096, -1), emb[ir[:4096]], itf[ir[:4096]]], 1)
    assert X.tobytes() == want.tobytes()
    p_all = eng.predict_idx(ur, ir, hist)
    sl = slice(30000, 31000)
    small = g.Engine(g.engine.default_config(g.MODEL_DIN_COS, uP=uP, S=S, D=D, cF=cF, batch=1000, pred_batch=1000))
    small.table_upload(g.TABLE_USER_FEAT, uf); small.table_upload(g.TABLE_ITEM_FEAT, itf); small.table_upload(g.TABLE_ITEM_EMB, emb)
    small.set_weights(*eng.get_weights())
    assert small.predict_idx(ur[sl], ir[sl], hist[sl]).tobytes() == p_all[sl].tobytes()
    # mass conservation per table row on uniform ids (with Zipf ids and lr=1 the hottest row moves by
    # ~10% inside one step and the documented Hogwild read-after-update window becomes first-order)
    ur, ir, hist, y = make_batch(rng, U, I, B, S, zipf=False)
    grads = eng.debug_grads_idx(ur, ir, hist, y)
    valid = hist >= 0
    want = np.bincount(hist[valid], weights=grads["dUb"].sum(-1, dtype=np.float64)[valid], minlength=I)
    want += np.bincount(ir, weights=grads["dIt"].sum(-1, dtype=np.float64), minlength=I)
    eng.train_step_idx(ur, ir, hist, y)
    got = (eng.table_download(g.TABLE_ITEM_EMB, I, D).astype(np.float64) - emb).sum(1)
    scale = np.abs(want).max()
    assert scale > 0
    np.testing.assert_allclose(got, -100.0 * want, rtol=2e-2, atol=2e-2 * 100.0 * scale)
    assert abs(got.sum() + 100.0 * want.sum()) <= 2e-3 * 100.0 * np.abs(want).sum()


def test_pipelined_epoch_entry_matches_per_batch_steps():
    """ctr_train_idx (one pass over n samples, H2D of batch i+1 overlapping batch i, ragged tail zero-padded
    with label 0) == the same batches through ctr_train_step_idx."""
    B, nfull = 256, 3
    engA, cfg, ocfg, W, (uf, itf, emb), _ = setup(g.MODEL_DIN_COS, "ref", B, seed=11)
    engB, *_ = setup(g.MODEL_DIN_COS, "ref", B, seed=11)
    rng = np.random.default_rng(5)
    n = nfull * B + 100
    ur, ir, hist, y = make_batch(rng, uf.shape[0], itf.shape[0], n, cfg.S)
    costs = engA.train_idx(ur, ir, hist, y)
    assert costs.shape == (nfull + 1,)
    want = []
    for b in range(nfull):
        sl = slice(b * B, (b + 1) * B)
        want.append(engB.train_step_idx(ur[sl], ir[sl], hist[sl], y[sl]).cost)
    # tail: pad explicitly with missing rows (zeros) and label 0
    pad = B - 100
    urt = np.concatenate([ur[nfull * B:], np.full(pad, -1, np.int32)]); irt = np.concatenate([ir[nfull * B:], np.full(pad, -1, np.int32)])
    ht = np.concatenate([hist[nfull * B:], np.full((pad, cfg.S), -1, np.int32)]); yt = np.concatenate([y[nfull * B:], np.zeros(pad, np.float32)])
    want.append(engB.train_step_idx(urt, irt, ht, yt).cost)
    np.testing.assert_allclose(costs, np.array(want, np.float32), rtol=2e-5, atol=1e-6)
    for a, b_ in zip(engA.get_weights(), engB.get_weights()):
        assert_mostly_close(a, b_, 1e-3, 1e-4, 0.995, "weights after pipelined pass")


def test_ubcache_window_on_device_matches_timeseq_filter():
    """feature/ubcache TimeSeq.Filter (cache.go:71-94) for a batch on the device vs the oracle, including
    the reference's own table (cache_test.go:9-38), maxTs == 0, unknown users and short histories."""
    eng = g.Engine(g.engine.default_config(g.MODEL_DIN_COS, S=5, batch=8, pred_batch=8))
    ts0 = np.array([10, 9, 8, 7, 6, 5, 4, 3, 2, 1], np.int64)
    eng.ubcache_upload([0, 10], ts0, ts0.astype(np.int32))
    got = eng.ubcache_window(np.zeros(4, np.int32), np.array([0, 5, 100, -3], np.int64))
    assert got[0].tolist() == [10, 9, 8, 7, 6]            # Filter(0, 5)
    assert got[1].tolist() == [5, 4, 3, 2, 1]             # Filter(5, 5)
    assert got[2].tolist() == [10, 9, 8, 7, 6]
    assert got[3].tolist() == [-1] * 5                    # nothing that old
    rng = np.random.default_rng(0)
    U, S = 300, 7
    eng = g.Engine(g.engine.default_config(g.MODEL_DIN_COS, S=S, batch=8, pred_batch=8))
    lens = rng.integers(0, 40, U); off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    ts = np.concatenate([np.sort(rng.integers(1, 1000, n))[::-1] for n in lens]).astype(np.int64)
    items = rng.integers(0, 5000, ts.size).astype(np.int32)
    eng.ubcache_upload(off, ts, items)
    ub = rng.integers(-1, U + 2, 2000).astype(np.int32); mt = rng.integers(0, 1100, 2000).astype(np.int64); mt[::9] = 0
    got = eng.ubcache_window(ub, mt)
    for b in range(2000):
        want = [-1] * S
        if 0 <= ub[b] < U and lens[ub[b]] > 0:
            seg = ts[off[ub[b]]:off[ub[b] + 1]]
            start, cnt = orc.ub_filter(seg, int(mt[b]), S)
            want[:cnt] = items[off[ub[b]] + start: off[ub[b]] + start + cnt].tolist()
        assert got[b].tolist() == want, (b, ub[b], mt[b])
