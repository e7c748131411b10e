"""The kernel matrix: every attention family and every wgmma GEMM tile width the engine dispatches on one GPU, forward
and backward, against the double-accumulating oracle, and against the fp32 FFMA engine wherever the wgmma engine runs.

The engine picks its kernels from the model dims (engine.cu attn_forward / attn_backward, umma_supported,
use_umma_dw).  Each case turns profiling on and asserts the profile keys of the kernel family and of the GEMMs it
means to cover, so that a change of the dispatch rules cannot silently move a case onto another kernel."""
import numpy as np
import pytest

import go_ctr_b200 as g
from oracle import oracle as orc
from tests.test_gpu_parity import GRAD_ATOL, GRAD_RTOL, SCORE_RTOL, setup
from tests.util import assert_mostly_close, make_batch, scaled_init

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]

MODELS = [g.MODEL_YOUTUBE, g.MODEL_DIN_COS, g.MODEL_DIN_EUC]
DIN = [g.MODEL_DIN_COS, g.MODEL_DIN_EUC]
MNAME = {g.MODEL_YOUTUBE: "youtube", g.MODEL_DIN_COS: "cos", g.MODEL_DIN_EUC: "euc"}
UM_KEYS = ("umma_fwd0_sigmoid", "umma_fwd1_sigmoid", "umma_dW1_splitk", "umma_dZ0_dsigmoid", "umma_dW0_splitk", "umma_dX")


def ru(x, m):
    return (x + m - 1) // m * m


def gemm_mode(dims, H0, H1, B=None, batch=None):
    """Which GEMM engine runs (DESIGN.md §4): wgmma when the padded widths H0p, H1p and round_up(2D, 16) fit 8 column
    chunks of 32, with the weight gradients on wgmma too when Kp <= 256 and the batch is the configured one; fp32 FFMA
    otherwise."""
    uP, S, D, cF = dims
    if ru(H0, 32) > 256 or ru(H1, 32) > 256 or ru(2 * D, 16) > 256:
        return "fp32"
    return "umma" if ru(uP + 2 * D + cF, 32) <= 256 and B == batch else "umma_fp32dw"


def gemm_keys(mode, dx=True):
    keys = {k if mode == "umma" or (mode == "umma_fp32dw" and "dW" not in k) else "sgemm_" + k[5:] for k in UM_KEYS}
    return keys if dx else {k for k in keys if not k.endswith("_dX")}


def assert_dispatch(eng, fwd, bwd, mode, dx=True):
    """The attention launches are exactly attn_fwd_<fwd> (and attn_bwd_<bwd>); the GEMM launches exactly `mode`'s."""
    prof = eng.profile_dump()
    attn = {k for k in prof if k.startswith("attn_")}
    assert attn == {"attn_fwd_" + fwd} | ({"attn_bwd_" + bwd} if bwd else set()), sorted(prof)
    mm = {k for k in prof if k.startswith(("umma_", "sgemm_"))}
    assert mm == gemm_keys(mode, dx), sorted(prof)
    return prof


def edges(batch):
    """Edge rows: an all-missing history, a missing item, the item's own row in its history (u == v: the euclid
    distance is 0 and both sides take its gradient as 0), one row repeated across a whole history."""
    ur, ir, hist, y = batch
    if len(y) >= 4:
        hist[0] = -1
        ir[1] = -1
        ir[2] = 5; hist[2, ::2] = 5
        hist[3] = 7
    return batch


def oracle(model, dims, H0, H1, W, tabs, batch, training=False, seed=0, drop=(0.0, 0.0), step=0):
    """The oracle's forward and backward of one batch; `step` is the handle's step counter (the dropout stream)."""
    uP, S, D, cF = dims
    (uf, itf, emb), (ur, ir, hist, y) = tabs, batch
    o = orc.make_cfg(model, uP, S, D, cF, H0, H1, *drop)
    ws = orc.Workspace(o, len(y))
    p, z = orc.forward(o, W, orc.gather_rows(uf, itf, emb, ur, ir, hist), orc.make_ranges(uP, S, D, cF),
                       training=training, seed=seed, step=step, ws=ws)
    ref = orc.backward(o, W, ws, y)
    ref.update(p=p, logit=z)
    return ref


def assert_matches(out, ref, model, batch, what):
    """Everything ctr_debug_grads_idx returns, at the parity bars of tests/test_gpu_parity.py."""
    ur, ir, hist, y = batch
    np.testing.assert_allclose(out["logit"], ref["logit"], rtol=SCORE_RTOL, atol=2e-5, err_msg=what + ": logit")
    np.testing.assert_allclose(out["p"], ref["p"], rtol=SCORE_RTOL, atol=1e-7, err_msg=what + ": p")
    assert abs(out["cost"] - ref["cost"]) <= 1e-5 * max(1.0, abs(ref["cost"])), (what, out["cost"], ref["cost"])
    for k in ("dW0", "dW1", "dW2"):
        scale = np.abs(ref[k]).max()
        np.testing.assert_allclose(out[k], ref[k], rtol=GRAD_RTOL, atol=GRAD_ATOL * scale + 1e-12, err_msg=what + ": " + k)
    item = ir >= 0                                      # a missing item has no row to receive its gradient
    np.testing.assert_allclose(out["dIt"][item], ref["dIt"][item], rtol=2e-3, atol=1e-4 * np.abs(ref["dIt"]).max() + 1e-12,
                               err_msg=what + ": dIt")
    if model != g.MODEL_YOUTUBE:
        np.testing.assert_allclose(out["datt"], ref["datt"], rtol=2e-3, atol=2e-5 * np.abs(ref["datt"]).max() + 1e-12,
                                   err_msg=what + ": datt")
    valid = hist >= 0                                   # gradients of padded slots are never scattered
    np.testing.assert_allclose(out["dUb"][valid], ref["dUb"][valid], rtol=2e-3, atol=2e-5 * np.abs(ref["dUb"]).max() + 1e-12,
                               err_msg=what + ": dUb")


def run_case(model, dims, B, fwd, bwd, H0=200, H1=80, seed=1, training=False, what="", **kw):
    """One batch through ctr_debug_grads_idx on the default (AUTO) engine, checked against the oracle and, when the
    wgmma engine ran, against the fp32 engine on the same state."""
    eng, cfg, ocfg, W, tabs, batch = setup(model, dims, B, seed=seed, H0=H0, H1=H1, **kw)
    edges(batch)
    eng.profile(True)
    out = eng.debug_grads_idx(*batch, training=training)
    mode = gemm_mode(dims, H0, H1, B, B)
    assert_dispatch(eng, fwd, bwd, mode)
    drop = (cfg.dropout0, cfg.dropout1) if training else (0.0, 0.0)
    assert_matches(out, oracle(model, dims, H0, H1, W, tabs, batch, training, cfg.seed, drop), model, batch, what)
    if mode != "fp32":
        fp, *_ = setup(model, dims, B, seed=seed, H0=H0, H1=H1, gemm=g.GEMM_FP32, **kw)
        fp.profile(True)
        out32 = fp.debug_grads_idx(*batch, training=training)
        assert_dispatch(fp, fwd, bwd, "fp32")
        assert_matches(out, out32, model, batch, what + " vs the fp32 engine")
        fp.close()
    eng.close()
    return mode


# ---- a. attention families x models ------------------------------------------------------------------------------
# (id, (uP, S, D, cF), forward family, backward family).  S = 32/33 is where the second prefetched history id per lane
# starts, S = 64 where it ends; (Kp - 2D)/4 is the number of lanes uP + cF take in the _idx forward (at most 32).
ATTN = ([("idx_D%d_S%d" % (D, S), (8, S, D, 7), "idx", "idx") for D in (16, 32, 64, 128) for S in (1, 31, 32, 33, 64)] + [
    ("lanes32", (64, 20, 32, 60), "idx", "idx"),          # Kp=192: (Kp-2D)/4 == 32, uP + cF fill all 32 lanes
    ("lanes24", (32, 20, 32, 60), "idx", "idx"),          # Kp=160: 24 lanes, just under
    ("lanes40", (64, 20, 32, 96), "vec", "idx"),          # Kp=224: 40 lanes, past what the _idx forward takes
    ("uP5", (5, 20, 32, 7), "vec", "idx"),                # uP % 4 != 0
    ("uP0", (0, 20, 32, 7), "vec", "idx"),                # no user features
] + [("vec_D%d_S%d" % (D, S), (8, S, D, 7), "vec", "vec") for D in (16, 32, 64, 128) for S in (65, 100)]
  + [("gen_D%d" % D, (5, 10, D, 7), "gen", "gen") for D in (7, 130, 256)])     # D=130/256: fp32 GEMMs (round_up(2D,16) > 256)


@pytest.mark.parametrize("model", MODELS, ids=MNAME.get)
@pytest.mark.parametrize("name,dims,fwd,bwd", ATTN, ids=[c[0] for c in ATTN])
def test_attention_family_against_oracle(name, dims, fwd, bwd, model):
    run_case(model, dims, 150, fwd, bwd, what=name)


@pytest.mark.parametrize("model", MODELS, ids=MNAME.get)
@pytest.mark.parametrize("D", [16, 32, 64, 128])
def test_dense_route_takes_the_vec_kernels(model, D):
    """ctr_train_dense / ctr_predict_dense with 16-byte aligned SampleInfo ranges: one epoch of exactly one batch from
    known weights == model.Train, then model.Predict."""
    uP, S, cF, B = 8, 10, 8, 200
    xcols = uP + S * D + D + cF                         # a multiple of 4, as are the range starts
    rng = np.random.default_rng(D)
    X = rng.random((B, xcols), np.float32)
    Y = (rng.random(B) > 0.5).astype(np.float32)
    cfg = g.engine.default_config(model, uP=uP, S=S, D=D, cF=cF, batch=B, pred_batch=B, seed=17)
    eng = g.Engine(cfg)
    ocfg = orc.make_cfg(model, uP, S, D, cF, 200, 80, cfg.dropout0, cfg.dropout1)
    W = scaled_init(orc, ocfg, 4)
    eng.set_weights(*W)
    ranges = [0, uP, uP, uP + S * D, uP + S * D, uP + S * D + D, uP + S * D + D, xcols]
    eng.profile(True)
    ep, cost = eng.train_dense(X, Y, ranges, 1)
    # a dense YouTube step has no attention weights and no rows to learn: no attention backward, no dX
    yt = model == g.MODEL_YOUTUBE
    assert_dispatch(eng, "vec", None if yt else "vec", gemm_mode((uP, S, D, cF), 200, 80, B, B), dx=not yt)
    Wo = [w.copy() for w in W]
    oep, ocost = orc.train_dense(ocfg, orc.default_solver(seed=cfg.seed), Wo, X, Y, orc.make_ranges(uP, S, D, cF), B, 1, 0)
    assert ep == oep == 1
    assert abs(cost - ocost) <= 2e-4 * max(1.0, abs(ocost)), (cost, ocost)
    got_w = eng.get_weights()
    for a, b, name in zip(got_w, Wo, ("mlp0", "mlp1", "mlp2", "att0")):
        assert_mostly_close(a, b, 2e-3, 2e-4, 0.995, name)
    eng.profile_reset()
    got = eng.predict_dense(X, ranges)
    assert {k for k in eng.profile_dump() if k.startswith("attn_")} == {"attn_fwd_vec"}
    want = orc.predict_dense(orc.make_cfg(model, uP, S, D, cF, 200, 80), [np.ascontiguousarray(w) for w in got_w], X,
                             orc.make_ranges(uP, S, D, cF), B)
    np.testing.assert_allclose(got, want, rtol=SCORE_RTOL, atol=1e-7)


# ---- b. ragged tail of the epoch entry, per family ------------------------------------------------------------------
@pytest.mark.parametrize("fam,dims", [("idx", (8, 20, 32, 7)), ("vec", (8, 70, 32, 7)), ("gen", (5, 6, 7, 5))], ids=["idx", "vec", "gen"])
def test_ragged_tail_of_the_epoch_entry_against_oracle(fam, dims):
    """ctr_train_idx over n % batch != 0 samples == the oracle stepping the same batches with the tail padded
    explicitly (missing ids, label 0): step costs, dense weights and the table rows (deterministic row SGD)."""
    B = 128
    n = 2 * B + 37
    eng, cfg, ocfg, W, tabs, _ = setup(g.MODEL_DIN_EUC, dims, B, seed=4, table_opt=g.TABLE_SGD_DETERMINISTIC, table_lr=0.5)
    uf, itf, emb = tabs
    ur, ir, hist, y = make_batch(np.random.default_rng(5), uf.shape[0], emb.shape[0], n, dims[1], zipf=True)
    eng.profile(True)
    costs = eng.train_idx(ur, ir, hist, y)
    assert_dispatch(eng, fam, fam, gemm_mode(dims, 200, 80, B, B))
    tr = orc.IdxTrainer(ocfg, orc.default_solver(seed=cfg.seed), W, uf, itf, emb)
    want = []
    for s in range(0, n, B):
        e = min(n, s + B); pad = B - (e - s)
        want.append(tr.step(np.concatenate([ur[s:e], np.full(pad, -1, np.int32)]), np.concatenate([ir[s:e], np.full(pad, -1, np.int32)]),
                            np.concatenate([hist[s:e], np.full((pad, dims[1]), -1, np.int32)]), np.concatenate([y[s:e], np.zeros(pad, np.float32)]),
                            table_lr=0.5)[0])
    np.testing.assert_allclose(costs, np.array(want, np.float32), rtol=2e-4, atol=1e-6)
    for a, b, name in zip(eng.get_weights(), tr.W, ("mlp0", "mlp1", "mlp2", "att0")):
        assert_mostly_close(a, b, 2e-3, 2e-4, 0.995, name)
    got = eng.table_download(g.TABLE_ITEM_EMB, *emb.shape)
    assert np.abs(tr.emb - emb).max() > 1e-5
    np.testing.assert_allclose(got, tr.emb, rtol=2e-3, atol=2e-5)


# ---- c. wgmma tile widths and batch edges ---------------------------------------------------------------------------
REF = (52, 10, 16, 53)           # in = 137, Kp = 160; the _idx kernels
# H0 -> NCH 1..8 of fwd0 / dZ0 / dW0; H1 -> NCH 1, 3, 4 of fwd1 / dW1 and k-loops of one, odd and even length;
# 33/17 and 200/80 pad inside a chunk; H0 = 300 does not fit (fp32 fallback)
WIDTHS = [(h0, h1) for h0 in (32, 64, 96, 128, 160, 192, 224, 256) for h1 in (32, 96, 128)] + [(33, 17), (200, 80), (300, 80)]


@pytest.mark.parametrize("model", DIN, ids=MNAME.get)
@pytest.mark.parametrize("H0,H1", WIDTHS, ids=["%dx%d" % w for w in WIDTHS])
def test_wgmma_tile_widths(H0, H1, model):
    mode = run_case(model, REF, 200, "idx", "idx", H0=H0, H1=H1, what="H0=%d H1=%d" % (H0, H1))
    assert mode == ("fp32" if H0 > 256 else "umma")


# dX: N = round_up(2D, 16) -> NCH 1..8 of k_umma_gemm<STORE>.  D = 48/80/96/112 take the _gen attention kernels; D = 128
# has Kp = 288 > 256, so its weight gradients run on the fp32 engine
DX = [(16, "idx"), (32, "idx"), (48, "gen"), (64, "idx"), (80, "gen"), (96, "gen"), (112, "gen"), (128, "idx")]


@pytest.mark.parametrize("model", DIN, ids=MNAME.get)
@pytest.mark.parametrize("D,fam", DX, ids=["D%d" % d for d, _ in DX])
def test_wgmma_dx_widths(D, fam, model):
    mode = run_case(model, (8, 10, D, 7), 200, fam, fam, what="D=%d" % D)
    assert mode == ("umma_fp32dw" if D == 128 else "umma")


@pytest.mark.parametrize("model", DIN, ids=MNAME.get)
def test_wgmma_long_k_loop(model):
    """uP = cF = 100, D = 64: Kp = 352, a long forward k-loop; the weight gradients fall back to fp32 (Kp > 256), and
    uP + cF need more lanes than the _idx forward has."""
    assert run_case(model, (100, 10, 64, 100), 200, "vec", "idx", what="Kp=352") == "umma_fp32dw"


@pytest.mark.parametrize("model", DIN, ids=MNAME.get)
@pytest.mark.parametrize("B", [1, 31, 127, 128, 129, 257, 1000])
def test_wgmma_batch_edges(B, model):
    """batch == B: k_umma_dw runs with a ragged last k-block of samples (B % 32 != 0) or with fewer than 32; the
    forward GEMMs with a partial last 128-row tile."""
    assert run_case(model, REF, B, "idx", "idx", what="B=%d" % B) == "umma"


@pytest.mark.timeout(600)
def test_wgmma_persistent_loop_matches_fp32_engine():
    """B = 40000 > 2 x 128 x SMs: every CTA of the persistent GEMMs walks several tiles.  wgmma vs fp32 engine on every
    output of the step."""
    B = 40000
    res = []
    for gm in (g.GEMM_AUTO, g.GEMM_FP32):
        eng, cfg, ocfg, W, tabs, batch = setup(g.MODEL_DIN_COS, REF, B, seed=2, U=5000, I=40000, gemm=gm)
        edges(batch)
        eng.profile(True)
        res.append(eng.debug_grads_idx(*batch))
        assert_dispatch(eng, "idx", "idx", "umma" if gm == g.GEMM_AUTO else "fp32")
        eng.close()
    assert_matches(res[0], res[1], g.MODEL_DIN_COS, batch, "B=40000 vs the fp32 engine")


@pytest.mark.parametrize("model", DIN, ids=MNAME.get)
@pytest.mark.parametrize("H0,H1", [(256, 80), (33, 17)], ids=["256x80", "33x17"])
def test_wgmma_dropout_masks(H0, H1, model):
    """Dropout on: the wgmma and fp32 engines and the oracle draw the same masks (counter = sample * H + column, H the
    unpadded width), forward and backward."""
    run_case(model, REF, 200, "idx", "idx", H0=H0, H1=H1, training=True, dropout0=0.3, dropout1=0.2, what="dropout")


# ---- d. table optimisers x families --------------------------------------------------------------------------------
TABLE_OPTS = [("sgd_hot100", g.TABLE_SGD, 100, 0.5),        # 600 Zipf rows, 100 replicated: the touched rows straddle hot_rows
              ("sgd_nohot", g.TABLE_SGD, -1, 0.5),          # every row through red.add
              ("sgd_sorted", g.TABLE_SGD_DETERMINISTIC, 0, 0.5),
              ("adam", g.TABLE_ADAM, 0, 0.01)]
TABLE_SHAPES = [("idx_D32", (8, 20, 32, 7), "idx"), ("idx_D128", (8, 20, 128, 7), "idx"), ("vec_S70", (8, 70, 32, 7), "vec"),
                ("gen_D7", (5, 6, 7, 5), "gen")]


@pytest.mark.parametrize("shape,dims,fam", TABLE_SHAPES, ids=[s[0] for s in TABLE_SHAPES])
@pytest.mark.parametrize("opt_name,opt,hot,lr", TABLE_OPTS, ids=[o[0] for o in TABLE_OPTS])
def test_table_optimisers_against_oracle(opt_name, opt, hot, lr, shape, dims, fam):
    """Three train steps with Zipf ids: step costs, dense weights and the downloaded table against the oracle's row
    solver.  The row gradients carry the 1/B of the mean cost, so a step moves a row by ~1e-4 and the fused scatter's
    Hogwild read-after-update window is second order."""
    B, I, steps = 256, 600, 3
    eng, cfg, ocfg, W, tabs, _ = setup(g.MODEL_DIN_COS, dims, B, seed=9, I=I, table_opt=opt, table_lr=lr, hot_rows=hot)
    uf, itf, emb = tabs
    tr = orc.IdxTrainer(ocfg, orc.default_solver(seed=cfg.seed), W, uf, itf, emb)
    rng = np.random.default_rng(99)
    eng.profile(True)
    hits = np.zeros(I, np.int64)                        # scatter-adds per row over the steps
    for step in range(steps):
        batch = make_batch(rng, uf.shape[0], I, B, dims[1], zipf=True)
        hits += np.bincount(np.concatenate([batch[2][batch[2] >= 0], batch[1]]), minlength=I)
        st = eng.train_step_idx(*batch)
        ocost, _ = tr.step(*batch, table_lr=lr, table_adam=opt == g.TABLE_ADAM)
        assert abs(st.cost - ocost) <= 2e-4 * max(1.0, abs(ocost)), (step, st.cost, ocost)
    prof = assert_dispatch(eng, fam, fam, gemm_mode(dims, 200, 80, B, B))
    # the replica accumulators serve the _idx / _vec scatters (row-aligned float4 lanes), not the _gen one
    assert ("hot_rows_apply" in prof) == (opt == g.TABLE_SGD and hot > 0 and fam != "gen"), sorted(prof)
    assert ("segment_sgd" in prof) == (opt == g.TABLE_SGD_DETERMINISTIC) and ("segment_adam" in prof) == (opt == g.TABLE_ADAM)
    for a, b, name in zip(eng.get_weights(), tr.W, ("mlp0", "mlp1", "mlp2", "att0")):
        assert_mostly_close(a, b, 2e-3, 2e-4, 0.995, name)
    assert_table_matches(opt, eng.table_download(g.TABLE_ITEM_EMB, *emb.shape), tr.emb, emb, hits)


def assert_table_matches(opt, got, want, start, hits):
    """Rows trained from `start` by the engine (got) against a reference trajectory (want) at the bars of the row
    optimiser `opt`; hits[i] = the scatter-adds row i received over the steps."""
    moved = np.abs(want - start).max()
    assert moved > 1e-5
    if opt == g.TABLE_ADAM:
        # an Adam step is ~lr * sign(g) at first: elements whose tiny gradient flips sign inside fp32 noise may differ
        assert_mostly_close(got, want, 2e-3, 2e-4, 0.995, "ITEM_EMB")
        return
    if opt == g.TABLE_SGD:
        np.testing.assert_allclose(got, want, rtol=1e-3, atol=1e-6)       # the fused-scatter bar
    else:
        np.testing.assert_allclose(got, want, rtol=2e-4, atol=2e-6)       # the sorted-update bar
    # the movement itself, which the bars on the row values above (~0.2) barely resolve: within 1 % of the largest
    # movement, plus, where rows are added to one sample at a time (red.add straight into the table), half an ulp of
    # the row value per add: a per-sample step of a few ulps is rounded once per add, which no summation order avoids
    tol = 1e-2 * moved + 1e-2 * np.abs(want - start)
    if opt == g.TABLE_SGD:
        tol = tol + 0.5 * hits[:, None] * np.spacing(np.abs(want))
    err = np.abs((got - start) - (want - start))
    assert (err <= tol).all(), (np.unravel_index(np.argmax(err - tol), err.shape), float((err - tol).max()), moved)
