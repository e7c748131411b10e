"""Multi-step training against the oracle at every wgmma tile width, and what the steps leave behind.

tests/test_gpu_paths.py checks one step from freshly set weights.  From the second step on three more mechanisms
matter, and each case here reaches them:
  * the wgmma GEMMs read TF32 hi/lo operand copies of W0 and W1 that k_adam writes as it updates the weights
    (engine.cu step_core, split_in_adam); k_split_weights runs only after set_weights or a checkpoint load, so
    every step after the first reads the optimiser's copies, whose layouts depend on Kp, H0p, H1p, uP and 2D;
  * the dropout masks follow the step counter (counter stream step * 4 + {0, 1});
  * the state after training: Adam moments at padded strides, predict with pred_batch != batch, checkpoint resume.
Each case trains with dropout on and with learnable rows, so that the dX GEMM, and with it the W0 rows [uP, uP + 2D)
copy, matters for every model, YouTube included."""
import numpy as np
import pytest

import go_ctr_b200 as g
from oracle import oracle as orc
from tests.test_gpu_parity import SCORE_RTOL, setup
from tests.test_gpu_paths import (ATTN, DIN, DX, MNAME, MODELS, REF, WIDTHS, assert_dispatch, assert_matches, edges,
                                  gemm_mode, oracle)
from tests.util import assert_mostly_close, make_batch, scaled_init

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]

STEPS = 4
TRAIN = dict(dropout0=0.3, dropout1=0.2, table_opt=g.TABLE_SGD_DETERMINISTIC, table_lr=0.5)
PRED_BATCH, NPRED = 300, 1000               # 1000 = 3 x 300 + a ragged chunk of 100
WEIGHTS = ("mlp0", "mlp1", "mlp2", "att0")


def batches(rng, tabs, B, S, n):
    uf, _, emb = tabs
    return [edges(make_batch(rng, uf.shape[0], emb.shape[0], B, S, zipf=True)) for _ in range(n)]


def assert_launches(prof, mode, steps):
    """The optimiser ran once per step, and the weights were split into TF32 copies once, for the first step after
    set_weights: every later step read the copies k_adam wrote.  The fp32 engine has no copies."""
    assert prof["adam_dense"][1] == steps, sorted(prof)
    assert prof.get("split_weights_tf32", (0, 0))[1] == (0 if mode == "fp32" else 1), sorted(prof)


def assert_trained_like(eng, W, emb, what):
    """Dense weights and the learnt table at the bars of test_index_train_steps_with_deterministic_row_update."""
    for a, b, name in zip(eng.get_weights(), W, WEIGHTS):
        assert_mostly_close(a, b, 2e-3, 2e-4, 0.995, what + ": " + name)
    got = eng.table_download(g.TABLE_ITEM_EMB, *emb.shape)
    np.testing.assert_allclose(got, emb, rtol=2e-4, atol=2e-6, err_msg=what + ": ITEM_EMB")


def assert_costs(costs, want, what):
    for step, (c, w) in enumerate(zip(costs, want)):
        assert abs(c - w) <= 2e-4 * max(1.0, abs(w)), (what, step, c, w)


def run_trajectory(model, dims, B, fwd, bwd, H0=200, H1=80, seed=1, what=""):
    """STEPS train steps on the default (AUTO) engine against the oracle stepping the same batches; then every output
    of ctr_debug_grads_idx at the step counter STEPS against the oracle on the state the engine holds, and predict
    on that state.  Where the wgmma engine ran, the same on the fp32 engine, and the two trajectories to each other."""
    mode = gemm_mode(dims, H0, H1, B, B)
    trained = {}
    for gemm in (g.GEMM_AUTO,) if mode == "fp32" else (g.GEMM_AUTO, g.GEMM_FP32):
        m = mode if gemm == g.GEMM_AUTO else "fp32"
        tag = "%s [%s]" % (what, m)
        eng, cfg, ocfg, W, tabs, _ = setup(model, dims, B, seed=seed, H0=H0, H1=H1, pred_batch=PRED_BATCH, gemm=gemm, **TRAIN)
        uf, itf, emb0 = tabs
        rng = np.random.default_rng(seed + 100)
        bs = batches(rng, tabs, B, dims[1], STEPS)
        eng.profile(True)
        costs = [eng.train_step_idx(*b).cost for b in bs]
        assert_launches(assert_dispatch(eng, fwd, bwd, m), m, STEPS)
        tr = orc.IdxTrainer(ocfg, orc.default_solver(seed=cfg.seed), W, uf, itf, emb0)
        assert_costs(costs, [tr.step(*b, table_lr=TRAIN["table_lr"])[0] for b in bs], tag + ": cost")
        assert_trained_like(eng, tr.W, tr.emb, tag)
        Wt, emb = eng.get_weights(), eng.table_download(g.TABLE_ITEM_EMB, *emb0.shape)
        # the masks of step STEPS, on the operand copies the last optimiser step wrote
        batch = batches(rng, tabs, B, dims[1], 1)[0]
        out = eng.debug_grads_idx(*batch, training=True)
        ref = oracle(model, dims, H0, H1, Wt, (uf, itf, emb), batch, True, cfg.seed, (cfg.dropout0, cfg.dropout1), step=STEPS)
        assert_matches(out, ref, model, batch, tag + " at step %d" % STEPS)
        if gemm == g.GEMM_AUTO:
            ur, ir, hist, _ = batches(rng, tabs, NPRED, dims[1], 1)[0]
            got = eng.predict_idx(ur, ir, hist)
            o0 = orc.make_cfg(model, *dims, H0, H1)
            want, _ = orc.forward(o0, Wt, orc.gather_rows(uf, itf, emb, ur, ir, hist), orc.make_ranges(*dims))
            np.testing.assert_allclose(got, want, rtol=SCORE_RTOL, atol=1e-7, err_msg=tag + ": predict")
        assert_launches(eng.profile_dump(), m, STEPS)          # neither the gradients nor predict split the weights again
        trained[m] = (eng, costs, emb)
    if len(trained) == 2:
        (eng, costs, _), (fp, costs32, emb32) = trained[mode], trained["fp32"]
        assert_costs(costs, costs32, what + ": cost vs the fp32 engine")
        assert_trained_like(eng, fp.get_weights(), emb32, what + " vs the fp32 engine")
    for eng, *_ in trained.values():
        eng.close()
    return mode


# ---- the matrix ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", MODELS, ids=MNAME.get)
@pytest.mark.parametrize("H0,H1", WIDTHS, ids=["%dx%d" % w for w in WIDTHS])
def test_trajectory_at_the_wgmma_tile_widths(H0, H1, model):
    mode = run_trajectory(model, REF, 200, "idx", "idx", H0=H0, H1=H1, what="H0=%d H1=%d" % (H0, H1))
    assert mode == ("fp32" if H0 > 256 else "umma")


@pytest.mark.parametrize("model", DIN, ids=MNAME.get)
@pytest.mark.parametrize("D,fam", DX, ids=["D%d" % d for d, _ in DX])
def test_trajectory_at_the_dx_widths(D, fam, model):
    """k_adam writes the W0 rows [uP, uP + 2D) the dX GEMM reads at NCH 1..8."""
    mode = run_trajectory(model, (8, 10, D, 7), 200, fam, fam, what="D=%d" % D)
    assert mode == ("umma_fp32dw" if D == 128 else "umma")


@pytest.mark.parametrize("model", DIN, ids=MNAME.get)
def test_trajectory_with_a_long_k_loop(model):
    """Kp = 352: the W0ᵀ copy k_adam writes has 352-float rows; the weight gradients run on the fp32 engine."""
    assert run_trajectory(model, (100, 10, 64, 100), 200, "vec", "idx", what="Kp=352") == "umma_fp32dw"


@pytest.mark.parametrize("model", DIN, ids=MNAME.get)
@pytest.mark.parametrize("B", [1, 31, 129, 257])
def test_trajectory_at_batch_edges(B, model):
    """The optimiser's 1/B, and k_umma_dw with a ragged or sub-32 last k-block of samples, over several steps."""
    assert run_trajectory(model, REF, B, "idx", "idx", what="B=%d" % B) == "umma"


# att0 has S entries stored with stride Sp = round_up(S, 4): the _idx kernels at D = 32 over their S list, the _vec
# kernels past S = 64, the _gen kernels above D = 128 (fp32 GEMMs)
ATT_S = [c for c in ATTN if c[0] in {"idx_D32_S%d" % s for s in (1, 31, 32, 33, 64)} | {"vec_D32_S65", "vec_D32_S100", "gen_D130", "gen_D256"}]


@pytest.mark.parametrize("model", DIN, ids=MNAME.get)
@pytest.mark.parametrize("name,dims,fwd,bwd", ATT_S, ids=[c[0] for c in ATT_S])
def test_trajectory_of_the_attention_weights(name, dims, fwd, bwd, model):
    run_trajectory(model, dims, 200, fwd, bwd, what=name)


# ---- resume ------------------------------------------------------------------------------------------------------------
RESUME = [("33x17", REF, 33, 17, "idx", "idx"), ("256x128", REF, 256, 128, "idx", "idx"),
          ("D48", (8, 10, 48, 7), 200, 80, "gen", "gen"), ("Kp352", (100, 10, 64, 100), 200, 80, "vec", "idx")]


@pytest.mark.parametrize("name,dims,H0,H1,fwd,bwd", RESUME, ids=[r[0] for r in RESUME])
def test_checkpoint_resume_splits_the_loaded_weights(name, dims, H0, H1, fwd, bwd, tmp_path):
    """Save after step 2 and load into a handle that has trained a step of its own on other weights and another
    table: its TF32 operand copies are current for its own weights and stale for the snapshot's, so only a load
    that marks them for a new split continues the run.  Both handles continue 2 steps: to each other at the bars of
    test_checkpoint_resume_continues_the_same_run, and the loaded one to the oracle."""
    B, model = 200, g.MODEL_DIN_COS
    a, cfg, ocfg, W, tabs, _ = setup(model, dims, B, seed=3, H0=H0, H1=H1, **TRAIN)
    uf, itf, emb0 = tabs
    rng = np.random.default_rng(7)
    bs = batches(rng, tabs, B, dims[1], 4)
    tr = orc.IdxTrainer(ocfg, orc.default_solver(seed=cfg.seed), W, uf, itf, emb0)
    ocosts = [tr.step(*b, table_lr=TRAIN["table_lr"])[0] for b in bs]
    for b in bs[:2]:
        a.train_step_idx(*b)
    path = tmp_path / "snap.ctr"
    a.checkpoint_save(path)
    # same config (and so the same dropout seed) as `a`, other weights and another table
    b_eng, *_ = setup(model, dims, B, seed=3, H0=H0, H1=H1, **TRAIN)
    b_eng.set_weights(*scaled_init(orc, ocfg, 77))
    b_eng.table_upload(g.TABLE_ITEM_EMB, (rng.standard_normal(emb0.shape) / np.sqrt(dims[2])).astype(np.float32))
    b_eng.train_step_idx(*batches(rng, tabs, B, dims[1], 1)[0])
    b_eng.profile(True)
    b_eng.checkpoint_load(path)
    costs_a = [a.train_step_idx(*b).cost for b in bs[2:]]
    costs_b = [b_eng.train_step_idx(*b).cost for b in bs[2:]]
    np.testing.assert_allclose(costs_a, costs_b, rtol=1e-5)
    for x, y in zip(a.get_weights(), b_eng.get_weights()):
        np.testing.assert_allclose(x, y, rtol=1e-4, atol=2e-5)
    np.testing.assert_allclose(a.table_download(g.TABLE_ITEM_EMB, *emb0.shape), b_eng.table_download(g.TABLE_ITEM_EMB, *emb0.shape),
                               rtol=1e-4, atol=1e-6)
    assert_costs(costs_b, ocosts[2:], name + ": resumed cost")
    assert_trained_like(b_eng, tr.W, tr.emb, name + ": resumed")
    mode = gemm_mode(dims, H0, H1, B, B)
    assert mode != "fp32"
    assert_launches(assert_dispatch(b_eng, fwd, bwd, mode), mode, 2)


# ---- device entry points -----------------------------------------------------------------------------------------------
def test_device_entry_points_follow_the_host_entry_points():
    """ctr_train_step_idx_dev and ctr_predict_idx_dev on device buffers made as bench.py makes them (torch tensors
    copied from the host batches, passed by data_ptr) == ctr_train_step_idx and ctr_predict_idx on the same batches,
    at the bars of test_pipelined_epoch_entry_matches_per_batch_steps."""
    import torch
    model, dims, B, H0, H1 = g.MODEL_DIN_EUC, REF, 200, 256, 128
    host, cfg, ocfg, W, tabs, _ = setup(model, dims, B, seed=5, H0=H0, H1=H1, pred_batch=PRED_BATCH, **TRAIN)
    dev_eng, *_ = setup(model, dims, B, seed=5, H0=H0, H1=H1, pred_batch=PRED_BATCH, **TRAIN)
    rng = np.random.default_rng(55)
    bs = batches(rng, tabs, B, dims[1], STEPS)
    dev = torch.device("cuda", 0)
    devb = [tuple(torch.from_numpy(a).to(dev) for a in b) for b in bs]
    torch.cuda.synchronize()                                # the engine's stream does not wait for torch's
    dev_eng.profile(True)
    costs_h, costs_d = [], []
    for b, (ur, ir, hist, y) in zip(bs, devb):
        costs_h.append(host.train_step_idx(*b).cost)
        dev_eng.train_step_idx_dev(ur.data_ptr(), ir.data_ptr(), hist.data_ptr(), y.data_ptr(), B)
        costs_d.append(dev_eng.last_cost())
    mode = gemm_mode(dims, H0, H1, B, B)
    assert_launches(assert_dispatch(dev_eng, "idx", "idx", mode), mode, STEPS)
    np.testing.assert_allclose(costs_d, costs_h, rtol=2e-5, atol=1e-6)
    for a, b in zip(dev_eng.get_weights(), host.get_weights()):
        assert_mostly_close(a, b, 1e-3, 1e-4, 0.995, "weights after the device-entry steps")
    emb_shape = tabs[2].shape
    np.testing.assert_allclose(dev_eng.table_download(g.TABLE_ITEM_EMB, *emb_shape), host.table_download(g.TABLE_ITEM_EMB, *emb_shape),
                               rtol=1e-4, atol=1e-6)
    ur, ir, hist, _ = batches(rng, tabs, NPRED, dims[1], 1)[0]
    want = host.predict_idx(ur, ir, hist)
    du, di, dh = (torch.from_numpy(a).to(dev) for a in (ur, ir, hist))
    out = torch.full((NPRED,), -1.0, dtype=torch.float32, device=dev)
    torch.cuda.synchronize()
    for s in range(0, NPRED, PRED_BATCH):                   # chunks of pred_batch, the last one ragged
        dev_eng.predict_idx_dev(du[s:].data_ptr(), di[s:].data_ptr(), dh[s:].data_ptr(), min(PRED_BATCH, NPRED - s), out[s:].data_ptr())
    dev_eng.sync()
    np.testing.assert_allclose(out.cpu().numpy(), want, rtol=SCORE_RTOL, atol=1e-7)
