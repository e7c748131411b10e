"""The table kernels at element offsets past 2^31 and 2^32: tables of 34 to 46 M rows (17 to 27 GB of HBM), as large as
the 100 M-row tables bench.py fills with ctr_table_fill, checked row by row.

Every kernel that touches a table addresses a row as (long)row * ld.  One int in such a product would wrap at 2^31
(a signed product: an address before the table) or at 2^32 (an unsigned or narrower one: the wrong row of the same
table), and nothing at the suite's small table sizes would notice.  Each case here therefore runs a real kernel at a
real large offset and compares it with a compact twin of the table:

* the big engine fills its tables on the device as bench.py does (ctr_table_fill: features U[0, 1), ITEM_EMB
  N(0, 1/D)), or uploads a mostly zero host table whose pages are never touched;
* R is a sorted set of about 4000 rows: rows 0-63, the hot-row boundary 32767-32769, the rows whose element offset
  straddles 2^31 and 2^32 in every table, the last three rows, the rows whose offsets alias the high rows' modulo
  2^32 (where an unsigned 32-bit wrap would land), and random rows; the rows are read back with ctr_gather_rows and
  held to a numpy restatement of k_table_fill;
* the twin engine holds exactly R's rows, with the same config, weights and seed, and sees every batch with its ids
  mapped by searchsorted(R, id).  The map is monotone, so the segment order of the sorted row update and every
  (score, row) tie-break are the same on both sides, and the twin's hot-row count is |R n [0, 32768)|, so the same
  rows are hot;
* the oracle runs on the compact tables.

A row's computation depends on its values, never on its id, so the big engine's per-sample outputs must equal the
twin's bit for bit, its atomically reduced outputs must agree at float32 summation-order tolerance, and both must
meet the suite's oracle bars."""
import numpy as np
import pytest

import go_ctr_b200 as g
from oracle import knn_oracle as ko
from oracle import oracle as orc
from tests.test_gpu_parity import SCORE_RTOL
from tests.test_gpu_paths import assert_dispatch, assert_matches, assert_table_matches, gemm_mode, oracle
from tests.test_gpu_recommend import engine_forward
from tests.util import assert_mostly_close, fill_normal_tol, fill_rows, mix64, scaled_init

GB = 1 << 30
B31, B32 = 1 << 31, 1 << 32
HOT = 32768                       # the automatic hot-row count of a large table (engine.cu ensure_hot)
U, H0, H1 = 1000, 200, 80
BATCH, PRED_BATCH = 512, 384
MODELS = [g.MODEL_YOUTUBE, g.MODEL_DIN_COS, g.MODEL_DIN_EUC]
MNAME = {g.MODEL_YOUTUBE: "youtube", g.MODEL_DIN_COS: "cos", g.MODEL_DIN_EUC: "euc"}
# bench.py's fill: table -> (seed, dist); the stream is the table index
FILL = {g.TABLE_USER_FEAT: (3, 0), g.TABLE_ITEM_FEAT: (4, 0), g.TABLE_ITEM_EMB: (5, 1)}

I_BIG = 2**25 + 2**20 + 7
# (uP, S, D, cF), I.  A: ITEM_EMB 4.43e9 > 2^32 and ITEM_FEAT 2.21e9 > 2^31 elements; B, C: ITEM_EMB > 2^32 on the
# _vec and _gen kernels (D = 96 is not a power of two: 2^32 is not a row boundary); D: ITEM_EMB 2.2e9 > 2^31, three
# times over with the row-Adam moments; E, F: ITEM_EMB > 2^32, uploaded
CASES = {"A": ((4, 8, 128, 64), I_BIG), "B": ((4, 65, 128, 4), I_BIG), "C": ((4, 8, 96, 4), -(-B32 // 96) + 2**20 + 5),
         "D": ((4, 8, 64, 4), I_BIG), "E": ((4, 8, 128, 4), I_BIG)}


def ld(width):
    return (width + 3) // 4 * 4


def straddles(I, width):
    """Per boundary 2^31, 2^32 inside a table of I rows: the rows ceil(b / ld) - 2 ... + 2, whose element offsets
    lie on both sides of b."""
    out = {}
    for b in (B31, B32):
        c = -(-b // ld(width))
        if c + 3 < I:
            out[b] = np.arange(c - 2, c + 3, dtype=np.int64)
    return out


def outside_rows(I, widths):
    """Rows no batch may touch: the rows just outside every straddle window and the last row's neighbour."""
    rows = [I - 4]
    for w in widths:
        for s in straddles(I, w).values():
            rows += [int(s[0]) - 1, int(s[-1]) + 1]
    return np.unique(np.array(rows, np.int64)).astype(np.int32)


def row_set(rng, I, widths, n=4000, high=0.0, alias=True):
    """R (sorted int32) and the rows a Zipf stream should hit first (the edges, then the rest in random order).
    high: the share of the random rows drawn from above the 2^32 straddle of ITEM_EMB (widths[0]); alias: add the
    rows whose offsets equal the high rows' modulo 2^32."""
    edges = [np.arange(64), np.array([HOT - 1, HOT, HOT + 1]), np.arange(I - 3, I)]
    for w in widths:
        edges += list(straddles(I, w).values())
    edges = np.unique(np.concatenate(edges).astype(np.int64))
    lo32 = -(-B32 // ld(widths[0]))
    m = n - edges.size
    nh = int(m * high)
    rest = np.concatenate([rng.integers(0, I, m - nh), rng.integers(lo32, I, nh)])
    R = np.union1d(edges, rest)
    if alias and B32 % ld(widths[0]) == 0:          # where an unsigned 32-bit product would put the high rows
        R = np.union1d(R, R[R >= lo32] - B32 // ld(widths[0]))
    R = R.astype(np.int32)
    first = np.concatenate([edges[edges >= 64], edges[edges < 64]])
    pop = np.concatenate([first, rng.permutation(np.setdiff1d(R, first))]).astype(np.int32)
    return R, pop


def assert_straddled(R, I, widths, need32=True):
    """The table really passes 2^32 elements (2^31 where need32 is False), and R holds rows on both sides of every
    boundary of every table."""
    assert I * ld(widths[0]) > (B32 if need32 else B31), (I, widths[0])
    for w in widths:
        for b, s in straddles(I, w).items():
            assert np.isin(s, R).all()
            assert (s.astype(np.int64) * ld(w) < b).any() and (s.astype(np.int64) * ld(w) >= b).any(), (w, b)


def remap(R, I, ids):
    """Big-table ids -> twin rows: searchsorted(R, id); -1 and ids >= I -> -1.  Every other id must be in R."""
    ids = np.asarray(ids)
    ok = (ids >= 0) & (ids < I)
    j = np.searchsorted(R, np.where(ok, ids, 0))
    assert (R[j[ok]] == ids[ok]).all(), "a batch id outside R"
    return np.where(ok, j, -1).astype(np.int32)


def rbatch(rng, pop, I, B, S):
    """Zipf ids over R (hottest first in `pop`), a -1 padded history tail on a fifth of the samples, and -1 and
    ids >= I sprinkled over items and history."""
    ir = pop[(rng.zipf(1.05, B) - 1) % pop.size]
    hist = pop[(rng.zipf(1.05, (B, S)) - 1) % pop.size]
    lens = np.where(rng.random(B) < 0.2, rng.integers(0, S + 1, B), S)
    hist[np.arange(S)[None, :] >= lens[:, None]] = -1
    hist[rng.random((B, S)) < 0.02] = I + 3
    ir[rng.random(B) < 0.02] = -1
    ir[rng.random(B) < 0.02] = I
    ur = rng.integers(0, U, B).astype(np.int32)
    y = (rng.random(B) > 0.5).astype(np.float32)
    return ur, ir.astype(np.int32), hist.astype(np.int32), y


@pytest.fixture
def own():
    """Engines made by a test are closed when it ends, pass or fail, so that one case's tables never overlap the
    next case's in HBM."""
    engs = []

    def add(e):
        engs.append(e)
        return e
    yield add
    for e in reversed(engs):
        e.close()


def require_hbm(need):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < need + 2 * GB:
        pytest.skip("needs %.1f GB + 2 GB of free HBM, %.1f GB free" % (need / GB, free / GB))


def make_cfg(model, dims, **kw):
    uP, S, D, cF = dims
    return g.engine.default_config(model, uP=uP, S=S, D=D, cF=cF, H0=H0, H1=H1, batch=BATCH, pred_batch=PRED_BATCH, seed=21, **kw)


def read_rows(eng, cfg, rows):
    """ITEM_EMB and ITEM_FEAT rows through ctr_gather_rows (item = rows, empty history)."""
    n = len(rows)
    X = eng.gather_rows(np.zeros(n, np.int32), rows, np.full((n, cfg.S), -1, np.int32))
    c = cfg.uP + cfg.S * cfg.D
    return X[:, c:c + cfg.D], X[:, c + cfg.D:]


def assert_fill(emb, feat, rows, D, cF):
    """Rows of the bench fill == the numpy restatement of k_table_fill: features bit for bit, N(0, 1/D) rows within
    the device's __logf / __cosf error."""
    want = fill_rows(rows, cF, FILL[g.TABLE_ITEM_FEAT][0], g.TABLE_ITEM_FEAT, 0, 1.0)
    assert feat.tobytes() == want.tobytes(), "ITEM_FEAT rows differ from the fill"
    scale = float(1.0 / np.sqrt(D))
    v, r = fill_rows(rows, D, FILL[g.TABLE_ITEM_EMB][0], g.TABLE_ITEM_EMB, 1, scale)
    err = np.abs(emb - v)
    tol = fill_normal_tol(r, scale)
    assert (err <= tol).all(), (rows[np.argmax((err - tol).max(1))], float((err - tol).max()))


class Pair:
    """The big engine (bench fill), R, the twin engine over R's rows, and the compact tables the oracle uses."""

    def __init__(self, own, case, model, seed=0, moments=False, **kw):
        dims, I = CASES[case]
        uP, S, D, cF = dims
        self.dims, self.I, self.widths = dims, I, (D, cF)
        need = 4 * (I * ld(D) * (3 if moments else 1) + I * ld(cF) + U * ld(uP))
        require_hbm(need)
        rng = np.random.default_rng(seed)
        self.R, self.pop = row_set(rng, I, self.widths)
        assert_straddled(self.R, I, self.widths, need32=case != "D")
        self.cfg = make_cfg(model, dims, **kw)
        self.cfg.reserved[0] = 0                                 # automatic: 32768 hot rows on the big table
        self.big = own(g.Engine(self.cfg))
        for t, w, n in ((g.TABLE_USER_FEAT, uP, U), (g.TABLE_ITEM_FEAT, cF, I), (g.TABLE_ITEM_EMB, D, I)):
            seed_, dist = FILL[t]
            self.big.table_fill(t, n, w, seed=seed_, dist=dist, scale=float(1.0 / np.sqrt(D)) if dist else 1.0)
        self.emb, self.feat = read_rows(self.big, self.cfg, self.R)
        assert_fill(self.emb, self.feat, self.R, D, cF)
        self.outside = outside_rows(I, self.widths)
        self.out_emb, out_feat = read_rows(self.big, self.cfg, self.outside)
        assert_fill(self.out_emb, out_feat, self.outside, D, cF)
        self.tcfg = make_cfg(model, dims, **kw)
        self.tcfg.reserved[0] = int((self.R < HOT).sum())       # the same rows hot; 0 would mean "automatic"
        assert self.tcfg.reserved[0] > 0
        self.twin = own(g.Engine(self.tcfg))
        self.twin.table_fill(g.TABLE_USER_FEAT, U, uP, seed=FILL[g.TABLE_USER_FEAT][0], dist=0, scale=1.0)
        self.twin.table_upload(g.TABLE_ITEM_FEAT, self.feat)
        self.twin.table_upload(g.TABLE_ITEM_EMB, self.emb)
        self.uf = self.twin.table_download(g.TABLE_USER_FEAT, U, uP)
        self.ocfg = orc.make_cfg(model, uP, S, D, cF, H0, H1, self.cfg.dropout0, self.cfg.dropout1)
        self.W = scaled_init(orc, self.ocfg, seed + 1)
        self.big.set_weights(*self.W); self.twin.set_weights(*self.W)
        self.rng = rng

    def batch(self, B):
        b = rbatch(self.rng, self.pop, self.I, B, self.dims[1])
        return b, (b[0], remap(self.R, self.I, b[1]), remap(self.R, self.I, b[2]), b[3])

    def hits(self, cb):
        """Scatter-adds per twin row of a compact batch."""
        ur, ir, hist, _ = cb
        return np.bincount(np.concatenate([hist[hist >= 0], ir[ir >= 0]]), minlength=self.R.size)

    def assert_untouched(self, touched):
        """Rows of R no batch touched, and the rows just outside every straddle window and next to the last row, are
        bit for bit what the fill wrote."""
        emb, _ = read_rows(self.big, self.cfg, self.R)
        keep = touched == 0
        assert keep.any()
        assert emb[keep].tobytes() == self.emb[keep].tobytes(), "an untouched row of R changed"
        out, _ = read_rows(self.big, self.cfg, self.outside)
        assert out.tobytes() == self.out_emb.tobytes(), "a row next to a straddle window or the last row changed"
        return emb


def assert_bitwise(a, b, what):
    a = np.ascontiguousarray(a); b = np.ascontiguousarray(b)
    assert a.shape == b.shape and a.tobytes() == b.tobytes(), (what, int(np.sum(a != b)), a.size)


def assert_reduced(a, b, what):
    """Outputs summed with atomics: the same terms in another order."""
    np.testing.assert_allclose(a, b, rtol=1e-5, atol=1e-5 * np.abs(b).max() + 1e-12, err_msg=what)


# ---- the restatement itself ---------------------------------------------------------------------------------------
def test_mix64_restatement_matches_the_oracle():
    L = orc.lib()
    rng = np.random.default_rng(1)
    ctr = np.concatenate([np.array([0, 1, B31 - 1, B31, B32 - 1, B32, 2**63, 2**64 - 1], np.uint64),
                          rng.integers(0, 2**64, 200, dtype=np.uint64)])
    for seed, stream in ((0, 0), (5, 2), (3, 0), (0xFFFFFFFF, 0xFFFFFFFF)):
        got = mix64(seed, stream, ctr)
        want = np.array([L.orc_mix64(seed, stream, int(c)) for c in ctr], np.uint64)
        assert np.array_equal(got, want), (seed, stream)


def test_fill_restatement_tells_neighbouring_rows_apart():
    """At every straddle of every case, row r's restated fill differs from rows r - 1 and r + 1 in every table: a
    kernel that reads or writes a neighbour is seen."""
    for dims, I in CASES.values():
        uP, S, D, cF = dims
        for w, t in ((D, g.TABLE_ITEM_EMB), (cF, g.TABLE_ITEM_FEAT)):
            seed, dist = FILL[t]
            for s in straddles(I, w).values():
                rows = np.arange(s[0] - 1, s[-1] + 2)
                v = fill_rows(rows, w, seed, t, dist, 1.0)
                v = v[0] if dist else v
                assert (v[1:] != v[:-1]).any(axis=1).all(), (dims, w)


# ---- forward and gradients ---------------------------------------------------------------------------------------
FWD = [("A", "idx"), ("B", "vec"), ("C", "gen")]


@pytest.mark.gpu
@pytest.mark.timeout(300)
@pytest.mark.parametrize("model", MODELS, ids=MNAME.get)
@pytest.mark.parametrize("case,fam", FWD, ids=["%s_%s" % c for c in FWD])
def test_forward_and_gradients_against_the_twin_and_oracle(case, fam, model, own):
    p = Pair(own, case, model, seed=ord(case) + model)
    dims, cfg = p.dims, p.cfg
    uP, S, D, cF = dims
    # predict over pred_batch != batch with a ragged tail
    (ur, ir, hist, y), (_, ic, hc, _) = p.batch(2 * PRED_BATCH + 77)
    assert (ir >= B32 // ld(D)).sum() > 10
    p.big.profile(True)
    got = p.big.predict_idx(ur, ir, hist)
    assert {k for k in p.big.profile_dump() if k.startswith("attn_")} == {"attn_fwd_" + fam}
    assert_bitwise(got, p.twin.predict_idx(ur, ic, hc), "predict")
    o0 = orc.make_cfg(model, uP, S, D, cF, H0, H1)
    po, _ = orc.forward(o0, p.W, orc.gather_rows(p.uf, p.feat, p.emb, ur, ic, hc), orc.make_ranges(uP, S, D, cF))
    np.testing.assert_allclose(got, po, rtol=SCORE_RTOL, atol=1e-7)
    # the comparison resolves single rows: R shifted by one row scores differently almost everywhere
    sh = lambda a: np.where((a >= 0) & (a < p.I - 1), a + 1, a)
    moved = p.big.predict_idx(ur, sh(ir), sh(hist)) != got
    assert moved[(ir >= 0) & (ir < p.I)].mean() > 0.95
    # one training-mode batch through ctr_debug_grads_idx
    batch, cb = p.batch(BATCH)
    p.big.profile_reset()
    out = p.big.debug_grads_idx(*batch, training=True)
    assert_dispatch(p.big, fam, fam, gemm_mode(dims, H0, H1, BATCH, BATCH))
    tw = p.twin.debug_grads_idx(*cb, training=True)
    valid = cb[2] >= 0; item = cb[1] >= 0
    assert_bitwise(out["p"], tw["p"], "p"); assert_bitwise(out["logit"], tw["logit"], "logit")
    assert_bitwise(out["dUb"][valid], tw["dUb"][valid], "dUb"); assert_bitwise(out["dIt"][item], tw["dIt"][item], "dIt")
    for k in ("dW0", "dW1", "dW2") + (("datt",) if model != g.MODEL_YOUTUBE else ()):
        assert_reduced(out[k], tw[k], k)
    assert abs(out["cost"] - tw["cost"]) <= 1e-6 * max(1.0, abs(tw["cost"]))
    ref = oracle(model, dims, H0, H1, p.W, (p.uf, p.feat, p.emb), cb, True, cfg.seed, (cfg.dropout0, cfg.dropout1))
    assert_matches(out, ref, model, cb, "%s %s" % (case, MNAME[model]))


# ---- training ----------------------------------------------------------------------------------------------------
def train_pair(p, opt, lr, steps=4):
    """`steps` train steps on both engines and the oracle; the rows after step 1 are returned for the bitwise check."""
    tr = orc.IdxTrainer(p.ocfg, orc.default_solver(seed=p.cfg.seed), p.W, p.uf, p.feat, p.emb)
    hits = np.zeros(p.R.size, np.int64)
    first = None
    for step in range(steps):
        batch, cb = p.batch(BATCH)
        hits += p.hits(cb)
        st = p.big.train_step_idx(*batch)
        st2 = p.twin.train_step_idx(*cb)
        ocost, _ = tr.step(*cb, table_lr=lr, table_adam=opt == g.TABLE_ADAM)
        assert abs(st.cost - ocost) <= 2e-4 * max(1.0, abs(ocost)), (step, st.cost, ocost)
        assert abs(st.cost - st2.cost) <= 1e-5 * max(1.0, abs(st2.cost)), (step, st.cost, st2.cost)
        if step == 0:
            first = (read_rows(p.big, p.cfg, p.R)[0], p.twin.table_download(g.TABLE_ITEM_EMB, p.R.size, p.dims[2]))
    return tr, hits, first


def assert_trained(p, tr, hits, opt):
    emb = p.assert_untouched(hits)
    tw = p.twin.table_download(g.TABLE_ITEM_EMB, p.R.size, p.dims[2])
    assert_table_matches(opt, emb, tr.emb, p.emb, hits)
    assert_table_matches(opt, emb, tw, p.emb, hits)
    for a, b, c, name in zip(p.big.get_weights(), tr.W, p.twin.get_weights(), ("mlp0", "mlp1", "mlp2", "att0")):
        assert_mostly_close(a, b, 2e-3, 2e-4, 0.995, name)
        assert_mostly_close(a, c, 2e-3, 2e-4, 0.995, name + " (twin)")


@pytest.mark.gpu
@pytest.mark.timeout(300)
def test_sorted_row_sgd_and_epoch_entry_past_2_32(own):
    """A with CTR_TABLE_SGD_DETERMINISTIC: four steps, then one ctr_train_idx epoch with n % batch != 0."""
    lr = 0.5
    p = Pair(own, "A", g.MODEL_DIN_COS, seed=11, table_opt=g.TABLE_SGD_DETERMINISTIC, table_lr=lr)
    p.big.profile(True)
    tr, hits, (b1, t1) = train_pair(p, g.TABLE_SGD_DETERMINISTIC, lr)
    assert_bitwise(b1, t1, "rows after step 1")
    assert not np.array_equal(b1, p.emb)
    prof = assert_dispatch(p.big, "idx", "idx", gemm_mode(p.dims, H0, H1, BATCH, BATCH))
    assert "segment_sgd" in prof and "hot_rows_apply" not in prof, sorted(prof)
    assert_trained(p, tr, hits, g.TABLE_SGD_DETERMINISTIC)
    # the bench's id-fed epoch entry, ragged tail padded with missing ids and label 0 on the oracle's side
    n = 2 * BATCH + 37
    (ur, ir, hist, y), (_, ic, hc, _) = p.batch(n)
    costs = p.big.train_idx(ur, ir, hist, y)
    np.testing.assert_allclose(costs, p.twin.train_idx(ur, ic, hc, y), rtol=1e-5, atol=1e-7)
    want = []
    for s in range(0, n, BATCH):
        e = min(n, s + BATCH); pad = BATCH - (e - s)
        cat = lambda a, v: np.concatenate([a[s:e], np.full((pad,) + a.shape[1:], v, a.dtype)])
        want.append(tr.step(cat(ur, -1), cat(ic, -1), cat(hc, -1), cat(y, 0), table_lr=lr)[0])
        hits += p.hits((None, ic[s:e], hc[s:e], None))
    np.testing.assert_allclose(costs, np.array(want, np.float32), rtol=2e-4, atol=1e-6)
    assert_trained(p, tr, hits, g.TABLE_SGD_DETERMINISTIC)


@pytest.mark.gpu
@pytest.mark.timeout(300)
def test_fused_row_sgd_with_automatic_hot_rows_past_2_32(own):
    """A with CTR_TABLE_SGD and reserved[0] = 0: rows [0, 32768) go through 4 replica accumulators (64 MB / 32768 rows
    of 512 B), the rest of the table, including every row past 2^31 and 2^32, through red.add."""
    lr = 0.5
    p = Pair(own, "A", g.MODEL_DIN_COS, seed=12, table_opt=g.TABLE_SGD, table_lr=lr)
    p.big.profile(True)
    tr, hits, _ = train_pair(p, g.TABLE_SGD, lr)
    prof = assert_dispatch(p.big, "idx", "idx", gemm_mode(p.dims, H0, H1, BATCH, BATCH))
    assert "hot_rows_apply" in prof, sorted(prof)
    assert hits[p.R < HOT].sum() > 0 and hits[(p.R >= HOT) & (p.R < 2 * HOT)].sum() > 0
    assert hits[p.R >= B32 // 128].sum() > 0
    assert_trained(p, tr, hits, g.TABLE_SGD)


@pytest.mark.gpu
@pytest.mark.timeout(300)
def test_row_adam_past_2_31(own):
    """D with CTR_TABLE_ADAM: the table and both moment tables pass 2^31 elements."""
    lr = 0.01
    p = Pair(own, "D", g.MODEL_DIN_COS, seed=13, moments=True, table_opt=g.TABLE_ADAM, table_lr=lr)
    p.big.profile(True)
    tr, hits, (b1, t1) = train_pair(p, g.TABLE_ADAM, lr)
    assert_bitwise(b1, t1, "rows after step 1")
    prof = assert_dispatch(p.big, "idx", "idx", gemm_mode(p.dims, H0, H1, BATCH, BATCH))
    assert "segment_adam" in prof, sorted(prof)
    assert hits[p.R >= B31 // 64].sum() > 0
    assert_trained(p, tr, hits, g.TABLE_ADAM)


# ---- search and recommendation over uploaded, mostly zero tables -------------------------------------------------
def sparse_engine(own, cfg, I, tables):
    """An engine whose item tables are zero except R's rows: host tables from np.zeros, whose untouched pages are never
    materialised, with only R's rows written."""
    eng = own(g.Engine(cfg))
    for t, (R, vals) in tables.items():
        host = np.zeros((I, vals.shape[1]), np.float32)
        host[R] = vals
        eng.table_upload(t, host)
        del host
    return eng


def map_back(R, rows):
    return np.where(rows >= 0, R[np.maximum(rows, 0)], -1).astype(np.int32)


@pytest.mark.gpu
@pytest.mark.timeout(300)
def test_knn_search_past_2_32(own):
    dims, I = CASES["E"]
    D = dims[2]
    require_hbm(4 * I * D)
    rng = np.random.default_rng(14)
    R, _ = row_set(rng, I, (D,))
    assert_straddled(R, I, (D,))
    vals = fill_rows(R, D, FILL[g.TABLE_ITEM_EMB][0], g.TABLE_ITEM_EMB, 1, 1.0)[0].astype(np.float32)
    cfg = g.engine.default_config(g.MODEL_DIN_COS, uP=0, cF=0, S=1, D=D, batch=1, pred_batch=1)
    eng = sparse_engine(own, cfg, I, {g.TABLE_ITEM_EMB: (R, vals)})
    qj = np.concatenate([np.arange(R.size - 6, R.size), np.flatnonzero(np.isin(R, straddles(I, D)[B32]))])
    assert (R[qj].astype(np.int64) * D >= B32).sum() >= 8
    q = rng.standard_normal((7, D))                      # float64 queries, not float32-representable
    for k in (10, 1024):
        r, s, c = eng.knn_search(k, rows=R[qj])
        orow, osim, ocnt = ko.search(vals, vals[qj].astype(np.float64), k, qj.astype(np.int32))
        assert np.array_equal(c, ocnt) and np.array_equal(r, map_back(R, orow)) and s.tobytes() == osim.tobytes(), k
        r, s, c = eng.knn_search(k, queries=q)
        orow, osim, ocnt = ko.search(vals, q, k)
        assert np.array_equal(c, ocnt) and np.array_equal(r, map_back(R, orow)) and s.tobytes() == osim.tobytes(), k


def expected_list(R, z, p, z0, I, k, hist, exclude):
    """The (logit desc, row asc) list over all I rows when every row outside R has the logit and score of the zero row
    z0 (a member of R): R's rows above that logit, then the tie run in row order."""
    j0 = int(np.searchsorted(R, z0))
    L0, P0 = z[j0], p[j0]
    ex = set(hist[(hist >= 0) & (hist < I)].tolist()) if exclude else set()
    keep = np.array([r not in ex for r in R.tolist()])
    above = np.flatnonzero((z > L0) & keep)
    above = above[np.lexsort((R[above], -z[above].astype(np.float64)))]
    inR = dict(zip(R.tolist(), range(R.size)))
    ties = []
    row = 0
    while len(above) + len(ties) < k:
        j = inR.get(row)
        if row not in ex and (j is None or z[j] == L0):
            ties.append(row)
        row += 1
    rows = np.concatenate([R[above], np.array(ties, np.int64)])[:k].astype(np.int32)
    zz = np.array([z[inR[r]] if r in inR else L0 for r in rows.tolist()], np.float32)
    pp = np.array([p[inR[r]] if r in inR else P0 for r in rows.tolist()], np.float32)
    return rows, zz, pp, above.size


@pytest.mark.gpu
@pytest.mark.timeout(300)
def test_recommend_topk_past_2_32(own):
    dims, I = CASES["E"]
    uP, S, D, cF = dims
    require_hbm(4 * I * (ld(D) + ld(cF)))
    rng = np.random.default_rng(15)
    R, _ = row_set(rng, I, (D, cF), n=600, high=0.9, alias=False)
    hi = -(-B32 // D)
    z0 = int(np.setdiff1d(np.arange(hi + 100, hi + 200), R)[0])         # the all-zero row of R
    R = np.union1d(R, [z0]).astype(np.int32)
    assert_straddled(R, I, (D, cF))
    emb = fill_rows(R, D, FILL[g.TABLE_ITEM_EMB][0], g.TABLE_ITEM_EMB, 1, float(1 / np.sqrt(D)))[0].astype(np.float32)
    feat = fill_rows(R, cF, FILL[g.TABLE_ITEM_FEAT][0], g.TABLE_ITEM_FEAT, 0, 1.0)
    j0 = int(np.searchsorted(R, z0))
    emb[j0] = 0; feat[j0] = 0
    # recommend_topk scores pred_batch items per chunk: the bench tools' chunk, not thousands of tiny ones
    cfg = g.engine.default_config(g.MODEL_DIN_COS, uP=uP, S=S, D=D, cF=cF, H0=H0, H1=H1, batch=256, pred_batch=65536, seed=5)
    big = sparse_engine(own, cfg, I, {g.TABLE_ITEM_FEAT: (R, feat), g.TABLE_ITEM_EMB: (R, emb)})
    twin = own(g.Engine(cfg))
    twin.table_upload(g.TABLE_ITEM_FEAT, feat); twin.table_upload(g.TABLE_ITEM_EMB, emb)
    for e in (big, twin):
        e.table_fill(g.TABLE_USER_FEAT, U, uP, seed=FILL[g.TABLE_USER_FEAT][0], dist=0, scale=1.0)
        e.set_weights(*scaled_init(orc, orc.make_cfg(g.MODEL_DIN_COS, uP, S, D, cF, H0, H1), 16))
    user = 7
    zero_rows = np.setdiff1d(np.arange(64, 200), R)[:2]                  # zero rows at the head of the tie run
    high = R[R >= hi]
    hist = np.array([high[-1], high[0], zero_rows[0], high[5], z0, zero_rows[1], -1, -1], np.int32)
    # the twin scores a zero row of the history as z0: the same values
    inR = np.isin(hist, R)
    hc = np.where(hist < 0, -1, np.where(inR, np.searchsorted(R, hist), j0)).astype(np.int32)
    z, pz = engine_forward(twin, cfg, user, hc, R.size)
    probe = np.setdiff1d([zero_rows[0], I // 2, I - 5, hi + 1], R).astype(np.int32)
    zb = big.debug_grads_idx(np.full(probe.size, user, np.int32), probe, np.tile(hist, (probe.size, 1)),
                             np.zeros(probe.size, np.float32))["logit"]
    assert (zb == z[j0]).all(), "rows outside R do not score as the zero row"
    for k, exclude in ((50, False), (1024, False), (1024, True)):
        rows, scores, logits, cnt = (a[0] for a in big.recommend_topk([user], hist[None, :], k, exclude_history=exclude))
        wr, wz, wp, n_above = expected_list(R, z, pz, z0, I, k, hist, exclude)
        assert cnt == k
        assert_bitwise(rows, wr, "rows k=%d exclude=%s" % (k, exclude))
        assert_bitwise(logits, wz, "logits"); assert_bitwise(scores, wp, "scores")
        if k == 50:
            assert (rows >= hi).sum() >= 25, rows                         # a list of rows past 2^32
        else:
            assert n_above < k                                            # the list runs into the tie run
        if exclude:
            assert not np.isin(rows, hist).any()
