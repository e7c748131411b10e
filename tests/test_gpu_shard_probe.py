"""The row-sharded kernels on one GPU: W = 2, 4 and 8 ranks emulated as W shards of one device, launched through the
kernel-level probe tests/cuda/shard_probe.cu (the engine's headers, not copies), checked against their single-table
twins and plain float64 references.

These kernels need nothing from the other ranks but addresses (RowSrc::peer_emb[], BwdOut::peer_adam[], the hot-row
buffers), so separately allocated shards on one device are, for them, separate ranks.  One stream reproduces the order
the engine's barriers give a sharded step: every rank's forward, every rank's backward, the hot-row fold, the all-reduce
(here a torch sum over the ranks' buffers, written back to each), each owner's update.  The barrier kernel, the peer
mappings and NCCL are not exercised here (tests/test_gpu_multi.py and the other multi-GPU tests keep those).

Global row g lives on rank g % W as local row g // W (table[r::W]).  Every shard buffer (table, moments, ITEM_FEAT,
gradient buffer) is sized for the largest shard plus CANARY rows of NaN, and the rows a short shard does not own are
NaN too: a stray read shows as a NaN in X0, a stray write as a changed canary.  The shard copies of the replicated hot
rows are NaN as well during training (the engine leaves them stale while the replicas train): nothing may read them.

Bars.  Exact (bit for bit): X0 against the twin, rows_cache, the touched-row counts / lists / flags / hot-row marks, the
untouched rows and canaries, the cleared buffers, the hot replicas against each other, the hot-row round trip, the
serving rows, the search and recommendation lists.  Summation bound n·2^-23·Σ|term| (tests/shard_ref.py): a gradient
row that red.add accumulated in any order, against the float64 sum of the twin's terms, and an SGD row against its
start plus that sum.  A few float32 roundings: the Adam moments and weights against row_adam_elem in float64.  The
oracle's attention bar (tests/test_gpu_paths.py): X0 of the 8×2 PEER forward lane map at D = 64."""
import numpy as np
import pytest
import torch

from tests import shard_probe as sp
from tests import shard_ref as ref

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

YT, COS, EUC = 0, 1, 2
MNAME = {YT: "youtube", COS: "cos", EUC: "euc"}
CANARY = 8
UP, CF, LDI = 8, 7, 8            # ITEM_FEAT rows are zero-padded to a multiple of 4 floats, as ctr_table_upload pads them
U = 50
I_ROWS = 203                     # not a multiple of 2, 4 or 8
B = 48
HOT_REPS = 16
LR_SGD = 0.125                   # a power of two: −lr/world scales the twin's terms exactly
ADAM = dict(lr=0.01, b1=0.9, b2=0.999, eps=1e-8)
DEV = "cuda"
NAN = float("nan")


def ru(x, m):
    return (x + m - 1) // m * m


def kp_of(D):
    return ru(UP + 2 * D + CF, 32)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def bits(t):
    return t.contiguous().view(torch.int32).cpu().numpy()


def host(t):
    return t.cpu().numpy()


class Box:
    """W ranks' shards of ITEM_EMB (and its row-Adam moments, ITEM_FEAT), each rank's hot-row replica, hot-row gradient
    buffers and owner-side gradient buffer, all on one device."""

    def __init__(self, table, W, hot_k, moments=None, ifeat=None, ifeat_sharded=False, poison_hot=True):
        I, D = table.shape
        self.I, self.D, self.W, self.hot_k = I, D, W, hot_k
        self.lde = D
        self.local = [len(range(r, I, W)) for r in range(W)]
        self.rows_max = self.local[0]
        self.emb = self._shards(table, poison_hot)
        self.m, self.v = (self._shards(x, poison_hot) for x in moments) if moments is not None else (None, None)
        hk = max(hot_k, 1)
        self.hot_tab = [self._padded(table[:hot_k], hk) for _ in range(W)]
        self.hot_m = [self._padded(moments[0][:hot_k], hk) for _ in range(W)] if moments is not None else None
        self.hot_v = [self._padded(moments[1][:hot_k], hk) for _ in range(W)] if moments is not None else None
        # hot_sum: [hot_k, D] gradient sums, then [hot_k] row-Adam touch marks, then NaN canaries
        self.hot_sum = [torch.cat([torch.zeros(hk * (D + 1), device=DEV), torch.full((CANARY * D,), NAN, device=DEV)]) for _ in range(W)]
        self.hot_acc = [torch.zeros(HOT_REPS * hk * D, device=DEV) for _ in range(W)]
        self.ifeat_full = dev(ifeat)
        self.ifeat_sharded = ifeat_sharded
        self.ifeat = self._shards(ifeat, False) if ifeat_sharded else None
        self.lay = sp.grad_layout(self.rows_max, self.lde)
        self.gbuf = []
        for _ in range(W):
            g = torch.zeros(self.lay["bytes"] + CANARY * self.lde * 4, dtype=torch.uint8, device=DEV)
            g[self.lay["bytes"]:].view(torch.float32).fill_(NAN)
            self.gbuf.append(g)

    def _padded(self, a, rows):
        t = torch.full((rows + CANARY, a.shape[1] if a.ndim == 2 else self.D), NAN, device=DEV)
        t[:a.shape[0]] = dev(a)
        return t

    def _shards(self, a, poison_hot):
        out = []
        for r in range(self.W):
            t = torch.full((self.rows_max + CANARY, a.shape[1]), NAN, device=DEV)
            loc = a[r::self.W].copy()
            if poison_hot:
                loc[np.arange(r, self.I, self.W)[:len(loc)] < self.hot_k] = NAN
            t[:len(loc)] = dev(loc)
            out.append(t)
        return out

    def assemble(self, shards, hot=None):
        """the global [I, width] table: rows from their owners, hot rows from rank 0's replica"""
        out = np.empty((self.I, shards[0].shape[1]), np.float32)
        for r in range(self.W):
            out[r::self.W] = host(shards[r][:self.local[r]])
        if hot is not None and self.hot_k:
            out[:self.hot_k] = host(hot[0][:self.hot_k])
        return out

    def table(self):
        return self.assemble(self.emb, self.hot_tab)

    def moments(self):
        return self.assemble(self.m, self.hot_m), self.assemble(self.v, self.hot_v)

    def gviews(self, r):
        g, L = self.gbuf[r], self.lay
        n = self.rows_max
        return dict(count=g[0:4].view(torch.int32), ticket=g[4:8].view(torch.int32),
                    flag=g[L["flag_off"]:L["flag_off"] + 4 * n].view(torch.int32),
                    list=g[L["list_off"]:L["list_off"] + 4 * n].view(torch.int32),
                    grad=g[L["grad_off"]:L["grad_off"] + 4 * n * self.lde].view(torch.float32).reshape(n, self.lde),
                    canary=g[L["bytes"]:])

    def peer_rows(self, r, batch, uf, rows_cache=None):
        ur, ir, hist, nvalid = batch[:4]
        return sp.rows(emb=self.emb[r], lde=self.lde, ufeat=uf, ldu=UP,
                       ifeat=self.ifeat[r] if self.ifeat_sharded else self.ifeat_full, ldi=LDI,
                       user_row=ur, item_row=ir, hist=hist, rows_cache=rows_cache, hot_tab=self.hot_tab[r],
                       peer_emb=self.emb, peer_ifeat=self.ifeat if self.ifeat_sharded else (),
                       nvalid=nvalid, n_emb=self.I, n_user=U, n_ifeat=self.I, world=self.W,
                       ifeat_sharded=int(self.ifeat_sharded), hot_k=self.hot_k)

    def twin_rows(self, emb, batch, uf):
        ur, ir, hist, nvalid = batch[:4]
        return sp.rows(emb=emb, lde=self.lde, ufeat=uf, ldu=UP, ifeat=self.ifeat_full, ldi=LDI, user_row=ur, item_row=ir,
                       hist=hist, nvalid=nvalid, n_emb=self.I, n_user=U, n_ifeat=self.I, world=1)

    def all_reduce_hot(self):
        n = max(self.hot_k, 1) * (self.D + 1)
        s = torch.stack([h[:n] for h in self.hot_sum]).sum(0)
        for h in self.hot_sum:
            h[:n] = s


def make_tables(rng, I, D):
    table = (rng.standard_normal((I, D)) * 0.5).astype(np.float32)
    uf = rng.random((U, UP), np.float32)
    itf = np.zeros((I, LDI), np.float32); itf[:, :CF] = rng.random((I, CF), np.float32)
    return table, uf, itf


def make_batches(rng, W, S, I, D, reserved):
    """One batch per rank.  Zipf-skewed ids (the hot rows are hit), ids −1, I … I+W−1 (rows a short shard would own),
    2^30 and −7 sprinkled in; sample 0 repeats one row across its whole history; sample 2 has dX = 0 and rows of its own
    (reserved[r]), so those rows are touched with a zero gradient sum; odd ranks have nvalid = B − 5 with valid ids left
    in the tail, which must not be touched."""
    pool = np.setdiff1d(np.arange(I), reserved)
    edges = np.array([-1, 2 ** 30, -7] + [I + j for j in range(W)], np.int32)

    def ids(n):
        z = np.minimum(rng.zipf(1.5, n) - 1, len(pool) - 1)
        u = rng.integers(0, len(pool), n)
        return pool[np.where(rng.random(n) < 0.5, z, u)].astype(np.int32)

    out = []
    for r in range(W):
        hist = ids(B * S).reshape(B, S)
        mask = rng.random((B, S)) < 0.1
        hist[mask] = rng.choice(edges, int(mask.sum()))
        item = ids(B)
        item[5] = -1; item[6] = I + (r % W); item[7] = 2 ** 30
        hist[0] = pool[(r * 7) % len(pool)]
        z = reserved[r]
        hist[2] = z; item[2] = z
        ur = rng.integers(0, U, B).astype(np.int32); ur[3] = -1
        nvalid = B if r % 2 == 0 else B - 5
        dX = rng.standard_normal((B, 2 * D)).astype(np.float32)
        dX[2] = 0.0
        out.append((ur, item, hist, nvalid, dX))
    return out


def one_row_batches(W, S, D, row, rng):
    """every history slot and every item of every rank is `row`"""
    out = []
    for r in range(W):
        hist = np.full((B, S), row, np.int32); item = np.full(B, row, np.int32)
        ur = rng.integers(0, U, B).astype(np.int32)
        out.append((ur, item, hist, B, rng.standard_normal((B, 2 * D)).astype(np.float32)))
    return out


def valid_terms(batch, dUb, dIt, I, scale):
    """(rows, terms·scale) of every slot the kernels scatter: b < nvalid, a history slot or the item, id in [0, I)"""
    ur, ir, hist, nvalid, _ = batch
    S = hist.shape[1]
    h = hist[:nvalid]; it = ir[:nvalid]
    hv = (h >= 0) & (h < I); iv = (it >= 0) & (it < I)
    rows = np.concatenate([h[hv], it[iv]])
    terms = np.concatenate([dUb[:nvalid][hv], dIt[:nvalid][iv]]).astype(np.float64) * scale
    return rows, terms


def expected_sums(rows_terms, I, D):
    """float64 per-row sums, Σ|term| and term counts over every rank's terms"""
    G = np.zeros((I, D)); A = np.zeros((I, D)); n = np.zeros(I, np.int64)
    for rows, terms in rows_terms:
        np.add.at(G, rows, terms); np.add.at(A, rows, np.abs(terms)); np.add.at(n, rows, 1)
    return G, A, n


def run_forward(box, batches, model, dims, att, uf_d):
    """every rank's PEER forward, each checked bit for bit against its twin on the assembled table; rows_cache
    against the table.  Returns the device batches and rows caches for the backward."""
    uP, S, D, cF = dims
    Kp = kp_of(D)
    table = box.table()
    emb_twin = dev(table)
    out = []
    for r, (ur, ir, hist, nvalid, dX) in enumerate(batches):
        db = (dev(ur), dev(ir), dev(hist), nvalid)
        cache = torch.full((B, S + 1, D), NAN, device=DEV)
        X0 = torch.full((B, Kp), NAN, device=DEV); X0t = torch.full((B, Kp), NAN, device=DEV)
        sp.fwd_idx(box.peer_rows(r, db, uf_d, cache), model, dims, att, X0, Kp, B, peer=True)
        sp.fwd_idx(box.twin_rows(emb_twin, db, uf_d), model, dims, att, X0t, Kp, B, peer=False, lane_peer=True)
        x = host(X0)
        assert not np.isnan(x).any(), ("rank %d: X0 holds a NaN: a read outside the valid rows" % r, np.argwhere(np.isnan(x))[:4])
        assert np.array_equal(bits(X0), bits(X0t)), ("rank %d: PEER X0 != twin" % r, np.argwhere(bits(X0) != bits(X0t))[:4])
        ids = np.concatenate([hist, ir[:, None]], 1)[:nvalid]
        ok = (ids >= 0) & (ids < box.I)
        c = host(cache)[:nvalid]
        assert np.array_equal(c[ok].view(np.int32), table[ids[ok]].view(np.int32)), "rank %d: rows_cache" % r
        out.append((db, cache, dev(dX)))
    return out, table, emb_twin


def run_backward(box, batches, fwd, model, dims, att, uf_d, emb_twin, adam):
    """every rank's fused PEER backward (SGD into the owners' rows, or row Adam into the owners' gradient buffers), then
    the twin's dUb / dIt.  Returns the (rows, scaled terms) of each rank."""
    uP, S, D, cF = dims
    W, hk = box.W, box.hot_k
    scale = 1.0 / W if adam else -LR_SGD / W
    for r, (db, cache, dX) in enumerate(fwd):
        a = None
        if adam:
            a = sp.Adam()
            for j in range(W):
                a.peer_adam[j] = box.gbuf[j].data_ptr()
            a.rows = box.rows_max
            a.hot_touch = box.hot_sum[r].data_ptr() + 4 * hk * D if hk else 0
        sp.bwd_idx(box.peer_rows(r, db, uf_d, cache), model, dims, att, dX, B, True, torch.zeros(S, device=DEV), neg_lr=scale,
                   hot_acc=box.hot_acc[r] if hk else None, hot_rows=hk, hot_reps=HOT_REPS if hk else 0, adam=a)
    rt = []
    for r, (db, cache, dX) in enumerate(fwd):
        dUb = torch.full((B, S, D), NAN, device=DEV); dIt = torch.full((B, D), NAN, device=DEV)
        sp.bwd_idx(box.twin_rows(emb_twin, db, uf_d), model, dims, att, dX, B, False, torch.zeros(S, device=DEV), dUb=dUb, dIt=dIt)
        rt.append(valid_terms(batches[r], host(dUb), host(dIt), box.I, scale))
    return rt


def check_sums(got, G, A, n, extra, what):
    ok = ref.within_sum_bound(got, G, n[:, None] + extra, A)
    assert ok.all(), (what, np.argwhere(~ok)[:4], float(np.abs(got - G)[~ok].max()))


def adam_consts(t, batch):
    a = sp.RowAdam()
    a.lr, a.b1, a.b2, a.eps = ADAM["lr"], ADAM["b1"], ADAM["b2"], ADAM["eps"]
    a.c1 = float(np.float32(1.0 - np.float64(np.float32(ADAM["b1"])) ** t))     # as row_adam_of forms them
    a.c2 = float(np.float32(1.0 - np.float64(np.float32(ADAM["b2"])) ** t))
    a.inv_batch = float(np.float32(1.0) / np.float32(batch))
    return a


def check_adam(w0, m0, v0, g, w, m, v, a, what):
    """the device's update of rows with gradient sums g against row_adam_elem in float64"""
    _, m_ref, v_ref, tm, tv = ref.row_adam64(w0, m0, v0, g, a.lr, a.b1, a.b2, a.eps, a.c1, a.c2, a.inv_batch)
    assert (np.abs(m - m_ref) <= tm).all(), (what, "m", float(np.abs(m - m_ref).max()))
    assert (np.abs(v - v_ref) <= tv).all(), (what, "v", float(np.abs(v - v_ref).max()))
    w_ref, tw = ref.adam_weight_from(w0, m, v, a.lr, a.eps, a.c1, a.c2)
    assert (np.abs(w - w_ref) <= tw).all(), (what, "w", float(np.abs(w - w_ref).max()))


def adam_step(box, batches, model, dims, att, uf_d, t):
    """one emulated row-Adam step with every check of the step"""
    uP, S, D, cF = dims
    W, I, hk, lde = box.W, box.I, box.hot_k, box.lde
    w_start, (m_start, v_start) = box.table(), box.moments()
    shard_bits = [bits(x) for x in box.emb]; m_bits = [bits(x) for x in box.m]; v_bits = [bits(x) for x in box.v]
    fwd, table, emb_twin = run_forward(box, batches, model, dims, att, uf_d)
    rt = run_backward(box, batches, fwd, model, dims, att, uf_d, emb_twin, adam=True)
    G, A, n = expected_sums(rt, I, D)
    hot_rows = np.arange(I) < hk
    # ---- the owners' gradient buffers before the update
    gsum = []
    for r in range(W):
        gv = box.gviews(r)
        want = [g for g in range(r, I, W) if n[g] > 0 and not hot_rows[g]]
        cnt = int(host(gv["count"])[0])
        assert cnt == len(want), ("owner %d: count" % r, cnt, len(want))
        lst = host(gv["list"])[:cnt]
        assert sorted(lst.tolist()) == sorted(g // W for g in want), ("owner %d: list" % r)
        flag = host(gv["flag"]); fw = np.zeros(box.rows_max, np.int32); fw[[g // W for g in want]] = 1
        assert np.array_equal(flag, fw), ("owner %d: flags" % r, np.argwhere(flag != fw)[:4])
        grad = host(gv["grad"])
        touched = np.zeros(box.rows_max, bool); touched[[g // W for g in want]] = True
        assert (bits(gv["grad"])[~touched] == 0).all(), ("owner %d: an untouched gradient row is not 0" % r)
        if want:
            check_sums(grad[[g // W for g in want]], G[want], A[want], n[want], 0, "owner %d: gradient rows" % r)
        assert np.isnan(host(gv["canary"].view(torch.float32))).all(), ("owner %d: gradient-buffer canary" % r)
        gsum.append(grad.copy())
    # ---- the hot rows: this rank's touch marks, the fold, the all-reduce
    for r in range(W):
        if hk:
            sp.hot_fold(box.hot_sum[r], box.hot_acc[r], hk, HOT_REPS, D)
            touch = host(box.hot_sum[r][hk * D:hk * D + hk])
            rows_r, _ = rt[r]
            tw = np.zeros(hk, np.float32); tw[np.unique(rows_r[rows_r < hk])] = 1.0
            assert np.array_equal(touch, tw), ("rank %d: hot_touch" % r, np.argwhere(touch != tw)[:4])
            assert (bits(box.hot_acc[r]) == 0).all(), "the fold leaves the replica accumulators at 0"
    if hk:
        box.all_reduce_hot()
        hs = host(box.hot_sum[0][:hk * D]).reshape(hk, D)
        check_sums(hs, G[:hk], A[:hk], n[:hk], HOT_REPS + W, "all-reduced hot-row sums")
        hsum = hs.copy(); htouch = host(box.hot_sum[0][hk * D:hk * D + hk]).copy()
    # ---- each owner's update, each rank's hot-row update
    a = adam_consts(t, B * W)
    for r in range(W):
        sp.shard_adam(box.gbuf[r], box.rows_max, box.emb[r], box.m[r], box.v[r], lde, D, a)
        if hk:
            sp.hot_adam(box.hot_tab[r], box.hot_sum[r], box.hot_sum[r][hk * D:], box.hot_m[r], box.hot_v[r], hk, D, a)
    for r in range(W):
        gv = box.gviews(r)
        assert int(host(gv["count"])[0]) == 0 and int(host(gv["ticket"])[0]) == 0, ("owner %d: count / ticket not reset" % r)
        assert (host(gv["flag"]) == 0).all() and (bits(gv["grad"]) == 0).all(), ("owner %d: flags / gradient rows not cleared" % r)
        assert np.isnan(host(gv["canary"].view(torch.float32))).all()
        gl = np.arange(r, I, W)
        touched = np.array([n[g] > 0 and not hot_rows[g] for g in gl], bool)
        nb = bits(box.emb[r]); mb = bits(box.m[r]); vb = bits(box.v[r])
        keep = np.ones(box.rows_max + CANARY, bool); keep[:len(gl)][touched] = False
        for now, before, name in ((nb, shard_bits[r], "table"), (mb, m_bits[r], "m"), (vb, v_bits[r], "v")):
            assert np.array_equal(now[keep], before[keep]), "owner %d: untouched %s rows or canaries changed" % (r, name)
        li = np.flatnonzero(touched)
        if li.size:
            gi = gl[li]
            check_adam(w_start[gi], m_start[gi], v_start[gi], gsum[r][li],
                       host(box.emb[r])[li], host(box.m[r])[li], host(box.v[r])[li], a, "owner %d" % r)
    if hk:
        for r in range(1, W):
            for x in (box.hot_tab, box.hot_m, box.hot_v):
                assert np.array_equal(bits(x[r]), bits(x[0])), "the hot replicas differ between ranks"
        assert (bits(box.hot_sum[0][:hk * (D + 1)]) == 0).all(), "k_hot_adam leaves the sums and marks at 0"
        tch = htouch > 0
        ht, hm, hv = host(box.hot_tab[0]), host(box.hot_m[0]), host(box.hot_v[0])
        assert np.array_equal(ht[:hk][~tch].view(np.int32), w_start[:hk][~tch].view(np.int32))
        assert np.array_equal(hm[:hk][~tch].view(np.int32), m_start[:hk][~tch].view(np.int32))
        assert np.isnan(ht[hk:]).all() and np.isnan(hm[hk:]).all()
        if tch.any():
            check_adam(w_start[:hk][tch], m_start[:hk][tch], v_start[:hk][tch], hsum[tch], ht[:hk][tch], hm[:hk][tch], hv[:hk][tch], a, "hot rows")
    return n


def setup_box(rng, W, D, hot_k, ifeat_sharded, adam=True):
    table, uf, itf = make_tables(rng, I_ROWS, D)
    mom = None
    if adam:
        mom = ((rng.standard_normal((I_ROWS, D)) * 1e-3).astype(np.float32), (rng.random((I_ROWS, D)) * 1e-5).astype(np.float32))
    box = Box(table, W, hot_k, mom, itf, ifeat_sharded)
    return box, dev(uf)


def att_of(rng, S):
    return dev((0.5 + rng.random(S)).astype(np.float32))


# (model, D, W, S, hot_k): every D x W for DIN-cos, every model at D = 64, the S edges at D = 64 with W = 4;
# hot_k walks 0, 1, a count that is not a multiple of W, and the whole table
HOTS = [0, 1, 5, I_ROWS]
CASES = ([(COS, D, W, 20, HOTS[(i + j) % 4]) for i, D in enumerate((16, 32, 64, 128)) for j, W in enumerate((2, 4, 8))]
         + [(m, 64, 4, 20, 5) for m in (YT, EUC)]
         + [(COS, 64, 4, S, HOTS[i % 4]) for i, S in enumerate((1, 31, 32, 33, 64))])
IDS = ["%s_D%d_W%d_S%d_hot%d" % (MNAME[m], D, W, S, h) for m, D, W, S, h in CASES]


@pytest.mark.parametrize("model,D,W,S,hot_k", CASES, ids=IDS)
def test_three_row_adam_steps(model, D, W, S, hot_k):
    """Three consecutive row-Adam steps (t = 1, 2, 3), each checked from the emulation's own start state: the forward
    against the twin, the owners' gradient buffers, the hot-row marks and sums, the owners' and the replicas' updates.
    The buffers must be clean between steps, and the bias corrections follow t."""
    rng = np.random.default_rng(1000 * D + 10 * W + S)
    box, uf_d = setup_box(rng, W, D, hot_k, ifeat_sharded=(W != 2))
    att = att_of(rng, S)
    reserved = np.array([I_ROWS - 1 - r for r in range(W)])
    zero_rows_seen = False
    for t in (1, 2, 3):
        batches = make_batches(rng, W, S, I_ROWS, D, reserved)
        n = adam_step(box, batches, model, (UP, S, D, CF), att, uf_d, t)
        zero_rows_seen |= bool((n[reserved] > 0).all())
    assert zero_rows_seen


@pytest.mark.parametrize("W", [2, 4, 8])
def test_one_cold_row_hit_by_every_slot(W):
    """Every history slot and every item of every rank is one cold row: its owner's count is exactly 1, the others' 0."""
    rng = np.random.default_rng(W)
    S, D, row = 33, 32, 77
    box, uf_d = setup_box(rng, W, D, 1, ifeat_sharded=True)
    n = adam_step(box, one_row_batches(W, S, D, row, rng), COS, (UP, S, D, CF), att_of(rng, S), uf_d, 1)
    assert n[row] == W * B * (S + 1)
    for r in range(W):
        assert int(host(box.gviews(r)["count"])[0]) == 0          # reset by the update
    assert np.count_nonzero(n) == 1


@pytest.mark.parametrize("model,D,W,S,hot_k", CASES, ids=IDS)
def test_sgd_step(model, D, W, S, hot_k):
    """One sharded SGD step: each owner's rows = start + Σ(−lr/world)·terms within the summation bound, every other row
    and canary keeps its bits; the hot rows go fold → all-reduce → k_apply_table_grad and the replicas stay identical."""
    rng = np.random.default_rng(7 + 1000 * D + 10 * W + S)
    box, uf_d = setup_box(rng, W, D, hot_k, ifeat_sharded=(W == 8), adam=False)
    att = att_of(rng, S)
    I = box.I
    start = box.table()
    before = [bits(x) for x in box.emb]
    batches = make_batches(rng, W, S, I, D, np.array([I - 1 - r for r in range(W)]))
    fwd, table, emb_twin = run_forward(box, batches, model, (UP, S, D, CF), att, uf_d)
    rt = run_backward(box, batches, fwd, model, (UP, S, D, CF), att, uf_d, emb_twin, adam=False)
    G, A, n = expected_sums(rt, I, D)
    hot = np.arange(I) < hot_k
    for r in range(W):
        gl = np.arange(r, I, W)
        now = host(box.emb[r])
        touched = np.array([n[g] > 0 and not hot[g] for g in gl], bool)
        keep = np.ones(box.rows_max + CANARY, bool); keep[:len(gl)][touched] = False
        assert np.array_equal(bits(box.emb[r])[keep], before[r][keep]), "owner %d: untouched rows or canaries changed" % r
        li = np.flatnonzero(touched)
        gi = gl[li]
        check_sums(now[li].astype(np.float64), start[gi] + G[gi], A[gi] + np.abs(start[gi]), n[gi], 1, "owner %d rows" % r)
    if hot_k:
        for r in range(W):
            sp.hot_fold(box.hot_sum[r], box.hot_acc[r], hot_k, HOT_REPS, D)
        box.all_reduce_hot()
        for r in range(W):
            sp.hot_apply_sgd(box.hot_tab[r], box.hot_sum[r], hot_k * D)
        for r in range(1, W):
            assert np.array_equal(bits(box.hot_tab[r]), bits(box.hot_tab[0])), "the hot replicas differ between ranks"
        ht = host(box.hot_tab[0])
        assert np.isnan(ht[hot_k:]).all()
        check_sums(ht[:hot_k].astype(np.float64), start[:hot_k] + G[:hot_k], A[:hot_k] + np.abs(start[:hot_k]), n[:hot_k],
                   HOT_REPS + W + 1, "hot rows")
        assert (bits(box.hot_sum[0][:hot_k * D]) == 0).all()


@pytest.mark.parametrize("model", [YT, COS, EUC], ids=MNAME.get)
@pytest.mark.parametrize("W", [2, 4, 8])
def test_peer_forward_d64_against_oracle(model, W):
    """X0 of the PEER forward at D = 64 — its own 8×2 lane map — against the oracle's attention (activation.go's cosine /
    Euclidean distance, gorgonia's sigmoid, the mean over S) at the attention family's bar of tests/test_gpu_paths.py."""
    from oracle import oracle as orc
    assert sp.lanes(False, True, 64) == (8, 2) and sp.lanes(False, False, 64) == (4, 4)
    rng = np.random.default_rng(64 + W + 10 * model)
    S, D = 33, 64
    box, uf_d = setup_box(rng, W, D, 5, ifeat_sharded=True, adam=False)
    att = (0.5 + rng.random(S)).astype(np.float32)
    batches = make_batches(rng, W, S, box.I, D, np.array([box.I - 1 - r for r in range(W)]))
    table = box.table(); uf = host(uf_d); itf = host(box.ifeat_full)
    Kp = kp_of(D)
    for r, (ur, ir, hist, nvalid, _) in enumerate(batches):
        db = (dev(ur), dev(ir), dev(hist), nvalid)
        X0 = torch.full((B, Kp), NAN, device=DEV)
        sp.fwd_idx(box.peer_rows(r, db, uf_d, None), model, (UP, S, D, CF), dev(att), X0, Kp, B, peer=True)
        clean = lambda a, n: np.where((a >= 0) & (a < n), a, -1).astype(np.int32)
        h, it, u = clean(hist, box.I), clean(ir, box.I), clean(ur, U)
        h[nvalid:] = -1; it[nvalid:] = -1; u[nvalid:] = -1
        X = orc.gather_rows(uf, itf[:, :CF], table, u, it, h)
        us = X[:, UP:UP + S * D].reshape(B, S, D); v = X[:, UP + S * D:UP + S * D + D]
        if model == YT:
            a = np.ones((B, S))
        else:
            x = orc.cosine(us, v[:, None, :]) if model == COS else orc.euc_distance(us, v[:, None, :])
            arg = ((x.astype(np.float32) + np.float32(1)) * np.float32(0.5) if model == COS else np.float32(1) - x.astype(np.float32)) * att
            a = np.vectorize(orc.sigmoid32)(arg.astype(np.float32)).astype(np.float64)
        pooled = (a[:, :, None] * us).sum(1) / S
        want = np.zeros((B, Kp)); want[:, :UP] = X[:, :UP]; want[:, UP:UP + D] = pooled; want[:, UP + D:UP + 2 * D] = v
        want[:, UP + 2 * D:UP + 2 * D + CF] = X[:, UP + S * D + D:]
        np.testing.assert_allclose(host(X0), want, rtol=2e-3, atol=2e-5 * np.abs(want).max(), err_msg="rank %d" % r)


@pytest.mark.parametrize("W,hot_k", [(2, 5), (4, 5), (8, 5), (4, I_ROWS), (8, I_ROWS)])
def test_hot_row_round_trip(W, hot_k):
    """k_hot_pull → k_hot_writeback gives back the shards bit for bit, k_hot_own + the sum over ranks gives back the
    moments; a changed replica lands in exactly its owners' rows."""
    rng = np.random.default_rng(W * 31 + hot_k)
    D = 32
    table, _, itf = make_tables(rng, I_ROWS, D)
    mom = (rng.standard_normal((I_ROWS, D)).astype(np.float32), rng.random((I_ROWS, D)).astype(np.float32))
    box = Box(table, W, hot_k, mom, itf, poison_hot=False)
    for r in range(W):
        box.hot_tab[r].fill_(NAN)
        sp.hot_pull(sp.rows(lde=D, peer_emb=box.emb, world=W), box.hot_tab[r], hot_k, D)
        assert np.array_equal(bits(box.hot_tab[r][:hot_k]), table[:hot_k].view(np.int32))
        assert np.isnan(host(box.hot_tab[r][hot_k:])).all()
    before = [bits(x) for x in box.emb]
    for r in range(W):
        sp.hot_writeback(box.emb[r], D, box.hot_tab[r], hot_k, D, W, r)
        assert np.array_equal(bits(box.emb[r]), before[r])
    for mo in (box.m, box.v):
        own = [torch.full((hot_k + CANARY, D), NAN, device=DEV) for _ in range(W)]
        for r in range(W):
            sp.hot_own(own[r], mo[r], D, hot_k, D, W, r)
        s = torch.stack([o[:hot_k] for o in own]).sum(0)
        assert np.array_equal(bits(s), box.assemble(mo)[:hot_k].view(np.int32))
        assert all(np.isnan(host(o[hot_k:])).all() for o in own)
    new = (table[:hot_k] + 1.0).astype(np.float32)
    for r in range(W):
        box.hot_tab[r][:hot_k] = dev(new)
        sp.hot_writeback(box.emb[r], D, box.hot_tab[r], hot_k, D, W, r)
    want = table.copy(); want[:hot_k] = new
    assert np.array_equal(box.assemble(box.emb).view(np.int32), want.view(np.int32))
    for r in range(W):
        assert np.isnan(host(box.emb[r][box.local[r]:])).all()


USER_CASES = ([(COS, 64, W, sh) for W in (2, 4, 8) for sh in (False, True)]
              + [(YT, 64, 4, True), (EUC, 64, 4, False), (COS, 128, 8, True), (COS, 16, 2, False)])


@pytest.mark.parametrize("model,D,W,sharded", USER_CASES,
                         ids=["%s_D%d_W%d_%s" % (MNAME[m], D, W, "ifeat_sharded" if s else "ifeat_replicated") for m, D, W, s in USER_CASES])
def test_fwd_user_peer_rows_equal_single_table(model, D, W, sharded):
    """k_attn_fwd_user<PEER> rows of rank r's local item l == k_attn_fwd_user<false> rows of global row l·W + r on the
    assembled table, bit for bit; the history holds hot rows (read from the replica), other ranks' rows and missing ids."""
    rng = np.random.default_rng(D + W + 100 * model + sharded)
    S = 33
    table, uf, itf = make_tables(rng, I_ROWS, D)
    box = Box(table, W, 5, None, itf, sharded, poison_hot=False)
    att = att_of(rng, S); uf_d = dev(uf)
    hist = rng.integers(0, I_ROWS, S).astype(np.int32)
    hist[:4] = [0, 3, -1, I_ROWS + W - 1]; hist[10] = 2 ** 30
    hist_d = dev(hist)
    Kp = kp_of(D)
    user = 7
    X0t = torch.full((I_ROWS, Kp), NAN, device=DEV)
    twin = sp.rows(emb=dev(table), lde=D, ufeat=uf_d, ldu=UP, ifeat=box.ifeat_full, ldi=LDI, n_emb=I_ROWS, n_user=U, n_ifeat=I_ROWS, world=1)
    sp.fwd_user(twin, model, (UP, S, D, CF), att, user, hist_d, 0, 0, X0t, Kp, I_ROWS, peer=False)
    xt = bits(X0t)
    for r in range(W):
        n = box.local[r]
        X0 = torch.full((n, Kp), NAN, device=DEV)
        pr = sp.rows(emb=box.emb[r], lde=D, ufeat=uf_d, ldu=UP, ifeat=box.ifeat[r] if sharded else box.ifeat_full, ldi=LDI,
                     hot_tab=box.hot_tab[r], peer_emb=box.emb, peer_ifeat=box.ifeat if sharded else (), n_emb=I_ROWS, n_user=U,
                     n_ifeat=I_ROWS, world=W, ifeat_sharded=int(sharded), hot_k=5)
        sp.fwd_user(pr, model, (UP, S, D, CF), att, user, hist_d, 0, r, X0, Kp, n, peer=True)
        assert np.array_equal(bits(X0), xt[np.arange(n) * W + r]), "rank %d" % r


@pytest.mark.parametrize("W", [2, 4, 8])
def test_gather_rows_f64(W):
    """k_gather_rows_f64 == the assembled table widened to float64; hot rows come from the replica (their shard copies
    are NaN here)"""
    rng = np.random.default_rng(W + 5)
    D = 32
    table, _, itf = make_tables(rng, I_ROWS, D)
    box = Box(table, W, 5, None, itf)
    rows = rng.permutation(I_ROWS).astype(np.int32)
    out = torch.full((I_ROWS, D), NAN, dtype=torch.float64, device=DEV)
    sp.gather_rows_f64(sp.rows(lde=D, peer_emb=box.emb, world=W, hot_k=5, hot_tab=box.hot_tab[0], n_emb=I_ROWS), dev(rows), D, out)
    assert np.array_equal(host(out), table[rows].astype(np.float64))


def _knn_single(table_d, I, D, nq, k, qrow=None, qvec=None, excl=None):
    rps = 256
    slices = max(1, (I + rps - 1) // rps)
    ls = torch.empty((nq, slices, k), dtype=torch.float64, device=DEV); lr = torch.empty((nq, slices, k), dtype=torch.int32, device=DEV)
    sp.knn_scan(table_d, I, 1, 0, D, nq, k, rps, slices, ls, lr, qvec=qvec, qrow=qrow, excl=excl)
    o_r = torch.empty((nq, k), dtype=torch.int32, device=DEV); o_s = torch.empty((nq, k), dtype=torch.float64, device=DEV)
    o_c = torch.empty(nq, dtype=torch.int32, device=DEV)
    sp.knn_merge(0, ls, lr, slices, k, slices * k, k, nq, o_r, o_s, o_c)
    return host(o_r), host(o_s), host(o_c)


def _knn_sharded(box, nq, k, qvec, excl):
    W, D = box.W, box.D
    rps = 256
    gs = torch.full((W, nq, k), NAN, dtype=torch.float64, device=DEV); gr = torch.full((W, nq, k), -5, dtype=torch.int32, device=DEV)
    for r in range(W):
        slices = max(1, (box.local[r] + rps - 1) // rps)
        ls = torch.empty((nq, slices, k), dtype=torch.float64, device=DEV); lr = torch.empty((nq, slices, k), dtype=torch.int32, device=DEV)
        sp.knn_scan(box.emb[r], box.local[r], W, r, D, nq, k, rps, slices, ls, lr, qvec=qvec, excl=excl)
        sp.knn_merge(0, ls, lr, slices, k, slices * k, k, nq, gr[r], gs[r])
    o_r = torch.empty((nq, k), dtype=torch.int32, device=DEV); o_s = torch.empty((nq, k), dtype=torch.float64, device=DEV)
    o_c = torch.empty(nq, dtype=torch.int32, device=DEV)
    sp.knn_merge(0, gs, gr, W, k, k, nq * k, nq, o_r, o_s, o_c)       # the ranks' gathered [W][n][k] lists
    return host(o_r), host(o_s), host(o_c)


@pytest.mark.parametrize("W,I,k", [(2, 1100, 40), (4, 203, 60), (8, 203, 30), (8, 37, 8)])
def test_knn_sharded_equals_single_table(W, I, k):
    """Per-rank k_knn_scan, the slice merge, then k_knn_merge over the ranks' gathered lists (sstride = n·k) == the
    single-table scan: rows exact, similarities bit-identical, counts equal.  Duplicate rows sit in different shards (the
    row-ascending tie-break crosses ranks); k may exceed a shard's rows (lists with empty entries).  Row queries take the
    engine's sharded route: the rows gathered by k_gather_rows_f64, scanned as vectors that exclude their own row."""
    rng = np.random.default_rng(W * 100 + I + k)
    D = 32
    table = (rng.standard_normal((I, D)) * 0.5).astype(np.float32)
    table[11] = table[10]; table[13] = table[10]; table[20] = table[10]
    box = Box(table, W, 0, None, np.zeros((I, LDI), np.float32), poison_hot=False)
    table_d = dev(table)
    qrows = np.array([10, 11, 0, I - 1, 13, 5, 20, 7, 3], np.int32)[:min(9, I)]
    nq = len(qrows)
    want = _knn_single(table_d, I, D, nq, k, qrow=dev(qrows))
    qv = torch.empty((nq, D), dtype=torch.float64, device=DEV)
    sp.gather_rows_f64(sp.rows(lde=D, peer_emb=box.emb, world=W, n_emb=I), dev(qrows), D, qv)
    got = _knn_sharded(box, nq, k, qv, dev(qrows))
    for g, w, name in zip(got, want, ("rows", "sims", "counts")):
        assert np.array_equal(np.asarray(g).view(np.int64 if g.dtype == np.float64 else np.int32),
                              np.asarray(w).view(np.int64 if w.dtype == np.float64 else np.int32)), name
    tie = list(want[0][0][:3])
    assert tie == [11, 13, 20], tie                        # the query row itself is excluded, the equal rows ascend
    vec = dev(rng.standard_normal((5, D)))
    want = _knn_single(table_d, I, D, 5, k, qvec=vec)
    got = _knn_sharded(box, 5, k, vec, None)
    assert all(np.array_equal(a, b) for a, b in zip(got, want))


@pytest.mark.parametrize("W,k", [(2, 25), (4, 25), (8, 30)])
def test_rec_sharded_equals_numpy_topk(W, k):
    """Per-rank k_rec_scan over the rank's local logits (several slices), the slice merge, then k_knn_merge<LogitKey>
    over the ranks' gathered [W][users][k] lists == numpy's top-k of (logit descending, global row ascending).  NaN
    logits never enter; tied logits sit on different ranks; the exclusion list names rows of every rank, duplicates and
    rows outside the table."""
    rng = np.random.default_rng(W * 7 + k)
    I, nu, nex = I_ROWS, 3, 12
    z = rng.standard_normal((nu, I)).astype(np.float32)
    z[:, rng.integers(0, I, 15)] = np.nan
    z[:, 40:48] = np.float32(2.5)                            # ties across ranks, near the top
    z[1, 60] = -np.inf
    z[2] = np.nan; z[2, :10] = rng.standard_normal(10)       # fewer qualifying rows than k
    excl = np.stack([np.concatenate([[41, 43, 41, -1, I + 2, 2 ** 30], rng.integers(0, I, nex - 6)]) for _ in range(nu)]).astype(np.int32)
    gs = torch.empty((W, nu, k), device=DEV); gr = torch.empty((W, nu, k), dtype=torch.int32, device=DEV)
    rps = 40
    for r in range(W):
        n = len(range(r, I, W))
        slices = (n + rps - 1) // rps
        for u in range(nu):
            ls = torch.empty((slices, k), device=DEV); lr = torch.empty((slices, k), dtype=torch.int32, device=DEV)
            sp.rec_scan(dev(z[u, r::W].copy()), n, 0, W, r, rps, dev(excl[u]), nex, k, ls, lr)
            sp.knn_merge(1, ls, lr, slices, k, slices * k, k, 1, gr[r, u], gs[r, u])
    o_r = torch.empty((nu, k), dtype=torch.int32, device=DEV); o_s = torch.empty((nu, k), device=DEV)
    o_c = torch.empty(nu, dtype=torch.int32, device=DEV)
    sp.knn_merge(1, gs, gr, W, k, k, nu * k, nu, o_r, o_s, o_c)
    for u in range(nu):
        keep = ~np.isin(np.arange(I), excl[u])
        wr, ws, wc = ref.topk(z[u][keep], np.arange(I)[keep], k, lambda s: s == s)
        assert int(host(o_c)[u]) == wc, (u, int(host(o_c)[u]), wc)
        assert np.array_equal(host(o_r)[u], wr), (u, host(o_r)[u], wr)
        assert np.array_equal(host(o_s)[u].view(np.int32), ws.view(np.int32)), u
        if u == 2:
            assert wc < k                                    # the list ends in empty entries
