"""The float64 MLP's serving kernels on a row-sharded ITEM_EMB, on one GPU: W = 2, 4 and 8 ranks emulated as W shards of
one device through the kernel-level probe tests/cuda/shard_mlp_probe.cu (attn.cuh, mlp64.cuh and rec.cuh themselves,
not copies).  Global row g of a table is local row g // W of shard g % W; RowSrc::peer_emb[j] points at shard j.

Bars, all bit for bit against the single-table kernels over the assembled tables:
  * the key-fed gather k_gather_rows<PEER>: -1 and past-the-table ids, hot rows whose shard copies are NaN (a read
    from the shard instead of the hot-row replica shows), ITEM_FEAT sharded and replicated, shorter than ITEM_EMB;
  * the prefix k_mlp64_prefix<true>, for windows that mix hot, remote, local and missing rows;
  * layer 0 and the later layers: each rank's logits of its local rows, chunk by chunk, stitched back into global
    order, for both SMEM_W forms, chunks that do not divide the shard, empty shards (I < W), ITEM_FEAT sharded and
    replicated, NaN and -0 logits;
  * the Logit64Key selection and rank at (world, rank), the engine's exchanges emulated as [W] stacks, equal to
    world = 1 under CTR_EXCLUDE_NONE, _WINDOW and _SEEN, and under SEEN to the owner-rule numpy model of
    test_gpu_shard_seen_probe.py."""
import numpy as np
import pytest
import torch

from tests import shard_mlp_probe as mp
from tests import shard_probe as sp
from tests import shard_ref as ref
from tests import shard_seen_probe as ssp
from tests.test_gpu_shard_seen_probe import cache_dev, make_cache, seen_mask

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

DEV = "cuda"
WS = [2, 4, 8]
MAXK = 1024
RPS = 40
UP, S, D, CF = 4, 6, 16, 3


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def bits(t):
    a = t.cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)
    return np.ascontiguousarray(a).view(np.int64 if a.dtype == np.float64 else np.int32)


def shard(tab, W, r):
    """rank r's shard of a [rows, w] float32 table (one zero row when it owns none, so the pointer is valid)"""
    s = tab[r::W]
    return dev(s if s.shape[0] else np.zeros((1, tab.shape[1]), np.float32))


def tables(rng, I, n_user, n_ifeat):
    emb = rng.standard_normal((I, D)).astype(np.float32)
    ufeat = rng.standard_normal((n_user, UP)).astype(np.float32)
    ifeat = rng.standard_normal((n_ifeat, CF)).astype(np.float32)
    return emb, ufeat, ifeat


def peer_rows(emb, ifeat, W, hot_k, ifeat_sharded, **kw):
    """a RowSrc of a row-sharded ITEM_EMB (the hot rows' shard copies poisoned with NaN) and the buffers it points at"""
    I = emb.shape[0]
    poisoned = emb.copy()
    poisoned[:hot_k] = np.nan
    shards = [shard(poisoned, W, r) for r in range(W)]
    hot = dev(emb[:max(hot_k, 1)])
    if ifeat_sharded:
        feat = [shard(ifeat, W, r) for r in range(W)]
        extra = dict(peer_ifeat=feat, ldi=CF)
    else:
        feat = dev(ifeat)
        extra = dict(ifeat=feat, ldi=CF)
    keep = [shards, hot, feat]                                          # the row source holds only their addresses
    r = sp.rows(lde=D, peer_emb=shards, n_emb=I, n_ifeat=ifeat.shape[0], world=W, ifeat_sharded=int(ifeat_sharded), hot_k=hot_k,
                hot_tab=hot, **extra, **kw)
    return r, keep


def ids(rng, n, I, special):
    a = rng.integers(-1, I + 4, n).astype(np.int32)
    a[:len(special)] = special
    return a


@pytest.mark.parametrize("W", WS)
def test_key_fed_gather(W):
    rng = np.random.default_rng(W)
    I, n_user, hot_k, B = 203, 40, 20, 96
    emb, ufeat, ifeat = tables(rng, I, n_user, I - 30)          # ITEM_FEAT shorter than ITEM_EMB
    user = dev(ids(rng, B, n_user, [-1, n_user, n_user + 9, 0]))
    item = dev(ids(rng, B, I, [-1, I, I + 3, 0, 1, hot_k - 1, hot_k, I - 1, I - 31, I - 30]))
    hist = dev(ids(rng, B * S, I, [-1, I, 3, hot_k - 1, hot_k, W, W + 1, I - 1]))
    nin = UP + S * D + D + CF
    want = torch.full((B, nin + 3), -7.0, dtype=torch.float64, device=DEV)
    buf = [dev(emb), dev(ufeat), dev(ifeat)]
    r1 = sp.rows(emb=buf[0], lde=D, ufeat=buf[1], ldu=UP, ifeat=buf[2], ldi=CF, user_row=user, item_row=item, hist=hist, nvalid=B, n_emb=I,
                 n_user=n_user, n_ifeat=I - 30)
    mp.gather(r1, False, (UP, S, D, CF), want, B)
    assert not torch.isnan(want).any()
    for fsh in (False, True):
        for hk in (0, hot_k):                                           # 0: no replica, the shards hold every row
            rw, keep = peer_rows(emb, ifeat, W, hk, fsh, ufeat=buf[1], ldu=UP, user_row=user, item_row=item, hist=hist, nvalid=B, n_user=n_user)
            got = torch.full_like(want, -7.0)
            mp.gather(rw, True, (UP, S, D, CF), got, B)
            assert np.array_equal(bits(got), bits(want)), (W, fsh, hk)


def net_params(rng, units, scale=0.3):
    n = sum(units[l + 1] * (1 + units[l]) for l in range(len(units) - 1))
    return rng.standard_normal(n) * scale


@pytest.mark.parametrize("W", WS)
def test_prefix(W):
    rng = np.random.default_rng(20 + W)
    I, hot_k = 203, 20
    emb, ufeat, ifeat = tables(rng, I, 8, I)
    units = [UP + S * D + D + CF, 37, 9, 1]
    net = mp.Net(units)
    params = dev(net_params(rng, units))
    buf = [dev(emb)]
    r1 = sp.rows(emb=buf[0], lde=D, n_emb=I)
    urow = dev(ufeat[3])
    windows = [[0, hot_k - 1, hot_k, 1 + W, -1, I + 2],               # hot, remote and local rows, missing ones
               [-1] * S, [I - 1, I - 2, 5, 5, hot_k, 2 ** 30]]
    for win in windows:
        h = dev(np.array(win, np.int32))
        for u in (urow, None):
            want = torch.empty(37, dtype=torch.float64, device=DEV)
            mp.prefix(False, params, net, u, UP, r1, h, S, D, want)
            rw, keep = peer_rows(emb, ifeat, W, hot_k, False)
            got = torch.empty_like(want)
            mp.prefix(True, params, net, u, UP, rw, h, S, D, got)
            assert np.array_equal(bits(got), bits(want)), (W, win)


def score_single(smem_w, params, net, pre, pcols, emb, ifeat, n_ifeat, I, acts_n):
    z = torch.full((max(I, 1),), -5.0, dtype=torch.float64, device=DEV)
    acts = torch.empty(acts_n, dtype=torch.float64, device=DEV)
    mp.score(smem_w, params, net, pre, pcols, dev(emb), None if ifeat is None else dev(ifeat), n_ifeat, 1, 0, D, CF, 0, I, 4, acts, z)
    return z[:I]


def score_sharded(smem_w, params, net, pre, pcols, emb, ifeat, W, fsh, bc, acts_n):
    """every rank scores its local rows chunk by chunk; the logits stitched back into global order"""
    I = emb.shape[0]
    out = torch.full((I,), -5.0, dtype=torch.float64, device=DEV)
    acts = torch.empty(acts_n, dtype=torch.float64, device=DEV)
    full_f = dev(ifeat)
    for r in range(W):
        e = shard(emb, W, r)
        n = len(range(r, I, W))
        f = shard(ifeat, W, r) if fsh else full_f
        nf = len(range(r, ifeat.shape[0], W)) if fsh else ifeat.shape[0]
        for i0 in range(0, n, bc):
            nb = min(bc, n - i0)
            z = torch.empty(nb, dtype=torch.float64, device=DEV)
            mp.score(smem_w, params, net, pre, pcols, e, f, nf, 1 if fsh else W, 0 if fsh else r, D, CF, i0, nb, min(4, (nb + 127) // 128), acts, z)
            out[torch.arange(r + i0 * W, r + (i0 + nb) * W, W, device=DEV)] = z
    return out


@pytest.mark.parametrize("W", WS)
def test_layer0_and_later_layers(W):
    rng = np.random.default_rng(30 + W)
    pcols = UP + S * D
    for units, hidden_act in (([pcols + D + CF, 37, 9, 1], 0), ([pcols + D + CF, 12, 1], 3), ([pcols + D + CF, 1], 0)):
        net = mp.Net(units, hidden_act=hidden_act)
        params = dev(net_params(rng, units))
        pre = dev(rng.standard_normal(units[1]))
        acts_n = 4096 * sum(units[1:])
        for I in sorted({1, W - 1, 203, 1000}):
            if I < 1:
                continue
            emb, _, ifeat = tables(rng, I, 1, max(1, I - 7))
            if I > 10:
                emb[5] = np.nan                                         # a NaN logit
            for smem_w in (0, 1):
                want = score_single(smem_w, params, net, pre, pcols, emb, ifeat, ifeat.shape[0], I, acts_n)
                if I > 10:
                    assert torch.isnan(want[5])
                for fsh in (False, True):
                    for bc in (37, 128, 4096):                          # chunks that do and do not divide the shard
                        got = score_sharded(smem_w, params, net, pre, pcols, emb, ifeat, W, fsh, bc, acts_n)
                        assert np.array_equal(bits(got), bits(want)), (W, units, I, smem_w, fsh, bc)


@pytest.mark.parametrize("W", WS)
def test_negative_zero_logits(W):
    """A network without hidden layers whose item columns underflow to -0 in every FMA and whose bias is -0: the
    items whose columns are all positive and tiny get the logit -0, the others +0 or a finite value."""
    rng = np.random.default_rng(40 + W)
    pcols = UP + S * D
    units = [pcols + D + CF, 1]
    net = mp.Net(units)
    p = np.zeros(1 + units[0])
    p[0] = -0.0
    p[1 + pcols:] = -1e-300
    params = dev(p)
    pre = dev(np.zeros(1))
    I = 203
    emb = np.full((I, D), 1e-30, np.float32)
    ifeat = np.full((I - 50, CF), 1e-30, np.float32)
    emb[::3] = 0.0
    ifeat[::3] = 0.0                                                    # rows 0, 3, 6, ...: every product +0, the logit +0
    emb[7] = 1.0
    want = score_single(0, params, net, pre, pcols, emb, ifeat, I - 50, I, 4096)
    w = want.cpu().numpy()
    assert (np.signbit(w) & (w == 0)).sum() > 50 and ((~np.signbit(w)) & (w == 0)).sum() > 50
    for smem_w in (0, 1):
        for fsh in (False, True):
            got = score_sharded(smem_w, params, net, pre, pcols, emb, ifeat, W, fsh, 37, 4096)
            assert np.array_equal(bits(got), bits(want)), (W, smem_w, fsh)


# ---- the Logit64Key selection and rank, as RecTopk::user / RecRank::pass launch them on every rank
def run_topk(z, W, k, bc, excl=None, seens=None):
    I = z.size
    nex = 0 if excl is None else excl.numel()
    gs = torch.empty((W, k), dtype=torch.float64, device=DEV); gr = torch.empty((W, k), dtype=torch.int32, device=DEV)
    maxsl = (bc + RPS - 1) // RPS
    for r in range(W):
        n = len(range(r, I, W))
        zr = dev(z[r::W].copy() if n else np.zeros(1))
        sl_s = torch.empty((1 + maxsl) * k, dtype=torch.float64, device=DEV); sl_r = torch.empty((1 + maxsl) * k, dtype=torch.int32, device=DEV)
        nch = (n + bc - 1) // bc
        for c in range(nch):
            i0 = c * bc; nb = min(bc, n - i0)
            slices = (nb + RPS - 1) // RPS
            first, last = c == 0, c == nch - 1
            mp.scan(zr[i0:], nb, i0, W, r, RPS, excl, nex, None if seens is None else seens[r], k, None if first else sl_s,
                    None if first else sl_r, sl_s[k:], sl_r[k:])
            ns = slices if first else slices + 1
            src_s, src_r = (sl_s[k:], sl_r[k:]) if first else (sl_s, sl_r)
            mp.merge(src_s, src_r, ns, k, ns * k, k, 1, gr[r] if last else sl_r, gs[r] if last else sl_s)
        if nch == 0:
            mp.merge(sl_s, sl_r, 0, k, 0, 0, 1, gr[r], gs[r])
    o_r = torch.empty(k, dtype=torch.int32, device=DEV); o_s = torch.empty(k, dtype=torch.float64, device=DEV)
    o_c = torch.empty(1, dtype=torch.int32, device=DEV)
    mp.merge(gs, gr, W, k, k, k, 1, o_r, o_s, o_c)                     # the ranks' gathered [W][k] lists, merged
    return o_r.cpu().numpy(), o_s.cpu().numpy(), int(o_c.item())


def run_ranks(z, rows, W, bc, excl=None, seens=None):
    I, m = z.size, rows.size
    nex = 0 if excl is None else excl.numel()
    rows_d = dev(rows.astype(np.int32))
    shards = [dev(z[r::W].copy() if len(range(r, I, W)) else np.zeros(1)) for r in range(W)]
    tl = torch.full((W, m), float("nan"), dtype=torch.float64, device=DEV)
    flag = torch.full((W, m), 7, dtype=torch.int32, device=DEV)
    for r in range(W):
        n = len(range(r, I, W))
        for c in sorted({(int(t) // W) // bc for t in rows if 0 <= t < I and t % W == r}):
            i0 = c * bc; nb = min(bc, n - i0)
            mp.target_logits(shards[r][i0:], nb, i0, W, r, rows_d, m, tl[r], None if seens is None else seens[r], None if seens is None else flag[r])
    states, bins = [], []
    for r in range(W):
        st = dict(place=torch.empty(m, dtype=torch.int32, device=DEV), nvalid=torch.empty(1, dtype=torch.int32, device=DEV),
                  ss=torch.empty(MAXK, dtype=torch.float64, device=DEV), sr=torch.empty(MAXK, dtype=torch.int32, device=DEV),
                  bins=torch.full((MAXK + 1,), -1, dtype=torch.int64, device=DEV))
        mp.sort(rows_d, tl, m, W, m, I, excl, nex, None if seens is None else flag, st["place"], st["nvalid"], st["ss"], st["sr"], st["bins"])
        n = len(range(r, I, W))
        for i0 in range(0, n, bc):
            mp.count(shards[r][i0:], min(bc, n - i0), i0, W, r, excl, nex, None if seens is None else seens[r], st["ss"], st["sr"], st["nvalid"],
                     st["bins"])
        states.append(st); bins.append(st["bins"][:m + 1])
    total = torch.stack(bins).sum(0)                                      # the all-reduce
    ranks, logits = [], []
    for r in range(W):
        o_r = torch.empty(m, dtype=torch.int64, device=DEV); o_l = torch.empty(m, dtype=torch.float64, device=DEV)
        mp.finish(rows_d, tl, m, W, states[r]["place"], m, I, total.clone(), o_r, o_l)
        ranks.append(o_r.cpu().numpy()); logits.append(o_l.cpu().numpy())
    return np.stack(ranks), np.stack(logits)


def numpy_ranks(z, mask, rows):
    I = z.size
    keep = ~np.isnan(z) & ~mask
    idx = np.arange(I)
    ranks, logits = [], []
    for t in rows:
        t = int(t)
        if t < 0 or t >= I:
            ranks.append(-1); logits.append(np.nan); continue
        logits.append(z[t])
        if np.isnan(z[t]) or mask[t]:
            ranks.append(-1); continue
        ranks.append(1 + int((keep & ((z > z[t]) | ((z == z[t]) & (idx < t)))).sum()))
    return np.array(ranks, np.int64), np.array(logits, np.float64)


def logits64(rng, I):
    z = rng.standard_normal(I)
    z[rng.integers(0, I, max(1, I // 20))] = np.nan
    if I > 60:
        z[40:48] = 2.5                                                  # equal logits on every rank
        z[50:54] = -0.0
        z[54:58] = 0.0                                                  # -0 and +0 tie, the row decides
    return z


def bitmaps(I, W, caches_d, u, max_ts, hist_d, nh):
    out = []
    for r in range(W):
        n = len(range(r, I, W))
        seen = torch.full((max(1, (n + 31) // 32),), -1, dtype=torch.int32, device=DEV)
        ssp.build_seen(caches_d[r], u, max_ts, hist_d, nh, I, W, r, n, seen)
        out.append(seen)
    return out


def check_mode(z, W, rows, hist, mode, caches=None, u=0, max_ts=0, ks=(1, 25, 300), bc=37):
    I = z.size
    hist_d = dev(np.asarray(hist if len(hist) else [-1], np.int32))
    mask = np.zeros(I, bool)
    excl = seens = seens1 = None
    if mode == "window":
        excl = hist_d if len(hist) else None
        mask = seen_mask(I, 1, [None], u, max_ts, hist)
    elif mode == "seen":
        caches_d = [cache_dev(c) for c in caches]
        seens = bitmaps(I, W, caches_d, u, max_ts, hist_d, len(hist))
        mask = seen_mask(I, W, caches, u, max_ts, hist)
        if all(c is caches[0] for c in caches):
            seens1 = bitmaps(I, 1, caches_d[:1], u, max_ts, hist_d, len(hist))
    for k in ks:
        got = run_topk(z, W, k, bc, excl, seens)
        wr, ws, wc = ref.topk(z[~mask], np.arange(I)[~mask], k, lambda s: s == s)
        assert got[2] == wc and np.array_equal(got[0], wr), (W, k, mode)
        assert np.array_equal(bits(got[1]), bits(ws)), (W, k, mode)
        if mode != "seen" or seens1 is not None:
            one = run_topk(z, 1, k, bc * W, excl, seens1)
            assert one[2] == got[2] and np.array_equal(one[0], got[0]) and np.array_equal(bits(one[1]), bits(got[1]))
    want_r, want_l = numpy_ranks(z, mask, rows)
    got_r, got_l = run_ranks(z, rows, W, bc, excl, seens)
    for r in range(W):
        assert np.array_equal(got_r[r], want_r), (W, r, mode, np.argwhere(got_r[r] != want_r)[:5].ravel())
        assert np.array_equal(bits(got_l[r]), bits(want_l)), (W, r, mode)
    if mode != "seen" or seens1 is not None:
        o_r, o_l = run_ranks(z, rows, 1, bc * W, excl, seens1)
        assert np.array_equal(o_r[0], got_r[0]) and np.array_equal(bits(o_l[0]), bits(got_l[0]))


def targets(rng, I, z):
    rows = rng.integers(-3, I + 5, 200).astype(np.int32)
    nan = np.flatnonzero(np.isnan(z))[:5]
    extra = np.concatenate([nan, [40, 41, 47, 50, 51, 55, 13, -1, I, I + 7, 2 ** 30]]).astype(np.int32)
    rows[:extra.size] = extra
    rows[extra.size] = rows[0]                                          # a target named twice
    return rows


@pytest.mark.parametrize("W", WS)
def test_selection_and_rank_logit64(W):
    rng = np.random.default_rng(50 + W)
    for I in (203, 5003):
        z = logits64(rng, I)
        rows = targets(rng, I, z)
        hist = [45, -1, I + 1, 45, 13, 51]
        check_mode(z, W, rows, hist, "none")
        check_mode(z, W, rows, hist, "window")
        seqs = make_cache(rng, 4, I)
        for mt in (0, 5, -3):
            check_mode(z, W, rows, hist, "seen", caches=[seqs] * W, u=1, max_ts=mt)
        divergent = [make_cache(rng, 4, I) for _ in range(W)]
        divergent[1] = None                                             # a rank without a cache
        check_mode(z, W, rows, hist, "seen", caches=divergent, u=2, max_ts=0, ks=(25,))
    for I in sorted({1, W - 1}):                                        # empty shards
        z = rng.standard_normal(I)
        rows = np.array([0, I - 1, I, -1, W], np.int32)
        for mode in ("none", "window"):
            check_mode(z, W, rows, [I + 3, 0], mode, ks=(1, 5))
