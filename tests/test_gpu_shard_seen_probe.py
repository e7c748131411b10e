"""The CTR_EXCLUDE_SEEN kernels on a row-sharded ITEM_EMB, on one GPU: W = 2, 4 and 8 ranks emulated as W shards of
one device through the kernel-level probe tests/cuda/shard_seen_probe.cu (ubcache.cuh and rec.cuh themselves, not
copies).

Rank r holds the logits z[r::W] (global row g is local row g // W of rank g % W) and its own behaviour cache.  Each rank
builds the seen bitmap over its local rows with k_ub_seen, then runs RecTopk::user (k_rec_scan_seen and the slice
merges, chunk by chunk) and RecRank::pass (k_rec_target_logits with the owner's flags, k_rec_rank_sort_seen,
k_rec_rank_seen, k_rec_rank_finish) as the engine launches them.  The engine's exchanges are emulated: the all-gathers
of the lists, target logits and flags are [W] stacks, the all-reduce of the bins a torch sum.  A slot a rank does not
own stays NaN (logits) or set (flags), so a value read from the wrong rank shows.

Bars, exact:
  * the same cache on every rank: every rank's lists and ranks equal, bit for bit, those of the single-table kernels
    (world = 1, a bitmap over the global rows) over the whole table and that cache;
  * caches that differ: a numpy model of the owner rule — row g is seen when it is a valid row of the window, or when
    rank g % W's cache holds an event of the user with ts <= the cut (0: every event) whose item is g."""
import numpy as np
import pytest
import torch

from tests import shard_ref as ref
from tests import shard_seen_probe as sp

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

DEV = "cuda"
MAXK = 1024
BC = 37                          # local rows per chunk: neither a divisor nor a multiple of kRankRows (2048)
RPS = 40                         # rows per selection slice
I64_MIN, I64_MAX = -2 ** 63, 2 ** 63 - 1
WS = [2, 4, 8]


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def f32bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.int32)


# ---- behaviour caches: per user a time-descending list of (ts, item)
def make_cache(rng, n_users, I, lens=None, ts_pool=None):
    """lists of (ts, item) per user, time-descending with tied runs; items include -1, repeats and rows past the table"""
    seqs = []
    for u in range(n_users):
        n = int(rng.integers(0, 40)) if lens is None else lens[u]
        pool = np.arange(1, 12) if ts_pool is None else ts_pool
        ts = np.sort(rng.choice(pool, n))[::-1].astype(np.int64)       # few distinct values: tied runs
        items = rng.integers(-1, I + 3, n).astype(np.int64)
        if n > 3:
            items[1] = items[0]                                         # a repeated row
        seqs.append(list(zip(ts.tolist(), items.tolist())))
    return seqs


def cache_dev(seqs):
    if seqs is None:
        return None
    off = np.concatenate([[0], np.cumsum([len(s) for s in seqs])]).astype(np.int64)
    ts = np.array([t for s in seqs for t, _ in s], np.int64)
    items = np.array([i for s in seqs for _, i in s], np.int32)
    if ts.size == 0:                                                    # keep a valid pointer
        ts = np.zeros(1, np.int64); items = np.zeros(1, np.int32)
    return dev(off), dev(ts), dev(items)


def seen_mask(I, W, caches, u, max_ts, hist):
    """the owner rule in numpy"""
    mask = np.zeros(I, bool)
    for h in hist:
        if 0 <= h < I:
            mask[h] = True
    for r in range(W):
        seqs = caches[r]
        if seqs is None or not 0 <= u < len(seqs):
            continue
        for t, it in seqs[u]:
            if (max_ts == 0 or t <= max_ts) and 0 <= it < I and it % W == r:
                mask[it] = True
    return mask


def numpy_topk(z, mask, k):
    keep = ~mask
    return ref.topk(z[keep], np.arange(z.size)[keep], k, lambda s: s == s)


def numpy_ranks(z, mask, rows):
    I = z.size
    keep = ~np.isnan(z) & ~mask
    idx = np.arange(I)
    ranks, logits = [], []
    for t in rows:
        t = int(t)
        if t < 0 or t >= I:
            ranks.append(-1); logits.append(np.float32(np.nan)); continue
        logits.append(z[t])
        if np.isnan(z[t]) or mask[t]:
            ranks.append(-1); continue
        before = keep & ((z > z[t]) | ((z == z[t]) & (idx < t)))
        ranks.append(1 + int(before.sum()))
    return np.array(ranks, np.int64), np.array(logits, np.float32)


# ---- the engine's passes on W emulated ranks
def seen_bitmaps(I, W, caches_d, u, max_ts, hist_d, S):
    out = []
    for r in range(W):
        n = len(range(r, I, W))
        seen = torch.full((max(1, (n + 31) // 32),), -1, dtype=torch.int32, device=DEV)
        sp.build_seen(caches_d[r], u, max_ts, hist_d, S, I, W, r, n, seen)
        out.append(seen)
    return out


def run_topk(z, caches_d, u, max_ts, hist, W, k, bc, one=False):
    """RecTopk::user on every rank, then the merge of the ranks' lists.  Returns (rows, logits, count)."""
    I = z.size
    hist_d = dev(np.asarray(hist, np.int32))
    seens = seen_bitmaps(I, W, caches_d, u, max_ts, hist_d, len(hist))
    gs = torch.empty((W, k), device=DEV); gr = torch.empty((W, k), dtype=torch.int32, device=DEV)
    maxsl = (bc + RPS - 1) // RPS
    for r in range(W):
        n = len(range(r, I, W))
        zr = dev(z[r::W].copy())
        sl_s = torch.empty((1 + maxsl) * k, device=DEV); sl_r = torch.empty((1 + maxsl) * k, dtype=torch.int32, device=DEV)
        nch = (n + bc - 1) // bc
        for c in range(nch):
            i0 = c * bc; nb = min(bc, n - i0)
            slices = (nb + RPS - 1) // RPS
            first, last = c == 0, c == nch - 1
            sp.scan(one, zr[i0:], nb, i0, W, r, RPS, seens[r], k, None if first else sl_s, None if first else sl_r, sl_s[k:], sl_r[k:])
            ns = slices if first else slices + 1
            src_s, src_r = (sl_s[k:], sl_r[k:]) if first else (sl_s, sl_r)
            sp.merge(src_s, src_r, ns, k, ns * k, k, 1, gr[r] if last else sl_r, gs[r] if last else sl_s)
        if nch == 0:                                                    # an empty shard: an empty list
            sp.merge(sl_s, sl_r, 0, k, 0, 0, 1, gr[r], gs[r])
    o_r = torch.empty(k, dtype=torch.int32, device=DEV); o_s = torch.empty(k, device=DEV); o_c = torch.empty(1, dtype=torch.int32, device=DEV)
    sp.merge(gs, gr, W, k, k, k, 1, o_r, o_s, o_c)                     # the ranks' gathered [W][k] lists
    return o_r.cpu().numpy(), o_s.cpu().numpy(), int(o_c.item())


def run_ranks(z, caches_d, u, max_ts, hist, rows, W, bc, one=False):
    """RecRank::pass on every rank.  Returns (ranks [W][m], logits [W][m])."""
    I, m = z.size, rows.size
    rows_d = dev(rows.astype(np.int32))
    hist_d = dev(np.asarray(hist, np.int32))
    seens = seen_bitmaps(I, W, caches_d, u, max_ts, hist_d, len(hist))
    shards = [dev(z[r::W].copy()) for r in range(W)]
    tl = torch.full((W, m), float("nan"), device=DEV)                     # [W][m]: the all-gathered target logits ...
    flag = torch.full((W, m), 7, dtype=torch.int32, device=DEV)         # ... and seen flags
    for r in range(W):
        n = len(range(r, I, W))
        for c in sorted({(int(t) // W) // bc for t in rows if 0 <= t < I and t % W == r}):
            i0 = c * bc; nb = min(bc, n - i0)
            sp.target_logits(shards[r][i0:], nb, i0, W, r, rows_d, m, tl[r], seens[r], flag[r])
    states, bins = [], []
    for r in range(W):
        st = dict(place=torch.empty(m, dtype=torch.int32, device=DEV), nvalid=torch.empty(1, dtype=torch.int32, device=DEV),
                  ss=torch.empty(MAXK, device=DEV), sr=torch.empty(MAXK, dtype=torch.int32, device=DEV),
                  bins=torch.full((MAXK + 1,), -1, dtype=torch.int64, device=DEV))
        sp.sort(one, rows_d, tl, m, W, m, I, flag, seens[r], st["place"], st["nvalid"], st["ss"], st["sr"], st["bins"])
        n = len(range(r, I, W))
        for i0 in range(0, n, bc):
            sp.count(one, shards[r][i0:], min(bc, n - i0), i0, W, r, seens[r], st["ss"], st["sr"], st["nvalid"], st["bins"])
        states.append(st); bins.append(st["bins"][:m + 1])
    total = torch.stack(bins).sum(0)                                      # the all-reduce
    ranks, logits = [], []
    for r in range(W):
        o_r = torch.empty(m, dtype=torch.int64, device=DEV); o_l = torch.empty(m, device=DEV)
        sp.finish(rows_d, tl, m, W, states[r]["place"], m, I, total.clone(), o_r, o_l)
        ranks.append(o_r.cpu().numpy()); logits.append(o_l.cpu().numpy())
    return np.stack(ranks), np.stack(logits)


def check(z, caches, u, max_ts, hist, rows, W, ks=(1, 25, 300), bc=BC):
    """caches: W per-rank caches (lists of sequences, or None).  When they are all the same, the single-table kernels
    over that cache are the reference too."""
    I = z.size
    caches_d = [cache_dev(c) for c in caches]
    mask = seen_mask(I, W, caches, u, max_ts, hist)
    same = all(c is caches[0] for c in caches)
    if same:
        assert np.array_equal(mask, seen_mask(I, 1, caches[:1], u, max_ts, hist))
    for k in ks:
        got = run_topk(z, caches_d, u, max_ts, hist, W, k, bc)
        wr, ws, wc = numpy_topk(z, mask, k)
        assert got[2] == wc and np.array_equal(got[0], wr), (W, k, u, max_ts, got[0][:8], wr[:8])
        assert np.array_equal(f32bits(got[1]), f32bits(ws)), (W, k)
        if same:
            for one in (True, False):                                   # both world = 1 forms
                o = run_topk(z, caches_d[:1], u, max_ts, hist, 1, k, bc * W, one=one)
                assert o[2] == got[2] and np.array_equal(o[0], got[0]) and np.array_equal(f32bits(o[1]), f32bits(got[1]))
    want_r, want_l = numpy_ranks(z, mask, rows)
    got_r, got_l = run_ranks(z, caches_d, u, max_ts, hist, rows, W, bc)
    for r in range(W):
        assert np.array_equal(got_r[r], want_r), (W, r, u, max_ts, np.argwhere(got_r[r] != want_r)[:5].ravel())
        assert np.array_equal(f32bits(got_l[r]), f32bits(want_l)), (W, r)
    if same:
        for one in (True, False):
            o_r, o_l = run_ranks(z, caches_d[:1], u, max_ts, hist, rows, 1, bc * W, one=one)
            assert np.array_equal(o_r[0], got_r[0]) and np.array_equal(f32bits(o_l[0]), f32bits(got_l[0]))
    # the rank/list invariant: a target ranked r <= k sits at place r - 1 of the top-k list
    lr, _, lc = run_topk(z, caches_d, u, max_ts, hist, W, MAXK, bc)
    for t, rk in zip(rows, want_r):
        if 0 < rk <= lc:
            assert lr[rk - 1] == t
        elif 0 <= t < I:
            assert t not in lr[:lc].tolist()
    return mask, want_r


def logits(rng, I):
    z = rng.standard_normal(I).astype(np.float32)
    z[rng.integers(0, I, max(1, I // 20))] = np.nan
    if I > 48:
        z[40:48] = np.float32(2.5)                                      # equal logits on every rank
    return z


def cuts(seq):
    """0, the int64 extremes, and every tied run's ts with its edges ±1"""
    out = {0, I64_MIN, I64_MAX}
    for t, _ in seq:
        out |= {t, t - 1, t + 1}
    return sorted(c for c in out if I64_MIN <= c <= I64_MAX)


def targets(rng, I, mask, z, hist):
    rows = rng.integers(-3, I + 5, 200).astype(np.int32)
    seen = np.flatnonzero(mask)[:20]
    nan = np.flatnonzero(np.isnan(z))[:5]
    extra = np.concatenate([seen, nan, [h for h in hist if 0 <= h < I][:3], [40, 41, 47, -1, I, I + 7, 2 ** 30]]).astype(np.int32)
    rows[:extra.size] = extra
    rows[extra.size] = rows[extra.size + 1] = rows[0]                   # a target named twice
    return rows


@pytest.mark.parametrize("W", WS)
def test_same_cache_on_every_rank(W):
    """Every rank holds the same cache: every user, every cut (0, the int64 extremes, inside tied runs and at their
    edges), users outside the cache; lists for k in {1, 25, 300}, ranks of seen, NaN, tied, window and out-of-table
    targets — equal to the single-table kernels and to numpy."""
    rng = np.random.default_rng(W)
    I = 203                                                             # uneven shards
    z = logits(rng, I)
    seqs = make_cache(rng, 6, I, lens=[40, 12, 0, 0, 25, 30])
    seqs[2] = [(I64_MAX, 5), (I64_MAX, 44), (3, 45), (3, 46), (I64_MIN, 47), (I64_MIN, 100)]      # events at the extremes
    seqs[3] = []                                                        # a user with no events
    hist = [45, -1, I + 1, 45, 13]
    caches = [seqs] * W
    n_seen = 0
    for u in (0, 2, 3, 6, -1):                                          # 6, -1: outside the cache
        seq = seqs[u] if 0 <= u < len(seqs) else []
        for mt in cuts(seq):
            mask = seen_mask(I, 1, [seqs], u, mt, hist)
            ks = (1, 25, 300) if mt in (0, I64_MAX) else (25,)
            check(z, caches, u, mt, hist, targets(rng, I, mask, z, hist), W, ks=ks)
            n_seen = max(n_seen, int(mask.sum()))
    assert n_seen > 20


@pytest.mark.parametrize("W", WS)
def test_divergent_caches_follow_the_owner(W):
    """Every rank holds a different cache, one rank none and one a cache that ends before the user: each row's
    verdict is its owner's, and every rank returns the same complete result."""
    rng = np.random.default_rng(10 + W)
    I = 203
    z = logits(rng, I)
    caches = [make_cache(rng, 5, I) for _ in range(W)]
    caches[1] = None                                                    # a rank with no cache
    caches[W - 1] = make_cache(rng, 2, I)                               # users 2.. are outside this rank's cache
    hist = [7, 8, -1]
    for u in (0, 3):
        for mt in (0, 5, 6, I64_MIN, I64_MAX):
            mask = seen_mask(I, W, caches, u, mt, hist)
            check(z, caches, u, mt, hist, targets(rng, I, mask, z, hist), W, ks=(25, 300))
    # the union of the caches would differ: a row seen only in a non-owner's cache is not excluded
    full = make_cache(rng, 1, I, lens=[60])
    caches = [full if r == 0 else [[]] for r in range(W)]
    mask = seen_mask(I, W, caches, 0, 0, [])
    owned = {it for _, it in full[0] if 0 <= it < I and it % W == 0}
    assert set(np.flatnonzero(mask).tolist()) == owned
    check(z, caches, 0, 0, [], targets(rng, I, mask, z, []), W, ks=(300,))


@pytest.mark.parametrize("W", WS)
def test_empty_shards(W):
    """I < W: the ranks past I hold no rows, build empty bitmaps, score nothing and add empty lists and zero bins."""
    rng = np.random.default_rng(30 + W)
    for I in sorted({1, W - 1}):
        z = rng.standard_normal(I).astype(np.float32)
        seqs = [[(5, 0), (4, I - 1), (4, I + 2), (1, -1)]]
        rows = np.array([0, I - 1, I, -1, W], np.int32)
        for mt in (0, 4, 3):
            check(z, [seqs] * W, 0, mt, [I + 3], rows, W, ks=(1, 5))
        check(z, [seqs] + [None] * (W - 1), 0, 0, [], rows, W, ks=(5,))


@pytest.mark.parametrize("W", WS)
def test_large_table_chunks_across_count_slices(W):
    """I = 20 011 in chunks of 3001 local rows (several kRankRows slices per chunk, ending mid-slice) and a user
    who has seen several thousand rows, ties at the top of the list."""
    rng = np.random.default_rng(40 + W)
    I = 20_011
    z = logits(rng, I)
    z[1000:1016] = np.float32(3.75)
    seqs = make_cache(rng, 3, I, lens=[5000, 0, 300], ts_pool=np.arange(-50, 50))
    seqs[0][:8] = [(60, 1000 + i) for i in range(8)]                    # half the tied top run seen
    hist = list(range(1008, 1012))
    for mt in (0, 60, 59, -3):
        mask = seen_mask(I, 1, [seqs], 0, mt, hist)
        rows = np.concatenate([targets(rng, I, mask, z, hist), np.arange(1000, 1016)]).astype(np.int32)
        check(z, [seqs] * W, 0, mt, hist, rows, W, ks=(100, 1024), bc=3001)
    divergent = [make_cache(rng, 1, I, lens=[3000], ts_pool=np.arange(0, 30)) for _ in range(W)]
    mask = seen_mask(I, W, divergent, 0, 12, [])
    check(z, divergent, 0, 12, [], targets(rng, I, mask, z, []), W, ks=(1024,), bc=3001)
