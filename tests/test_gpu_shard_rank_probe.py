"""The rank kernels of ctr_rank_items on a row-sharded ITEM_EMB, on one GPU: W = 2, 4 and 8 ranks emulated as W shards
of one device through the kernel-level probe tests/cuda/shard_rank_probe.cu (rec.cuh itself, not a copy).

Rank r holds the logits z[r::W] (global row g is local row g // W of rank g % W) and scores them in chunks of BC local
rows, which do not line up with kRankRows.  The engine's two exchanges per pass are emulated: the all-gather of the
ranks' target logits is the [W][m] stack of their buffers, the all-reduce of the bins a torch sum.  A slot a rank does
not own stays NaN, so a logit read from the wrong rank shows.

Bars, exact: every emulated rank's ranks and logit bits equal those of the same kernels at world = 1 over the whole z,
and a numpy count of the list order (logit descending, then row ascending; NaN and excluded rows never counted);
every rank's sorted-target state (places, valid count, sorted logits and rows) is the same."""
import numpy as np
import pytest
import torch

from tests import shard_rank_probe as rp

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

DEV = "cuda"
MAXK = 1024
BC = 37                          # local rows per chunk: neither a divisor nor a multiple of kRankRows (2048)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def f32bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.int32)


def numpy_ranks(z, rows, excl):
    """rank of each target in z's list order, -1 outside the table, NaN or excluded; logit NaN outside the table"""
    I = z.size
    ex = set(int(e) for e in excl)
    keep = ~np.isnan(z)
    keep[[e for e in ex if 0 <= e < I]] = False
    idx = np.arange(I)
    ranks, logits = [], []
    for t in rows:
        t = int(t)
        if t < 0 or t >= I:
            ranks.append(-1); logits.append(np.float32(np.nan)); continue
        logits.append(z[t])
        if np.isnan(z[t]) or t in ex:
            ranks.append(-1); continue
        before = keep & ((z > z[t]) | ((z == z[t]) & (idx < t)))
        ranks.append(1 + int(before.sum()))
    return np.array(ranks, np.int64), np.array(logits, np.float32)


def run_ranks(z, rows, excl, W, bc):
    """The pass of RecRank on W emulated ranks.  Returns (ranks [W][m], logits [W][m], sorted-target states per rank)."""
    I, m, nex = z.size, rows.size, excl.size
    rows_d = dev(rows.astype(np.int32))
    excl_d = dev(excl.astype(np.int32)) if nex else None
    shards = [dev(z[r::W].copy()) if len(range(r, I, W)) else None for r in range(W)]
    tl = torch.full((W, m), float("nan"), device=DEV)                     # [W][m]: the all-gathered target logits
    for r in range(W):
        n = len(range(r, I, W))
        chunks = sorted({(int(t) // W) // bc for t in rows if 0 <= t < I and t % W == r})
        for c in chunks:
            i0 = c * bc; nb = min(bc, n - i0)
            rp.target_logits(shards[r][i0:], nb, i0, W, r, rows_d, m, tl[r])
    states, bins = [], []
    for r in range(W):
        st = dict(place=torch.empty(m, dtype=torch.int32, device=DEV), nvalid=torch.empty(1, dtype=torch.int32, device=DEV),
                  ss=torch.empty(MAXK, device=DEV), sr=torch.empty(MAXK, dtype=torch.int32, device=DEV),
                  bins=torch.full((MAXK + 1,), -1, dtype=torch.int64, device=DEV))
        rp.sort(rows_d, tl, m, W, m, I, excl_d, nex, st["place"], st["nvalid"], st["ss"], st["sr"], st["bins"])
        n = len(range(r, I, W))
        for i0 in range(0, n, bc):
            nb = min(bc, n - i0)
            rp.count(shards[r][i0:], nb, i0, W, r, excl_d, nex, st["ss"], st["sr"], st["nvalid"], st["bins"])
        states.append(st); bins.append(st["bins"][:m + 1])
    total = torch.stack(bins).sum(0)                                      # the all-reduce
    ranks, logits = [], []
    for r in range(W):
        o_r = torch.empty(m, dtype=torch.int64, device=DEV); o_l = torch.empty(m, device=DEV)
        rp.finish(rows_d, tl, m, W, states[r]["place"], m, I, total.clone(), o_r, o_l)
        ranks.append(o_r.cpu().numpy()); logits.append(o_l.cpu().numpy())
    return np.stack(ranks), np.stack(logits), states


def check(z, rows, excl, W, bc=BC):
    got_r, got_l, states = run_ranks(z, rows, excl, W, bc)
    one_r, one_l, _ = run_ranks(z, rows, excl, 1, bc * W)                 # the single-table kernels
    want_r, want_l = numpy_ranks(z, rows, excl)
    assert np.array_equal(one_r[0], want_r), np.argwhere(one_r[0] != want_r)[:5]
    assert np.array_equal(f32bits(one_l[0]), f32bits(want_l))
    for r in range(W):
        assert np.array_equal(got_r[r], want_r), (r, np.argwhere(got_r[r] != want_r)[:5].ravel(), got_r[r][:8], want_r[:8])
        assert np.array_equal(f32bits(got_l[r]), f32bits(want_l)), r
    v = int(states[0]["nvalid"].item())
    assert v == int((want_r > 0).sum())
    for st in states[1:]:
        assert int(st["nvalid"].item()) == v
        assert torch.equal(st["place"], states[0]["place"])
        assert torch.equal(st["ss"][:v].view(torch.int32), states[0]["ss"][:v].view(torch.int32))
        assert torch.equal(st["sr"][:v], states[0]["sr"][:v])
    return want_r


def logits(rng, I):
    z = rng.standard_normal(I).astype(np.float32)
    z[rng.integers(0, I, max(1, I // 20))] = np.nan
    return z


WS = [2, 4, 8]


@pytest.mark.parametrize("W", WS)
def test_one_target_and_a_full_pass(W):
    """m = 1 and m = 1024 over I = 203 (uneven shards): targets on every rank, named twice, outside the table; the
    exclusion list holds targets, duplicates, -1 and rows past the table."""
    rng = np.random.default_rng(W)
    I = 203
    z = logits(rng, I)
    z[40:48] = np.float32(2.5)                                            # equal logits on different ranks ...
    excl = np.array([41, 43, 41, -1, I + 2, 2 ** 30, 7, 7, 150], np.int32)
    for t in (44, 45, 0, I - 1):                                          # ... right at a target
        check(z, np.array([t]), excl, W)
        check(z, np.array([t]), np.zeros(0, np.int32), W)
    rows = rng.integers(-3, I + 5, MAXK).astype(np.int32)
    rows[:12] = [40, 41, 42, 43, 44, 45, 46, 47, 7, 150, -1, I]           # ties, excluded targets, outside the table
    rows[12] = rows[13] = 100                                              # a target named twice
    r = check(z, rows, excl, W)
    assert (r == -1).any() and (r > 0).any() and len({int(t) % W for t in rows if 0 <= t < I}) == W
    check(z, rows, np.zeros(0, np.int32), W)


@pytest.mark.parametrize("W", WS)
def test_special_logits(W):
    """NaN and -inf logits, a -0 target logit beside +0 logits on other ranks."""
    rng = np.random.default_rng(10 + W)
    I = 203
    z = logits(rng, I)
    z[60] = -np.inf; z[61] = -np.inf
    z[70] = np.float32(-0.0); z[71] = np.float32(0.0); z[77] = np.float32(0.0)
    z[90] = np.nan
    rows = np.array([60, 61, 70, 71, 77, 90, 0, 1, 2], np.int32)
    _, got_l, _ = run_ranks(z, rows, np.zeros(0, np.int32), W, BC)
    assert f32bits(got_l[0])[2] == np.int32(-2 ** 31)                    # the -0 logit keeps its sign
    r = check(z, rows, np.array([61, -1], np.int32), W)
    assert r[1] == -1 and r[5] == -1 and r[0] > 0 and r[2] < r[3] < r[4]


@pytest.mark.parametrize("W", WS)
def test_targets_owned_by_one_rank(W):
    """Every target on rank 0: the other ranks own none, score no target chunk and still count their shards."""
    rng = np.random.default_rng(20 + W)
    I = 203
    z = logits(rng, I)
    rows = np.arange(0, I, W, dtype=np.int32)[:50]
    check(z, rows, np.array([W, 3 * W, 1], np.int32), W)
    rows = np.arange(W - 1, I, W, dtype=np.int32)[:50]                     # only the last rank
    check(z, rows, np.zeros(0, np.int32), W)


@pytest.mark.parametrize("W", WS)
def test_empty_shards(W):
    """I < W: the ranks past I hold no rows, score nothing and add zero bins."""
    rng = np.random.default_rng(30 + W)
    for I in sorted({1, W - 1}):
        z = rng.standard_normal(I).astype(np.float32)
        rows = np.array([0, I - 1, I, -1, W], np.int32)
        check(z, rows, np.array([I + 3], np.int32), W)
        check(z, rows, np.array([0], np.int32), W)


@pytest.mark.parametrize("W", WS)
def test_large_table_chunks_across_count_slices(W):
    """Chunks of 3001 local rows: several kRankRows slices per chunk, ending mid-slice."""
    rng = np.random.default_rng(40 + W)
    I = 20_011
    z = logits(rng, I)
    z[1000:1016] = np.float32(1.75)
    rows = np.concatenate([rng.integers(0, I, 300), np.arange(1000, 1016)]).astype(np.int32)
    excl = np.concatenate([rng.integers(0, I, 20), [1003, 1003, -1, I + 1]]).astype(np.int32)
    check(z, rows, excl, W, bc=3001)
