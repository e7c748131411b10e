"""The key-fed fit's minibatch gather on a row-sharded ITEM_EMB, on one GPU: W = 2, 4 and 8 ranks emulated as W shards of
one device through the kernel-level probe tests/cuda/mlp_fit_probe.cu (attn.cuh itself, not a copy).  Global row g of a
table is local row g // W of shard g % W; RowSrc::peer_emb[j] points at shard j.

ctr_mlp_fit_keys_dist trains every rank on the same survivor records in the same shuffled order, so its parity with one
GPU rests on k_gather_rows<double, RowsByIdx, true> writing, for every minibatch, the float64 rows the local
k_gather_rows<double, RowsByIdx> writes over the whole table.  Bars, all bit for bit: the survivors in a shuffled order,
minibatches of 64 with a short last one, -1 and past-the-table ids (user, item and history), hot rows whose shard copies
are NaN (a read from the shard instead of the hot-row replica shows), no hot rows, ITEM_FEAT sharded and replicated and
shorter than ITEM_EMB; and the local gather itself against a numpy assembly of the same rows."""
import numpy as np
import pytest
import torch

from tests import mlp_fit_probe as fp
from tests import shard_probe as sp

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

DEV = "cuda"
WS = [2, 4, 8]
UP, S, D, CF = 4, 6, 16, 3
NIN = UP + S * D + D + CF
BS = 64


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def bits(t):
    return np.ascontiguousarray(t.cpu().numpy()).view(np.int64)


def shard(tab, W, r):
    """rank r's shard of a [rows, w] float32 table (one zero row when it owns none, so the pointer is valid)"""
    s = tab[r::W]
    return dev(s if s.shape[0] else np.zeros((1, tab.shape[1]), np.float32))


def ids(rng, n, top, special):
    a = rng.integers(-1, top + 4, n).astype(np.int32)
    a[:len(special)] = special
    return a


def assemble(ufeat, emb, ifeat, user, item, hist):
    """numpy GetSampleVector over the whole tables: a missing row (-1 or past the end) is zeros"""
    def take(tab, r):
        out = np.zeros((r.size, tab.shape[1]), np.float64)
        ok = (r >= 0) & (r < tab.shape[0])
        out[ok] = tab[r[ok]]
        return out
    T = user.size
    return np.concatenate([take(ufeat, user), take(emb, hist.ravel()).reshape(T, S * D), take(emb, item), take(ifeat, item)], axis=1)


def gather_all(r, peer, bi, T):
    """the epoch's minibatches in order, each written to its own rows of X (as mlp_epochs walks them)"""
    X = torch.full((T, NIN + 5), -7.0, dtype=torch.float64, device=DEV)
    for b0 in range(0, T, BS):
        rows = min(BS, T - b0)
        fp.gather(r, peer, (UP, S, D, CF), bi[b0:], X[b0:], rows)
    return X


@pytest.mark.parametrize("W", WS)
def test_fit_gather_by_index(W):
    rng = np.random.default_rng(60 + W)
    I, n_user, hot_k, T = 203, 40, 20, 501                              # 501 = 7 full minibatches of 64 and one of 53
    emb = rng.standard_normal((I, D)).astype(np.float32)
    ufeat = rng.standard_normal((n_user, UP)).astype(np.float32)
    ifeat = rng.standard_normal((I - 30, CF)).astype(np.float32)        # ITEM_FEAT shorter than ITEM_EMB
    user = ids(rng, T, n_user, [-1, n_user, n_user + 9, 0])
    item = ids(rng, T, I, [-1, I, I + 3, 0, 1, hot_k - 1, hot_k, I - 1, I - 31, I - 30])
    hist = ids(rng, T * S, I, [-1, I, 3, hot_k - 1, hot_k, W, W + 1, I - 1]).reshape(T, S)
    order = rng.permutation(T).astype(np.int64)                         # the epoch's shuffled survivor order
    u_d, i_d, h_d, bi = dev(user), dev(item), dev(hist), dev(order)
    whole = [dev(emb), dev(ufeat), dev(ifeat)]
    r1 = sp.rows(emb=whole[0], lde=D, ufeat=whole[1], ldu=UP, ifeat=whole[2], ldi=CF, user_row=u_d, item_row=i_d, hist=h_d, nvalid=T,
                 n_emb=I, n_user=n_user, n_ifeat=ifeat.shape[0])
    want = gather_all(r1, False, bi, T)
    assert not torch.isnan(want).any()
    X = assemble(ufeat, emb, ifeat, user, item, hist)[order]
    assert np.array_equal(want[:, :NIN].cpu().numpy().view(np.int64), X.view(np.int64))
    assert (want[:, NIN:] == -7.0).all()                                # nothing past a row's nin columns
    for fsh in (False, True):
        for hk in (0, hot_k):                                           # 0: no replica, the shards hold every row
            poisoned = emb.copy()
            poisoned[:hk] = np.nan
            shards = [shard(poisoned, W, r) for r in range(W)]
            hot = dev(emb[:max(hk, 1)])
            if fsh:
                feat = [shard(ifeat, W, r) for r in range(W)]
                extra = dict(peer_ifeat=feat, ldi=CF)
            else:
                feat = dev(ifeat)
                extra = dict(ifeat=feat, ldi=CF)
            rw = sp.rows(lde=D, peer_emb=shards, ufeat=whole[1], ldu=UP, user_row=u_d, item_row=i_d, hist=h_d, nvalid=T, n_emb=I,
                         n_user=n_user, n_ifeat=ifeat.shape[0], world=W, ifeat_sharded=int(fsh), hot_k=hk, hot_tab=hot, **extra)
            got = gather_all(rw, True, bi, T)
            assert np.array_equal(bits(got), bits(want)), (W, fsh, hk)
