"""ctr_item_emb_train's numbering over the ranks' streams and its owner-written rows on one GPU: W = 2, 4 and 8 ranks
emulated in one device through the kernel-level probe tests/cuda/i2v_shard_probe.cu (item2vec.cuh and idmap.cuh
themselves, not copies, through the inline host steps the collective path calls).  The min all-reduce of the row tags
becomes an elementwise minimum and the all-gather of the side lists a padded concatenation.  Bit for bit against the
one-GPU numbering of the concatenated stream (and the numpy model of tests/item_emb_shard_model.py):
  * vocab_ids, V, word of every row and the side tables (ids and words);
  * the ranks' documents, which concatenated equal the one-GPU document;
  * the sharded scatter's W shards, interleaved, equal the single table: R not divisible by W, R < W (empty shards) and
    rows whose id never occurs (zeros)."""
import numpy as np
import pytest
import torch

from tests import i2v_shard_probe as ip
from tests import item_emb_shard_model as m
from tests.util import INT64_MAX, INT64_MIN

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

DEV = "cuda"
NEVER = -1                                      # kI2vNever as int64 bits


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def cap_for(n):
    cap = 64
    while cap < 2 * n:
        cap <<= 1
    return cap


def make_map(imap):
    cap = cap_for(imap.size)
    keys = torch.empty(cap, dtype=torch.int64, device=DEV); vals = torch.empty(cap, dtype=torch.int32, device=DEV)
    ip.build_map(dev(imap), keys, vals, torch.zeros(1, dtype=torch.int32, device=DEV))
    return keys, vals


def local(keys, vals, s, R, rank):
    n = s.size
    ids = dev(s) if n else torch.empty(0, dtype=torch.int64, device=DEV)
    rows = torch.empty(max(n, 1), dtype=torch.int32, device=DEV)
    tag = torch.empty(max(R, 1), dtype=torch.int64, device=DEV)
    sid = torch.empty(max(n, 1), dtype=torch.int64, device=DEV); spos = torch.empty(max(n, 1), dtype=torch.int32, device=DEV)
    u = ip.local(keys, vals, ids, R, rank, rows, tag, sid, spos)
    return ids, rows, tag[:R], sid[:u], spos[:u]


def number(keys, vals, imap, streams):
    """the collective path's steps on W emulated ranks: (vocab, V, word_of_row, side_id, word_of_side, docs)"""
    W, R = len(streams), imap.size
    loc = [local(keys, vals, s, R, r) for r, s in enumerate(streams)]
    tags = np.stack([l[2].cpu().numpy().view(np.uint64) for l in loc])
    row_tag = dev(tags.min(axis=0).view(np.int64))                        # the min all-reduce
    cnt = [int(l[3].numel()) for l in loc]
    stride = max(cnt)
    g_ids = torch.full((W, max(stride, 1)), 0x5A5A5A5A5A5A5A5A, dtype=torch.int64, device=DEV)     # padding: never read
    g_pos = torch.full((W, max(stride, 1)), 0x5A5A5A5A, dtype=torch.int32, device=DEV)
    for r, l in enumerate(loc):
        g_ids[r, :cnt[r]] = l[3]; g_pos[r, :cnt[r]] = l[4]
    mt = sum(cnt)
    side_id = torch.empty(max(mt, 1), dtype=torch.int64, device=DEV); side_tag = torch.empty(max(mt, 1), dtype=torch.int64, device=DEV)
    u = ip.merge(g_ids, g_pos, stride, cnt, side_id, side_tag) if mt else 0
    wor = torch.empty(max(R, 1), dtype=torch.int32, device=DEV); wos = torch.empty(max(u, 1), dtype=torch.int32, device=DEV)
    vocab = torch.empty(max(R + u, 1), dtype=torch.int64, device=DEV)
    V = ip.order(keys, vals, row_tag, R, side_id, side_tag, u, W, wor, wos, vocab)
    docs = []
    for l in loc:
        ids, rows = l[0], l[1]
        if ids.numel():
            ip.doc(rows, ids, wor, side_id, u, wos)
        docs.append(rows[:ids.numel()].cpu().numpy().astype(np.int64))
    return (vocab[:V].cpu().numpy(), V, wor[:R].cpu().numpy(), side_id[:u].cpu().numpy(), wos[:u].cpu().numpy(), docs,
            row_tag.cpu().numpy(), side_tag[:u].cpu().numpy())


def corpus(rng, n, n_items, n_side):
    items = rng.permutation(np.unique(rng.integers(INT64_MIN + 1, INT64_MAX, n_items + n_side + 50, dtype=np.int64)))
    mapped, side, never = items[:n_items], items[n_items:n_items + n_side], items[n_items + n_side:]
    pool = np.concatenate([mapped, side])
    s = pool[(rng.zipf(1.2, n) - 1) % pool.size]
    for _ in range(8):                                                    # runs of one id
        p = int(rng.integers(0, n - 200)); s[p:p + int(rng.integers(10, 200))] = pool[int(rng.integers(0, pool.size))]
    s[int(0.9 * n)] = INT64_MIN                                            # first seen on a late rank
    s[int(0.95 * n)] = side[-1] if side[-1] not in s[:int(0.95 * n)] else s[int(0.95 * n)]
    imap = rng.permutation(np.concatenate([mapped, never]))
    return s, imap


CASES = [(2, "even"), (2, "empty"), (4, "random"), (4, "empty"), (8, "random"), (8, "empty")]


@pytest.mark.parametrize("W,kind", CASES)
def test_numbering_across_ranks_equals_one_gpu(W, kind):
    rng = np.random.default_rng(W * 31 + len(kind))
    s, imap = corpus(rng, 200_000, 20_000, 3000)
    n = s.size
    c = sorted(rng.integers(0, n + 1, W - 1).tolist()) if kind != "even" else [n * (r + 1) // W for r in range(W - 1)]
    if kind == "empty":
        c[0] = 0; c[-1] = n
        if W >= 4:
            c[2] = c[1]
    streams = m.split(s, c)
    keys, vals = make_map(imap)
    one = number(keys, vals, imap, [s])
    many = number(keys, vals, imap, streams)
    vocab, V, wor, sid, wos, docs, row_tag, side_tag = many
    assert V == one[1] and vocab.tobytes() == one[0].tobytes()
    assert wor.tobytes() == one[2].tobytes()
    assert sid.tobytes() == one[3].tobytes() and wos.tobytes() == one[4].tobytes()
    assert np.concatenate(docs).tobytes() == one[5][0].tobytes()
    for r, d in enumerate(docs):
        assert d.size == streams[r].size
    # the tags are (rank << 32) | position of the first occurrence
    bounds = np.concatenate([[0], np.cumsum([x.size for x in streams])])
    seen = row_tag != NEVER
    rt = row_tag[seen].view(np.uint64)
    gpos = bounds[(rt >> np.uint64(32)).astype(np.int64)] + (rt & np.uint64(0xFFFFFFFF)).astype(np.int64)
    assert (s[gpos] == imap[seen]).all()
    # the numpy model and dictionary.Add over the concatenation
    want_vocab, want_doc = m.dictionary_add(s)
    assert vocab.tolist() == want_vocab.tolist() and np.concatenate(docs).tolist() == want_doc.tolist()
    assert INT64_MIN in sid and (wor < 0).sum() >= 40


@pytest.mark.parametrize("W", [2, 4, 8])
@pytest.mark.parametrize("R", [1, 3, 7, 1000, 1001, 4099])
@pytest.mark.parametrize("D", [4, 64])
def test_sharded_scatter_interleaves_to_the_single_table(W, R, D):
    rng = np.random.default_rng(R * W + D)
    V = max(2, R // 2)
    syn0 = dev(rng.standard_normal((V, D)).astype(np.float32))
    wor_h = rng.integers(0, V, R).astype(np.int32)
    wor_h[rng.random(R) < 0.3] = -1                                       # rows whose id never occurs
    wor = dev(wor_h)
    one = torch.full((R, D), float("nan"), device=DEV)
    ip.scatter(syn0, wor, R, D, 1, 0, one)
    want = syn0.cpu().numpy()[np.maximum(wor_h, 0)]
    want[wor_h < 0] = 0
    assert one.cpu().numpy().tobytes() == want.tobytes()
    stitched = np.full((R, D), np.nan, np.float32)
    for r in range(W):
        local = (R - r + W - 1) // W
        sh = torch.full((max(local, 1) + 1, D), float("nan"), device=DEV)  # one spare row: must stay untouched
        ip.scatter(syn0, wor, R, D, W, r, sh)
        got = sh.cpu().numpy()
        assert np.isnan(got[local:]).all()
        stitched[r::W] = got[:local]
    assert stitched.tobytes() == want.tobytes()
