"""The collective live id maps and table writes on one GPU: W = 2, 4 and 8 ranks emulated in one device through the
kernel-level probe tests/cuda/live_shard_probe.cu (idmap.cuh, item2vec.cuh, attn.cuh and vmm.cuh themselves, not copies).
The test plays the all-gathers and the owner routing with plain copies; every bar is bit for bit against the single-GPU
twin, and against the numpy model of tests/live_shard_model.py:
  * insert: each rank's numbering, the gathered lists padded to the longest and the rank merge (idmap_merge_ranks) give
    the ids, the map (download, lookups, digest) and the rehash capacity of the single-GPU insert of the concatenation;
    ids new on several ranks, ids new on one rank and repeated on later ones, empty ranks, a rehash the merge triggers,
    all ids present, no map yet;
  * write: k_shard_write_rows on each rank's routed rows equals k_table_write_rows on the single table, hot rows in
    every rank's replica, row-Adam moments zeroed on the owner and in the hot-moment replicas only for written rows;
  * growth: vmm_grow_rows keeps the live rows, zeroes the gap (a shard's spare bytes are not zero) and reallocates at
    max(new rows, 2 x old rows) only when the new rows do not fit."""
import numpy as np
import pytest
import torch

from tests import live_shard_model as lm
from tests import live_shard_probe as lp

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

DEV = "cuda"
WS = [2, 4, 8]


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def u64(a):
    return dev(np.asarray(a, np.int64))                     # the probe reads int64 ids as uint64 bits


class Map:
    """a device map: keys [cap] (uint64 bits in int64), vals [cap]"""

    def __init__(self):
        self.keys = self.vals = None
        self.n = 0

    def add(self, fresh, u):
        """as ctr_idmap_insert writes: a larger table (cleared, the old map rehashed) when the count needs one"""
        cap = lm.idmap_capacity(self.n + u)
        keys, vals = self.keys, self.vals
        if cap > (keys.numel() if keys is not None else 0):
            keys = torch.empty(cap, dtype=torch.int64, device=DEV); vals = torch.empty(cap, dtype=torch.int32, device=DEV)
        if u or keys is not self.keys:
            lp.add(self.keys, self.vals, keys, vals, fresh, u, self.n, torch.zeros(1, dtype=torch.int32, device=DEV))
        self.keys, self.vals = keys, vals
        self.n += u

    def ids(self):
        out = torch.empty(max(self.n, 1), dtype=torch.int64, device=DEV)
        if self.n:
            lp.dump(self.keys, self.vals, out)
        return out[:self.n].cpu().numpy()

    def rows(self, ids):
        ids = u64(ids)
        out = torch.empty(max(ids.numel(), 1), dtype=torch.int32, device=DEV)
        if ids.numel():
            lp.lookup(self.keys, self.vals, ids, out)
        return out[:ids.numel()].cpu().numpy()

    def digest(self):
        out = torch.zeros(1, dtype=torch.int64, device=DEV)
        lp.digest(self.keys, self.vals, out)
        return int(out.item())


def number(m, ids):
    ids = u64(ids)
    n = max(ids.numel(), 1)
    rows = torch.empty(n, dtype=torch.int32, device=DEV)
    out_ids = torch.empty(n, dtype=torch.int64, device=DEV); out_pos = torch.empty(n, dtype=torch.int32, device=DEV)
    _, u = lp.number(m.keys, m.vals, ids, rows, out_ids, out_pos)
    return out_ids[:u], out_pos[:u], u


def insert_single(m, ids):
    """the single-GPU insert: numbering, the sort by first position, the write"""
    k, p, u = number(m, ids)
    fresh = torch.empty(max(u, 1), dtype=torch.int64, device=DEV)
    if u:
        lp.order(k, p, u, fresh)
    m.add(fresh, u)
    return fresh[:u].cpu().numpy()


def insert_ranks(m, per_rank):
    """the collective insert: every rank numbers its own ids on the shared map, the lists are gathered padded to the longest,
    every rank merges (the merge is deterministic: run once per rank and compared) and writes"""
    lists = [number(m, a) for a in per_rank]
    cnt = [u for _, _, u in lists]
    stride = max(cnt + [0])
    W = len(per_rank)
    fresh = None
    if stride:
        g_ids = torch.full((W * stride,), -1, dtype=torch.int64, device=DEV)       # padding: never read
        g_pos = torch.full((W * stride,), -7, dtype=torch.int32, device=DEV)
        for j, (k, p, u) in enumerate(lists):
            g_ids[j * stride:j * stride + u] = k; g_pos[j * stride:j * stride + u] = p
        outs = []
        for _ in range(W):
            out = torch.empty(sum(cnt), dtype=torch.int64, device=DEV)
            u = lp.merge(g_ids, g_pos, stride, cnt, out)
            outs.append(out[:u].cpu().numpy())
        assert all(o.tobytes() == outs[0].tobytes() for o in outs)
        fresh = outs[0]
    u = 0 if fresh is None else fresh.size
    m.add(u64(fresh if u else [0]), u)
    return np.zeros(0, np.int64) if fresh is None else fresh


def scenarios(rng, W):
    base = rng.choice(10**9, 300, replace=False).astype(np.int64) - 5 * 10**8
    shared = rng.choice(10**9, 50, replace=False).astype(np.int64) + 10**10
    def ranks(k, empty=(1,)):
        out = []
        for j in range(W):
            own = rng.choice(10**6, k, replace=False).astype(np.int64) + (j + 2) * 10**12
            a = np.concatenate([own, rng.choice(shared, 20), rng.choice(base, 10), own[::3], [np.int64(-1), np.int64(2**63 - 1)]])
            rng.shuffle(a)
            out.append(np.zeros(0, np.int64) if j in empty else a)
        return out
    return base, [
        ("no map yet", None, ranks(40)),
        ("shared, one-rank and present ids", base, ranks(25)),
        ("empty ranks", base, ranks(5, empty=range(1, W))),
        ("rehash by the merge", base[:31], [np.array([base[0], 10**15 + j, 10**15], np.int64) for j in range(W)]),
        ("all present", base, [rng.choice(base, 17) for _ in range(W)]),
        ("large", base, ranks(5000)),
    ]


@pytest.mark.parametrize("W", WS)
def test_rank_merge_equals_the_single_gpu_insert_of_the_concatenation(W):
    rng = np.random.default_rng(40 + W)
    base, cases = scenarios(rng, W)
    for name, start, per_rank in cases:
        one, many, model = Map(), Map(), lm.SingleMap()
        if start is not None:
            for m in (one, many):
                insert_single(m, start)
            model.insert(start)
        cap0 = many.keys.numel() if many.keys is not None else 0
        want = insert_single(one, np.concatenate(per_rank))
        got = insert_ranks(many, per_rank)
        assert got.tobytes() == want.tobytes(), name
        rows = lm.insert_ranks(model, per_rank)
        assert many.ids().tobytes() == one.ids().tobytes() == model.ids().tobytes(), name
        assert many.keys.numel() == one.keys.numel() == lm.idmap_capacity(many.n), name
        if name == "rehash by the merge":
            assert cap0 == 64 and many.keys.numel() == 128
        if name == "all present":
            assert got.size == 0 and many.n == len(base)
        for j, a in enumerate(per_rank):
            assert many.rows(a).tobytes() == rows[j].tobytes(), (name, j)
        assert many.digest() == one.digest(), name
    # the digest tells maps apart: one pair moved to another row
    a, b = Map(), Map()
    insert_single(a, base[:40]); insert_single(b, np.concatenate([base[1:2], base[:1], base[2:40]]))
    assert a.digest() != b.digest()


def shards_of(tab, W, ld):
    out = []
    for r in range(W):
        s = np.zeros((max(tab[r::W].shape[0], 1), ld), np.float32)
        s[:tab[r::W].shape[0], :tab.shape[1]] = tab[r::W]
        out.append(dev(s))
    return out


@pytest.mark.parametrize("W", WS)
@pytest.mark.parametrize("width,hot_k,adam", [(8, 0, False), (8, 6, True), (6, 0, True), (8, 0, True)])
def test_owner_routed_writes_equal_the_single_table(W, width, hot_k, adam):
    rng = np.random.default_rng(W * 10 + width + hot_k)
    N, ld = 203, (width + 3) // 4 * 4
    tab = rng.standard_normal((N, width)).astype(np.float32)
    full = np.zeros((N, ld), np.float32); full[:, :width] = tab
    twin = dev(full)
    tm, tv = (dev(np.ones((N, ld), np.float32)), dev(np.ones((N, ld), np.float32))) if adam else (None, None)
    shards = shards_of(tab, W, ld)
    ones = np.ones((N, ld), np.float32)
    ms = shards_of(ones, W, ld) if adam else [None] * W
    vs = shards_of(ones, W, ld) if adam else [None] * W
    hot = [dev(tab[:hot_k]) for _ in range(W)] if hot_k else [None] * W
    hm = [dev(np.ones((hot_k, width), np.float32)) for _ in range(W)] if hot_k and adam else [None] * W
    hv = [dev(np.ones((hot_k, width), np.float32)) for _ in range(W)] if hot_k and adam else [None] * W
    rows = rng.permutation(np.unique(np.concatenate([[0, 1, N - 1], rng.permutation(N)[:90]])))
    per = [(p.astype(np.int32), rng.standard_normal((p.size, width)).astype(np.float32)) for p in np.array_split(rows, W)]
    per[-1] = (np.zeros(0, np.int32), np.zeros((0, width), np.float32))                   # a rank that writes nothing
    all_rows = np.concatenate([r for r, _ in per]); all_data = np.concatenate([d for _, d in per])
    lp.write(twin, dev(all_rows), dev(all_data), mo=tm, vo=tv)
    model = lm.ShardedTable(tab, W, hot_k=hot_k, adam=adam)
    for k, (rr, dd) in enumerate(model.route(per)):
        if rr:
            lp.write(shards[k], dev(np.array(rr, np.int32)), dev(np.array(dd, np.float32)), W, k, ms[k], vs[k], hot[k], hot_k, hm[k], hv[k])
    model.write(per)
    want = twin.cpu().numpy()
    for k in range(W):
        got = shards[k].cpu().numpy()[:want[k::W].shape[0]]
        assert got.tobytes() == want[k::W].tobytes(), k
        if adam:
            assert ms[k].cpu().numpy()[:want[k::W].shape[0]].tobytes() == tm.cpu().numpy()[k::W].tobytes()
            assert vs[k].cpu().numpy()[:want[k::W].shape[0]].tobytes() == tv.cpu().numpy()[k::W].tobytes()
        if hot_k:
            assert hot[k].cpu().numpy().tobytes() == want[:hot_k, :width].tobytes(), k
            if adam:
                assert hm[k].cpu().numpy().tobytes() == tm.cpu().numpy()[:hot_k, :width].tobytes()
    assert model.assembled().tobytes() == want[:, :width].tobytes()
    if adam:
        written = np.zeros(N, bool); written[all_rows] = True
        m = tm.cpu().numpy()
        assert (m[written] == 0).all() and (m[~written] == 1).all()


@pytest.mark.parametrize("rows,want,width", [(1000, 2000, 16), (1000, 40000, 16), (40000, 70000, 16), (0, 5, 16), (3, 3, 6)])
def test_shard_growth_keeps_rows_zeroes_the_gap_and_doubles(rows, want, width):
    rng = np.random.default_rng(rows + want)
    host = rng.standard_normal((rows, width)).astype(np.float32)
    out, ob, nb, gran = lp.grow(host, want)
    assert out[:rows].tobytes() == host.tobytes()
    assert not out[rows:].any()
    row_b = width * 4
    if want * row_b <= ob:
        assert nb == ob                                                           # in place
    else:                                                                         # max(new rows, 2 x old rows), granule-rounded
        need = max(want, 2 * rows) * row_b
        assert nb == (need + gran - 1) // gran * gran
