"""The numpy model of the collective live id maps and table writes (tests/live_shard_model.py) against the single-GPU
semantics restated on the host: an insert at W ranks equals one insert of the rank concatenation (rows, map, rehash
capacity), a sharded write equals one write of the concatenation (rows, growth with zero gaps, moments zeroed only for
written rows, hot-row replicas), and the shard capacity rule reallocates O(log n) times.  No GPU."""
import numpy as np
import pytest

from tests import live_shard_model as lm

WS = [2, 4, 8]


def rank_ids(rng, W, base):
    """ids per rank: some new on several ranks, some new on one rank and present in the map, an empty rank"""
    shared = rng.choice(10**6, 30, replace=False).astype(np.int64) + 10**7
    out = []
    for j in range(W):
        own = rng.choice(10**6, int(rng.integers(0, 40)), replace=False).astype(np.int64) + 10**8 * (j + 2)
        a = np.concatenate([own, rng.choice(shared, 10), rng.choice(base, 5), own[:3]])
        rng.shuffle(a)
        out.append(a if j != 1 else np.zeros(0, np.int64))
    return out


@pytest.mark.parametrize("W", WS)
def test_insert_ranks_equals_one_insert_of_the_concatenation(W):
    rng = np.random.default_rng(W)
    for base_n in (0, 1, 31, 500):
        base = rng.choice(10**6, base_n, replace=False).astype(np.int64) - 5 * 10**5
        one, many = lm.SingleMap(), lm.SingleMap()
        if base_n:
            one.insert(base); many.insert(base)
        for _ in range(3):
            per = rank_ids(rng, W, base if base_n else np.array([7], np.int64))
            want = one.insert(np.concatenate(per))
            got = lm.insert_ranks(many, per)
            assert np.concatenate(got).tobytes() == want.tobytes()
            assert many.ids().tobytes() == one.ids().tobytes() and many.cap == one.cap == lm.idmap_capacity(len(one.row))
    # everything already present: nothing changes
    m = lm.SingleMap(); m.insert([5, 6, 7]); cap = m.cap
    assert [r.tolist() for r in lm.insert_ranks(m, [[7, 5]] + [[]] * (W - 1))] == [[2, 0]] + [[]] * (W - 1)
    assert m.ids().tolist() == [5, 6, 7] and m.cap == cap
    # a merge that crosses a capacity doubling: 31 ids (64 slots) + 2 new on two ranks -> 128 slots
    m = lm.SingleMap(); m.insert(np.arange(31)); assert m.cap == 64
    lm.insert_ranks(m, [[100]] + [[101, 100]] + [[]] * (W - 2))
    assert m.cap == 128 and m.ids()[31:].tolist() == [100, 101]


def test_insert_ranks_refusals_change_nothing():
    m = lm.SingleMap(); m.insert([1, 2])
    with pytest.raises(lm.Refused):
        lm.insert_ranks(m, [[3], [4, lm.INT64_MIN]])
    assert m.ids().tolist() == [1, 2]


def test_numbering_is_ascending_uint64_with_first_positions():
    ids, pos = lm.number({}, [5, -1, 5, 3, -1, 9])
    assert ids.tolist() == [3, 5, 9, -1] and pos.tolist() == [3, 0, 5, 1]


@pytest.mark.parametrize("W", WS)
@pytest.mark.parametrize("hot_k", [0, 5])
@pytest.mark.parametrize("adam", [False, True])
def test_sharded_write_equals_one_write_of_the_concatenation(W, hot_k, adam):
    rng = np.random.default_rng(100 + W + hot_k)
    w = 6
    tab = rng.standard_normal((37, w)).astype(np.float32)
    one, sh = lm.SingleTable(tab, adam=adam), lm.ShardedTable(tab, W, hot_k=hot_k, adam=adam)
    for top in (37, 38, 60, 200, 201, 1000):              # overwrites, then growth past the end
        rows = rng.permutation(top)[:min(top, 3 * W)]
        parts = np.array_split(rows, W)
        per = [(p, rng.standard_normal((p.size, w)).astype(np.float32)) for p in parts]
        one.write(np.concatenate([p for p, _ in per]), np.concatenate([d for _, d in per]))
        sh.write(per)
        assert sh.assembled().tobytes() == one.t.tobytes()
        if adam:
            assert sh.assembled("m").tobytes() == one.m.tobytes() and sh.assembled("v").tobytes() == one.v.tobytes()
    # the moments of rows never written keep their values
    if adam:
        untouched = np.setdiff1d(np.arange(37), np.concatenate([r for r, _ in per]))
        assert (one.m[untouched] != 0).any()


def test_hot_rows_reach_every_replica():
    W, tab = 4, np.arange(40, dtype=np.float32).reshape(20, 2)
    sh = lm.ShardedTable(tab, W, hot_k=6, adam=True)
    sh.write([(np.array([1, 9]), np.full((2, 2), -1, np.float32)), (np.array([4]), np.full((1, 2), -2, np.float32))] + [(np.zeros(0, np.int64), np.zeros((0, 2), np.float32))] * 2)
    for k in range(W):
        assert (sh.hot[k][[1, 4]] == [[-1, -1], [-2, -2]]).all() and (sh.hot[k][[0, 2, 3, 5]] == tab[[0, 2, 3, 5]]).all()
        assert (sh.hm[k][[1, 4]] == 0).all() and (sh.hm[k][[0, 2, 3, 5]] == 1).all()
    assert (sh.shard[1][0] == -1).all() and (sh.shard[1][2] == -1).all() and (sh.shard[0][1] == -2).all()


def test_duplicates_across_ranks_are_refused():
    sh = lm.ShardedTable(np.zeros((8, 2), np.float32), 2)
    with pytest.raises(lm.Refused):
        sh.write([(np.array([3]), np.ones((1, 2), np.float32)), (np.array([3]), np.ones((1, 2), np.float32))])
    assert not sh.assembled().any()


def test_growth_zeroes_the_gap():
    one = lm.SingleTable(np.ones((3, 2), np.float32))
    one.write([10], np.full((1, 2), 7, np.float32))
    assert one.t.shape == (11, 2) and not one.t[3:10].any() and (one.t[10] == 7).all()


@pytest.mark.parametrize("W", WS)
def test_shard_capacity_grows_geometrically(W):
    sh = lm.ShardedTable(np.zeros((1, 2), np.float32), W)
    n = 1
    for _ in range(5000):                                   # one new row per call
        sh.write([(np.array([n]), np.ones((1, 2), np.float32))] + [(np.zeros(0, np.int64), np.zeros((0, 2), np.float32))] * (W - 1))
        n += 1
    assert all(c >= s.shape[0] for c, s in zip(sh.cap, sh.shard))
    assert sh.reallocs <= W * (int(np.log2(5000 / W)) + 2)
    assert lm.shard_capacity(10, 10, 11) == 20 and lm.shard_capacity(10, 8, 10) == 10 and lm.shard_capacity(4, 4, 30) == 30
