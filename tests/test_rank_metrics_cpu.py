"""ctr_rank_metrics (HR@k, Recall@k, NDCG@k, MRR of full-catalogue ranks) against a plain Python restatement, and the
argument refusals of ctr_rank_items / ctr_mlp_rank_items, which come before any device is needed."""
import ctypes as C
import math

import numpy as np
import pytest

import go_ctr_b200 as g

_lp = C.POINTER(C.c_int64)
_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int32)


def restated(ranks, groups, ks):
    """The definitions, with math.fsum: groups in order of first appearance, misses (-1) in every denominator."""
    order, members = [], {}
    for r, gid in zip(ranks, groups):
        if gid not in members:
            order.append(gid); members[gid] = []
        members[gid].append(int(r))
    n, G = len(ranks), len(order)
    hit, recall, ndcg = [], [], []
    for k in ks:
        h = lambda r: 0 < r <= k
        hit.append(math.fsum(1.0 for r in ranks if h(int(r))) / n)
        recall.append(math.fsum(sum(h(r) for r in members[gid]) / len(members[gid]) for gid in order) / G)
        terms = []
        for gid in order:
            ms = members[gid]
            dcg = math.fsum(1.0 / math.log2(r + 1) for r in ms if h(r))
            idcg = math.fsum(1.0 / math.log2(j + 1) for j in range(1, min(len(ms), k) + 1))
            terms.append(dcg / idcg)
        ndcg.append(math.fsum(terms) / G)
    mrr = math.fsum(1.0 / int(r) for r in ranks if int(r) > 0) / n
    return np.array(hit), np.array(recall), np.array(ndcg), mrr


def check(ranks, groups, ks):
    got = g.rank_metrics(ranks, groups, ks)
    want = restated(list(ranks), list(groups), ks)
    for a, b in zip(got[:3], want[:3]):
        np.testing.assert_allclose(a, b, rtol=1e-12, atol=1e-15)
    assert abs(got[3] - want[3]) <= 1e-12 * max(1.0, abs(want[3]))
    again = g.rank_metrics(ranks, groups, ks)
    for a, b in zip(got[:3], again[:3]):
        assert a.tobytes() == b.tobytes()
    assert np.float64(got[3]).tobytes() == np.float64(again[3]).tobytes()
    return got


def test_one_key_per_group():
    rng = np.random.default_rng(1)
    n = 5000
    ranks = rng.integers(1, 3000, n).astype(np.int64)
    ranks[rng.random(n) < 0.1] = -1
    hit, recall, ndcg, mrr = check(ranks, np.arange(n) * 7 - 100, [1, 10, 100, 1024, 5000])
    np.testing.assert_array_equal(hit, recall)          # one key per group: HR and Recall agree


def test_many_keys_per_group_beyond_k():
    rng = np.random.default_rng(2)
    n = 4000
    groups = rng.integers(-50, 50, n) * 1_000_003          # ~100 groups of ~40 keys, interleaved
    ranks = rng.integers(1, 60, n).astype(np.int64)
    ranks[rng.random(n) < 0.2] = -1
    check(ranks, groups, [1, 5, 10, 20, 100])


def test_known_values():
    # group 7: ranks 1 and 3 at k = 2 -> one hit of two; group 9: one miss
    hit, recall, ndcg, mrr = g.rank_metrics([1, 3, -1], [7, 7, 9], [2])
    assert hit[0] == 1 / 3 and recall[0] == 0.25
    assert abs(ndcg[0] - (1.0 / (1.0 + 1.0 / math.log2(3))) / 2) < 1e-15
    assert abs(mrr - (1 + 1 / 3) / 3) < 1e-15


def test_all_misses():
    hit, recall, ndcg, mrr = check(np.full(100, -1, np.int64), np.arange(100) % 7, [1, 10])
    assert not hit.any() and not recall.any() and not ndcg.any() and mrr == 0.0


def test_ranks_up_to_2_to_the_31():
    ranks = np.array([1, 2**31, 2**31 - 1, 2**31 + 5, 1024, 1025, -1], np.int64)
    check(ranks, [1, 1, 2, 2, 3, 3, 3], [1, 1024, 2**31 - 1])


def _raw(ranks, groups, ks, n=None, nks=None, null=None):
    r = np.ascontiguousarray(ranks, np.int64); gr = np.ascontiguousarray(groups, np.int64); k = np.ascontiguousarray(ks, np.int32)
    outs = [np.full(max(k.size, 1), 5.5) for _ in range(3)]
    mrr = C.c_double(5.5)
    ptr = {"rank": r.ctypes.data_as(_lp), "group": gr.ctypes.data_as(_lp), "ks": k.ctypes.data_as(_ip)}
    if null:
        ptr[null] = None
    L = g.load_library()
    rc = L.ctr_rank_metrics(ptr["rank"], ptr["group"], C.c_int64(r.size if n is None else n), ptr["ks"],
                            C.c_int32(k.size if nks is None else nks), *[o.ctypes.data_as(_dp) for o in outs], C.byref(mrr))
    untouched = all((o == 5.5).all() for o in outs) and mrr.value == 5.5
    return rc, untouched


def test_refusals_write_nothing():
    assert _raw([1, 2], [0, 0], [3]) == (0, False)
    for case in (dict(ranks=[1, 0], groups=[0, 0], ks=[3]), dict(ranks=[1, -2], groups=[0, 0], ks=[3]),
                 dict(ranks=[1, 2], groups=[0, 0], ks=[3, 0]), dict(ranks=[1, 2], groups=[0, 0], ks=[-1])):
        rc, ok = _raw(**case)
        assert rc == g.EINVAL and ok, case
    assert _raw([1, 2], [0, 0], [3], n=0) == (g.EINVAL, True)
    assert _raw([1, 2], [0, 0], [3], nks=0) == (g.EINVAL, True)
    for null in ("rank", "group", "ks"):
        assert _raw([1, 2], [0, 0], [3], null=null) == (g.EINVAL, True), null
    assert b"rank" in g.load_library().ctr_last_error(None)
    L = g.load_library()
    r = np.array([3], np.int64); gr = np.array([0], np.int64); k = np.array([1], np.int32)
    assert L.ctr_rank_metrics(r.ctypes.data_as(_lp), gr.ctypes.data_as(_lp), C.c_int64(1), k.ctypes.data_as(_ip), C.c_int32(1),
                              None, None, None, None) == 0                       # every output may be NULL
    with pytest.raises(g.CtrError) as e:
        g.rank_metrics([1, 0], [0, 0], [1])
    assert e.value.code == g.EINVAL


def test_rank_item_calls_refuse_bad_arguments_without_a_device():
    L = g.load_library()
    i32 = np.zeros(4, np.int32); i64 = np.zeros(4, np.int64); rk = np.full(4, 9, np.int64)
    lf = np.full(4, 9.0, np.float32); ld = np.full(4, 9.0)
    # a null handle
    assert L.ctr_rank_items(None, i32.ctypes.data_as(_ip), i32.ctypes.data_as(_ip), i32.ctypes.data_as(_ip), C.c_int64(1), C.c_int32(1),
                            rk.ctypes.data_as(_lp), lf.ctypes.data_as(C.POINTER(C.c_float))) == g.EINVAL
    assert L.ctr_mlp_rank_items(None, None, i64.ctypes.data_as(_lp), i64.ctypes.data_as(_lp), i64.ctypes.data_as(_lp), C.c_int64(1), C.c_int32(1),
                                rk.ctypes.data_as(_lp), ld.ctypes.data_as(_dp)) == g.EINVAL
    assert (rk == 9).all() and (lf == 9).all() and (ld == 9).all()


def test_new_symbols_are_exported():
    for name in ("ctr_rank_items", "ctr_mlp_rank_items", "ctr_rank_metrics"):
        assert name in g.engine.EXPORTS
        assert hasattr(g.load_library(), name)
    assert "rank_metrics" in g.engine.__all__ and g.rank_metrics is g.engine.rank_metrics
