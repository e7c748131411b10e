"""ctr_knn_search (search.Searcher on the device) against the search.go oracle: bit-identical similarities and the
same neighbour lists, in both query modes, plus the reference's known answers through the Searcher mirror."""
import io
import json
import os

import numpy as np
import pytest

import go_ctr_b200 as g
from oracle import knn_oracle as ko
from tests.test_oracle_knn import ordered_topk

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]
KAT = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "search_kat.json")))


def table_engine(tab):
    eng = g.Engine(g.engine.default_config(g.MODEL_DIN_COS, uP=0, cF=0, S=1, D=tab.shape[1], batch=1, pred_batch=1))
    eng.table_upload(g.TABLE_ITEM_EMB, tab)
    return eng


def assert_same(dev, orc, ctx):
    (r, s, c), (orow, osim, ocnt) = dev, orc
    assert np.array_equal(c, ocnt), ctx
    assert np.array_equal(r, orow), ctx
    assert s.tobytes() == osim.tobytes(), ctx


def test_reference_known_answers_through_searcher():
    for key in ("search_internal", "search_vector"):
        for case in KAT[key]:
            s = g.Searcher.New(*[g.Embedding(it["Word"], it["Vector"]) for it in case["items"]])
            got = s.SearchInternal(case["word"], case["k"]) if key == "search_internal" else s.SearchVector(case["query"], case["k"])
            assert got == [g.Neighbor(e["Word"], e["Rank"], e["Similarity"]) for e in case["expect"]], (case["cite"], got)
    with pytest.raises(ValueError, match="is not found in searcher"):
        s.SearchInternal("elderberry", 1)


CASES = [  # D, N, nq, k
    (5, 1, 1, 1), (5, 1000, 7, 10), (16, 1000, 300, 100), (256, 1000, 300, 1024), (64, 1000, 300, 1),
    (64, 100_003, 7, 1024), (256, 100_003, 7, 10), (5, 100_003, 300, 10), (16, 100_003, 1, 100),
    (16, 4_000_000, 7, 100), (5, 4_000_000, 1, 10), (64, 4_000_000, 1, 1024),
]


@pytest.mark.parametrize("D,N,nq,k", CASES)
def test_bit_exact_against_the_oracle(D, N, nq, k):
    rng = np.random.default_rng(D * 7 + N + nq + k)
    tab = rng.standard_normal((N, D), dtype=np.float32)
    eng = table_engine(tab)
    q = rng.standard_normal((nq, D))                          # float64 queries, not float32-representable
    assert_same(eng.knn_search(k, queries=q), ko.search(tab, q, k), ("vector", D, N, nq, k))
    rows = rng.integers(0, N, nq).astype(np.int32)
    assert_same(eng.knn_search(k, rows=rows), ko.search(tab, tab[rows].astype(np.float64), k, rows), ("row", D, N, nq, k))
    eng.close()


def test_exact_ties_rank_by_row_and_batching_does_not_change_a_result():
    rng = np.random.default_rng(3)
    tab = rng.integers(-2, 3, (3000, 4)).astype(np.float32)   # a few hundred distinct directions: ties everywhere
    tab[1000:1100] = tab[:100]                               # plus exact duplicates
    eng = table_engine(tab)
    items = [[float(x) for x in r] for r in tab]
    q = rng.integers(-2, 3, (300, 4)).astype(np.float64)
    k = 50
    r, s, c = eng.knn_search(k, queries=q)
    orow, osim, ocnt = ko.search(tab, q, k)
    assert np.array_equal(c, ocnt) and s.tobytes() == osim.tobytes()       # the same similarities as search.go
    for i in (0, 1, 77, 299):
        wr, ws, wc = ordered_topk(items, q[i].tolist(), k)
        assert r[i].tolist() == wr and s[i].tobytes() == np.array(ws).tobytes() and c[i] == wc
        r1, s1, c1 = eng.knn_search(k, queries=q[i])
        assert r1[0].tolist() == r[i].tolist() and s1.tobytes() == s[i].tobytes() and c1[0] == c[i]
    rr, rs, rc = eng.knn_search(k, rows=np.arange(300, dtype=np.int32))
    for i in (0, 5, 299):
        wr, ws, wc = ordered_topk(items, items[i], k, ignore=i)
        assert rr[i].tolist() == wr and rs[i].tobytes() == np.array(ws).tobytes()


def test_zero_query_nan_rows_and_short_results():
    rng = np.random.default_rng(4)
    tab = rng.standard_normal((500, 8)).astype(np.float32)
    tab[::9] = np.nan; tab[3] = 0
    eng = table_engine(tab)
    r, s, c = eng.knn_search(10, queries=np.zeros((1, 8)))
    assert c[0] == 0 and (r == -1).all() and (s == 0).all()
    q = rng.standard_normal((3, 8))
    r, s, c = eng.knn_search(1024, queries=q)
    assert not np.isin(r, np.arange(0, 500, 9)).any() and not np.isin(r, [3]).any()
    for i in range(3):
        n = c[i]
        assert 0 < n < 500 and (r[i, :n] >= 0).all() and (s[i, :n] > 0).all()
        assert (r[i, n:] == -1).all() and (s[i, n:] == 0).all()
    assert_same((r, s, c), ko.search(tab, q, 1024), "nan")
    # one positive item and k = 5: the true count, padded
    t2 = np.array([[1, 0], [-1, 0], [0, -1]], np.float32)
    e2 = table_engine(t2)
    r, s, c = e2.knn_search(5, queries=np.array([[1.0, 0.5]]))
    assert c[0] == 1 and r[0].tolist() == [0, -1, -1, -1, -1] and s[0, 1:].tolist() == [0.0] * 4


def test_live_table_after_sgd_steps():
    rng = np.random.default_rng(5)
    U, I, uP, cF, D, S, B = 200, 3000, 8, 4, 32, 10, 256
    cfg = g.engine.default_config(g.MODEL_DIN_COS, uP=uP, S=S, D=D, cF=cF, batch=B, pred_batch=B, table_opt=g.TABLE_SGD, table_lr=0.5, seed=3)
    eng = g.Engine(cfg)
    eng.table_upload(g.TABLE_USER_FEAT, rng.random((U, uP), np.float32))
    eng.table_upload(g.TABLE_ITEM_FEAT, rng.random((I, cF), np.float32))
    eng.table_upload(g.TABLE_ITEM_EMB, rng.standard_normal((I, D)).astype(np.float32))
    for _ in range(5):
        eng.train_step_idx(rng.integers(0, U, B), rng.integers(0, I, B), rng.integers(-1, I, (B, S)), (rng.random(B) > 0.5).astype(np.float32))
    rows = rng.integers(0, I, 20).astype(np.int32)
    got = eng.knn_search(10, rows=rows)
    tab = eng.table_download(g.TABLE_ITEM_EMB, I, D)
    assert_same(got, ko.search(tab, tab[rows].astype(np.float64), 10, rows), "live")
    s = g.Searcher.from_engine(eng, [str(i) for i in range(I)])
    nb = s.SearchInternal(str(rows[0]), 10)
    assert [n.Word for n in nb] == [str(x) for x in got[0][0]]


def test_text_loaded_vectors_match_a_float64_search():
    words = [str(100 + (i * 7919) % 211) for i in range(30000)]
    m = g.TrainEmbedding(iter(words), 5, 16, 1)
    buf = io.StringIO()
    g.SaveVectors(buf, m.id2word, m.emb)
    embs = g.LoadVectors(buf.getvalue())
    s = g.Searcher.New(*embs)
    V = np.stack([e.Vector for e in embs]); nv = np.linalg.norm(V, axis=1)
    for w in ("100", "107", "250"):
        i = [e.Word for e in embs].index(w)
        sims = V @ V[i] / nv / nv[i]; sims[i] = -np.inf
        order = np.argsort(-sims, kind="stable")[:10]
        got = s.SearchInternal(w, 10)
        assert len(got) == 10
        for j, n in enumerate(got):
            want = embs[order[j]].Word
            assert abs(n.Similarity - sims[order[j]]) < 1e-6
            if n.Word != want:                       # a swap only between near-equal similarities
                assert abs(sims[[e.Word for e in embs].index(n.Word)] - sims[order[j]]) < 1e-6


def test_errors_do_not_fault():
    tab = np.random.default_rng(6).standard_normal((100, 8)).astype(np.float32)
    eng = table_engine(tab)
    for k in (0, 1025):
        with pytest.raises(g.CtrError) as e:
            eng.knn_search(k, queries=np.ones((1, 8)))
        assert e.value.code == g.EINVAL
    with pytest.raises(g.CtrError) as e:
        eng.knn_search(5, rows=[100])
    assert e.value.code == g.ENOTFOUND and "100 is not found in searcher" in str(e.value)
    bare = g.Engine(g.engine.default_config(g.MODEL_DIN_COS, uP=0, cF=0, S=1, D=8, batch=1, pred_batch=1))
    with pytest.raises(g.CtrError) as e:
        bare.knn_search(5, queries=np.ones((1, 8)))
    assert e.value.code == g.ESTATE
    r, s, c = eng.knn_search(3, rows=[7])                    # the handle still works
    assert c[0] == 3 and 7 not in r[0]
