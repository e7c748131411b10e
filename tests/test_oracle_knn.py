"""search.Searcher oracle (oracle/knn_oracle.c) against a line-by-line Python transliteration of search.go and the
reference's own known answers (tests/golden/search_kat.json).  Also pins where the device's order differs from the
bubble insertion: only the order of exactly equal similarities."""
import json
import math
import os

import numpy as np
import pytest

from go_ctr_b200.item2vec import Neighbor, neighbors_from_result
from oracle import knn_oracle as ko

KAT = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "search_kat.json")))


def go_norm(v):                                    # embutil.go:21-27
    n = 0.0
    for x in v:
        n += x * x
    return math.sqrt(n)


def go_cosine(v1, v2, n1, n2):                     # searchutil.go:17-26
    if n1 == 0 or n2 == 0:
        return 0.0
    dot = 0.0
    for a, b in zip(v1, v2):
        dot += a * b
    return dot / n1 / n2


def search_go(items, query, k, ignore=-1):
    """search.go:94-134 over items (list of float lists); returns (rows, sims, count) with empty slots -1 / 0."""
    qn = go_norm(query)
    rows, sims = [-1] * k, [0.0] * k
    low = 0.0
    for it, v in enumerate(items):
        if it == ignore:
            continue
        score = go_cosine(query, v, qn, go_norm(v))
        if score > low:
            tr, ts = it, score
            for i in range(k):
                if ts > sims[i]:
                    rows[i], tr = tr, rows[i]
                    sims[i], ts = ts, sims[i]
            low = sims[k - 1]
    return rows, sims, sum(r != -1 for r in rows)


def ordered_topk(items, query, k, ignore=-1):
    """The device's selection: the first k items under (similarity descending, row ascending), similarity > 0."""
    qn = go_norm(query)
    sc = [(go_cosine(query, v, qn, go_norm(v)), it) for it, v in enumerate(items) if it != ignore]
    sc = sorted((s for s in sc if s[0] > 0), key=lambda p: (-p[0], p[1]))[:k]
    rows = [r for _, r in sc] + [-1] * (k - len(sc))
    sims = [s for s, _ in sc] + [0.0] * (k - len(sc))
    return rows, sims, len(sc)


def _tables():
    rng = np.random.default_rng(7)
    t = {}
    t["random"] = rng.standard_normal((300, 16)).astype(np.float32)
    base = rng.standard_normal((40, 8)).astype(np.float32)
    t["duplicated"] = base[rng.integers(0, 40, 200)]                                  # exact ties everywhere
    t["quantised"] = rng.integers(-2, 3, (250, 4)).astype(np.float32)                  # few distinct directions
    z = rng.standard_normal((120, 6)).astype(np.float32); z[::7] = 0                   # zero rows: similarity 0
    z[5, 2] = np.nan; z[50, :] = np.nan                                                # NaN rows never qualify
    t["zero_nan"] = z
    t["tiny"] = rng.standard_normal((3, 5)).astype(np.float32)                         # k > N
    t["mostly_negative"] = -np.abs(rng.standard_normal((60, 5))).astype(np.float32)    # fewer than k positives
    t["mostly_negative"][[3, 17, 41]] = np.abs(t["mostly_negative"][[3, 17, 41]])
    return t


TABLES = _tables()


@pytest.mark.parametrize("name", sorted(TABLES))
@pytest.mark.parametrize("k", [1, 5, 64])
def test_oracle_is_search_go(name, k):
    tab = TABLES[name]
    items = [[float(x) for x in r] for r in tab]
    rng = np.random.default_rng(len(name) * 100 + k)
    qv = np.concatenate([rng.standard_normal((4, tab.shape[1])), np.abs(rng.standard_normal((1, tab.shape[1]))),
                         np.zeros((1, tab.shape[1]))])
    rows = np.array([0, len(tab) - 1, len(tab) // 2], np.int64)
    # vector queries (SearchVector: nothing ignored) and row queries (SearchInternal: the row itself ignored)
    cases = [(q, -1) for q in qv] + [(tab[r].astype(np.float64), int(r)) for r in rows]
    Q = np.stack([c[0] for c in cases]); ig = np.array([c[1] for c in cases], np.int32)
    orow, osim, ocnt = ko.search(tab, Q, k, ig)
    for i, (q, r) in enumerate(cases):
        wr, ws, wc = search_go(items, [float(x) for x in q], k, r)
        assert orow[i].tolist() == wr and ocnt[i] == wc, (name, i)
        assert osim[i].tobytes() == np.array(ws, np.float64).tobytes(), (name, i)
        assert all(s > 0 for s in ws[:wc]) and all(s == 0 for s in ws[wc:])
        # the device's order names the same similarities; with no exact tie among them or at the k-th place, the
        # same rows too
        dr, ds, dc = ordered_topk(items, [float(x) for x in q], k + 1, r)
        assert min(dc, k) == wc and np.array(ds[:k]).tobytes() == np.array(ws).tobytes()
        if len(set(ws[:wc])) == wc and (dc <= k or ds[k] != ds[k - 1]):
            assert dr[:k] == wr


def test_bubble_insertion_rotates_equal_similarities():
    """search.go's bubble keeps equal similarities in a rotating queue: an item inserted above a run of ties pushes
    the run's FIRST member behind the others (or out, at the end of the list).  The device orders ties by row."""
    items = [[1.0, 0.0], [1.0, 0.0], [1.0, 1.0]]     # rows 0 and 1 tie; row 2 scores higher against [1, 1]
    q = [1.0, 1.0]
    assert search_go(items, q, 2)[0] == [2, 1]           # row 0 dropped, although it came first
    assert ordered_topk(items, q, 2)[0] == [2, 0]
    assert search_go(items, q, 3)[0] == [2, 1, 0]        # rotated, not dropped
    assert ordered_topk(items, q, 3)[0] == [2, 0, 1]
    assert ko.search(np.array(items, np.float32), np.array(q), 2)[0][0].tolist() == [2, 1]


def test_reference_known_answers():
    for case in KAT["cosine"]:
        assert go_cosine(case["v1"], case["v2"], go_norm(case["v1"]), go_norm(case["v2"])) == case["expect"]
        assert ko.cosine(case["v1"], case["v2"]) == case["expect"]
    for key in ("search_internal", "search_vector"):
        for case in KAT[key]:
            words = [it["Word"] for it in case["items"]]
            tab = np.array([it["Vector"] for it in case["items"]], np.float32)
            if key == "search_internal":
                row = words.index(case["word"]); q, ig = tab[row].astype(np.float64), row
            else:
                q, ig = np.array(case["query"], np.float64), -1
            r, s, c = ko.search(tab, q, case["k"], [ig])
            got = neighbors_from_result(words, r[0], s[0], c[0], case["k"])
            assert got == [Neighbor(e["Word"], e["Rank"], e["Similarity"]) for e in case["expect"]]


def test_list_shape_reproduces_the_short_result_quirk():
    words = ["a", "b", "c", "d"]
    # fewer than k qualify: k-1 entries, the tail zero Neighbor{} values (search.go:126-133)
    got = neighbors_from_result(words, [2, 0, -1, -1, -1], [0.9, 0.5, 0, 0, 0], 2, 5)
    assert got == [Neighbor("c", 1, 0.9), Neighbor("a", 2, 0.5), Neighbor("", 0, 0.0), Neighbor("", 0, 0.0)]
    assert neighbors_from_result(words, [-1, -1, -1], [0, 0, 0], 0, 3) == [Neighbor("", 0, 0.0)] * 2
    assert neighbors_from_result(words, [-1], [0.0], 0, 1) == []
    full = neighbors_from_result(words, [3, 1], [0.7, 0.2], 2, 2)
    assert full == [Neighbor("d", 1, 0.7), Neighbor("b", 2, 0.2)]
    # the oracle on a table with one positive item reproduces the same shape through the mirror
    tab = np.array([[1, 0], [-1, 0], [0, 1]], np.float32)
    r, s, c = ko.search(tab, np.array([1.0, -0.5]), 3)
    assert neighbors_from_result(["x", "y", "z"], r[0], s[0], c[0], 3) == [Neighbor("x", 1, 1 / math.sqrt(1.25)), Neighbor("", 0, 0.0)]
