"""ctr_item_emb_train over the ranks' streams (world > 1), without a GPU:
  * the numpy model of the device steps (tests/item_emb_shard_model.py: rank-tagged first positions, their minimum, the
    gathered side lists' min-tag merge, the sort by tag) equals dictionary.Add over the ranks' streams concatenated, for
    random cuts into 2, 4 and 8 ranks with empty shards, runs of one id across a cut, side ids first seen on a later
    rank and INT64_MIN;
  * Engine.item_emb_train's new keywords and the empty shard, against a stub library;
  * the probe's new kernel forms compile for sm_90a with no stack frame and no spill."""
import ctypes as C
import re
import subprocess
import types

import numpy as np
import pytest

import go_ctr_b200 as g
from tests import item_emb_shard_model as m
from tests.util import INT64_MAX, INT64_MIN


def corpus(rng, n, n_items, n_side):
    """a Zipf stream over mapped items and unmapped ids (INT64_MIN among them), runs of one id included, and a map that
    also holds ids the stream never has, in shuffled row order"""
    items = np.unique(rng.integers(INT64_MIN + 1, INT64_MAX, n_items + n_side + 10, dtype=np.int64))
    items = rng.permutation(items)
    mapped, side = items[:n_items], np.concatenate([[INT64_MIN], items[n_items:n_items + n_side - 1]])
    never = items[n_items + n_side - 1:]
    pool = np.concatenate([mapped, side])
    s = pool[(rng.zipf(1.3, n) - 1) % pool.size]
    for _ in range(4):                                                   # runs of one id
        p = int(rng.integers(0, n - 20)); s[p:p + int(rng.integers(3, 20))] = pool[int(rng.integers(0, pool.size))]
    s[s == INT64_MIN] = mapped[0]
    s[int(0.8 * n)] = INT64_MIN                                          # first seen late: on a later rank for most cuts
    imap = rng.permutation(np.concatenate([mapped, never]))
    return s, imap


def cuts(rng, n, W, kind):
    if kind == "even":
        return [n * (r + 1) // W for r in range(W - 1)]
    c = sorted(rng.integers(0, n + 1, W - 1).tolist())
    if kind == "empty":                                                  # empty shards first, last and (W >= 4) between
        c[0] = 0
        if W > 2:
            c[-1] = n
        if W >= 4:
            c[2] = c[1]
    return c


@pytest.mark.parametrize("W", [2, 4, 8])
@pytest.mark.parametrize("kind", ["even", "random", "empty"])
def test_model_equals_dictionary_add_over_the_concatenation(W, kind):
    rng = np.random.default_rng(100 * W + len(kind))
    s, imap = corpus(rng, 3000, 300, 40)
    c = cuts(rng, s.size, W, kind)
    assert len(c) == W - 1
    streams = m.split(s, c)
    if kind == "empty":
        assert any(x.size == 0 for x in streams)
    vocab, word_of_row, side_ids, word_of_side, docs = m.numbering(streams, imap)
    want_vocab, want_doc = m.dictionary_add(s)
    assert vocab.tolist() == want_vocab.tolist()
    assert np.concatenate(docs).tolist() == want_doc.tolist()
    word = {int(v): w for w, v in enumerate(want_vocab)}
    assert word_of_row.tolist() == [word.get(int(v), -1) for v in imap]
    assert (word_of_row < 0).any()                                       # map rows whose id never occurs
    assert side_ids.tolist() == sorted(set(s.tolist()) - set(imap.tolist()), key=lambda v: v & (2 ** 64 - 1))
    assert word_of_side.tolist() == [word[int(v)] for v in side_ids]
    assert INT64_MIN in side_ids


def test_model_edges():
    """a side id and a mapped id first seen on a later rank, a run across every cut, INT64_MIN on the last rank only"""
    imap = np.array([50, 40, 30], np.int64)
    s = np.array([30, 30, 30, 7, 7, 7, 40, 7, 9, INT64_MIN], np.int64)
    for c in ([3], [4, 6], [1, 2, 8], [0, 0, 10], [5, 5, 5, 5, 5, 5, 9]):
        streams = m.split(s, c)
        vocab, word_of_row, side_ids, word_of_side, docs = m.numbering(streams, imap)
        want_vocab, want_doc = m.dictionary_add(s)
        assert vocab.tolist() == want_vocab.tolist() == [30, 7, 40, 9, INT64_MIN]
        assert word_of_row.tolist() == [-1, 2, 0]
        assert np.concatenate(docs).tolist() == want_doc.tolist()
        assert side_ids.tolist() == [7, 9, INT64_MIN] and word_of_side.tolist() == [1, 3, 4]


class _Stub:
    """records ctr_item_emb_train's arguments; world, the item map's size and V are the test's"""

    def __init__(self, n_map, V):
        self.calls, self.n_map, self.V, self.reads = [], n_map, V, 0

    def ctr_idmap_download(self, h, which, ids, cap, n):
        n._obj.value = self.n_map
        return 0

    def ctr_item_emb_train(self, h, cfg, ids, n, vocab, cap, V, st):
        self.calls.append(dict(cfg=cfg._obj, ids=ids, n=n.value, cap=cap.value))
        out = np.ctypeslib.as_array(vocab, (cap.value,))
        out[:min(cap.value, self.V)] = 1000 + np.arange(min(cap.value, self.V))
        V._obj.value = self.V
        return 0

    def ctr_item_emb_vocab(self, h, vocab, cap, V):
        self.reads += 1
        out = np.ctypeslib.as_array(vocab, (cap.value,))
        out[:min(cap.value, self.V)] = 1000 + np.arange(min(cap.value, self.V))
        V._obj.value = self.V
        return 0

    def ctr_last_error(self, h):
        return b""


def _engine(world, n_map=10, V=3):
    e = object.__new__(g.Engine)
    e.L = _Stub(n_map, V); e.h = C.c_void_p(1)
    e.cfg = types.SimpleNamespace(D=16, world=world)
    return e


def test_sync_every_keyword_and_the_empty_shard():
    e = _engine(world=4)
    cfg = g.i2v_default_config(dim=16)
    vocab, _ = e.item_emb_train(np.zeros(0, np.int64), cfg=cfg, sync_every=1000)
    c = e.L.calls[-1]
    assert c["n"] == 0 and c["ids"] is None and c["cfg"].reserved[1] == 1000
    assert c["cap"] == 10                                                 # the item map's rows plus this rank's tokens
    assert cfg.reserved[1] == 0                                           # the caller's configuration is not touched
    assert vocab.tolist() == [1000, 1001, 1002] and e.L.reads == 0
    e.item_emb_train([5, 6, 7], window=3)
    c = e.L.calls[-1]
    assert c["n"] == 3 and c["cfg"].reserved[1] == 0 and c["cfg"].window == 3 and c["cap"] == 13
    e.item_emb_train([5, 6], sync_every=np.int64(7))
    assert e.L.calls[-1]["cfg"].reserved[1] == 7
    for bad in (-1, 2 ** 31, 1.5, True, "8"):
        with pytest.raises(ValueError, match="sync_every"):
            e.item_emb_train([5], sync_every=bad)
    one = _engine(world=1)
    one.item_emb_train([5, 6, 7])
    assert one.L.calls[-1]["cap"] == 3                                    # one GPU: V <= n


def test_a_vocabulary_longer_than_the_rank_could_size_is_read_back():
    """other ranks' unmapped ids: V exceeds this rank's cap, and the whole list comes back through ctr_item_emb_vocab"""
    e = _engine(world=2, n_map=4, V=50)
    vocab, _ = e.item_emb_train([5, 6])
    assert e.L.calls[-1]["cap"] == 6 and e.L.reads == 1
    assert vocab.tolist() == (1000 + np.arange(50)).tolist()


PROPS = re.compile(r"Function properties for (\S+)\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads")


def test_probe_kernels_compile_without_spills():
    from tests import i2v_shard_probe
    _, log = i2v_shard_probe.build_probe(force=True)
    assert "sm_90a" in log
    found = {m_.group(1): tuple(int(x) for x in m_.groups()[1:]) for m_ in PROPS.finditer(log)}
    names = subprocess.run(["c++filt"], input="\n".join(found), capture_output=True, text=True, check=True).stdout.split("\n")
    props = {n.replace("void ", ""): v for n, v in zip(names, found.values())}
    want = ["ctr::k_i2v_first_tag(", "ctr::k_i2v_dict_rank_keys(", "ctr::k_i2v_dict_rank(", "ctr::k_i2v_dict_doc(", "ctr::k_i2v_dict_side(",
            "ctr::k_i2v_emb_scatter(", "ctr::k_idmap_first_pos(", "ctr::k_idmap_dump("]
    for prefix in want:
        got = {k: v for k, v in props.items() if k.startswith(prefix)}
        assert len(got) == 1, (prefix, sorted(props))
        for name, v in got.items():
            assert v == (0, 0, 0), (name, v)
    # the scatter takes (world, rank); the rank keys are 64-bit tags
    assert any(n.startswith("ctr::k_i2v_emb_scatter(float const*, int const*, long, int, int, int, float*)") for n in props), sorted(props)
    assert any(n.startswith("ctr::k_i2v_dict_rank_keys(unsigned long long const*, long, unsigned long long const*, long") for n in props)
