"""ctr_item_emb_vocab: the vocabulary ctr_item_emb_train keeps when its vocab_ids cannot take all of it (cap < V), read
back whole; nothing kept when vocab_ids took every id, when the caller passed none, or after a refused call."""
import ctypes as C

import numpy as np
import pytest

import go_ctr_b200 as g
from tests.test_gpu_item_emb_train import host_route, make_stream, store

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

LP = C.POINTER(C.c_int64)


def _train(L, eng, cfg, ids, out, cap):
    V = C.c_int32(-1)
    rc = L.ctr_item_emb_train(eng.h, C.byref(cfg), ids.ctypes.data_as(LP), C.c_int64(ids.size), out.ctypes.data_as(LP) if out is not None else None,
                              C.c_int64(cap), C.byref(V), None)
    return rc, V.value


def _read(L, eng, cap):
    out = np.full(max(cap, 1), 77, np.int64); V = C.c_int32(-1)
    rc = L.ctr_item_emb_vocab(eng.h, out.ctypes.data_as(LP), C.c_int64(cap), C.byref(V))
    return rc, V.value, out


def test_a_short_vocab_ids_keeps_the_whole_vocabulary_on_the_handle():
    D = 16
    rng = np.random.default_rng(3)
    ids, imap = make_stream(rng, 20_000, 800, 1.3)
    cfg = g.i2v_default_config(dim=D, window=3, seed=2)
    vocab_h = host_route(ids, imap, cfg)[0]
    L = g.load_library()
    eng = store(D)
    eng.idmap_build(g.IDMAP_ITEM, imap)
    assert _read(L, eng, 4)[0] == g.ESTATE                                   # no call yet
    short = np.empty(10, np.int64)
    assert _train(L, eng, cfg, ids, short, 10) == (0, vocab_h.size)
    assert short.tolist() == vocab_h[:10].tolist()
    rc, V, out = _read(L, eng, vocab_h.size + 1)
    assert rc == 0 and V == vocab_h.size and out[:V].tolist() == vocab_h.tolist() and out[V] == 77
    rc, V, out = _read(L, eng, 5)                                            # a read-back cut at its own cap
    assert rc == 0 and V == vocab_h.size and out[:5].tolist() == vocab_h[:5].tolist()
    assert L.ctr_item_emb_vocab(eng.h, None, C.c_int64(0), C.byref(C.c_int32())) == 0
    full = np.empty(vocab_h.size, np.int64)
    assert _train(L, eng, cfg, ids, full, full.size) == (0, vocab_h.size)   # every id returned: nothing kept
    assert _read(L, eng, 4)[0] == g.ESTATE
    assert _train(L, eng, cfg, ids, short, 10)[0] == 0
    assert _train(L, eng, cfg, ids, None, 0)[0] == 0                         # no vocab_ids: nothing kept, the old one dropped
    assert _read(L, eng, 4)[0] == g.ESTATE
    assert _train(L, eng, cfg, ids, short, 10)[0] == 0
    bad = g.i2v_default_config(dim=2 * D)
    assert _train(L, eng, bad, ids, short, 10)[0] == g.EINVAL                # a refusal drops it too
    assert _read(L, eng, 4)[0] == g.ESTATE
    assert L.ctr_item_emb_vocab(eng.h, None, C.c_int64(3), C.byref(C.c_int32())) == g.EINVAL
    vocab, _ = eng.item_emb_train(ids, cfg=cfg)                              # the Python call returns the whole list
    assert vocab.tolist() == vocab_h.tolist()
