"""ctr_item_emb_train: recommend.Train's embedding stage straight into ITEM_EMB, against the host route it replaces —
words numbered by first appearance in numpy, ctr_i2v_train on the word ids, the table remapped into item rows (zeros
for items the stream never holds) and uploaded with ctr_table_upload."""
import ctypes as C

import numpy as np
import pytest

import go_ctr_b200 as g
from oracle import oracle as orc
from tests.util import INT64_MAX, INT64_MIN

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

NEG = -1234567890123


def make_stream(rng, n, n_items, a, n_never=40):
    """A Zipf stream of sparse int64 item ids and an item map for it.  The stream holds INT64_MIN, INT64_MAX and a
    negative id from its first tokens on, and eight ids that occur once or twice.  INT64_MIN (never a map key), catalog
    items spread over the frequency ranks and four of the rare ids have no map entry; the map also holds n_never ids the
    stream never has, and is shuffled so that rows are not in first-appearance order."""
    draw = np.unique(rng.integers(INT64_MIN + 1, INT64_MAX, 2 * n_items + 8, dtype=np.int64))
    draw = rng.permutation(draw[~np.isin(draw, [NEG, INT64_MAX])])
    cat, rare = np.concatenate([draw[:n_items - 3], [INT64_MAX, INT64_MIN, NEG]]), draw[n_items - 3:n_items + 5]
    ids = cat[(rng.zipf(a, n) - 1) % cat.size]
    ids[[3, 11, 29]] = [INT64_MIN, INT64_MAX, NEG]
    for k, v in enumerate(rare):
        ids[rng.integers(40, n, 1 + k % 2)] = v
    unmapped = np.concatenate([[INT64_MIN], cat[[r for r in (1, 5, 12, 25, 40, 55) if r < n_items - 3]], rare[4:]])
    never = rng.integers(INT64_MIN + 1, INT64_MAX, n_never, dtype=np.int64)
    never = never[~np.isin(never, np.concatenate([cat, rare]))]
    imap = rng.permutation(np.concatenate([cat[~np.isin(cat, unmapped)], rare[:4], never]))
    return ids, imap


def host_route(ids, imap, cfg):
    """Numbering by first appearance in numpy, ctr_i2v_train, remap into item rows with zeros elsewhere."""
    uniq, first = np.unique(ids, return_index=True)
    order = np.argsort(first, kind="stable")
    word_of_uniq = np.empty(uniq.size, np.int64); word_of_uniq[order] = np.arange(uniq.size)
    tok = word_of_uniq[np.searchsorted(uniq, ids)].astype(np.int32)
    emb, st = g.i2v_train_ids(tok, uniq.size, cfg=cfg)
    pos = np.minimum(np.searchsorted(uniq, imap), uniq.size - 1)
    hit = uniq[pos] == imap
    table = np.zeros((imap.size, cfg.dim), np.float32)
    table[hit] = emb[word_of_uniq[pos[hit]]]
    words_of_rows = np.full(imap.size, -1, np.int64); words_of_rows[hit] = word_of_uniq[pos[hit]]
    return uniq[order], tok, table, st, words_of_rows


def store(D, **kw):
    return g.Engine(g.engine.default_config(g.MODEL_DIN_COS, uP=0, cF=0, S=1, D=D, batch=1, pred_batch=1, **kw))


def seq_cfg(**kw):
    cfg = g.i2v_default_config(**kw)
    cfg.reserved[0] = 1
    return cfg


def same_stats(a, b, fields):
    return {f: (getattr(a, f), getattr(b, f)) for f in fields if getattr(a, f) != getattr(b, f)}


@pytest.mark.parametrize("D,W,iters,n,n_items,a,extra", [
    (16, 5, 1, 30_000, 3000, 1.3, {}),
    (64, 3, 2, 20_000, 2000, 1.2, {}),
    (16, 2, 3, 12_000, 500, 1.5, {"min_count": 3}),
    # past one 32 MB staging chunk of the int64 stream (4 Mi tokens); a heavy head and a large subsample threshold keep
    # the sequential trainer's share of the run short
    (16, 1, 1, 4_200_000, 60, 2.0, {"subsample": 1.0e5}),
])
def test_sequential_mode_equals_the_host_route_bit_for_bit(D, W, iters, n, n_items, a, extra):
    rng = np.random.default_rng(n + D)
    ids, imap = make_stream(rng, n, n_items, a)
    cfg = seq_cfg(dim=D, window=W, iter=iters, seed=17, update_lr_batch=1000, **extra)
    vocab_h, tok, table_h, st_h, word_row = host_route(ids, imap, cfg)
    cnt = np.bincount(tok, minlength=vocab_h.size)
    rare = cnt < cfg.min_count
    assert rare.any() and (~rare).any()                                      # words below min_count, and trained ones
    in_map = np.isin(vocab_h, imap)
    assert (~in_map).sum() >= 2 and INT64_MIN in vocab_h and INT64_MAX in vocab_h and NEG in vocab_h
    assert (word_row < 0).sum() >= 30                                        # rows whose item never occurs
    assert (rare & in_map).any() and (rare & ~in_map).any()
    eng = store(D)
    eng.idmap_build(g.IDMAP_ITEM, imap)
    vocab_d, st_d = eng.item_emb_train(ids, cfg=cfg)
    assert vocab_d.tolist() == vocab_h.tolist()
    assert not same_stats(st_d, st_h, ("doc_len", "trained_positions", "pairs", "node_visits"))
    got = eng.table_download(g.TABLE_ITEM_EMB, imap.size, D)
    assert got.tobytes() == table_h.tobytes()
    assert not got[word_row < 0].any()


def test_parallel_mode_numbers_like_the_host_route():
    D = 32
    rng = np.random.default_rng(7)
    ids, imap = make_stream(rng, 300_000, 20_000, 1.1)
    cfg = g.i2v_default_config(dim=D, window=5, iter=2, seed=23)
    vocab_h, tok, _, st_h, word_row = host_route(ids, imap, cfg)
    eng = store(D)
    eng.idmap_build(g.IDMAP_ITEM, imap)
    vocab_d, st_d = eng.item_emb_train(ids, cfg=cfg)
    assert vocab_d.tolist() == vocab_h.tolist()
    assert not same_stats(st_d, st_h, ("doc_len", "trained_positions", "pairs"))
    got = eng.table_download(g.TABLE_ITEM_EMB, imap.size, D)
    cnt = np.bincount(tok, minlength=vocab_h.size)
    rows = np.nonzero(word_row >= 0)[0]
    rare_rows = rows[cnt[word_row[rows]] < cfg.min_count]
    assert rare_rows.size > 100
    init = orc.lib().orc_i2v_init
    for r in rare_rows[:: max(1, rare_rows.size // 200)]:                    # never trained: the initial vector of the word
        w = int(word_row[r])
        want = np.array([init(23, w * D + k, D) for k in range(D)], np.float32)
        assert got[r].tobytes() == want.tobytes(), (r, w)
    assert not got[word_row < 0].any()
    assert np.isfinite(got).all() and np.abs(got[rows]).sum(axis=1).min() > 0


def test_end_to_end_state_equals_an_upload_of_the_host_table():
    """Handle A (row Adam, trained already) runs ctr_item_emb_train; handle B uploads the host route's table.  After the
    same ctr_set_weights both train the same keys identically: the call reset the row moments and hot rows as an
    upload does.  YouTube DNN at batch 32: no attention-weight or split-K gradient sums whose order could vary."""
    rng = np.random.default_rng(41)
    U, D, uP, cF, S, B = 50, 16, 4, 4, 3, 32
    ids, imap = make_stream(rng, 40_000, 400, 1.3)
    I = imap.size
    uid = rng.permutation(np.arange(1000, 1000 + U, dtype=np.int64) * 7919)
    uf = rng.random((U, uP), np.float32); itf = rng.random((I, cF), np.float32)
    emb0 = (rng.standard_normal((I, D)) / 4).astype(np.float32)
    kw = dict(uP=uP, S=S, D=D, cF=cF, batch=B, pred_batch=B, table_opt=g.TABLE_ADAM, table_lr=0.01, seed=3, dropout0=0.0, dropout1=0.0)
    n_keys = 10 * B
    ku = uid[rng.integers(0, U, n_keys)]; ki = imap[rng.integers(0, I, n_keys)]
    kt = np.zeros(n_keys, np.int64); y = (rng.random(n_keys) > 0.5).astype(np.float32)

    def engine():
        e = g.Engine(g.engine.default_config(g.MODEL_YOUTUBE, **kw))
        e.table_upload(g.TABLE_USER_FEAT, uf); e.table_upload(g.TABLE_ITEM_FEAT, itf)
        e.idmap_build(g.IDMAP_USER, uid); e.idmap_build(g.IDMAP_ITEM, imap)
        return e

    A = engine()
    W = A.get_weights()
    A.table_upload(g.TABLE_ITEM_EMB, emb0)
    A.train_keys(ku, ki, kt, y, epochs=2)
    assert not np.array_equal(A.table_download(g.TABLE_ITEM_EMB, I, D), emb0)          # row Adam moved rows: moments are live
    cfg = seq_cfg(dim=D, window=5, iter=1, seed=5)
    A.item_emb_train(ids, cfg=cfg)
    _, _, table_h, _, _ = host_route(ids, imap, cfg)
    assert A.table_download(g.TABLE_ITEM_EMB, I, D).tobytes() == table_h.tobytes()
    Bh = engine()
    Bh.table_upload(g.TABLE_ITEM_EMB, table_h)
    for e in (A, Bh):
        e.set_weights(*W)
    for _ in range(3):
        ca = A.train_keys(ku, ki, kt, y, epochs=1); cb = Bh.train_keys(ku, ki, kt, y, epochs=1)
        assert np.float32(ca[1]).tobytes() == np.float32(cb[1]).tobytes() and ca == cb, (ca, cb)
    for wa, wb in zip(A.get_weights(), Bh.get_weights()):
        assert wa.tobytes() == wb.tobytes()
    assert A.table_download(g.TABLE_ITEM_EMB, I, D).tobytes() == Bh.table_download(g.TABLE_ITEM_EMB, I, D).tobytes()


def test_in_place_and_reallocated_tables_and_the_vocabulary_cap():
    """ITEM_EMB of the map's shape is rewritten in place; another shape (or none) is reallocated; vocab_ids stops at cap."""
    D = 16
    rng = np.random.default_rng(3)
    ids, imap = make_stream(rng, 20_000, 800, 1.3)
    cfg = g.i2v_default_config(dim=D, window=3, seed=2)
    vocab_h, _, _, _, word_row = host_route(ids, imap, cfg)
    for pre in (None, imap.size, imap.size + 5):
        eng = store(D)
        eng.idmap_build(g.IDMAP_ITEM, imap)
        if pre:
            eng.table_upload(g.TABLE_ITEM_EMB, np.full((pre, D), 9.0, np.float32))
        vocab, _ = eng.item_emb_train(ids, cfg=cfg)
        assert vocab.tolist() == vocab_h.tolist()
        got = eng.table_download(g.TABLE_ITEM_EMB, imap.size, D)
        assert not got[word_row < 0].any() and (got[word_row >= 0] != 9.0).all()
    L = g.load_library()
    cap = 10; out = np.full(cap + 1, 77, np.int64); V = C.c_int32(0)
    a = np.ascontiguousarray(ids)
    assert L.ctr_item_emb_train(eng.h, C.byref(cfg), a.ctypes.data_as(C.POINTER(C.c_int64)), C.c_int64(a.size),
                                out.ctypes.data_as(C.POINTER(C.c_int64)), C.c_int64(cap), C.byref(V), None) == 0
    assert V.value == vocab_h.size and out[:cap].tolist() == vocab_h[:cap].tolist() and out[cap] == 77


def test_refusals_leave_the_table_as_it_was():
    D = 16
    rng = np.random.default_rng(5)
    ids, imap = make_stream(rng, 5_000, 300, 1.3)
    emb0 = rng.random((imap.size, D), np.float32)
    L = g.load_library()
    lp = C.POINTER(C.c_int64)

    def call(eng, cfg, a, n):
        V = C.c_int32(-1)
        rc = L.ctr_item_emb_train(eng.h, C.byref(cfg) if cfg is not None else None, a.ctypes.data_as(lp) if a is not None else None,
                                  C.c_int64(n), None, C.c_int64(0), C.byref(V), None)
        return rc, V.value

    bare = store(D)                                                          # no item map
    bare.table_upload(g.TABLE_ITEM_EMB, emb0)
    assert call(bare, g.i2v_default_config(dim=D), ids, ids.size)[0] == g.ESTATE
    assert bare.table_download(g.TABLE_ITEM_EMB, imap.size, D).tobytes() == emb0.tobytes()
    eng = store(D, table_opt=g.TABLE_ADAM, table_lr=0.01)
    eng.idmap_build(g.IDMAP_ITEM, imap)
    eng.table_upload(g.TABLE_ITEM_EMB, emb0)
    one = np.full(100, imap[0], np.int64)
    cases = [(g.i2v_default_config(dim=2 * D), ids, ids.size),              # dim != D
             (g.i2v_default_config(dim=D, window=0), ids, ids.size),       # a configuration the trainer refuses
             (g.i2v_default_config(dim=D), one, one.size),                 # one distinct word
             (g.i2v_default_config(dim=D), ids, 0),                        # n = 0
             (None, ids, ids.size), (g.i2v_default_config(dim=D), None, ids.size)]
    for cfg, a, n in cases:
        rc, V = call(eng, cfg, a, n)
        assert rc == g.EINVAL, (rc, n)
        assert eng.table_download(g.TABLE_ITEM_EMB, imap.size, D).tobytes() == emb0.tobytes()
    assert call(eng, g.i2v_default_config(dim=D), one, one.size)[1] == 1   # V is reported with the refusal
    with pytest.raises(g.CtrError):
        g.TrainItemEmbedding(eng, ["5", "5", "5"])


def test_profile_keys_and_the_python_mirror():
    D = 16
    rng = np.random.default_rng(9)
    ids, imap = make_stream(rng, 8_000, 400, 1.3)
    eng = store(D)
    eng.idmap_build(g.IDMAP_ITEM, imap)
    eng.profile(True)
    vocab, st = g.TrainItemEmbedding(eng, [str(int(v)) for v in ids], window=5, iter=1)
    prof = eng.profile_dump()
    for k in ("i2v_dict_resolve", "i2v_dict_side", "i2v_dict_rank", "i2v_dict_doc", "i2v_emb_scatter"):
        assert k in prof, (k, sorted(prof))
    vocab2, _ = eng.item_emb_train(ids, window=5, iter=1)                    # ints and canonical strings: one stream
    assert vocab.tolist() == vocab2.tolist() and st.doc_len > 0
