"""item2vec on the device vs the oracle (BASELINE config 5).  The reference's own test asserts only shapes
(feature/embedding/wordemb_test.go:23) and its trainer is Hogwild, so parity here is: identical
deterministic bookkeeping (filtered document, subsampling decisions), and equal embedding quality."""
import numpy as np
import pytest

import go_ctr_b200 as g
from oracle import oracle as orc
from tests.test_oracle_i2v import neighbour_purity, planted_corpus

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]


def test_item2vec_counts_match_oracle_and_clusters_are_learned():
    rng = np.random.default_rng(2)
    toks, remap, nc, per = planted_corpus(rng)
    V = nc * per
    emb, st = g.i2v_train_ids(toks, V, dim=16, window=5, iter=3, seed=5)
    ocfg = orc.i2v_cfg(dim=16, window=5, iters=3, seed=5, rng_mode=1)
    oemb, otrained = orc.i2v_train(ocfg, toks, V)
    assert st.doc_len == toks.size                                  # every item is frequent enough here
    assert st.trained_positions == otrained                         # same subsampling decisions, position by position
    assert st.pairs > 0 and st.node_visits > 3 * st.pairs                     # paths are walked, not cut off at the root
    assert emb.shape == (V, 16) and np.isfinite(emb).all()
    pg, po = neighbour_purity(emb, remap, nc, per), neighbour_purity(oemb, remap, nc, per)
    assert pg > 0.9 and po > 0.9 and abs(pg - po) < 0.08, (pg, po)
    # the similarity structure agrees with the sequential float64 trainer
    def cosmat(e):
        e = e / (np.linalg.norm(e, axis=1, keepdims=True) + 1e-12); return e @ e.T
    corr = np.corrcoef(cosmat(emb).ravel(), cosmat(oemb).ravel())[0, 1]
    assert corr > 0.8, corr


def test_min_count_filter_keeps_rare_items_at_their_initial_vector():
    rng = np.random.default_rng(3)
    toks, remap, nc, per = planted_corpus(rng, n_clusters=4, per=6, n_users=100, seq=30)
    V = nc * per + 2
    toks = np.concatenate([toks, [V - 2, V - 1, V - 2]]).astype(np.int32)   # two items seen < 5 times
    emb, st = g.i2v_train_ids(toks, V, dim=16, window=5, iter=1, seed=9)
    assert st.doc_len == toks.size - 3                                       # memory.go:53-62
    for w in (V - 2, V - 1):
        want = np.array([orc.lib().orc_i2v_init(9, w * 16 + k, 16) for k in range(16)], np.float32)
        np.testing.assert_array_equal(emb[w], want)                          # word2vec.go:103-111, never trained


def test_train_embedding_mirror_and_dims():
    words = [str(100 + (i * 7) % 13) for i in range(4000)]
    m = g.TrainEmbedding(iter(words), 5, 16, 1)
    mp = m.GenEmbeddingMap32()
    assert len(mp) == 13 and all(v.shape == (16,) and v.dtype == np.float32 for v in mp.values())
    assert m.id2word[0] == "100"                                             # ids by first appearance
    for d in (4, 64):
        emb, st = g.i2v_train_ids(np.arange(2000, dtype=np.int32) % 50, 50, dim=d, window=3, iter=1)
        assert emb.shape == (50, d) and np.isfinite(emb).all() and st.trained_positions > 0
    with pytest.raises(g.CtrError):
        g.i2v_train_ids(np.zeros(10, np.int32), 5, dim=12)                   # not a power of two


@pytest.mark.parametrize("dim", [16, 64])
def test_sequential_float64_mode_reproduces_the_oracle_bit_for_bit(dim):
    """cfg.reserved[0] = 1: one warp walks the document in order with float64 tables — the reference's algorithm as a
    single goroutine runs it (word2vec.go:198-221, model.go:48-78, optimizer.go:107-129).  Same tokens, same counter-RNG
    draws: the embeddings equal oracle/i2v_oracle.c's exactly, which pins the MinCount filter, subsample thresholds,
    Huffman paths and lr schedule of the host plan both kernels are given.  The parallel kernel's own draws, window
    enumeration and update arithmetic are checked in tests/test_gpu_i2v_kernel.py."""
    rng = np.random.default_rng(12)
    toks, remap, nc, per = planted_corpus(rng, n_clusters=5, per=8, n_users=60, seq=40)
    V = nc * per + 3
    toks = np.concatenate([toks, [V - 1, V - 2, V - 1]]).astype(np.int32)      # rare words: filtered from the document
    cfg = g.i2v_default_config(dim=dim, window=5, iter=2, seed=21, update_lr_batch=500)
    cfg.reserved[0] = 1
    emb, st = g.i2v_train_ids(toks, V, cfg=cfg)
    ocfg = orc.i2v_cfg(dim=dim, window=5, iters=2, seed=21, rng_mode=1)
    ocfg.update_lr_batch = 500
    # the C ABI carries init_lr / min_lr / subsample as float32: give the float64 oracle the same values
    ocfg.init_lr = float(np.float32(cfg.init_lr)); ocfg.min_lr = float(np.float32(cfg.min_lr)); ocfg.subsample = float(np.float32(cfg.subsample))
    oemb, otrained = orc.i2v_train(ocfg, toks, V)
    assert st.trained_positions == otrained and st.doc_len == toks.size - 3
    assert np.abs(emb - orc.i2v_train(orc.i2v_cfg(dim=dim, window=5, iters=1, seed=21, rng_mode=1), toks, V)[0]).max() > 1e-4   # training moved them
    assert emb.tobytes() == oemb.tobytes()
