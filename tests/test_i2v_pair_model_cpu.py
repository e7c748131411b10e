"""The reference that judges the parallel item2vec kernel (tests/i2v_pair_model.py) is itself held to
oracle/i2v_oracle.c here, and the kernel probe (tests/cuda/i2v_probe.cu) is compiled.  No GPU: the compile shows
what ptxas made of every instantiation of k_i2v_skipgram_hs — it is not a run, tests/test_gpu_i2v_kernel.py is."""
import re

import numpy as np

import go_ctr_b200 as g
from oracle import oracle as orc
from tests import i2v_pair_model as pm
from tests import i2v_probe
from tests.test_oracle_i2v import planted_corpus


def test_mix64_equals_the_oracles_counter_rng():
    for seed, stream, ctr in [(0, 0, 0), (5, 200, 17), (0xFFFFFFFF, 301, 2 ** 40 + 3), (21, 100, 2 ** 63 + 1)]:
        assert pm.mix64(seed, stream, ctr) == orc.lib().orc_mix64(seed, stream, ctr)
    ctr = np.array([0, 17, 2 ** 40 + 3], np.int64)
    assert [int(x) for x in pm._mix64_np(5, 200, ctr)] == [pm.mix64(5, 200, int(c)) for c in ctr]


def test_sequential_model_reproduces_the_oracle_trainer():
    """Both scales absent, float64 f, each pair seeing every earlier update: the model over a whole corpus, two
    iterations with the oracle's learning-rate schedule, equals orc_i2v_train — syn1 bit for bit, the embeddings after
    the same rounding to float32, the trained count.  (Products and sums are rounded separately on both sides: the
    oracle is built without FMA contraction and numpy's element-wise loops do not fuse.)"""
    rng = np.random.default_rng(7)
    toks, _, nc, per = planted_corpus(rng, n_clusters=4, per=6, n_users=40, seq=30)
    V, D, W, iters, seed, upd = nc * per, 16, 5, 2, 11, 100
    cfg = orc.i2v_cfg(dim=D, window=W, iters=iters, seed=seed, rng_mode=1)
    cfg.update_lr_batch = upd
    oemb, osyn1, otrained = orc.i2v_train(cfg, toks, V, want_syn1=True)
    cnt = np.bincount(toks, minlength=V)
    assert cnt.min() >= cfg.min_count                                         # the MinCount filter keeps every token
    poff, pnode, pcode = g.i2v_paths(cnt, cfg.max_depth)
    z = np.maximum(0.0, 1.0 - np.sqrt(cfg.subsample / cnt))                   # subsample.go:34-38
    syn0 = np.array([orc.lib().orc_i2v_init(seed, i, D) for i in range(V * D)], np.float64).reshape(V, D)
    syn1 = np.zeros((V - 1, D), np.float64)
    n = toks.size
    lr, trained = cfg.init_lr, 0
    for it in range(iters):
        lr_tab = np.empty(n // upd + 1, np.float64)
        for k in range(lr_tab.size):                                          # observe(), word2vec.go:223-233
            lr_tab[k] = lr
            seen = (k + 1) * upd
            if seen <= n:
                lr = cfg.min_lr if lr < cfg.min_lr else cfg.init_lr * (1.0 - seen / n)
        a = pm.Launch(doc=toks, z=z, poff=poff, pnode=pnode, pcode=pcode, syn0=syn0, syn1=syn1, W=W, lr_tab=lr_tab, upd=upd, seed=seed, iter=it)
        r = pm.launch_model(a, "sequential", f32=False)
        syn0, syn1 = r.syn0, r.syn1
        trained += r.counters[0]
    assert trained == otrained and 0 < trained < iters * n                    # subsampling dropped some positions
    assert syn1.tobytes() == osyn1.tobytes()
    assert syn0.astype(np.float32).tobytes() == oemb.tobytes()
    assert np.abs(osyn1).max() > 1e-3


def small_launch(rng, V=30, D=8, nd=400, W=3):
    doc = rng.integers(0, V, nd).astype(np.int32)
    cnt = np.bincount(doc, minlength=V) + 1
    poff, pnode, pcode = g.i2v_paths(cnt, 100)
    return pm.Launch(doc=doc, z=rng.uniform(0.3, 1.2, V), poff=poff, pnode=pnode, pcode=pcode,
                     syn0=rng.uniform(-0.5, 0.5, (V, D)).astype(np.float32), syn1=rng.uniform(-0.25, 0.25, (V - 1, D)).astype(np.float32),
                     W=W, lr_tab=np.array([2.0 ** -12, 2.0 ** -13, 2.0 ** -12.5], np.float32), upd=150, seed=3, iter=1,
                     node_scale=rng.choice([1.0, 0.5, 1.0 / 3], V - 1).astype(np.float32), word_scale=rng.choice([1.0, 0.25], V).astype(np.float32),
                     pos_begin=7, pos_end=nd - 5)


def test_vectorised_stale_sum_equals_the_loop():
    a = small_launch(np.random.default_rng(1))
    r = pm.launch_model(a, "stale", f32=False)
    d0, d1, ctr = pm.stale_sum(a)
    assert ctr == r.counters and ctr[0] > 50 and ctr[2] > ctr[1] > ctr[0]
    for d, out, init in ((d0, r.syn0, a.syn0), (d1, r.syn1, a.syn1)):
        want = out - init.astype(np.float64)
        # the loop's f is float64 and takes the float64 bin, stale_sum's the kernel's float32 bin: they differ on the rare
        # f within a rounding of a bin edge, by one table step (3e-3 of one addend)
        assert np.abs(d - want).max() < 1e-4 * np.abs(want).max() and np.abs(want).max() > 1e-5


def test_orders_agree_to_second_order_in_the_learning_rate():
    a = small_launch(np.random.default_rng(2))
    seq, stale = pm.launch_model(a, "sequential"), pm.launch_model(a, "stale")
    assert seq.counters == stale.counters and seq.rows == stale.rows and seq.nodes == stale.nodes
    step = np.abs(stale.syn1 - a.syn1).max()
    assert 0 < np.abs(seq.syn1 - stale.syn1).max() < 0.05 * step


def test_probe_compiles_for_sm90a_without_spills():
    """A compile, not a run: ptxas reports no spill and no stack frame for any of the six vector widths."""
    so, log = i2v_probe.build_probe(force=True)
    found = {}
    for m in re.finditer(r"Function properties for _ZN3ctr17k_i2v_skipgram_hsILi(\d+)EE\S*\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads"
                         r"\s+ptxas info\s+: Used (\d+) registers", log):
        found[int(m.group(1))] = tuple(int(x) for x in m.groups()[1:])
    assert sorted(found) == [1, 2, 4, 8, 16, 32], log
    for lpr, (stack, st, ld, regs) in sorted(found.items()):
        print("k_i2v_skipgram_hs<%d>: %d registers" % (lpr, regs))
        assert (stack, st, ld) == (0, 0, 0) and regs <= 255, (lpr, stack, st, ld, regs)
    assert "sm_90a" in log
