"""ctr_item_emb_train on a multi-GPU handle (needs >= 2 GPUs; runs at W = 2, 4 and 8, as many as the box has), one
process per rank.  The planted corpus of tests/test_oracle_i2v.py, as sparse item ids with unmapped ids, rare items and
an INT64_MIN mixed in, is cut into the ranks' shards (one case leaves a rank empty) and trained into a replicated
ITEM_EMB, a row-sharded one and a row-sharded one with replicated hot rows.  Against a one-GPU ctr_item_emb_train on the
concatenated stream:
  * vocab_ids and V on every rank equal the one-GPU call's; the ranks' doc_len sum to its doc_len;
  * rows of words below min_count equal its rows (the seeded initial vector): bit for bit at W = 2, within 1e-6 at W > 2,
    where the replica average's sum of W equal floats can round (include/ctr_b200.h); rows of absent items are zero;
  * a replicated ITEM_EMB is byte-identical on every rank; the trained rows learn the clusters (neighbour purity > 0.9,
    within 0.08 of the float64 oracle);
  * right after the call, ctr_knn_search and ctr_recommend_topk on the handle equal, bit for bit and on every rank, a
    one-GPU handle holding the stitched table (the mappings republished, the hot rows pulled from the new rows); a
    sharded train step then matches that twin at the suite's training bars;
  * refusals (configurations that differ, item maps that differ, the sequential mode, one distinct word, every rank
    empty, no item map on one rank) give the same code on every rank and change no map or table."""
import os

import numpy as np
import pytest
import torch

import go_ctr_b200 as g
from oracle import oracle as orc
from tests import test_gpu_shard_rank as sr
from tests.test_oracle_i2v import neighbour_purity, planted_corpus
from tests.util import INT64_MIN, assert_mostly_close

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

UP, S, D, CF = 4, 5, 16, 3
B = 64
NC, PER = 8, 12
RARE = np.array([77_001, 77_002, 77_003], np.int64)          # mapped items seen fewer than min_count times
SIDE = np.array([88_001, 88_002], np.int64)                 # unmapped ids, frequent enough to train
NEVER = 5000 + np.arange(20, dtype=np.int64)                # mapped items the stream never holds
CASES = {"replicated": dict(policy=2, hot=-1, empty=None), "sharded": dict(policy=1, hot=-1, empty=None),
         "hot": dict(policy=1, hot=16, empty=1)}


def _corpus():
    rng = np.random.default_rng(2)
    toks, remap, nc, per = planted_corpus(rng)
    word_tok = np.empty(nc * per, np.int64); word_tok[remap] = np.arange(nc * per)
    item_of_tok = 1000 + 7 * np.arange(nc * per, dtype=np.int64)
    s = item_of_tok[word_tok[toks]]
    r2 = np.random.default_rng(3)
    for v, k in [(RARE[0], 1), (RARE[1], 2), (RARE[2], 3), (SIDE[0], 9), (SIDE[1], 12), (INT64_MIN, 6)]:
        s[r2.integers(0, s.size, k)] = v
    imap = np.random.default_rng(4).permutation(np.concatenate([item_of_tok, RARE, NEVER]))
    return s, imap, item_of_tok


def _cuts(n, W, empty):
    c = [n * (r + 1) // W for r in range(W - 1)]
    if empty is not None and empty < W - 1:                   # rank `empty` holds nothing: its end is its start
        c[empty] = c[empty - 1] if empty > 0 else 0
    elif empty is not None:                                   # the last rank: the cut before it moves to the end
        c[-1] = n
    return c


def _i2v(**kw):
    return g.i2v_default_config(**{"dim": D, "window": 5, "iter": 3, "seed": 5, **kw})


def _cfg(policy, hot, **kw):
    x = g.engine.default_config(g.MODEL_DIN_COS, uP=UP, S=S, D=D, cF=CF, pred_batch=128, table_opt=g.TABLE_SGD_DETERMINISTIC,
                                table_lr=0.5, dropout0=0.0, dropout1=0.0, seed=5, **kw)
    x.reserved[1] = policy; x.reserved[0] = hot
    return x


def _setup(eng, imap):
    rng = np.random.default_rng(1)
    eng.table_upload(g.TABLE_USER_FEAT, rng.standard_normal((30, UP)).astype(np.float32))
    eng.table_upload(g.TABLE_ITEM_FEAT, rng.standard_normal((imap.size, CF)).astype(np.float32))
    eng.table_upload(g.TABLE_ITEM_EMB, np.full((imap.size, D), 9.0, np.float32))
    eng.idmap_build(g.IDMAP_USER, 100 + np.arange(30, dtype=np.int64)); eng.idmap_build(g.IDMAP_ITEM, imap)


def _serve(eng, res, n_items):
    rng = np.random.default_rng(6)
    q = rng.integers(0, n_items, 12).astype(np.int32)
    res["knn.rows"], res["knn.sims"], res["knn.count"] = eng.knn_search(10, rows=q)
    urows = rng.integers(0, 30, 8).astype(np.int32); hist = rng.integers(-1, n_items, (8, S)).astype(np.int32)
    for j, part in enumerate(("rows", "scores", "logits", "count")):
        res["rec." + part] = eng.recommend_topk(urows, hist, 20)[j]


def _keys(W, n_items, rank):
    out = []
    for j in range(W):
        rng = np.random.default_rng(60 + j)
        out.append((100 + rng.integers(0, 30, B), rng.integers(0, n_items, B), rng.integers(1, 50, B).astype(np.int64),
                    (rng.random(B) > 0.5).astype(np.float32)))
    return out[rank] if rank is not None else tuple(np.concatenate([o[k] for o in out]) for k in range(4))


def _worker(rank, W, port, out_dir, case):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=W)
    torch.cuda.set_device(rank)
    c = CASES[case]
    s, imap, _ = _corpus()
    shard = np.split(s, _cuts(s.size, W, c["empty"]))[rank]
    eng = sr._engine(rank, lambda r: _cfg(c["policy"], c["hot"], batch=B, device=r, rank=r, world=W))
    _setup(eng, imap)
    res = {}
    eng.profile(True); eng.profile_reset()
    vocab, st = eng.item_emb_train(shard, cfg=_i2v(), sync_every=2000)
    res["prof"] = np.array(sorted(eng.profile_dump())); eng.profile(False)
    res["has_side"] = np.array(bool((~np.isin(shard, imap)).any()))      # i2v_dict_side runs only on such a rank
    res["vocab"], res["doc_len"] = vocab, np.array(st.doc_len)
    res["emb"] = eng.table_download(g.TABLE_ITEM_EMB, imap.size, D)
    _serve(eng, res, imap.size)
    ku, ki, kt, ky = _keys(W, imap.size, rank)
    _, cost, _ = eng.train_keys(ku, imap[ki], kt, ky, epochs=1)
    res["cost"] = np.array([cost], np.float32)
    res["emb.trained"] = eng.table_download(g.TABLE_ITEM_EMB, imap.size, D)
    for i, w in enumerate(eng.get_weights()):
        res["w%d" % i] = w
    # refusals: the same code everywhere, no map or table changed
    state = lambda: [eng.idmap_download(g.IDMAP_ITEM), eng.table_download(g.TABLE_ITEM_EMB, imap.size, D)]
    same = lambda a, b: all(x.tobytes() == y.tobytes() for x, y in zip(a, b))
    before = state()
    call = lambda ids, cfg: sr._err(lambda: eng.item_emb_train(ids, cfg=cfg))[0]
    seq = _i2v(); seq.reserved[0] = 1
    res["code.cfg"] = np.array(call(shard, _i2v(window=6 if rank == W - 1 else 5)))
    res["code.seq"] = np.array(call(shard, seq))
    res["code.one"] = np.array(call(np.full(3 if rank == 0 else 0, imap[0], np.int64), _i2v()))
    res["code.empty"] = np.array(call(np.zeros(0, np.int64), _i2v()))
    res["unchanged"] = np.array(same(before, state()))
    eng.idmap_build(g.IDMAP_ITEM, imap if rank == 0 else imap[::-1].copy())
    before = state()
    res["code.maps"] = np.array(call(shard, _i2v()))
    res["maps_unchanged"] = np.array(same(before, state()))
    eng.close()
    bare = sr._engine(rank, lambda r: _cfg(c["policy"], c["hot"], batch=B, device=r, rank=r, world=W))
    if rank == 0:
        bare.idmap_build(g.IDMAP_ITEM, imap)
    res["code.nomap"] = np.array(sr._err(lambda: bare.item_emb_train(shard, cfg=_i2v()))[0])
    bare.close()
    np.savez(os.path.join(out_dir, "emb_%s_%d_%d.npz" % (case, W, rank)), **res)
    dist.barrier(); dist.destroy_process_group()


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("W", [2, 4, 8])
def test_sharded_item_emb_train_equals_one_gpu(tmp_path, W, case):
    if W > torch.cuda.device_count():
        pytest.skip("needs %d GPUs" % W)
    import torch.multiprocessing as mp
    mp.spawn(_worker, args=(W, sr._free_port(), str(tmp_path), case), nprocs=W, join=True)
    _check([np.load(tmp_path / ("emb_%s_%d_%d.npz" % (case, W, r))) for r in range(W)], W, case)


def _check(rs, W, case, refusals=True):
    s, imap, item_of_tok = _corpus()
    one = g.Engine(_cfg(0, -1, batch=B * W))
    _setup(one, imap)
    vocab1, st1 = one.item_emb_train(s, cfg=_i2v())
    emb1 = one.table_download(g.TABLE_ITEM_EMB, imap.size, D)
    one.close()
    sharded = CASES[case]["policy"] == 1
    emb = np.zeros_like(emb1)
    keys = {"i2v_dict_resolve", "i2v_dict_rank", "i2v_dict_doc", "i2v_emb_scatter"} | ({"i2v_dict_ranks"} if W > 1 else set())
    for r, res in enumerate(rs):
        assert res["vocab"].tobytes() == vocab1.tobytes(), r
        prof = set(res["prof"].tolist())
        assert keys <= prof, (r, sorted(prof))
        assert ("i2v_dict_side" in prof) == bool(res["has_side"]), (r, sorted(prof))
        if sharded:
            emb[r::W] = res["emb"][r::W]
        else:
            assert res["emb"].tobytes() == rs[0]["emb"].tobytes(), r              # every rank holds the same replica
            emb = res["emb"]
    if CASES[case]["empty"] is not None and W > 1:
        assert not bool(rs[CASES[case]["empty"]]["has_side"]) and int(rs[CASES[case]["empty"]]["doc_len"]) == 0
    assert sum(int(res["doc_len"]) for res in rs) == st1.doc_len
    row = {int(v): i for i, v in enumerate(imap)}
    rare = [row[int(v)] for v in RARE]
    if W <= 2:      # x + x and a halving are exact: the rare words' initial vectors survive the averaging bit for bit
        assert emb[rare].tobytes() == emb1[rare].tobytes()
    else:           # a sum of W > 2 equal floats can round once per replica average
        np.testing.assert_allclose(emb[rare], emb1[rare], rtol=1e-6, atol=0)
    assert not emb[[row[int(v)] for v in NEVER]].any()
    rows = np.array([row[int(v)] for v in item_of_tok])
    pg = neighbour_purity(emb[rows], np.arange(NC * PER), NC, PER)
    toks, remap, nc, per = planted_corpus(np.random.default_rng(2))
    oemb, _ = orc.i2v_train(orc.i2v_cfg(dim=D, window=5, iters=3, seed=5, rng_mode=1), toks, nc * per)
    po = neighbour_purity(oemb, remap, nc, per)
    assert pg > 0.9 and abs(pg - po) < 0.08, (pg, po)
    # serving and training right after the call: a one-GPU twin holding the stitched table
    twin = g.Engine(_cfg(0, -1, batch=B * W))
    _setup(twin, imap)
    twin.table_upload(g.TABLE_ITEM_EMB, emb)
    want = {}
    _serve(twin, want, imap.size)
    ku, ki, kt, ky = _keys(W, imap.size, None)
    _, cost, _ = twin.train_keys(ku, imap[ki], kt, ky, epochs=1)
    want_emb = twin.table_download(g.TABLE_ITEM_EMB, imap.size, D)
    want_w = twin.get_weights()
    twin.close()
    for r, res in enumerate(rs):
        for key in ("knn.rows", "knn.sims", "knn.count", "rec.rows", "rec.scores", "rec.logits", "rec.count"):
            sr._assert_same(res[key], want[key], "%s (rank %d)" % (key, r))
    np.testing.assert_allclose(rs[0]["cost"], np.float32(cost), rtol=2e-4, atol=1e-6)
    for i in range(4):
        assert_mostly_close(rs[0]["w%d" % i], want_w[i], 2e-3, 2e-4, 0.995, "weights %d" % i)
    trained = np.zeros_like(want_emb)
    for r, res in enumerate(rs):
        trained[r::W] = res["emb.trained"][r::W]
    np.testing.assert_allclose(trained, want_emb, rtol=2e-3, atol=2e-5)
    if not refusals:
        return
    for r, res in enumerate(rs):
        for k in ("code.cfg", "code.seq", "code.one", "code.empty", "code.maps"):
            assert int(res[k]) == g.EINVAL, (k, r, int(res[k]))
        assert int(res["code.nomap"]) == g.ESTATE
        assert bool(res["unchanged"]) and bool(res["maps_unchanged"])
