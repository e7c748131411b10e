"""The key-fed float64 MLP served from a row-sharded feature store (needs >= 2 GPUs): predict_keys, recommend_topk_ex
and rank_items_ex on both ranks must equal, bit for bit, a single-GPU feature store holding the assembled tables, the
same id maps, rank 0's ubcache and the same parameters.

Cases, each of which first asserts its placement from the ranks' table downloads: ITEM_FEAT sharded beside a sharded
ITEM_EMB; the by-size placement with an ITEM_EMB above 32 MB (sharded, its popular rows replicated) beside a small,
replicated ITEM_FEAT; hot rows with sharded train steps queued right before the calls and no sync; a table of one row
(rank 1's shard is empty); ubcaches that differ across ranks (every rank returns the same result, the windows rank 0's
cache cuts).  A classifier and an identity-output regressor.  Refusals: a ts that differs on one rank (EINVAL on
both), id maps that resolve the same ids to other rows on one rank (EINVAL on both), a user missing from one rank's id
map (ENOTFOUND on both), fit_keys, a replicated ITEM_EMB beside a sharded ITEM_FEAT and a model with classes (ESTATE).
The profile keys of one call of each kind."""
import os

import numpy as np
import pytest

import go_ctr_b200 as g
from tests import test_gpu_shard_rank as sr

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200)]

WORLD = sr.WORLD
U = 40
UP, S, D, CF = 4, 5, 16, 3
NIN = UP + S * D + D + CF
# placement: reserved[1] 1 shards both ITEM tables; 0 shards a table above 32 MB (600 000 x 16 floats = 38.4 MB) and
# replicates the rest.  hot: reserved[0] (-1 none, 0 the default popular rows).  nu / nr: users per recommendation, keys
# per rank call.
CASES = {
    "feat_sharded": dict(N=1001, NF=900, policy=1, hot=-1, pb=128, train=False, nu=260, nr=120, emb="sharded", feat="sharded"),
    "feat_auto": dict(N=600_000, NF=5000, policy=0, hot=0, pb=8192, train=False, nu=12, nr=40, emb="sharded", feat="replicated"),
    "hot_trained": dict(N=777, NF=777, policy=1, hot=64, pb=96, train=True, nu=60, nr=120, emb="sharded", feat="sharded"),
    "one_row": dict(N=1, NF=1, policy=1, hot=-1, pb=64, train=False, nu=260, nr=120, emb="sharded", feat="sharded"),
}
MODES = {"none": dict(exclude_history=False), "window": dict(exclude_history=True), "seen": dict(exclude_seen=True)}


def _cfg(c, **kw):
    return g.engine.default_config(g.MODEL_DIN_COS, uP=UP, S=S, D=D, cF=CF, batch=64, pred_batch=c["pb"], table_opt=g.TABLE_SGD,
                                   table_lr=0.5, dropout0=0.0, dropout1=0.0, seed=5, **kw)


def _sharded(c, policy=None):
    def cfg(r):
        x = _cfg(c, device=r, rank=r, world=WORLD)
        x.reserved[1] = c["policy"] if policy is None else policy
        x.reserved[0] = c["hot"]
        return x
    return cfg


def _tables(name):
    c = CASES[name]
    rng = np.random.default_rng(sum(name.encode()))
    return (rng.standard_normal((U, UP)).astype(np.float32), rng.standard_normal((c["NF"], CF)).astype(np.float32),
            rng.standard_normal((c["N"], D)).astype(np.float32))


def _ids(c):
    return 1000 + np.arange(U, dtype=np.int64), 50_000 + 3 * np.arange(c["N"], dtype=np.int64)


def _cache(c, salt=0):
    rng = np.random.default_rng(7 + salt)
    seqs = []
    for u in range(U):
        n = int(rng.integers(0, 30))
        ts = np.sort(rng.integers(1, 40, n))[::-1].astype(np.int64)
        seqs.append(list(zip(ts.tolist(), rng.integers(-1, c["N"] + 2, n).tolist())))
    off = np.concatenate([[0], np.cumsum([len(s) for s in seqs])]).astype(np.int64)
    return off, np.array([t for s in seqs for t, _ in s], np.int64), np.array([i for s in seqs for _, i in s], np.int32)


def _setup(eng, name, salt=0, users=None, items=None):
    c = CASES[name]
    uf, itf, emb = _tables(name)
    eng.table_upload(g.TABLE_USER_FEAT, uf)
    eng.table_upload(g.TABLE_ITEM_FEAT, itf)
    eng.table_upload(g.TABLE_ITEM_EMB, emb)
    uid, iid = _ids(c)
    eng.idmap_build(0, uid if users is None else users)
    eng.idmap_build(1, iid if items is None else items)
    eng.ubcache_upload(*_cache(c, salt))


def _assert_placement(eng, rank, tables):
    """tables: (which, full table, "sharded" | "replicated").  A sharded table's download fills this rank's rows only."""
    for which, tab, want in tables:
        exp = tab.copy()
        if want == "sharded":
            exp[np.arange(tab.shape[0]) % WORLD != rank] = 0
        assert np.array_equal(eng.table_download(which, *tab.shape), exp), ("placement", which, want, rank)


def _case_placement(eng, name, rank):
    c = CASES[name]
    _, itf, emb = _tables(name)
    _assert_placement(eng, rank, [(g.TABLE_ITEM_EMB, emb, c["emb"]), (g.TABLE_ITEM_FEAT, itf, c["feat"])])


def _models(device):
    rng = np.random.default_rng(11)
    clf = g.engine.MLPClassifier(NIN, hidden=(24, 7), device=device)
    clf.set_params(rng.standard_normal(clf.get_params().size) * 0.2)
    reg = g.engine.MLPRegressor(NIN, hidden=(9,), device=device)
    reg.set_params(rng.standard_normal(reg.get_params().size) * 0.2, out_activation="identity")
    return {"clf": clf, "reg": reg}


def _keys(c):
    uid, iid = _ids(c)
    rng = np.random.default_rng(5)
    users = uid[rng.integers(0, U, 300)]
    ts = rng.integers(0, 45, 300).astype(np.int64)
    items = iid[rng.integers(0, c["N"], 300)]
    items[:3] = [7, iid[0], iid[-1]]                                  # an unknown item id
    return users, items, ts


def _calls(models, eng, c, res, tag):
    users, items, ts = _keys(c)
    nu, nr = c["nu"], c["nr"]
    for mn, m in models.items():
        res["%s.%s.pred" % (tag, mn)] = m.predict_keys(eng, users, items, ts)
        for md, kw in MODES.items():
            for k in (1, 100):
                out = m.recommend_topk(eng, users[:nu], ts[:nu], k, **kw)
                for j, part in enumerate(("rows", "scores", "logits", "count")):
                    res["%s.%s.rec.%s.%d.%s" % (tag, mn, md, k, part)] = out[j]
            r, l = m.rank_items(eng, users[:nr], items[:nr], ts[:nr], **kw)
            res["%s.%s.rank.%s" % (tag, mn, md)], res["%s.%s.rank.%s.logit" % (tag, mn, md)] = r, l


def _worker(rank, port, out_dir, names):
    import torch.distributed as dist
    sr._init(rank, port)
    models = _models(rank)
    for name in names:
        c = CASES[name]
        eng = sr._engine(rank, _sharded(c))
        _setup(eng, name)
        _case_placement(eng, name, rank)
        res = {}
        if c["train"]:                                                # sharded steps queued right before the calls
            rng = np.random.default_rng(3)
            for _ in range(2):
                ur = rng.integers(0, U, 128).astype(np.int32); ir = rng.integers(0, c["N"], 128).astype(np.int32)
                ir[:16] = np.arange(16)                                 # hot rows
                hist = rng.integers(-1, c["N"], (128, S)).astype(np.int32); y = (rng.random(128) > 0.5).astype(np.float32)
                sl = slice(rank * 64, (rank + 1) * 64)
                eng.train_step_idx(ur[sl], ir[sl], hist[sl], y[sl])
            users, items, ts = _keys(c)
            for mn, m in models.items():                                # no sync: the collective calls order themselves
                r, l = m.rank_items(eng, users[:50], items[:50], ts[:50])
                res["live.%s.rank" % mn], res["live.%s.logit" % mn] = r, l
            eng.sync(); dist.barrier()
        _calls(models, eng, c, res, "a")
        if name == "feat_sharded":
            eng.profile(True); eng.profile_reset()
            users, items, ts = _keys(c)
            models["clf"].recommend_topk(eng, users[:260], ts[:260], 10)
            models["clf"].rank_items(eng, users[:5], items[:5], ts[:5])
            prof = eng.profile_dump()
            eng.profile(False)
            for key in ("mlp_rec_prefix", "mlp_rec_layer0", "mlp_rec_topk", "mlp_rec_merge_ranks", "mlp_rec_finish", "mlp_rank_target",
                        "mlp_rank_count"):
                res["prof." + key] = np.array(prof.get(key, (0, 0))[1])
        sr._snapshot(eng, name, res)
        res["emb"] = eng.table_download(g.TABLE_ITEM_EMB, c["N"], D)
        np.savez(os.path.join(out_dir, "%s_%d.npz" % (name, rank)), **res)
        eng.close()
    dist.barrier(); dist.destroy_process_group()


def _load(tmp_path, name, N):
    r0, r1 = np.load(tmp_path / ("%s_0.npz" % name)), np.load(tmp_path / ("%s_1.npz" % name))
    emb = np.array(r0["emb"])
    if N > 1:
        emb[1::2] = r1["emb"][1::2]                                   # each rank's download holds its own rows
    return r0, r1, emb


def _reference(name, emb):
    c = CASES[name]
    ref = g.Engine(_cfg(c))
    _setup(ref, name)
    ref.table_upload(g.TABLE_ITEM_EMB, emb)
    return ref


def test_sharded_mlp_equals_single_gpu(tmp_path):
    sr._needs_two()
    import torch.multiprocessing as mp
    names = list(CASES)
    mp.spawn(_worker, args=(sr._free_port(), str(tmp_path), names), nprocs=WORLD, join=True)
    models = _models(0)
    for name in names:
        c = CASES[name]
        r0, r1, emb = _load(tmp_path, name, c["N"])
        ref = _reference(name, emb)
        want = {}
        _calls(models, ref, c, want, "a")
        for key, w in want.items():
            sr._assert_same(r0[key], r1[key], key + " (rank 0 vs rank 1)")
            sr._assert_same(r0[key], w, key)
        if c["train"]:
            for mn in models:
                sr._assert_same(r0["live.%s.rank" % mn], r1["live.%s.rank" % mn], "live rank")
                users, items, ts = _keys(c)
                r, l = models[mn].rank_items(ref, users[:50], items[:50], ts[:50])
                sr._assert_same(r0["live.%s.rank" % mn], r, "live rank")
                sr._assert_same(r0["live.%s.logit" % mn], l, "live logit")
        if name == "feat_sharded":                                    # 260 users: two list all-gathers, 260 prefixes
            for res in (r0, r1):
                assert 260 < int(res["prof.mlp_rec_prefix"]) <= 265               # and one per rank pass
                assert int(res["prof.mlp_rec_merge_ranks"]) == 2
                assert int(res["prof.mlp_rec_layer0"]) > 0 and int(res["prof.mlp_rank_count"]) > 0
        ref.close()


# ---- caches that differ, disagreements and refusals
NAME = "feat_sharded"


def _misc_worker(rank, port, out_dir):
    import torch.distributed as dist
    sr._init(rank, port)
    c = CASES[NAME]
    models = _models(rank)
    users, items, ts = _keys(c)
    res = {}
    eng = sr._engine(rank, _sharded(c))
    _setup(eng, NAME, salt=rank)                                       # a different ubcache on each rank
    _case_placement(eng, NAME, rank)
    clf = models["clf"]
    for md, kw in MODES.items():
        out = clf.recommend_topk(eng, users[:40], ts[:40], 50, **kw)
        res["div.rec.%s.rows" % md], res["div.rec.%s.logits" % md] = out[0], out[2]
        r, l = clf.rank_items(eng, users[:40], items[:40], ts[:40], **kw)
        res["div.rank.%s" % md], res["div.rank.%s.logit" % md] = r, l
    res["code.ts"] = np.array(sr._err(lambda: clf.recommend_topk(eng, users[:10], ts[:10] + rank, 5))[0])
    res["code.ts_rank"] = np.array(sr._err(lambda: clf.rank_items(eng, users[:10], items[:10], ts[:10] + rank))[0])
    res["code.fit"] = np.array(sr._err(lambda: clf.fit_keys(eng, users[:10], items[:10], ts[:10], np.ones(10, np.float32)))[0])
    res["fit_msg"] = np.array(sr._err(lambda: clf.fit_keys(eng, users[:10], items[:10], ts[:10], np.ones(10, np.float32)))[1])
    cls = g.engine.MLPClassifier(NIN, hidden=(5,), device=rank)
    cls.set_params(np.zeros(NIN * 5 + 5 + 3 * 6), classes=[1.0, 2.0, 3.0])
    res["code.classes"] = np.array(sr._err(lambda: cls.recommend_topk(eng, users[:10], ts[:10], 5))[0])
    eng.close()
    # a user missing from rank 1's id map
    uid, _ = _ids(c)
    eng = sr._engine(rank, _sharded(c))
    _setup(eng, NAME, users=uid if rank == 0 else uid[uid != users[3]])
    res["code.unknown"] = np.array(sr._err(lambda: clf.recommend_topk(eng, users[:10], ts[:10], 5))[0])
    res["code.unknown_rank"] = np.array(sr._err(lambda: clf.rank_items(eng, users[:10], items[:10], ts[:10]))[0])
    eng.close()
    # id maps holding the same ids at other rows on rank 1: every id is known everywhere, the resolved rows differ
    _, iid = _ids(c)
    eng = sr._engine(rank, _sharded(c))
    _setup(eng, NAME, items=iid if rank == 0 else iid[::-1].copy())
    res["code.items_permuted"] = np.array(sr._err(lambda: clf.rank_items(eng, users[:10], items[:10], ts[:10]))[0])
    eng.close()
    eng = sr._engine(rank, _sharded(c))
    _setup(eng, NAME, users=uid if rank == 0 else uid[::-1].copy())
    res["code.users_permuted"] = np.array(sr._err(lambda: clf.recommend_topk(eng, users[:10], ts[:10], 5))[0])
    res["code.users_permuted_rank"] = np.array(sr._err(lambda: clf.rank_items(eng, users[:10], items[:10], ts[:10]))[0])
    eng.close()
    # ITEM_EMB replicated (small) beside a sharded ITEM_FEAT (3 000 000 x 3 floats, 48 MB padded) under the by-size placement
    eng = sr._engine(rank, _sharded(c, policy=0))
    uf, _, emb = _tables(NAME)
    big = np.random.default_rng(2).standard_normal((3_000_000, CF)).astype(np.float32)
    eng.table_upload(g.TABLE_USER_FEAT, uf)
    eng.table_upload(g.TABLE_ITEM_EMB, emb)
    eng.table_upload(g.TABLE_ITEM_FEAT, big)
    _assert_placement(eng, rank, [(g.TABLE_ITEM_EMB, emb, "replicated"), (g.TABLE_ITEM_FEAT, big, "sharded")])
    eng.idmap_build(0, uid); eng.idmap_build(1, iid)
    res["code.mixed"] = np.array(sr._err(lambda: clf.predict_keys(eng, users[:10], items[:10], ts[:10]))[0])
    eng.close()
    np.savez(os.path.join(out_dir, "misc_%d.npz" % rank), **res)
    dist.barrier(); dist.destroy_process_group()


def test_sharded_mlp_divergent_caches_and_refusals(tmp_path):
    sr._needs_two()
    import torch.multiprocessing as mp
    mp.spawn(_misc_worker, args=(sr._free_port(), str(tmp_path)), nprocs=WORLD, join=True)
    r0, r1 = np.load(tmp_path / "misc_0.npz"), np.load(tmp_path / "misc_1.npz")
    for key in r0.files:
        if key.startswith("div."):
            sr._assert_same(r0[key], r1[key], key)
    # without exclusion or with the window, the windows are rank 0's: a single GPU with rank 0's cache
    c = CASES[NAME]
    ref = _reference(NAME, _tables(NAME)[2])
    clf = _models(0)["clf"]
    users, items, ts = _keys(c)
    for md in ("none", "window"):
        out = clf.recommend_topk(ref, users[:40], ts[:40], 50, **MODES[md])
        sr._assert_same(r0["div.rec.%s.rows" % md], out[0], md)
        sr._assert_same(r0["div.rec.%s.logits" % md], out[2], md)
        r, l = clf.rank_items(ref, users[:40], items[:40], ts[:40], **MODES[md])
        sr._assert_same(r0["div.rank.%s" % md], r, md)
    ref.close()
    for res in (r0, r1):
        assert int(res["code.ts"]) == g.EINVAL and int(res["code.ts_rank"]) == g.EINVAL
        assert int(res["code.unknown"]) == g.ENOTFOUND and int(res["code.unknown_rank"]) == g.ENOTFOUND
        assert int(res["code.items_permuted"]) == g.EINVAL
        assert int(res["code.users_permuted"]) == g.EINVAL and int(res["code.users_permuted_rank"]) == g.EINVAL
        assert int(res["code.fit"]) == g.ESTATE and "ctr_mlp_set_params" in str(res["fit_msg"])
        assert int(res["code.classes"]) == g.ESTATE
        assert int(res["code.mixed"]) == g.ESTATE
