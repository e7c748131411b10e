"""Live id maps and tables on a multi-GPU handle (needs >= 2 GPUs; runs at W = 2, 4 and 8, as many as the box has), one
process per rank: ctr_idmap_insert and ctr_table_write_rows are collective, ctr_idmap_download is local.  A one-GPU twin
performs the same calls on the ranks' arguments concatenated in rank order, and every rank must hold what it holds:

  * the id maps (idmap_download on every rank, the rows each rank's insert returned) and every table (table_download of
    each shard, USER_FEAT replicated), after inserts with ids new on several ranks, already present, repeated, and an
    empty rank;
  * a write that does not grow the tables and touches ITEM_EMB's hot rows while their replica is live (a collective call
    published the shards just before), with a rank that writes nothing (an empty array, and a width-less empty list);
  * a write that grows ITEM_EMB, ITEM_FEAT (row-sharded) and USER_FEAT; recommend_topk, rank_items, batch_predict_keys and
    the float64 MLP's predict_keys on the grown store, bit for bit, after each write;
  * a sharded ctr_train_keys step whose keys touch the new rows and the hot rows, then a growing write while the trained
    replica is live: costs, weights and tables at the suite's training bars (the twin trains the global batch under
    CTR_TABLE_SGD_DETERMINISTIC);
  * refusals (a row written by two ranks, maps that differ, INT64_MIN on one rank, a width mismatch on one rank): the
    same code on every rank, and the id maps and tables unchanged;
  * the profile keys of the collective calls."""
import os

import numpy as np
import pytest
import torch

import go_ctr_b200 as g
from tests import test_gpu_shard_rank as sr
from tests.util import assert_mostly_close

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

USER, ITEM = g.IDMAP_USER, g.IDMAP_ITEM
UP, S, D, CF = 4, 5, 16, 3
U0, I0 = 40, 300
NIN = UP + S * D + D + CF
B = 64                     # keys per rank in the training step
HOT = 32
WIDTH = {g.TABLE_USER_FEAT: UP, g.TABLE_ITEM_FEAT: CF, g.TABLE_ITEM_EMB: D}


def _cfg(**kw):
    return g.engine.default_config(g.MODEL_DIN_COS, uP=UP, S=S, D=D, cF=CF, pred_batch=128, table_opt=g.TABLE_SGD_DETERMINISTIC,
                                   table_lr=0.5, dropout0=0.0, dropout1=0.0, seed=5, **kw)


def _base():
    rng = np.random.default_rng(1)
    return (1000 + np.arange(U0, dtype=np.int64), 50_000 + 3 * np.arange(I0, dtype=np.int64),
            rng.standard_normal((U0, UP)).astype(np.float32), rng.standard_normal((I0, CF)).astype(np.float32),
            rng.standard_normal((I0, D)).astype(np.float32))


def _setup(eng):
    uid, iid, uf, itf, emb = _base()
    eng.table_upload(g.TABLE_USER_FEAT, uf); eng.table_upload(g.TABLE_ITEM_FEAT, itf); eng.table_upload(g.TABLE_ITEM_EMB, emb)
    eng.idmap_build(USER, uid); eng.idmap_build(ITEM, iid)


def _inserts(W):
    """per-rank ids: each rank's own new ids, ids new on several ranks, present ids, repeats; rank 1 passes nothing"""
    uid, iid, *_ = _base()
    rng = np.random.default_rng(7)
    shared_u, shared_i = 9_000_000 + np.arange(5), 8_000_000 + np.arange(40)
    us, its = [], []
    for j in range(W):
        own_u = 7_000_000 + 100 * j + np.arange(3 + j)
        own_i = 6_000_000 + 10_000 * j + np.arange(200 * (j + 1))
        u = np.concatenate([own_u, shared_u[j % 3:], uid[:2], own_u[:1]]).astype(np.int64)
        i = np.concatenate([shared_i[j:], own_i, iid[rng.integers(0, I0, 5)], own_i[:7]]).astype(np.int64)
        rng.shuffle(i)
        us.append(u if j != 1 else np.zeros(0, np.int64)); its.append(i if j != 1 else np.zeros(0, np.int64))
    return us, its


def _split(rows, W, seed, which, empty_rank=None):
    """rows [k] and their data, split across the ranks (row r by rank r % W; empty_rank's share goes to rank 0)"""
    data = np.random.default_rng(seed).standard_normal((rows.size, WIDTH[which])).astype(np.float32)
    owner = rows % W
    if empty_rank is not None:
        owner[owner == empty_rank] = 0
    return [(rows[owner == j].astype(np.int32), data[owner == j]) for j in range(W)]


def _writes_a(W):
    """no growth; ITEM_EMB's hot rows among the rows; rank 1 writes nothing"""
    emb_rows = np.array([0, 1, 2, 7, 30, 31, 33, 100, 150, I0 - 1])
    return {g.TABLE_ITEM_EMB: _split(emb_rows, W, 20, g.TABLE_ITEM_EMB, 1),
            g.TABLE_ITEM_FEAT: _split(np.array([3, 4, 5, 200]), W, 21, g.TABLE_ITEM_FEAT, 1),
            g.TABLE_USER_FEAT: _split(np.array([1, 2, 39]), W, 22, g.TABLE_USER_FEAT, 1)}


def _writes_b(W, n_users, n_items):
    """the new rows, a few old ones (hot rows among them), and rows past the id maps (ITEM_EMB 17 past the end, ITEM_FEAT 3
    past: growth with a zero gap)"""
    out = {}
    for which, old, n in ((g.TABLE_USER_FEAT, U0, n_users), (g.TABLE_ITEM_FEAT, I0, n_items + 3), (g.TABLE_ITEM_EMB, I0, n_items + 17)):
        gap = {g.TABLE_ITEM_FEAT: 3, g.TABLE_ITEM_EMB: 17}.get(which, 0)
        rows = np.concatenate([np.arange(old, n - gap), [n - 1], [0, 5, 40, 61]])
        out[which] = _split(rows, W, 30 + which, which)
    return out


def _writes_c(W, n_items):
    """after training, with the trained replica live: ITEM_FEAT grows first (its republish re-pulls ITEM_EMB's hot rows),
    then ITEM_EMB, a hot row among its rows"""
    return {g.TABLE_ITEM_FEAT: _split(np.array([n_items + 5, 9]), W, 40, g.TABLE_ITEM_FEAT),
            g.TABLE_ITEM_EMB: _split(np.array([n_items + 20, 2, I0 + 1]), W, 41, g.TABLE_ITEM_EMB)}


def _pick(per, rank):
    """rank's share of a per-rank argument list; rank None: the concatenation in rank order (the twin's argument)"""
    if rank is not None:
        return per[rank]
    if isinstance(per[0], tuple):
        return tuple(np.concatenate([p[k] for p in per]) for k in range(len(per[0])))
    return np.concatenate(per)


def _write(eng, per_table, rank):
    for which, per in per_table.items():
        rows, data = _pick(per, rank)
        if rows.size == 0 and which == g.TABLE_USER_FEAT:
            data = []                                       # an empty list: the width comes from the table
        eng.table_write_rows(which, rows, data)


def _train_keys(W, n_users, n_items):
    """every rank's B keys: users old and new, items new and hot"""
    uid_new = np.arange(U0, n_users); item_new = np.arange(I0, n_items)
    out = []
    for j in range(W):
        rng = np.random.default_rng(60 + j)
        u = np.concatenate([rng.integers(0, U0, B // 2), rng.choice(uid_new, B - B // 2)])
        i = np.concatenate([rng.integers(0, HOT, B // 4), rng.choice(item_new, B - B // 4)])
        out.append((u, i, rng.integers(1, 50, B).astype(np.int64), (rng.random(B) > 0.5).astype(np.float32)))
    return out


def _serve(eng, res, tag, n_users, n_items):
    rng = np.random.default_rng(11)
    uid, iid = eng.idmap_download(USER), eng.idmap_download(ITEM)
    users = uid[rng.integers(0, n_users, 120)]; items = iid[rng.integers(0, n_items, 120)]; ts = rng.integers(0, 50, 120).astype(np.int64)
    items[:3] = iid[-3:]
    items[3:6] = iid[:3]                                                          # hot rows
    res[tag + ".pred"] = eng.batch_predict_keys(users, items, ts)
    urows = eng.idmap_lookup(USER, users[:30]).astype(np.int32); hist = np.full((30, S), -1, np.int32)
    hist[:, :2] = eng.idmap_lookup(ITEM, items[30:90]).reshape(30, 2)
    for j, part in enumerate(("rows", "scores", "logits", "count")):
        res[tag + ".rec." + part] = eng.recommend_topk(urows, hist, 50)[j]
    res[tag + ".rank"], res[tag + ".rank.logit"] = eng.rank_items(urows, hist, eng.idmap_lookup(ITEM, items[:30]).astype(np.int32))
    clf = g.engine.MLPClassifier(NIN, hidden=(9,), device=torch.cuda.current_device())
    clf.set_params(np.random.default_rng(3).standard_normal(clf.get_params().size) * 0.2)
    res[tag + ".mlp"] = clf.predict_keys(eng, users, items, ts)


def _download_all(eng, shapes, tag=""):
    return {tag + "tab%d" % which: eng.table_download(which, *shape) for which, shape in shapes.items()}


def _shapes(n_users, n_items, grown_c=False):
    return {g.TABLE_USER_FEAT: (n_users, UP), g.TABLE_ITEM_FEAT: (n_items + (6 if grown_c else 3), CF),
            g.TABLE_ITEM_EMB: (n_items + (21 if grown_c else 17), D)}


def _script(eng, W, rank, res):
    """the calls of one rank (rank None: the twin, on the concatenated arguments); results into res"""
    us, its = _inserts(W)
    eng.profile(True); eng.profile_reset()
    res["urows"] = eng.idmap_insert(USER, _pick(us, rank)); res["irows"] = eng.idmap_insert(ITEM, _pick(its, rank))
    res["prof.insert"] = np.array(sorted(eng.profile_dump()))
    n_users, n_items = eng.idmap_download(USER).size, eng.idmap_download(ITEM).size
    sizes = _shapes(n_users, n_items)
    start = dict(sizes); start[g.TABLE_USER_FEAT] = (U0, UP); start[g.TABLE_ITEM_FEAT] = (I0, CF); start[g.TABLE_ITEM_EMB] = (I0, D)
    _serve(eng, res, "s0", n_users, n_items)                 # publishes the shards: the hot-row replica is live
    eng.profile_reset()
    _write(eng, _writes_a(W), rank)
    res["prof.write_a"] = np.array(sorted(eng.profile_dump()))
    res.update(_download_all(eng, start, "a."))
    _serve(eng, res, "s1", n_users, n_items)
    eng.profile_reset()
    _write(eng, _writes_b(W, n_users, n_items), rank)
    res["prof.write_b"] = np.array(sorted(eng.profile_dump()))
    eng.profile(False)
    res["uids"], res["iids"] = eng.idmap_download(USER), eng.idmap_download(ITEM)
    res.update(_download_all(eng, sizes, "b."))
    _serve(eng, res, "s2", n_users, n_items)
    uid, iid = res["uids"], res["iids"]
    ku, ki, kt, ky = _pick(_train_keys(W, n_users, n_items), rank)
    _, cost, used = eng.train_keys(uid[ku], iid[ki], kt, ky, epochs=1)
    res["cost"], res["used"] = np.array([cost], np.float32), np.array(used)
    _write(eng, _writes_c(W, n_items), rank)
    res.update(_download_all(eng, _shapes(n_users, n_items, True), "c."))
    for i, w in enumerate(eng.get_weights()):
        res["w%d" % i] = w
    return n_users, n_items


def _worker(rank, W, port, out_dir):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=W)
    torch.cuda.set_device(rank)

    def cfg(r):
        x = _cfg(batch=B, device=r, rank=r, world=W)
        x.reserved[1] = 1; x.reserved[0] = HOT               # both ITEM tables sharded, HOT replicated rows
        return x
    eng = sr._engine(rank, cfg)
    _setup(eng)
    res = {}
    n_users, n_items = _script(eng, W, rank, res)
    # refusals: the same code everywhere, the id maps and the tables unchanged
    shapes = _shapes(n_users, n_items, True)
    state = lambda: [eng.idmap_download(USER), eng.idmap_download(ITEM)] + list(_download_all(eng, shapes).values())
    same = lambda a, b: all(x.tobytes() == y.tobytes() for x, y in zip(a, b))
    before = state()
    w = lambda which, rows, data: sr._err(lambda: eng.table_write_rows(which, np.array(rows, np.int32), data))[0]
    res["code.dup"] = np.array(w(g.TABLE_ITEM_EMB, [3], np.ones((1, D), np.float32)))          # row 3 from every rank
    res["code.width"] = np.array(w(g.TABLE_ITEM_FEAT, [rank], np.ones((1, CF + (rank == W - 1)), np.float32)))
    bad = np.array([123_456_789, -2**63] if rank == W - 1 else [123_456_789], np.int64)
    res["code.min"] = np.array(sr._err(lambda: eng.idmap_insert(ITEM, bad))[0])
    res["unchanged"] = np.array(same(before, state()))
    uid = eng.idmap_download(USER)
    eng.idmap_build(USER, uid if rank == 0 else uid[::-1].copy())         # maps that differ on every rank but rank 0
    before = state()
    res["code.maps"] = np.array(sr._err(lambda: eng.idmap_insert(USER, np.array([5_555_555], np.int64)))[0])
    res["maps_unchanged"] = np.array(same(before, state()))
    np.savez(os.path.join(out_dir, "live_%d_%d.npz" % (W, rank)), **res)
    eng.close()
    dist.barrier(); dist.destroy_process_group()


def _own_rows(tab, W, r):
    exp = tab.copy()
    exp[np.arange(exp.shape[0]) % W != r] = 0
    return exp


@pytest.mark.parametrize("W", [2, 4, 8])
def test_sharded_live_tables_equal_a_single_gpu_twin(tmp_path, W):
    if W > torch.cuda.device_count():
        pytest.skip("needs %d GPUs" % W)
    import torch.multiprocessing as mp
    mp.spawn(_worker, args=(W, sr._free_port(), str(tmp_path)), nprocs=W, join=True)
    rs = [np.load(tmp_path / ("live_%d_%d.npz" % (W, r))) for r in range(W)]
    twin = g.Engine(_cfg(batch=B * W))
    _setup(twin)
    want = {}
    _script(twin, W, None, want)
    us, its = _inserts(W)
    off_u = np.cumsum([0] + [a.size for a in us]); off_i = np.cumsum([0] + [a.size for a in its])
    exact = ["uids", "iids"] + ["%s.%s" % (s, k) for s in ("s0", "s1", "s2") for k in
                                ("pred", "rec.rows", "rec.scores", "rec.logits", "rec.count", "rank", "rank.logit", "mlp")]
    for r, res in enumerate(rs):
        sr._assert_same(res["urows"], want["urows"][off_u[r]:off_u[r + 1]], "urows")
        sr._assert_same(res["irows"], want["irows"][off_i[r]:off_i[r + 1]], "irows")
        for key in exact:
            sr._assert_same(res[key], want[key], "%s (rank %d)" % (key, r))
        for stage in ("a.", "b.", "c."):
            sr._assert_same(res[stage + "tab%d" % g.TABLE_USER_FEAT], want[stage + "tab%d" % g.TABLE_USER_FEAT], stage + "USER_FEAT")
            sr._assert_same(res[stage + "tab%d" % g.TABLE_ITEM_FEAT], _own_rows(want[stage + "tab%d" % g.TABLE_ITEM_FEAT], W, r), stage + "ITEM_FEAT")
        for stage in ("a.", "b."):                                                 # before training: bit for bit
            sr._assert_same(res[stage + "tab%d" % g.TABLE_ITEM_EMB], _own_rows(want[stage + "tab%d" % g.TABLE_ITEM_EMB], W, r), stage + "ITEM_EMB")
        assert {"idmap_digest", "idmap_gather_ranks", "idmap_merge_ranks"} <= set(res["prof.insert"].tolist())
        assert {"table_write_ranks", "table_write_check", "table_write_shard"} <= set(res["prof.write_a"].tolist())
        assert not {"table_shard_grow", "table_grow"} & set(res["prof.write_a"].tolist())
        assert {"table_write_ranks", "table_write_check", "table_write_shard", "table_shard_grow", "table_grow"} <= set(res["prof.write_b"].tolist())
        assert int(res["code.dup"]) == g.EINVAL and int(res["code.width"]) == g.EINVAL and int(res["code.min"]) == g.EINVAL
        assert bool(res["unchanged"]) and int(res["code.maps"]) == g.EINVAL and bool(res["maps_unchanged"])
        assert int(res["used"]) == B
        assert res["cost"].tobytes() == rs[0]["cost"].tobytes() and res["w0"].tobytes() == rs[0]["w0"].tobytes()
    # the training step and the write after it: the suite's training bars
    np.testing.assert_allclose(rs[0]["cost"], want["cost"], rtol=2e-4, atol=1e-6)
    for i in range(4):
        assert_mostly_close(rs[0]["w%d" % i], want["w%d" % i], 2e-3, 2e-4, 0.995, "weights %d" % i)
    emb = np.zeros_like(want["c.tab%d" % g.TABLE_ITEM_EMB])
    for r, res in enumerate(rs):
        emb[r::W] = res["c.tab%d" % g.TABLE_ITEM_EMB][r::W]
    before = want["b.tab%d" % g.TABLE_ITEM_EMB]
    assert np.abs(want["c.tab%d" % g.TABLE_ITEM_EMB][:before.shape[0]] - before).max() > 1e-5           # the step moved rows
    np.testing.assert_allclose(emb, want["c.tab%d" % g.TABLE_ITEM_EMB], rtol=2e-3, atol=2e-5)
    twin.close()
