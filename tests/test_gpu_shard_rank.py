"""ctr_rank_items on a row-sharded ITEM_EMB (needs >= 2 GPUs): the call is collective — each rank counts the items of its
own shard against the targets, whose logits come from their owners, and the ranks' counts are summed.  Both ranks must
return the same ranks and logits, bit for bit, as a single-GPU handle holding the assembled table and the same weights.
Cases cover the placements (sharded with and without replicated hot rows, the automatic placement of a large filled
table beside a small replicated ITEM_FEAT, ITEM_FEAT shorter than ITEM_EMB, an empty shard), a call queued right
behind sharded train steps without a host sync, the invariant with the sharded recommendation lists, serving.Evaluate
on both ranks, argument disagreement and a verdict that fails on one rank, the replicated placement (served locally)
and the profile keys of a sharded pass."""
import os
import socket

import numpy as np
import pytest
import torch

import go_ctr_b200 as g
from go_ctr_b200 import serving

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

WORLD = 2
U = 50

# (model, dims, ITEM_EMB rows, ITEM_FEAT rows, placement policy (reserved[1]), hot rows (reserved[0]), pred_batch, filled)
CASES = {
    "din_cos_d16": dict(model=g.MODEL_DIN_COS, uP=8, S=50, D=16, cF=5, N=1001, NF=700, policy=1, hot=-1, pb=128, fill=False),
    "youtube_d64_hot": dict(model=g.MODEL_YOUTUBE, uP=4, S=1, D=64, cF=3, N=777, NF=777, policy=1, hot=64, pb=96, fill=False),
    "din_euc_auto": dict(model=g.MODEL_DIN_EUC, uP=4, S=50, D=64, cF=7, N=140_000, NF=90_000, policy=0, hot=0, pb=8192, fill=True),
    "tiny": dict(model=g.MODEL_DIN_COS, uP=4, S=1, D=16, cF=0, N=1, NF=0, policy=1, hot=-1, pb=64, fill=False),
}


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _needs_two():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")


def _tables(name):
    c = CASES[name]
    rng = np.random.default_rng(sum(name.encode()) + 1)          # the same tables in every process
    uf = rng.standard_normal((U, c["uP"])).astype(np.float32)
    itf = rng.standard_normal((c["NF"], c["cF"])).astype(np.float32) if c["cF"] else None
    emb = None if c["fill"] else rng.standard_normal((c["N"], c["D"])).astype(np.float32)
    if emb is not None and c["N"] > 10:
        emb[10] = emb[4]                                         # equal logits on the two ranks: ranked by row
    return uf, itf, emb


def _cfg(name, **kw):
    c = CASES[name]
    return g.engine.default_config(c["model"], uP=c["uP"], S=c["S"], D=c["D"], cF=c["cF"], batch=64, pred_batch=c["pb"],
                                   table_opt=g.TABLE_SGD, table_lr=0.5, dropout0=0.0, dropout1=0.0, seed=5, **kw)


def _sharded_cfg(name, policy=None, hot=None):
    c = CASES[name]

    def cfg(r):
        x = _cfg(name, device=r, rank=r, world=WORLD)
        x.reserved[1] = c["policy"] if policy is None else policy
        x.reserved[0] = c["hot"] if hot is None else hot
        return x
    return cfg


def _keys(name):
    """The rank_items calls of a case: (key, kwargs), the same list for the ranks and for the reference handle."""
    c = CASES[name]
    N, S = c["N"], c["S"]
    rng = np.random.default_rng(2000 + len(name))
    out = []
    if N == 1:
        out.append(("one", dict(user_rows=[0, 1, 0], hist=[[0], [-1], [-1]], item_rows=[0, 0, 1], exclude_history=True)))
        out.append(("keep", dict(user_rows=[0], hist=[[0]], item_rows=[0], exclude_history=False)))
        return out
    users = rng.integers(0, U, 6).astype(np.int32)
    users[1] = U + 5                                             # a user row outside USER_FEAT
    hist = rng.integers(-1, N + 40, (6, S)).astype(np.int32)     # both ranks' rows, -1, rows past the table
    hist[0, :min(S, 4)] = np.arange(min(S, 4))                   # hot rows
    hist[2] = -1
    n = 60
    ku = rng.integers(0, 6, n)
    items = rng.integers(0, N, n).astype(np.int32)
    items[:10] = [0, 1, 4, 10, N - 1, N - 2, -1, N, N + 7, 63]    # both ranks, tied rows, outside the table, a hot row
    items[10] = items[11] = 500 % N                              # a target named twice
    ku[:12] = 0
    items[12] = hist[0, 0]; ku[12] = 0                           # a row of its own window
    kw = dict(user_rows=users[ku], hist=hist[ku], item_rows=items)
    out.append(("excl", dict(kw, exclude_history=True)))
    out.append(("keep", dict(kw, exclude_history=False)))
    out.append(("m1", dict(user_rows=users[3:4], hist=hist[3:4], item_rows=items[20:21], exclude_history=True)))
    big = rng.integers(-2, N + 2, 1100).astype(np.int32)         # one (user, window) of 1100 targets: two passes
    out.append(("m1100", dict(user_rows=np.full(big.size, users[4], np.int32), hist=np.tile(hist[4], (big.size, 1)),
                              item_rows=big, exclude_history=True)))
    return out


def _profiled(name):
    """the call whose profile keys are checked: one (user, window), one pass"""
    keys = _keys(name)
    return keys[-1][1] if CASES[name]["N"] == 1 else keys[2][1]


def _run(eng, keys):
    res = {}
    for key, kw in keys:
        r, l = eng.rank_items(**kw)
        res[key + ".rank"], res[key + ".logit"] = r, l
    return res


def _engine(rank, cfg_fn):
    import torch.distributed as dist
    eng = g.Engine(cfg_fn(rank))
    ids = [eng.comm_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(ids, src=0)
    eng.comm_init(ids[0])
    return eng


def _upload(eng, name):
    c = CASES[name]
    uf, itf, emb = _tables(name)
    eng.table_upload(g.TABLE_USER_FEAT, uf)
    if itf is not None:
        eng.table_upload(g.TABLE_ITEM_FEAT, itf)
    if c["fill"]:
        eng.table_fill(g.TABLE_ITEM_EMB, c["N"], c["D"], seed=9, dist=1, scale=1.0)
    else:
        eng.table_upload(g.TABLE_ITEM_EMB, emb)


def _snapshot(eng, name, res):
    c = CASES[name]
    res["emb"] = eng.table_download(g.TABLE_ITEM_EMB, c["N"], c["D"])
    for i, w in enumerate(eng.get_weights()):
        res["w%d" % i] = w


def _init(rank, port):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=WORLD)
    torch.cuda.set_device(rank)


def _err(fn):
    try:
        fn()
    except g.CtrError as e:
        return e.code, str(e)
    return 0, ""


def _reference(name, emb, weights):
    uf, itf, _ = _tables(name)
    ref = g.Engine(_cfg(name))
    ref.table_upload(g.TABLE_USER_FEAT, uf)
    if itf is not None:
        ref.table_upload(g.TABLE_ITEM_FEAT, itf)
    ref.table_upload(g.TABLE_ITEM_EMB, emb)
    ref.set_weights(*weights)
    return ref


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view({8: np.int64, 4: np.int32}[a.dtype.itemsize]) if a.dtype.kind == "f" else a


def _assert_same(got, want, key):
    assert got.shape == want.shape, key
    assert np.array_equal(_bits(got), _bits(want)), "%s differs at %s" % (key, np.argwhere(_bits(got) != _bits(want))[:5].tolist())


def _load(tmp_path, tag, N):
    r0, r1 = np.load(tmp_path / ("%s_0.npz" % tag)), np.load(tmp_path / ("%s_1.npz" % tag))
    emb = np.array(r0["emb"])
    if N > 1:
        emb[1::2] = r1["emb"][1::2]                              # each rank's download holds its own rows
    return r0, r1, emb


def _check(tmp_path, tag, name, keys):
    r0, r1, emb = _load(tmp_path, tag, CASES[name]["N"])
    ref = _reference(name, emb, [r0["w%d" % i] for i in range(4)])
    want = _run(ref, keys)
    for key, w in want.items():
        _assert_same(r0[key], r1[key], key + " (rank 0 vs rank 1)")
        _assert_same(r0[key], w, key)
    assert any((want[k] > 0).any() for k in want if k.endswith(".rank"))
    return r0, want


# ---- every case: ranks, the lists' invariant and the profile keys
def _case_worker(rank, port, out_dir, names):
    import torch.distributed as dist
    _init(rank, port)
    for name in names:
        c = CASES[name]
        eng = _engine(rank, _sharded_cfg(name))
        _upload(eng, name)
        keys = _keys(name)
        res = _run(eng, keys)
        # the sharded lists: rank r <= k means the target at position r - 1 of recommend_topk(k), for k = 1024 and k = r
        kw = dict(keys[0][1])
        rows, _, logits, cnt = eng.recommend_topk(kw["user_rows"], kw["hist"], 1024, exclude_history=kw["exclude_history"])
        res["list.rows"], res["list.logits"], res["list.count"] = rows, logits, cnt
        for j, r in enumerate(res[keys[0][0] + ".rank"]):
            if 0 < r <= 1024:
                rr, _, ll, nn = eng.recommend_topk(kw["user_rows"][j:j + 1], np.asarray(kw["hist"])[j:j + 1], int(r),
                                                   exclude_history=kw["exclude_history"])
                res["at_rank.%d" % j] = np.array([rr[0, r - 1], nn[0]], np.int64)
        # profile keys of one sharded pass: this rank's target chunks and its local chunks
        eng.profile(True); eng.profile_reset()
        eng.rank_items(**_profiled(name))
        prof = eng.profile_dump()
        eng.profile(False)
        res["prof.target"] = np.array(prof.get("rank_target", (0, 0))[1]); res["prof.count"] = np.array(prof.get("rank_count", (0, 0))[1])
        res["prof.rec"] = np.array(int(bool({"rec_topk", "rec_merge", "rec_finish"} & set(prof))))
        _snapshot(eng, name, res)
        np.savez(os.path.join(out_dir, "%s_%d.npz" % (name, rank)), **res)
        eng.close()
    dist.barrier(); dist.destroy_process_group()


def test_sharded_rank_items_equal_single_gpu(tmp_path):
    _needs_two()
    import torch.multiprocessing as mp
    names = list(CASES)
    mp.spawn(_case_worker, args=(_free_port(), str(tmp_path), names), nprocs=WORLD, join=True)
    for name in names:
        c = CASES[name]
        keys = _keys(name)
        r0, want = _check(tmp_path, name, name, keys)
        k0 = keys[0][0]
        rows, cnt = r0["list.rows"], r0["list.count"]
        items = np.asarray(keys[0][1]["item_rows"])
        for j, (t, r) in enumerate(zip(items, r0[k0 + ".rank"])):
            if 0 < r <= 1024:
                assert rows[j, r - 1] == t and r0["list.logits"][j, r - 1].tobytes() == r0[k0 + ".logit"][j].tobytes()
                assert r0["at_rank.%d" % j][0] == t and r0["at_rank.%d" % j][1] == r
            else:
                assert t not in rows[j, :cnt[j]].tolist()
        # one pass per rank: the target chunks this rank owns + the sort; its local chunks + the finish
        Bc = c["pb"]
        kw = _profiled(name)
        for rk, res in ((0, r0), (1, np.load(tmp_path / ("%s_1.npz" % name)))):
            local = len(range(rk, c["N"], WORLD))
            owned = {(int(t) // WORLD) // Bc for t in kw["item_rows"] if 0 <= t < c["N"] and t % WORLD == rk}
            npass = len({(int(u), tuple(np.atleast_1d(h))) for u, h in zip(kw["user_rows"], np.asarray(kw["hist"]))})
            assert int(res["prof.target"]) == npass * (len(owned) + 1), (name, rk)
            assert int(res["prof.count"]) == npass * ((local + Bc - 1) // Bc + 1), (name, rk)
            assert int(res["prof.rec"]) == 0


# ---- a table trained right before the call, with no host sync in between
LIVE = "din_cos_d16"


def _live_worker(rank, port, out_dir):
    import torch.distributed as dist
    _init(rank, port)
    c = CASES[LIVE]
    eng = _engine(rank, _sharded_cfg(LIVE, hot=64))
    _upload(eng, LIVE)
    rng = np.random.default_rng(31)
    for step in range(3):
        ur = rng.integers(0, U, 128).astype(np.int32); ir = rng.integers(0, c["N"], 128).astype(np.int32)
        ir[:8] = np.arange(8)
        hist = rng.integers(-1, c["N"], (128, c["S"])).astype(np.int32); y = (rng.random(128) > 0.5).astype(np.float32)
        sl = slice(rank * 64, (rank + 1) * 64)
        if step < 2:
            eng.train_step_idx(ur[sl], ir[sl], hist[sl], y[sl])
        else:
            d = "cuda:%d" % rank
            t = [torch.from_numpy(np.ascontiguousarray(a[sl])).to(d) for a in (ur, ir, hist, y)]
            torch.cuda.synchronize(d)
            eng.train_step_idx_dev(t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), t[3].data_ptr(), 64)   # asynchronous
    res = _run(eng, _keys(LIVE)[:1])                             # queued right behind it
    _snapshot(eng, LIVE, res)
    np.savez(os.path.join(out_dir, "live_%d.npz" % rank), **res)
    eng.close()
    dist.barrier(); dist.destroy_process_group()


def test_sharded_rank_items_see_the_table_trained_just_before(tmp_path):
    _needs_two()
    import torch.multiprocessing as mp
    mp.spawn(_live_worker, args=(_free_port(), str(tmp_path)), nprocs=WORLD, join=True)
    _, _, emb = _load(tmp_path, "live", CASES[LIVE]["N"])
    _, _, emb0 = _tables(LIVE)
    assert np.abs(emb[:64] - emb0[:64]).max() > 1e-6 and np.abs(emb[64:] - emb0[64:]).max() > 1e-6
    _check(tmp_path, "live", LIVE, _keys(LIVE)[:1])


# ---- serving.Evaluate, argument agreement, a one-rank verdict, the replicated placement
def _serving_setup(eng, name):
    c = CASES[name]
    rng = np.random.default_rng(44)
    uid = rng.choice(10_000_000, U, replace=False).astype(np.int64) + 1
    iid = rng.choice(10_000_000, c["N"], replace=False).astype(np.int64) + 1
    serving.load_id_maps(eng, uid, iid)
    lens = rng.integers(0, 15, U); off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    ts = np.concatenate([np.sort(rng.integers(1, 1000, n))[::-1] for n in lens]).astype(np.int64)
    eng.ubcache_upload(off, ts, rng.integers(0, c["N"], ts.size).astype(np.int32))
    held = [serving.Sample(int(uid[rng.integers(0, U)]), int(iid[rng.integers(0, c["N"])]), int(rng.integers(0, 1000))) for _ in range(40)]
    held.append(serving.Sample(int(uid[0]), 10 ** 15, 500))     # an unknown item: a miss
    return held


def _agree_worker(rank, port, out_dir):
    import torch.distributed as dist
    _init(rank, port)
    name = "din_cos_d16"
    S = CASES[name]["S"]
    hist = np.full((1, S), -1, np.int32)
    res = {}
    eng = _engine(rank, _sharded_cfg(name))
    _upload(eng, name)
    res["eval"] = np.array(sorted(serving.Evaluate(eng, _serving_setup(eng, name), ks=(1, 10, 100)).items()), dtype=object).astype(str)
    res["items_code"] = np.array(_err(lambda: eng.rank_items([0], hist, [5 + rank]))[0])        # item rows differ
    res["hist_code"] = np.array(_err(lambda: eng.rank_items([0], hist + rank, [5]))[0])         # windows differ
    r, l = eng.rank_items([0, 0], np.tile(hist, (2, 1)), [5, 6])                               # a matching call afterwards
    res["after.rank"], res["after.logit"] = r, l
    _snapshot(eng, name, res)
    eng.close()

    half = _engine(rank, _sharded_cfg(name))                     # rank 1 has no USER_FEAT: both get its verdict
    uf, itf, emb = _tables(name)
    if rank == 0:
        half.table_upload(g.TABLE_USER_FEAT, uf)
    half.table_upload(g.TABLE_ITEM_FEAT, itf); half.table_upload(g.TABLE_ITEM_EMB, emb)
    code, msg = _err(lambda: half.rank_items([0], hist, [5]))
    res["state_code"] = np.array(code); res["state_msg"] = np.array(msg)
    half.close()

    rep = _engine(rank, _sharded_cfg(name, policy=2))           # replicated placement: local, no collective
    _upload(rep, name)
    dist.barrier()
    if rank == 0:
        r, l = rep.rank_items([0, 3], np.tile(hist, (2, 1)), [5, 900])
        res["rep.rank"], res["rep.logit"] = r, l
        w = rep.get_weights()
        for i in range(4):
            res["rep_w%d" % i] = w[i]
    dist.barrier()
    rep.close()
    np.savez(os.path.join(out_dir, "agree_%d.npz" % rank), **res)
    dist.barrier(); dist.destroy_process_group()


def test_sharded_rank_items_agreement_evaluate_and_replicated(tmp_path):
    _needs_two()
    import torch.multiprocessing as mp
    mp.spawn(_agree_worker, args=(_free_port(), str(tmp_path)), nprocs=WORLD, join=True)
    name = "din_cos_d16"
    S = CASES[name]["S"]
    hist = np.full((1, S), -1, np.int32)
    r0, r1, emb = _load(tmp_path, "agree", CASES[name]["N"])
    for r in (r0, r1):
        assert int(r["items_code"]) == g.EINVAL and int(r["hist_code"]) == g.EINVAL
        assert int(r["state_code"]) == g.ESTATE and "USER_FEAT" in str(r["state_msg"])
    ref = _reference(name, emb, [r0["w%d" % i] for i in range(4)])
    rr, ll = ref.rank_items([0, 0], np.tile(hist, (2, 1)), [5, 6])
    for key, w in (("after.rank", rr), ("after.logit", ll)):
        _assert_same(r0[key], r1[key], key)
        _assert_same(r0[key], w, key)
    want = np.array(sorted(serving.Evaluate(ref, _serving_setup(ref, name), ks=(1, 10, 100)).items()), dtype=object).astype(str)
    assert np.array_equal(r0["eval"], want) and np.array_equal(r1["eval"], want), (r0["eval"], want)
    _, _, emb_rep = _tables(name)
    rep = _reference(name, emb_rep, [r0["rep_w%d" % i] for i in range(4)])
    rr, ll = rep.rank_items([0, 3], np.tile(hist, (2, 1)), [5, 900])
    _assert_same(r0["rep.rank"], rr, "rep.rank")
    _assert_same(r0["rep.logit"], ll, "rep.logit")
