"""Search and top-k recommendation on a row-sharded ITEM_EMB (needs >= 2 GPUs): ctr_knn_search and ctr_recommend_topk are
collective there — each rank scans its own shard and the ranks' lists are merged.  Both ranks must return the same
result, bit for bit, as a single-GPU handle holding the assembled table and the same weights: rows, similarities /
logits / scores and counts.  Cases cover the placements (sharded with and without replicated hot rows, the automatic
placement of a large filled table beside a small replicated ITEM_FEAT, ITEM_FEAT shorter than ITEM_EMB, an empty
shard), a table trained right before the calls without a host sync, and argument disagreement and errors."""
import os
import socket

import numpy as np
import pytest
import torch

import go_ctr_b200 as g

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

WORLD = 2


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


# ---- cases: (model, dims, ITEM_EMB rows, ITEM_FEAT rows, placement policy, hot rows, pred_batch, filled table)
CASES = {
    # reserved[1] = 1 (sharded), hot rows off; odd N; ITEM_FEAT shorter than ITEM_EMB (missing features read as zeros)
    "din_cos_d16": dict(model=g.MODEL_DIN_COS, uP=8, S=50, D=16, cF=5, N=1001, NF=700, policy=1, hot=-1, pb=128, fill=False),
    # sharded with rows [0, 64) replicated on every rank; S = 1
    "youtube_d64_hot": dict(model=g.MODEL_YOUTUBE, uP=4, S=1, D=64, cF=3, N=777, NF=777, policy=1, hot=64, pb=96, fill=False),
    # automatic placement: a filled ITEM_EMB above 32 MB is sharded, the small ITEM_FEAT stays replicated
    "din_euc_auto": dict(model=g.MODEL_DIN_EUC, uP=4, S=50, D=64, cF=7, N=140_000, NF=90_000, policy=0, hot=0, pb=8192, fill=True),
    # the smallest table the sharded upload takes: rank 1's shard is empty
    "tiny": dict(model=g.MODEL_DIN_COS, uP=4, S=1, D=16, cF=0, N=1, NF=0, policy=1, hot=-1, pb=64, fill=False),
}
U = 50


def _tables(name):
    c = CASES[name]
    rng = np.random.default_rng(sum(name.encode()))          # the same tables in every process
    uf = rng.standard_normal((U, c["uP"])).astype(np.float32)
    itf = rng.standard_normal((c["NF"], c["cF"])).astype(np.float32) if c["cF"] else None
    emb = None if c["fill"] else rng.standard_normal((c["N"], c["D"])).astype(np.float32)
    if emb is not None and c["N"] > 10:
        emb[3] = 0.0                          # a zero row: similarity 0 with everything, never returned
        emb[10] = emb[4]                      # tied similarities: rank by row
    return uf, itf, emb


def _cfg(name, **kw):
    c = CASES[name]
    return g.engine.default_config(c["model"], uP=c["uP"], S=c["S"], D=c["D"], cF=c["cF"], batch=64, pred_batch=c["pb"],
                                   table_opt=g.TABLE_SGD, table_lr=0.5, dropout0=0.0, dropout1=0.0, seed=5, **kw)


def _calls(name):
    """The calls of a case: (key, kind, kwargs), the same list for the ranks and for the reference handle."""
    c = CASES[name]
    N, D, S = c["N"], c["D"], c["S"]
    rng = np.random.default_rng(1000 + len(name))
    out = []
    if N == 1:
        out.append(("knn_row", "knn", dict(k=4, rows=[0])))
        out.append(("knn_vec", "knn", dict(k=2, queries=rng.standard_normal((3, D)))))
        out.append(("rec", "rec", dict(user_rows=[0, 1], hist=[[0], [-1]], k=3, exclude_history=True)))
        out.append(("rec_keep", "rec", dict(user_rows=[0], hist=[[0]], k=1, exclude_history=False)))
        return out
    q = rng.standard_normal((1500, D))
    q[7] = 0.0                                                               # a zero query: count 0
    out.append(("knn_vec_1500_k10", "knn", dict(k=10, queries=q)))
    excl = rng.integers(-1, N, 1500).astype(np.int32)
    out.append(("knn_vec_excl_k10", "knn", dict(k=10, queries=q, rows=excl)))
    out.append(("knn_vec_1_k1", "knn", dict(k=1, queries=q[:1])))
    out.append(("knn_zero_query", "knn", dict(k=5, queries=np.zeros((1, D)))))
    rows = np.array([0, 1, 2, 3, 4, 10, 63, 64, 65, N - 1, N - 2, N // 2, N // 2 + 1], np.int32)   # both ranks' rows, hot rows
    out.append(("knn_rows_k10", "knn", dict(k=10, rows=rows)))
    out.append(("knn_rows_k1024", "knn", dict(k=1024, rows=rows[:4])))
    out.append(("knn_rows_1", "knn", dict(k=10, rows=[N - 1])))
    nu = 300 if N < 10_000 else 3                                            # two user groups of 256 on the small tables
    users = rng.integers(0, U, nu).astype(np.int32)
    users[1] = U + 5                                                         # a user row outside USER_FEAT
    hist = rng.integers(-1, N + 40, (nu, S)).astype(np.int32)                # both ranks' rows, -1, rows past the table
    hist[0, :min(S, 4)] = np.arange(min(S, 4))                               # hot rows
    hist[2] = -1
    out.append(("rec_k100_excl", "rec", dict(user_rows=users, hist=hist, k=100, exclude_history=True)))
    out.append(("rec_k100_keep", "rec", dict(user_rows=users, hist=hist, k=100, exclude_history=False)))
    out.append(("rec_k1", "rec", dict(user_rows=users[:5], hist=hist[:5], k=1, exclude_history=True)))
    out.append(("rec_k1024", "rec", dict(user_rows=users[:3], hist=hist[:3], k=1024, exclude_history=True)))
    return out


def _run(eng, calls):
    res = {}
    for key, kind, kw in calls:
        if kind == "knn":
            r, s, n = eng.knn_search(**kw)
            res[key + ".rows"], res[key + ".sims"], res[key + ".count"] = r, s, n
        else:
            r, s, l, n = eng.recommend_topk(**kw)
            res[key + ".rows"], res[key + ".scores"], res[key + ".logits"], res[key + ".count"] = r, s, l, n
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


def _save(out_dir, rank, tag, res):
    np.savez(os.path.join(out_dir, "%s_%d.npz" % (tag, rank)), **res)


def _err(fn):
    try:
        fn()
    except g.CtrError as e:
        return e.code, str(e)
    return 0, ""


def _case_worker(rank, world, port, out_dir, names):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.cuda.set_device(rank)
    for name in names:
        c = CASES[name]

        def cfg(r):
            x = _cfg(name, device=r, rank=r, world=world)
            x.reserved[1] = c["policy"]; x.reserved[0] = c["hot"]
            return x
        eng = _engine(rank, cfg)
        _upload(eng, name)
        res = _run(eng, _calls(name))
        res["emb"] = eng.table_download(g.TABLE_ITEM_EMB, c["N"], c["D"])
        for i, w in enumerate(eng.get_weights()):
            res["w%d" % i] = w
        _save(out_dir, rank, name, res)
        eng.close()
    dist.barrier(); dist.destroy_process_group()


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
    assert np.array_equal(_bits(got), _bits(want)), "%s differs from the single-GPU handle at %s" % (key, np.argwhere(_bits(got) != _bits(want))[:5].tolist())


def _assemble(tmp_path, tag, N):
    r0, r1 = np.load(tmp_path / ("%s_0.npz" % tag)), np.load(tmp_path / ("%s_1.npz" % tag))
    emb = np.array(r0["emb"])
    if N > 1:
        emb[1::2] = r1["emb"][1::2]
    return r0, r1, emb


def _check_case(tmp_path, name, calls):
    c = CASES[name]
    r0, r1, emb = _assemble(tmp_path, name, c["N"])
    if c["fill"]:
        assert np.abs(emb).max() > 0.5
    ref = _reference(name, emb, [r0["w%d" % i] for i in range(4)])
    want = _run(ref, calls)
    for key, w in want.items():
        _assert_same(r0[key], r1[key], key + " (rank 0 vs rank 1)")
        _assert_same(r0[key], w, key)
    counts = [want[k] for k in want if k.endswith(".count")]
    assert any((n > 0).any() for n in counts)


def _needs_two():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")


def test_sharded_search_and_recommend_equal_single_gpu(tmp_path):
    _needs_two()
    import torch.multiprocessing as mp
    names = list(CASES)
    mp.spawn(_case_worker, args=(WORLD, _free_port(), str(tmp_path), names), nprocs=WORLD, join=True)
    for name in names:
        _check_case(tmp_path, name, _calls(name))


# ---- a live table: sharded SGD steps with hot rows, then search and recommend with no host sync in between
LIVE = "din_cos_d16"


def _live_batches():
    c = CASES[LIVE]
    rng = np.random.default_rng(31)
    out = []
    for _ in range(3):
        B = 64
        ur = rng.integers(0, U, 2 * B).astype(np.int32)
        ir = rng.integers(0, c["N"], 2 * B).astype(np.int32)
        ir[:8] = np.arange(8)                                                # hot rows
        hist = rng.integers(-1, c["N"], (2 * B, c["S"])).astype(np.int32)
        y = (rng.random(2 * B) > 0.5).astype(np.float32)
        out.append((ur, ir, hist, y))
    return out


def _live_calls():
    c = CASES[LIVE]
    rng = np.random.default_rng(77)
    hist = rng.integers(-1, c["N"], (4, c["S"])).astype(np.int32)
    hist[:, :3] = [0, 1, 2]
    _, _, emb0 = _tables(LIVE)
    return [("knn_rows", "knn", dict(k=20, rows=np.array([0, 1, 5, 8, 500, 999], np.int32))),
            ("knn_vec", "knn", dict(k=20, queries=rng.standard_normal((4, c["D"])))),
            # the trained hot rows' starting values: each row itself must compete, with its current (trained) value
            ("knn_hot", "knn", dict(k=5, queries=emb0[:8].astype(np.float64))),
            ("rec", "rec", dict(user_rows=np.array([0, 1, 2, 3], np.int32), hist=hist, k=50, exclude_history=True))]


def _live_worker(rank, world, port, out_dir):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.cuda.set_device(rank)

    def cfg(r):
        x = _cfg(LIVE, device=r, rank=r, world=world)
        x.reserved[1] = 1; x.reserved[0] = 64
        return x
    eng = _engine(rank, cfg)
    _upload(eng, LIVE)
    batches = _live_batches()
    sl = slice(rank * 64, (rank + 1) * 64)
    for ur, ir, hist, y in batches[:-1]:
        eng.train_step_idx(ur[sl], ir[sl], hist[sl], y[sl])
    ur, ir, hist, y = batches[-1]
    dev = "cuda:%d" % rank
    t = [torch.from_numpy(np.ascontiguousarray(a[sl])).to(dev) for a in (ur, ir, hist, y)]
    torch.cuda.synchronize(dev)
    eng.train_step_idx_dev(t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), t[3].data_ptr(), 64)   # asynchronous
    res = _run(eng, _live_calls())                                           # queued right behind it, no sync
    res["emb"] = eng.table_download(g.TABLE_ITEM_EMB, CASES[LIVE]["N"], CASES[LIVE]["D"])
    for i, w in enumerate(eng.get_weights()):
        res["w%d" % i] = w
    _save(out_dir, rank, "live", res)
    eng.close()
    dist.barrier(); dist.destroy_process_group()


def test_sharded_serving_sees_the_table_trained_just_before(tmp_path):
    _needs_two()
    import torch.multiprocessing as mp
    mp.spawn(_live_worker, args=(WORLD, _free_port(), str(tmp_path)), nprocs=WORLD, join=True)
    r0, r1, emb = _assemble(tmp_path, "live", CASES[LIVE]["N"])
    _, _, emb0 = _tables(LIVE)
    assert np.abs(emb[:64] - emb0[:64]).max() > 1e-6 and np.abs(emb[64:] - emb0[64:]).max() > 1e-6   # hot and other rows moved
    trained = np.unique(np.concatenate([b[1] for b in _live_batches()]))
    hot_trained = trained[(trained < 8) & (trained != 3) & (trained != 4)]   # row 3 starts at zero, row 4 has an untrained twin (row 10)
    assert hot_trained.size > 0 and np.abs(emb[hot_trained] - emb0[hot_trained]).max() > 1e-6
    hot_hits = r0["knn_hot.rows"][hot_trained, 0]
    assert (hot_hits == hot_trained).all(), hot_hits                         # each trained hot row is its own query's best match
    assert (r0["knn_hot.sims"][hot_trained, 0] < 1.0).all()                  # ... scored with its trained value, not the start value
    ref = _reference(LIVE, emb, [r0["w%d" % i] for i in range(4)])
    for key, w in _run(ref, _live_calls()).items():
        _assert_same(r0[key], r1[key], key + " (rank 0 vs rank 1)")
        _assert_same(r0[key], w, key)


# ---- argument agreement and errors
def _agree_worker(rank, world, port, out_dir):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.cuda.set_device(rank)
    name = "din_cos_d16"
    N = CASES[name]["N"]

    def cfg(r):
        x = _cfg(name, device=r, rank=r, world=world)
        x.reserved[1] = 1; x.reserved[0] = -1
        return x
    eng = _engine(rank, cfg)
    _upload(eng, name)
    res = {}
    q = np.random.default_rng(3).standard_normal((2, CASES[name]["D"]))
    code, msg = _err(lambda: eng.knn_search(5 + rank, queries=q))                        # k differs between the ranks
    res["k_code"] = np.array(code)
    hist = np.full((1, CASES[name]["S"]), -1, np.int32)
    code, _ = _err(lambda: eng.recommend_topk([rank], hist, 5))                          # user row differs
    res["u_code"] = np.array(code)
    r, s, n = eng.knn_search(5, queries=q)                                                # a matching call afterwards
    res["after.rows"], res["after.sims"], res["after.count"] = r, s, n
    code, msg = _err(lambda: eng.knn_search(3, rows=[N]))                                 # the same bad row on both ranks
    res["nf_code"] = np.array(code); res["nf_msg"] = np.array(msg)
    res["emb"] = eng.table_download(g.TABLE_ITEM_EMB, N, CASES[name]["D"])
    for i, w in enumerate(eng.get_weights()):
        res["w%d" % i] = w
    eng.close()

    # a state check that fails on one rank only (rank 1 has no USER_FEAT): every rank returns rank 1's verdict
    half = _engine(rank, cfg)
    uf, itf, emb = _tables(name)
    if rank == 0:
        half.table_upload(g.TABLE_USER_FEAT, uf)
    half.table_upload(g.TABLE_ITEM_FEAT, itf); half.table_upload(g.TABLE_ITEM_EMB, emb)
    code, msg = _err(lambda: half.recommend_topk([0], hist, 5))
    res["state_code"] = np.array(code); res["state_msg"] = np.array(msg)
    half.close()

    def cfg_rep(r):                                                                       # replicated placement: local, no collective
        x = _cfg(name, device=r, rank=r, world=world)
        x.reserved[1] = 2
        return x
    rep = _engine(rank, cfg_rep)
    _upload(rep, name)
    dist.barrier()
    if rank == 0:
        r, s, n = rep.knn_search(7, queries=q)
        res["rep.rows"], res["rep.sims"], res["rep.count"] = r, s, n
        r, s, l, n = rep.recommend_topk([0], hist, 7)
        res["rep_rec.rows"], res["rep_rec.logits"], res["rep_rec.count"] = r, l, n
    dist.barrier()
    rep.close()
    _save(out_dir, rank, "agree", res)
    dist.barrier(); dist.destroy_process_group()


def test_sharded_serving_arguments_must_agree(tmp_path):
    _needs_two()
    import torch.multiprocessing as mp
    mp.spawn(_agree_worker, args=(WORLD, _free_port(), str(tmp_path)), nprocs=WORLD, join=True)
    name = "din_cos_d16"
    N = CASES[name]["N"]
    r0, r1, emb = _assemble(tmp_path, "agree", N)
    for r in (r0, r1):
        assert int(r["k_code"]) == g.EINVAL and int(r["u_code"]) == g.EINVAL
        assert int(r["nf_code"]) == g.ENOTFOUND
        assert int(r["state_code"]) == g.ESTATE and "USER_FEAT" in str(r["state_msg"])
    ref = _reference(name, emb, [r0["w%d" % i] for i in range(4)])
    want = _err(lambda: ref.knn_search(3, rows=[N]))
    assert str(r0["nf_msg"]) == str(r1["nf_msg"]) == want[1] and want[0] == g.ENOTFOUND
    q = np.random.default_rng(3).standard_normal((2, CASES[name]["D"]))
    rr, ss, nn = ref.knn_search(5, queries=q)
    for key, w in (("after.rows", rr), ("after.sims", ss), ("after.count", nn)):
        _assert_same(r0[key], r1[key], key)
        _assert_same(r0[key], w, key)
    rr, ss, nn = ref.knn_search(7, queries=q)
    for key, w in (("rep.rows", rr), ("rep.sims", ss), ("rep.count", nn)):
        _assert_same(r0[key], w, key)
    hist = np.full((1, CASES[name]["S"]), -1, np.int32)
    rr, _, ll, nn = ref.recommend_topk([0], hist, 7)
    for key, w in (("rep_rec.rows", rr), ("rep_rec.logits", ll), ("rep_rec.count", nn)):
        _assert_same(r0[key], w, key)
