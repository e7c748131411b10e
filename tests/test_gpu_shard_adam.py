"""CTR_TABLE_ADAM on a row-sharded ITEM_EMB (world ranks x batch B, placement 1) against one GPU x batch world*B on the
whole table, both with the lazy row Adam, dropout off: per-step costs, dense weights, the table assembled from the
shards (touched rows to float32 summation order, untouched rows bit-identical to the upload) and scores on a probe
batch.  Over DIN-cos and YouTube, uniform and Zipf ids, hot rows default (rows [0, 32768) replicated) and off; through
ctr_train_step_idx, ctr_train_idx with a ragged tail and ctr_train_keys; a checkpoint after 2 of 4 steps; the profile
keys of the owner update; table_download and sharded search after training.

One process group per world size runs every case (tests skip when fewer GPUs are visible); rank 0's outputs and each
rank's shard land in a temporary directory, the single-GPU references run in the test process."""
import os
import socket

import numpy as np
import pytest
import torch

import go_ctr_b200 as g
from tests.util import assert_mostly_close, close_frac, make_batch, make_tables

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200)]

DIMS = dict(uP=8, S=10, D=16, cF=12)
U, I, B, STEPS, LR = 97, 40000, 256, 4, 0.01          # I > 32768: the default hot range covers part of the table
CASES = [(m, z, hot) for m in ("din", "youtube") for z in (False, True) for hot in (0, -1)]
NEW_KEYS = {"shard_row_adam", "hot_rows_adam", "hot_moments_pull"}


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _tables():
    return make_tables(np.random.default_rng(11), U, I, DIMS["uP"], DIMS["cF"], DIMS["D"])


def _global_batches(ci, world, zipf, n=STEPS):
    """n global batches of world*B samples; a few history ids and target ids past the table (missing rows)."""
    rng = np.random.default_rng(100 + ci)
    out = []
    for _ in range(n):
        ur, ir, hist, y = make_batch(rng, U, I, world * B, DIMS["S"], zipf=zipf)
        hist[rng.random(hist.shape) < 0.01] = I + 3
        ir[rng.random(ir.shape) < 0.01] = I + 7
        out.append((ur, ir, hist, y))
    return out


def _probe():
    return make_batch(np.random.default_rng(9), U, I, B, DIMS["S"])[:3]


def _queries():
    return np.random.default_rng(5).standard_normal((3, DIMS["D"]))


def _cfg(model, batch, hot, world=1, rank=0, topt=g.TABLE_ADAM):
    m = g.MODEL_DIN_COS if model == "din" else g.MODEL_YOUTUBE
    cfg = g.engine.default_config(m, batch=batch, pred_batch=batch, table_opt=topt, table_lr=LR, dropout0=0.0, dropout1=0.0,
                                  seed=3, device=rank if world > 1 else 0, rank=rank, world=world, **DIMS)
    cfg.reserved[0] = hot
    cfg.reserved[1] = 1 if world > 1 else 0
    return cfg


def _upload(eng, tabs):
    uf, itf, emb = tabs
    eng.table_upload(g.TABLE_USER_FEAT, uf); eng.table_upload(g.TABLE_ITEM_FEAT, itf); eng.table_upload(g.TABLE_ITEM_EMB, emb)


def _sharded(dist, rank, world, model, hot, topt=g.TABLE_ADAM):
    eng = g.Engine(_cfg(model, B, hot, world, rank, topt))
    ids = [eng.comm_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(ids, src=0)
    eng.comm_init(ids[0])
    return eng


def _save(out_dir, name, rank, eng, **extra):
    eng.sync()
    np.savez(os.path.join(out_dir, "%s_r%d.npz" % (name, rank)), emb=eng.table_download(g.TABLE_ITEM_EMB, I, DIMS["D"]),
             **{"w%d" % i: w for i, w in enumerate(eng.get_weights())}, **extra)


def _ragged(world, ci):
    """per-rank sample arrays of 2B + 37 samples (ctr_train_idx: the last batch is a ragged tail)"""
    n = 2 * B + 37
    rng = np.random.default_rng(500 + ci)
    return [make_batch(rng, U, I, n, DIMS["S"]) for _ in range(world)]


def _keys(world, ci):
    """per-rank sample keys (2B each) over id maps user id = 1000 + row, item id = 50000 + row"""
    rng = np.random.default_rng(700 + ci)
    out = []
    for _ in range(world):
        ur, ir, _, y = make_batch(rng, U, I, 2 * B, DIMS["S"], zipf=True)
        out.append((ur.astype(np.int64) + 1000, ir.astype(np.int64) + 50000, np.arange(2 * B, dtype=np.int64), y))
    return out


def _worker(rank, world, port, out_dir):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.cuda.set_device(rank)
    tabs = _tables()
    sl = slice(rank * B, (rank + 1) * B)
    pu, pi, ph = _probe()
    for ci, (model, zipf, hot) in enumerate(CASES):
        batches = _global_batches(ci, world, zipf)
        eng = _sharded(dist, rank, world, model, hot)
        _upload(eng, tabs)
        costs = []
        for k, b in enumerate(batches):
            if k == STEPS - 1 and ci == 0:
                eng.profile(True); eng.profile_reset()
            costs.append(eng.train_step_idx(*(a[sl] for a in b)).cost)
        prof = sorted(eng.profile_dump()) if ci == 0 else []
        eng.profile(False)
        eng.sync(); dist.barrier()
        p = eng.predict_idx(pu, pi, ph)
        extra = {}
        if ci == 0:         # sharded search after training (collective) reads the trained rows, hot rows included
            kr, ks, _ = eng.knn_search(8, queries=_queries())
            extra = dict(knn_rows=kr, knn_sims=ks)
        _save(out_dir, "steps%d" % ci, rank, eng, costs=np.array(costs, np.float32), p=p, prof=np.array(prof), **extra)
        eng.close(); dist.barrier()
    # sharded SGD step: none of the row-Adam launches
    eng = _sharded(dist, rank, world, "din", 0, g.TABLE_SGD)
    _upload(eng, tabs)
    eng.profile(True)
    eng.train_step_idx(*(a[sl] for a in _global_batches(0, world, False, 1)[0]))
    np.save(os.path.join(out_dir, "sgdprof_r%d.npy" % rank), np.array(sorted(eng.profile_dump())))
    eng.close(); dist.barrier()
    # ctr_train_idx with a ragged tail, hot rows default and off
    for hot in (0, -1):
        eng = _sharded(dist, rank, world, "din", hot)
        _upload(eng, tabs)
        ur, ir, hist, y = _ragged(world, hot)[rank]
        costs = eng.train_idx(ur, ir, hist, y)
        _save(out_dir, "ragged%d" % hot, rank, eng, costs=costs)
        eng.close(); dist.barrier()
    # ctr_train_keys
    eng = _sharded(dist, rank, world, "din", 0)
    _upload(eng, tabs)
    eng.idmap_build(g.IDMAP_USER, np.arange(U, dtype=np.int64) + 1000)
    eng.idmap_build(g.IDMAP_ITEM, np.arange(I, dtype=np.int64) + 50000)
    ku, ki, kt, ky = _keys(world, 0)[rank]
    ep, cost, used = eng.train_keys(ku, ki, kt, ky, epochs=1)
    _save(out_dir, "keys", rank, eng, cost=np.array([cost], np.float32))
    eng.close(); dist.barrier()
    # checkpoint after 2 steps, fresh handles, 2 more steps (case 0: din, uniform ids, hot rows default)
    batches = _global_batches(0, world, False)
    eng = _sharded(dist, rank, world, "din", 0)
    _upload(eng, tabs)
    for b in batches[:2]:
        eng.train_step_idx(*(a[sl] for a in b))
    eng.sync()
    ck = os.path.join(out_dir, "ck%d.bin" % rank)
    eng.checkpoint_save(ck)
    eng.close(); dist.barrier()
    eng = _sharded(dist, rank, world, "din", 0)
    eng.checkpoint_load(ck)
    costs = [eng.train_step_idx(*(a[sl] for a in b)).cost for b in batches[2:]]
    _save(out_dir, "ckpt", rank, eng, costs=np.array(costs, np.float32))
    eng.close()
    dist.barrier()
    dist.destroy_process_group()


_RUNS = {}


def _run(world, tmp_path_factory):
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    if world not in _RUNS:
        import torch.multiprocessing as mp
        d = tmp_path_factory.mktemp("shard_adam_w%d" % world)
        mp.spawn(_worker, args=(world, _free_port(), str(d)), nprocs=world, join=True)
        _RUNS[world] = d
    return _RUNS[world]


def _assembled(d, name, world):
    emb = np.zeros((I, DIMS["D"]), np.float32)
    for r in range(world):
        emb[r::world] = np.load(d / ("%s_r%d.npz" % (name, r)))["emb"][r::world]
    return emb


def _touched(batches):
    t = np.zeros(I, bool)
    for ur, ir, hist, y in batches:
        for a in (hist.reshape(-1), ir):
            a = a[(a >= 0) & (a < I)]
            t[a] = True
    return t


def _reference(model, batches, hot=0):
    tabs = _tables()
    ref = g.Engine(_cfg(model, len(batches[0][0]), hot))
    _upload(ref, tabs)
    costs = [ref.train_step_idx(*b).cost for b in batches]
    return ref, costs


def _compare(d, name, world, ref, batches, what):
    emb0 = _tables()[2]
    got = _assembled(d, name, world)
    want = ref.table_download(g.TABLE_ITEM_EMB, I, DIMS["D"])
    t = _touched(batches)
    assert t.sum() > 100 and (~t).sum() > 100
    assert got[~t].tobytes() == emb0[~t].tobytes(), "%s: an untouched row changed" % what
    assert want[~t].tobytes() == emb0[~t].tobytes()
    assert np.abs(want[t] - emb0[t]).max() > 0.5 * LR                          # the rows did move
    assert_mostly_close(got[t], want[t], 2e-3, 2e-5, 0.995, "%s: touched rows" % what)
    r0 = np.load(d / ("%s_r0.npz" % name))
    for i, w in enumerate(ref.get_weights()):
        assert_mostly_close(r0["w%d" % i], w, 2e-3, 2e-4, 0.995, "%s: weights %d" % (what, i))
    return r0


WORLDS = [2, 4, 8]


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("ci", range(len(CASES)), ids=["%s-%s-hot%s" % (m, "zipf" if z else "uniform", "default" if h == 0 else "off") for m, z, h in CASES])
def test_sharded_adam_steps_equal_one_gpu_global_batch(world, ci, tmp_path_factory):
    d = _run(world, tmp_path_factory)
    model, zipf, hot = CASES[ci]
    batches = _global_batches(ci, world, zipf)
    ref, want = _reference(model, batches)
    r0 = _compare(d, "steps%d" % ci, world, ref, batches, CASES[ci])
    np.testing.assert_allclose(r0["costs"], np.array(want, np.float32), rtol=2e-4, atol=1e-6)
    for r in range(1, world):
        assert np.load(d / ("steps%d_r%d.npz" % (ci, r)))["costs"].tobytes() == r0["costs"].tobytes()
        assert np.load(d / ("steps%d_r%d.npz" % (ci, r)))["w0"].tobytes() == r0["w0"].tobytes()
    np.testing.assert_allclose(r0["p"], ref.predict_idx(*_probe()), rtol=2e-3, atol=1e-5)


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("hot", [0, -1], ids=["hot_default", "hot_off"])
def test_sharded_adam_train_idx_ragged_tail(world, hot, tmp_path_factory):
    d = _run(world, tmp_path_factory)
    per = _ragged(world, hot)
    glob = []
    for b in range(3):            # global batch b = every rank's batch b; a rank's tail padded with missing ids, label 0
        parts = []
        for ur, ir, hist, y in per:
            s = slice(b * B, min((b + 1) * B, ur.size)); pad = B - (s.stop - s.start)
            parts.append((np.concatenate([ur[s], np.full(pad, -1, np.int32)]), np.concatenate([ir[s], np.full(pad, -1, np.int32)]),
                          np.concatenate([hist[s], np.full((pad, DIMS["S"]), -1, np.int32)]), np.concatenate([y[s], np.zeros(pad, np.float32)])))
        glob.append(tuple(np.concatenate([p[k] for p in parts]) for k in range(4)))
    ref, want = _reference("din", glob)
    r0 = _compare(d, "ragged%d" % hot, world, ref, glob, "train_idx hot=%d" % hot)
    np.testing.assert_allclose(r0["costs"], np.array(want, np.float32), rtol=2e-4, atol=1e-6)


@pytest.mark.parametrize("world", WORLDS)
def test_sharded_adam_train_keys(world, tmp_path_factory):
    d = _run(world, tmp_path_factory)
    per = _keys(world, 0)
    glob = []
    for b in range(2):            # no behaviour cache: every history is empty
        s = slice(b * B, (b + 1) * B)
        ur = np.concatenate([k[0][s] - 1000 for k in per]).astype(np.int32); ir = np.concatenate([k[1][s] - 50000 for k in per]).astype(np.int32)
        glob.append((ur, ir, np.full((ur.size, DIMS["S"]), -1, np.int32), np.concatenate([k[3][s] for k in per])))
    ref, want = _reference("din", glob)
    r0 = _compare(d, "keys", world, ref, glob, "train_keys")
    np.testing.assert_allclose(r0["cost"][0], want[-1], rtol=2e-4, atol=1e-6)


@pytest.mark.parametrize("world", WORLDS)
def test_sharded_adam_checkpoint_resume(world, tmp_path_factory):
    """save after 2 steps, load into fresh handles, 2 more == 4 uninterrupted steps (case 0).  A restart that lost the
    moments (the hot rows' included) would move touched rows by about table_lr more than the uninterrupted run."""
    d = _run(world, tmp_path_factory)
    full, res = _assembled(d, "steps0", world), _assembled(d, "ckpt", world)
    batches = _global_batches(0, world, False)
    t = _touched(batches)
    assert res[~t].tobytes() == full[~t].tobytes()
    hot = np.zeros(I, bool); hot[:32768] = True
    for sel, what in ((t & hot, "hot rows"), (t & ~hot, "owner rows")):
        assert sel.sum() > 100
        assert close_frac(res[sel], full[sel], 1e-3, 1e-5) >= 0.995, what
        assert np.abs(res[sel] - full[sel]).max() < 0.2 * LR, what
    a, b = np.load(d / "ckpt_r0.npz"), np.load(d / "steps0_r0.npz")
    np.testing.assert_allclose(a["costs"], b["costs"][2:], rtol=2e-4, atol=1e-6)
    for i in range(4):
        assert_mostly_close(a["w%d" % i], b["w%d" % i], 2e-3, 2e-4, 0.995, "weights %d" % i)


@pytest.mark.parametrize("world", WORLDS)
def test_sharded_adam_profile_keys(world, tmp_path_factory):
    d = _run(world, tmp_path_factory)
    keys = set(np.load(d / "steps0_r0.npz")["prof"].tolist())
    assert {"shard_row_adam", "hot_rows_adam"} <= keys and "segment_adam" not in keys
    assert not NEW_KEYS & set(np.load(d / "sgdprof_r0.npy").tolist())
    ref = g.Engine(_cfg("din", world * B, 0))
    _upload(ref, _tables())
    ref.profile(True)
    ref.train_step_idx(*_global_batches(0, world, False, 1)[0])
    assert not NEW_KEYS & set(ref.profile_dump())


@pytest.mark.parametrize("world", WORLDS)
def test_sharded_adam_download_and_search_see_hot_rows(world, tmp_path_factory):
    """table_download and the sharded ctr_knn_search read the trained hot rows (written back from the replicas)."""
    d = _run(world, tmp_path_factory)
    emb = _assembled(d, "steps0", world)
    emb0 = _tables()[2]
    t = _touched(_global_batches(0, world, False))
    assert (np.abs(emb[:32768][t[:32768]] - emb0[:32768][t[:32768]]).max(axis=1) > 0).mean() > 0.99
    r0 = np.load(d / "steps0_r0.npz")
    one = g.Engine(_cfg("din", B, 0))           # one GPU holding the downloaded table: the sharded search is bit-identical to it
    one.table_upload(g.TABLE_ITEM_EMB, emb)
    kr, ks, _ = one.knn_search(8, queries=_queries())
    assert r0["knn_rows"].tolist() == kr.tolist()
    assert r0["knn_sims"].tobytes() == ks.tobytes()
