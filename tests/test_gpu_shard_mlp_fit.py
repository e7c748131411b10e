"""The key-fed float64 MLP trained on a multi-GPU feature store (ctr_mlp_fit_keys_dist; needs >= 2 GPUs): every rank
passes its own keys, and every rank's model must equal, bit for bit, fit_keys on one GPU over the ranks' keys
concatenated in rank order, against a single-GPU feature store holding the same tables, id maps and ubcache.

Cases (the placements of tests/test_gpu_shard_mlp.py, each asserted from the ranks' table downloads): a row-sharded
ITEM_EMB with hot rows beside a sharded ITEM_FEAT; the by-size placement, a sharded ITEM_EMB above 32 MB with the default
hot rows beside a replicated ITEM_FEAT; ITEM_EMB and ITEM_FEAT both sharded without hot rows, where rank 1 passes no
keys.  Models: a binary classifier (adam), a classifier on rating classes (sgd with momentum) and an identity-output
regressor (adam), each then fitted again with warm_start from its fitted state.  The keys of each rank differ, and some
unknown user and item ids appear on one rank only.  Checked on every rank: get_params, n_iter, loss_curve, rows_used,
classes_ / out_activation_, then predict_keys and recommend_topk against the one-GPU model's.  Refusals: a seed that
differs on one rank (EINVAL on both, the parameters unchanged), every key unknown (ENOTFOUND on both), a replicated
ITEM_EMB beside a sharded ITEM_FEAT (ESTATE on both), and ctr_mlp_fit_keys on the same handle (still ESTATE).  The
profile keys of one fit."""
import os

import numpy as np
import pytest

import go_ctr_b200 as g
from tests import test_gpu_shard_mlp as sm
from tests import test_gpu_shard_rank as sr

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200)]

WORLD = sr.WORLD
NIN = sm.NIN
CASES = {"hot_trained": dict(split=0.45), "feat_auto": dict(split=0.6), "feat_sharded": dict(split=1.0)}   # split: rank 0's share
MODELS = {
    "binary": (g.engine.MLPClassifier, dict(hidden=(12, 5), solver="adam", batch=32, max_iter=4, seed=3, lr_init=0.01)),
    "ratings": (g.engine.MLPClassifier, dict(hidden=(9,), solver="sgd", momentum=0.9, batch=40, max_iter=3, seed=4, lr_init=0.05)),
    "regressor": (g.engine.MLPRegressor, dict(hidden=(7,), solver="adam", batch=32, max_iter=3, seed=5, lr_init=0.01)),
}


def _labels(name, n, rng):
    if name == "binary":
        return (rng.random(n) < 0.4).astype(np.float32)
    return rng.integers(1, 6, n).astype(np.float32)                     # ratings: classes, or the regressor's targets


def _keys(name, call):
    """the concatenated keys of a case and call (0: first fit, 1: warm start) and where rank 1's part starts"""
    c = sm.CASES[name]
    uid, iid = sm._ids(c)
    rng = np.random.default_rng(100 * call + len(name))
    n = 300
    users = uid[rng.integers(0, sm.U, n)]
    items = iid[rng.integers(0, c["N"], n)]
    ts = rng.integers(0, 45, n).astype(np.int64)
    cut = int(n * CASES[name]["split"])
    users[5] = 99_999_999                                               # an unknown user on rank 0 only
    items[cut + 2 if cut + 2 < n else 7] = 7                            # an unknown item on rank 1 (or on rank 0 when rank 1 has none)
    return users, items, ts, cut


def _part(arr, cut, rank):
    return arr[:cut] if rank == 0 else arr[cut:]


def _model(mn, device, **kw):
    cls, base = MODELS[mn]
    return cls(NIN, device=device, **{**base, **kw})


def _state(m, res, tag):
    res[tag + ".params"] = m.get_params()
    res[tag + ".n_iter"] = np.array(m.n_iter)
    res[tag + ".loss"] = np.asarray(m.loss_curve)
    res[tag + ".rows_used"] = np.array(m.rows_used)
    res[tag + ".head"] = np.asarray(m.out_activation_ if isinstance(m, g.engine.MLPRegressor) else m.classes_)


def _fits(eng, name, device, rank, res):
    """the fits of one case; rank None: the one-GPU reference over the concatenated keys"""
    for mn in MODELS:
        m = _model(mn, device, warm_start=True)
        for call in (0, 1):
            users, items, ts, cut = _keys(name, call)
            y = _labels(mn, users.size, np.random.default_rng(call))
            if rank is None:
                m.fit_keys(eng, users, items, ts, y)
            else:
                m.fit_keys_dist(eng, *(_part(a, cut, rank) for a in (users, items, ts, y)))
            _state(m, res, "%s.%s.%d" % (name, mn, call))
        users, items, ts, _ = _keys(name, 0)
        res["%s.%s.pred" % (name, mn)] = m.predict_keys(eng, users[:50], items[:50], ts[:50])
        if mn != "ratings":                                             # a model with classes predicts labels: no ranking
            out = m.recommend_topk(eng, users[:20], ts[:20], 10)
            res["%s.%s.rec.rows" % (name, mn)], res["%s.%s.rec.logits" % (name, mn)] = out[0], out[2]


def _worker(rank, port, out_dir):
    import torch.distributed as dist
    sr._init(rank, port)
    res = {}
    for name in CASES:
        eng = sr._engine(rank, sm._sharded(sm.CASES[name]))
        sm._setup(eng, name)
        sm._case_placement(eng, name, rank)
        if name == "hot_trained":
            eng.profile(True); eng.profile_reset()
        _fits(eng, name, rank, rank, res)
        if name == "hot_trained":
            prof = eng.profile_dump()
            eng.profile(False)
            for key in ("mlp_fit_gather_peer", "mlp_fit_gather_ranks"):
                res["prof." + key] = np.array(prof.get(key, (0, 0))[1])
        if name == "feat_sharded":
            _refusals(eng, rank, res)
        eng.close()
    _mixed(rank, res)
    np.savez(os.path.join(out_dir, "fit_%d.npz" % rank), **res)
    dist.barrier(); dist.destroy_process_group()


def _refusals(eng, rank, res):
    users, items, ts, cut = _keys("feat_sharded", 0)
    y = _labels("binary", users.size, np.random.default_rng(0))
    m = _model("binary", rank, warm_start=True)
    m.fit_keys_dist(eng, users[:100], items[:100], ts[:100], y[:100])
    before = m.get_params()
    odd = _model("binary", rank, warm_start=True, seed=3 + rank)        # a configuration that differs on rank 1
    odd.set_params(before)
    res["code.config"] = np.array(sr._err(lambda: odd.fit_keys_dist(eng, users[:100], items[:100], ts[:100], y[:100]))[0])
    res["config.params"] = odd.get_params()
    unknown = np.full(20, 123_456_789, np.int64)
    res["code.unknown"] = np.array(sr._err(lambda: m.fit_keys_dist(eng, unknown, items[:20], ts[:20], y[:20]))[0])
    res["unknown.params"] = m.get_params()
    res["before.params"] = before
    res["code.fit_keys"] = np.array(sr._err(lambda: m.fit_keys(eng, users[:10], items[:10], ts[:10], y[:10]))[0])


def _mixed(rank, res):
    """ITEM_EMB replicated (small) beside a sharded ITEM_FEAT under the by-size placement"""
    c = sm.CASES["feat_sharded"]
    eng = sr._engine(rank, sm._sharded(c, policy=0))
    uf, _, emb = sm._tables("feat_sharded")
    big = np.random.default_rng(2).standard_normal((3_000_000, sm.CF)).astype(np.float32)
    eng.table_upload(g.TABLE_USER_FEAT, uf)
    eng.table_upload(g.TABLE_ITEM_EMB, emb)
    eng.table_upload(g.TABLE_ITEM_FEAT, big)
    sm._assert_placement(eng, rank, [(g.TABLE_ITEM_EMB, emb, "replicated"), (g.TABLE_ITEM_FEAT, big, "sharded")])
    uid, iid = sm._ids(c)
    eng.idmap_build(0, uid); eng.idmap_build(1, iid)
    users, items, ts, _ = _keys("feat_sharded", 0)
    m = _model("binary", rank)
    res["code.mixed"] = np.array(sr._err(lambda: m.fit_keys_dist(eng, users[:10], items[:10], ts[:10], np.ones(10, np.float32)))[0])
    eng.close()


def test_fit_keys_dist_equals_single_gpu(tmp_path):
    sr._needs_two()
    import torch.multiprocessing as mp
    mp.spawn(_worker, args=(sr._free_port(), str(tmp_path)), nprocs=WORLD, join=True)
    r0, r1 = np.load(tmp_path / "fit_0.npz"), np.load(tmp_path / "fit_1.npz")
    want = {}
    for name in CASES:
        ref = sm._reference(name, sm._tables(name)[2])
        _fits(ref, name, 0, None, want)
        ref.close()
    for key, w in want.items():
        sr._assert_same(r0[key], r1[key], key + " (rank 0 vs rank 1)")
        sr._assert_same(r0[key], w, key)
    for name in CASES:
        for mn in MODELS:
            assert int(r0["%s.%s.0.rows_used" % (name, mn)]) == 298       # one unknown user, one unknown item
    # one peer gather per minibatch of every epoch of the case's six fits, one record all-gather per fit
    batches = sum(int(r0["hot_trained.%s.%d.n_iter" % (mn, call)]) * -(-int(r0["hot_trained.%s.%d.rows_used" % (mn, call)]) // MODELS[mn][1]["batch"])
                  for mn in MODELS for call in (0, 1))
    for res in (r0, r1):
        assert int(res["prof.mlp_fit_gather_peer"]) == batches and int(res["prof.mlp_fit_gather_ranks"]) == 2 * len(MODELS)
        assert int(res["code.config"]) == g.EINVAL
        sr._assert_same(res["config.params"], res["before.params"], "params after a refused fit")
        assert int(res["code.unknown"]) == g.ENOTFOUND
        sr._assert_same(res["unknown.params"], res["before.params"], "params after ENOTFOUND")
        assert int(res["code.fit_keys"]) == g.ESTATE
        assert int(res["code.mixed"]) == g.ESTATE
