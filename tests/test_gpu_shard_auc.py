"""ROC AUC and GAUC over every rank's samples on a multi-GPU handle (ctr_roc_auc_dist, ctr_group_auc_dist; needs >= 2
GPUs): every rank passes its own samples, and every rank's result must equal, bit for bit, roc_auc / group_auc on one
GPU over the ranks' samples concatenated in rank order, the per-group arrays included.  Cases: random scores and groups,
tied scores, all scores equal, NaN / ±0 / ±inf scores, a group on every rank, group ids INT64_MIN and INT64_MAX, one
class absent, rank 0 passing no samples.  Refusals: bad arguments on rank 1 only (every rank returns rank 1's code and
message, nothing written), no samples on any rank, ranks in different calls, and a cap below the group count."""
import os

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

import go_ctr_b200 as g
from tests import test_gpu_shard_rank as sr

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

WORLD = sr.WORLD
CASES = ["random", "ties", "equal", "special", "every_rank", "extremes", "one_class", "empty_rank0"]


def _case(name):
    rng = np.random.default_rng(CASES.index(name))
    n = 50_000
    pred = rng.random(n).astype(np.float32)
    if name in ("ties", "every_rank", "extremes"):
        pred = (rng.integers(0, 15, n) / 14).astype(np.float32)
    if name == "equal":
        pred[:] = 1.0
    if name == "special":
        pool = np.r_[np.array([0.0, -0.0, np.inf, -np.inf, 0.5], np.float32), np.array([0x7fc00000, 0xffc00000, 0x7f800001], np.uint32).view(np.float32)]
        pred = pool[rng.integers(0, pool.size, n)]
    y = (rng.random(n) < 0.35).astype(np.float32)
    if name == "one_class":
        y[:] = 0.0
    grp = rng.integers(0, 3000, n).astype(np.int64)
    if name == "extremes":
        grp = rng.choice(np.array([np.iinfo(np.int64).min, np.iinfo(np.int64).max, -1, 0], np.int64), n)
    cut = 0 if name == "empty_rank0" else int(n * 0.4)
    if name == "every_rank":
        grp[0] = grp[cut] = 11
    return pred, y, grp, [0, cut, n]


def _cfg(r):
    return g.engine.default_config(g.MODEL_DIN_COS, batch=1, pred_batch=1, device=r, rank=r, world=WORLD)


def _bits(x):
    return np.asarray(x, np.float64).view(np.int64)


def _worker(rank, port, out_dir):
    sr._init(rank, port)
    eng = sr._engine(rank, _cfg)
    res = {}
    for name in CASES:
        pred, y, grp, cuts = _case(name)
        s = slice(cuts[rank], cuts[rank + 1])
        res[name + "_auc"] = np.float64(eng.roc_auc_dist(pred[s], y[s]))
        ga = eng.group_auc_dist(pred[s], y[s], grp[s], per_group=True)
        res[name + "_gauc"] = np.array([ga[0]]); res[name + "_counts"] = np.array(ga[1:3])
        for k, v in ga[3].items():
            res[name + "_pg_" + k] = v
    # refusals: rank 1's arguments are bad; every rank returns its code and message and writes nothing
    bad = None if rank == 1 else np.ones(3, np.float32)
    L, h = eng.L, eng.h
    import ctypes as C
    fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float)) if a is not None else None
    auc = C.c_double(-7.0)
    p3 = np.ones(3, np.float32)
    rc = L.ctr_roc_auc_dist(h, fp(p3), fp(bad), C.c_int64(3), C.byref(auc))
    res["bad_rc"] = np.array([rc, int(auc.value == -7.0)]); res["bad_msg"] = np.frombuffer(L.ctr_last_error(h), np.uint8)
    res["none"] = np.array([sr._err(lambda: eng.roc_auc_dist([], []))[0], sr._err(lambda: eng.group_auc_dist([], [], []))[0]])
    # rank 0 in roc_auc_dist, rank 1 in group_auc_dist: both refuse
    pred, y, grp, _ = _case("random")
    res["mixed"] = np.array([sr._err(lambda: eng.roc_auc_dist(pred[:10], y[:10]) if rank == 0 else eng.group_auc_dist(pred[:10], y[:10], grp[:10]))[0]])
    # cap 1 below the group count: refused on both, nothing written
    gauc = C.c_double(-7.0); og = np.full(4, -9, np.int64)
    rc = L.ctr_group_auc_dist(h, fp(pred[:100]), fp(y[:100]), grp[:100].ctypes.data_as(C.POINTER(C.c_int64)), C.c_int64(100), C.byref(gauc), None,
                              None, C.c_int64(1), og.ctypes.data_as(C.POINTER(C.c_int64)), None, None, None)
    res["cap"] = np.array([rc, int(gauc.value == -7.0), int((og == -9).all())])
    np.savez(os.path.join(out_dir, "rank%d.npz" % rank), **res)


def test_ranks_equal_one_gpu(tmp_path):
    sr._needs_two()
    mp.spawn(_worker, args=(sr._free_port(), str(tmp_path)), nprocs=WORLD, join=True)
    one = g.Engine(g.engine.default_config(g.MODEL_DIN_COS, batch=1, pred_batch=1))
    for rank in range(WORLD):
        got = np.load(os.path.join(tmp_path, "rank%d.npz" % rank))
        for name in CASES:
            pred, y, grp, _ = _case(name)
            assert _bits(got[name + "_auc"]) == _bits(one.roc_auc(pred, y)), (rank, name)
            want = one.group_auc(pred, y, grp, per_group=True)
            assert _bits(got[name + "_gauc"][0]) == _bits(want[0]) and tuple(got[name + "_counts"]) == want[1:3], (rank, name)
            for k in ("group", "n", "pos"):
                assert np.array_equal(got[name + "_pg_" + k], want[3][k]), (rank, name, k)
            assert np.array_equal(_bits(got[name + "_pg_auc"]), _bits(want[3]["auc"])), (rank, name)
        assert tuple(got["bad_rc"]) == (g.EINVAL, 1) and b"bad auc_dist arguments" in got["bad_msg"].tobytes(), rank
        assert tuple(got["none"]) == (g.EINVAL, g.EINVAL) and tuple(got["mixed"]) == (g.EINVAL,)
        assert tuple(got["cap"]) == (g.EINVAL, 1, 1)
