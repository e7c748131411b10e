"""world_size-2 gloo test (CPU) of CTR_TABLE_ADAM on the row-sharded placement (tests/shard_adam_model.py, built on tests/shard_model.py):
owner-side gradient sums, the touched set by occurrence, lazy Adam at the owner and the hot rows replicated with their
own moments == a numpy single-table lazy Adam on the global batch.  Covered: a touched row whose summed gradient is
exactly 0 (cold and hot), a ragged tail, ids of -1 and ids past the table, rows on both sides of hot_k."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests import shard_adam_model as sh
from tests import shard_model

WORLD, I, D, B, S, STEPS, HOT_K = 2, 241, 8, 13, 4, 3, 10
LR, B1, B2, EPS = 0.01, 0.9, 0.999, 1e-8
NVALID = {(2, 1): 7}                     # (step, rank) → valid samples of a ragged tail
ZERO_COLD, ZERO_HOT = 20, 3              # touched in step 1 with a gradient sum of exactly 0 (over both ranks)


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _table():
    return np.random.default_rng(123).standard_normal((I, D)).astype(np.float32)


def _step_data(step):
    """every rank's (lookups [B, S+1], grads [B, S+1, D]) of one step, the same on every process"""
    rng = np.random.default_rng(1000 + step)
    out = []
    for rank in range(WORLD):
        hist = rng.integers(-1, I + 3, (B, S))              # -1 and ids past the table included
        item = rng.integers(0, I + 2, B)
        grads = rng.standard_normal((B, S + 1, D)).astype(np.float32)
        out.append([hist, item, grads])
    gz = np.random.default_rng(7).standard_normal(D).astype(np.float32)
    for row, col in ((ZERO_COLD, 0), (ZERO_HOT, 1)):
        for rank in range(WORLD):
            h, it, gr = out[rank]
            h[h == row] = -1; it[it == row] = I + 1
            if step <= 1:                                   # step 0: one occurrence on rank 0; step 1: +gz on rank 0, -gz on rank 1
                if step == 1 or rank == 0:
                    h[0, col] = row
                    gr[0, col] = gz if rank == 0 else -gz
    res = []
    for rank, (h, it, gr) in enumerate(out):
        look = sh.valid_lookups(h, it, I, NVALID.get((step, rank), B))
        res.append((look, gr))
    return res


def _worker(rank, world, port, out_dir):
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    table = _table()
    shard = shard_model.shard_table(table, rank, world)
    st = dict(shard=shard.copy(), m=np.zeros_like(shard), v=np.zeros_like(shard),
              hot=table[:HOT_K].copy(), hot_m=np.zeros((HOT_K, D), np.float32), hot_v=np.zeros((HOT_K, D), np.float32))
    for step in range(STEPS):
        look, grads = _step_data(step)[rank]
        sh.adam_step_sharded(dist, torch, st, rank, world, look, grads, HOT_K, step + 1, LR, B1, B2, EPS, 1.0 / (world * B))
    np.savez(os.path.join(out_dir, "st%d.npz" % rank), **st)
    dist.barrier()
    dist.destroy_process_group()


def _reference():
    """one table, one process, the global batch: every distinct valid row once with its summed gradient"""
    w = _table(); m = np.zeros_like(w); v = np.zeros_like(w)
    trace = []
    for step in range(STEPS):
        g = np.zeros((I, D), np.float64); touched = np.zeros(I, bool)
        for look, grads in _step_data(step):
            f = look.reshape(-1); ok = f >= 0
            np.add.at(g, f[ok], grads.reshape(-1, D)[ok].astype(np.float64))
            touched[f[ok]] = True
        tr = np.nonzero(touched)[0]
        ww, mm, vv = w[tr], m[tr], v[tr]
        sh.row_adam(ww, mm, vv, g[tr].astype(np.float32), step + 1, LR, B1, B2, EPS, 1.0 / (WORLD * B))
        w[tr], m[tr], v[tr] = ww, mm, vv
        trace.append((touched, g, w.copy(), m.copy(), v.copy()))
    return w, m, v, trace


def test_valid_lookups_marks_missing_and_tail():
    hist = np.array([[4, -1, 9], [2, 12, 0]]); item = np.array([10, 3])
    look = sh.valid_lookups(hist, item, 11, 1)
    assert look.tolist() == [[4, -1, 9, 10], [-1, -1, -1, -1]]


def test_reference_touches_by_occurrence():
    """the reference itself: rows whose summed gradient is exactly 0 in step 1 are touched, their moments decay and
    they move; the sharded leg is compared against exactly this"""
    _, _, _, trace = _reference()
    (t0, _, w0, m0, v0), (t1, g1, w1, m1, v1) = trace[0], trace[1]
    for row in (ZERO_COLD, ZERO_HOT):
        assert t1[row] and not g1[row].any()
        assert np.array_equal(m1[row], np.float32(B1) * m0[row]) and np.abs(m0[row]).max() > 0
        assert np.abs(w1[row] - w0[row]).max() > 1e-4


@pytest.mark.timeout(120)
def test_sharded_row_adam_two_ranks_gloo(tmp_path):
    mp.spawn(_worker, args=(WORLD, _free_port(), str(tmp_path)), nprocs=WORLD, join=True)
    st = [dict(np.load(tmp_path / ("st%d.npz" % r))) for r in range(WORLD)]
    for k in ("hot", "hot_m", "hot_v"):                      # identical replicas of the hot rows and their moments
        assert st[0][k].tobytes() == st[1][k].tobytes()
    got = sh.assemble_sharded(st, WORLD, HOT_K)
    w, m, v, trace = _reference()
    ever = np.zeros(I, bool)
    for t, *_ in trace:
        ever |= t
    assert ever[:HOT_K].any() and ever[HOT_K:].any() and (~ever).any()
    table = _table()
    for a, b in ((got["shard"], table), (got["m"], np.zeros_like(table)), (got["v"], np.zeros_like(table))):
        assert a[~ever].tobytes() == b[~ever].astype(np.float32).tobytes()         # untouched rows: bit for bit
    np.testing.assert_allclose(got["shard"], w, rtol=1e-5, atol=1e-7)
    # the moments carry the replicated placement's scaling: gradients enter scaled by 1/world
    np.testing.assert_allclose(got["m"] * WORLD, m, rtol=1e-4, atol=1e-9)
    np.testing.assert_allclose(got["v"] * WORLD ** 2, v, rtol=1e-4, atol=1e-12)
    assert np.abs(w[ever] - table[ever]).max() > 0.5 * LR
