"""Times one epoch of ctr_mlp_fit_keys_dist (the key-fed float64 MLP trained on a multi-GPU feature store: every rank
resolves its own keys, the survivor records are all-gathered, and every rank runs the same fit, layer 0's rows read from
their owners through the peer gather) at world 1, 2, 4 and 8 over the same keys.
Store: the widths of the other sharded tools (uP 52, S 50, D 64, cF 53), ITEM_EMB and ITEM_FEAT ctr_table_fill'ed with
100 M rows by default, reserved[1] = 1 (both row-sharded when world > 1, the default 32 768 hot rows), an ubcache of 50
events for each of 10 000 users.  Keys: 100 000, every one known (so 100 000 survivors), cut into `world` equal
consecutive parts in rank order.  Model: the reference's classifier, hidden (100,), batch 200, max_iter 1 (one epoch).
Rounds alternate the worlds: in each round every world builds its store, fits once to warm up, times one fit (host wall
time around the call, which returns after the device has finished) and closes the store.  Reported per world: the median
over the rounds, and a profiled fit (mlp_fit_gather_peer / mlp_gather: one gather per minibatch; mlp_fit_gather_ranks:
the record all-gather).  One JSON line from rank 0, with the card's name and power limit.  Worlds above the launch's
process count are skipped.  Launch (one GPU: plain python):
    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 --master-port P \\
        tests/tools/shard_mlp_fit_time.py [--rows R] [--keys K] [--rounds n]"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import shard_rank_time as srt                    # noqa: E402  (the card helper)

g = srt.g
uP, S, D, cF = srt.uP, 50, 64, srt.cF
USERS = 10_000


def store(I, rank, world, local):
    cfg = g.engine.default_config(g.MODEL_DIN_COS, uP=uP, S=S, D=D, cF=cF, seed=3, device=local, rank=rank, world=world)
    cfg.reserved[1] = 1
    eng = g.Engine(cfg)
    if world > 1:
        ids = [eng.comm_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(ids, src=0, group=sub(world))
        eng.comm_init(ids[0])
    eng.table_fill(g.TABLE_USER_FEAT, USERS, uP, seed=1)
    eng.table_fill(g.TABLE_ITEM_FEAT, I, cF, seed=2)
    eng.table_fill(g.TABLE_ITEM_EMB, I, D, seed=3, dist=1, scale=1.0)
    eng.idmap_build(0, np.arange(USERS, dtype=np.int64))
    eng.idmap_build(1, np.arange(I, dtype=np.int64))
    rng = np.random.default_rng(4)
    off = np.arange(0, 50 * (USERS + 1), 50, dtype=np.int64)
    ts = np.tile(np.arange(100, 50, -1, dtype=np.int64), USERS)
    eng.ubcache_upload(off, ts, rng.integers(0, I, 50 * USERS).astype(np.int32))
    return eng


_groups = {}


def sub(world):
    """the process group of ranks [0, world) (created on every process, in the same order)"""
    return _groups[world]


def keys(n, I):
    rng = np.random.default_rng(6)
    return (rng.integers(0, USERS, n).astype(np.int64), rng.integers(0, I, n).astype(np.int64), rng.integers(60, 120, n).astype(np.int64),
            (rng.random(n) < 0.3).astype(np.float32))


def fit_once(eng, local, part, profile=False):
    m = g.engine.MLPClassifier(uP + S * D + D + cF, hidden=(100,), batch=200, max_iter=1, seed=7, device=local)
    if profile:
        eng.profile(True); eng.profile_reset()
    t0 = time.perf_counter()
    m.fit_keys_dist(eng, *part)
    ms = (time.perf_counter() - t0) * 1e3
    prof = None
    if profile:
        prof = {k: [round(v[0], 3), v[1]] for k, v in sorted(eng.profile_dump().items()) if k.startswith("mlp_")}
        eng.profile(False)
    used = m.rows_used
    m.close()
    return ms, used, prof


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--keys", type=int, default=100_000)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    launched = "RANK" in os.environ
    rank = int(os.environ.get("RANK", 0)); nproc = int(os.environ.get("WORLD_SIZE", 1)); local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    if launched:
        dist.init_process_group("gloo")
    worlds = [w for w in (1, 2, 4, 8) if w <= nproc]
    for w in worlds:
        if w > 1:
            _groups[w] = dist.new_group(list(range(w)))
    allk = keys(a.keys, a.rows)
    res = dict(card=srt.card(local), rows=a.rows, keys=a.keys, uP=uP, S=S, D=D, cF=cF, hidden=[100], batch=200, rounds=a.rounds, worlds={})
    times = {w: [] for w in worlds}
    prof = {}
    for rd in range(a.rounds):
        for w in worlds:
            if rank < w:
                lo, hi = rank * a.keys // w, (rank + 1) * a.keys // w
                part = [x[lo:hi] for x in allk]
                eng = store(a.rows, rank, w, local)
                fit_once(eng, local, part)                                     # warm-up: lazy buffers, the publish
                ms, used, _ = fit_once(eng, local, part)
                times[w].append(ms)
                if rd == 0:
                    _, _, prof[w] = fit_once(eng, local, part, profile=True)
                    assert used == a.keys, (used, a.keys)
                eng.close()
                torch.cuda.empty_cache()
            if launched:
                dist.barrier()
    if rank == 0:                                                              # rank 0 takes part in every world
        for w in worlds:
            res["worlds"][str(w)] = dict(fit_epoch_ms=round(float(np.median(times[w])), 2), runs_ms=[round(t, 2) for t in times[w]], profile=prof[w])
        print(json.dumps({"shard_mlp_fit_time": res}))
    if launched:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
