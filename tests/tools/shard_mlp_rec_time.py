"""Times the key-fed float64 MLP's recommendation and held-out rank on a row-sharded ITEM_EMB (collective: each rank
scores its own shard for rank 0's windows; per group of 256 users one window broadcast and one list all-gather, per rank
pass a target-logit all-gather and a bin sum) against the same calls on one GPU holding the whole table.
Table: ctr_table_fill N(0,1), D = 64, S = 50, 10 M and 100 M rows by default, reserved[1] = 1, pred_batch 65 536,
north-star uP / cF, hidden (100,), an ubcache of 50 events per user.  Calls: ctr_mlp_recommend_topk with k = 100 for 1 and
for 300 users, ctr_mlp_rank_items with 16 targets of one user (one pass).  Per call: CUDA events on the engine stream
and host wall time, median of several runs after a warm-up, and a profiled call.  Rank 0 then times the same calls on a
single-GPU store of the same rows (when the table fits one GPU).  One JSON line per rank, with the card's name and
power limit.  Needs 2, 4 or 8 GPUs.  Launch:
    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 --master-port P \\
        tests/tools/shard_mlp_rec_time.py [rows ...] [--reps R] [--no-single]"""
import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import shard_rank_time as srt                    # noqa: E402  (the card, timing and profile helpers)

g = srt.g
uP, S, D, cF, PRED_BATCH, K, USERS = srt.uP, 50, 64, srt.cF, srt.PRED_BATCH, 100, 1000


def store(I, rank=0, world=1, local=0):
    cfg = g.engine.default_config(g.MODEL_DIN_COS, uP=uP, S=S, D=D, cF=cF, pred_batch=PRED_BATCH, seed=3, device=local, rank=rank, world=world)
    cfg.reserved[1] = 1
    eng = g.Engine(cfg)
    if world > 1:
        ids = [eng.comm_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(ids, src=0)
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


def model(local):
    m = g.engine.MLPClassifier(uP + S * D + D + cF, hidden=(100,), device=local)
    m.set_params(np.random.default_rng(5).standard_normal(m.get_params().size) * 0.02)
    return m


def measure(eng, m, local, I, reps):
    stream = torch.cuda.ExternalStream(eng.stream, device=torch.device("cuda", local))
    rng = np.random.default_rng(6)
    users = rng.integers(0, USERS, 300).astype(np.int64); ts = np.full(300, 1000, np.int64)
    items = rng.integers(0, I, 16).astype(np.int64)
    calls = {
        "rec_1user": lambda: m.recommend_topk(eng, users[:1], ts[:1], K),
        "rec_300users": lambda: m.recommend_topk(eng, users, ts, K),
        "rank_16": lambda: m.rank_items(eng, np.full(16, users[0]), items, np.full(16, 1000, np.int64)),
    }
    out = {name: srt.timed(stream, f, reps) for name, f in calls.items()}
    out["profile_rec_1user"] = srt.profiled(eng, calls["rec_1user"])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("rows", type=int, nargs="*", default=[10_000_000, 100_000_000])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-single", action="store_true")
    a = ap.parse_args()
    rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"]); local = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")
    res = dict(rank=rank, world=world, card=srt.card(local), D=D, S=S, pred_batch=PRED_BATCH, k=K, targets=16, cases=[])
    m = model(local)
    for n in a.rows:
        eng = store(n, rank, world, local)
        case = dict(rows=n, sharded=measure(eng, m, local, n, a.reps))
        eng.close()
        dist.barrier()
        if rank == 0 and not a.no_single:
            try:
                one = store(n)
            except g.CtrError as e:                      # the whole table does not fit one GPU
                case["single"] = dict(error=str(e))
            else:
                case["single"] = measure(one, m, local, n, a.reps)
                one.close()
        dist.barrier()
        res["cases"].append(case)
    print(json.dumps({"shard_mlp_rec_time": res}))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
