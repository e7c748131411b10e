"""Times search and top-k recommendation on a row-sharded ITEM_EMB (ctr_knn_search / ctr_recommend_topk are collective
there: each rank scans its own shard, the ranks' lists are merged).  Table: ctr_table_fill N(0,1), 100 M x 64 by default,
reserved[1] = 1, pred_batch 65 536.  Calls: one vector query (k = 10), 1024 vector queries (k = 10), one user's
recommendation (k = 100) over 10 M and over the full table.  Per call: CUDA events on the engine stream and host wall
time around the call, median of several runs after a warm-up.  One JSON line per rank, with the card's name and power
limit.  Launch:
    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 --master-port P \\
        tests/tools/shard_serve_time.py [rows] [reps]"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import go_ctr_b200 as g          # noqa: E402

uP, S, D, cF, PRED_BATCH = 52, 50, 64, 53, 65_536


def card(local):
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(local), "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return dict(name=out[0].strip(), power_limit_w=float(out[1]), sm_max_mhz=float(out[2]))
    except Exception as e:          # noqa: BLE001
        return dict(error=str(e))


def engine(rank, world, local, I):
    cfg = g.engine.default_config(g.MODEL_DIN_COS, uP=uP, S=S, D=D, cF=cF, pred_batch=PRED_BATCH, seed=3,
                                  device=local, rank=rank, world=world)
    cfg.reserved[1] = 1
    eng = g.Engine(cfg)
    ids = [eng.comm_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(ids, src=0)
    eng.comm_init(ids[0])
    eng.table_fill(g.TABLE_USER_FEAT, 1000, uP, seed=1)
    eng.table_fill(g.TABLE_ITEM_FEAT, I, cF, seed=2)
    eng.table_fill(g.TABLE_ITEM_EMB, I, D, seed=3, dist=1, scale=1.0)
    return eng


def timed(eng, stream, f, reps):
    for _ in range(2):
        f()
    dev, wall = [], []
    for _ in range(reps):
        dist.barrier()
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record(stream); f(); e1.record(stream); e1.synchronize()
        wall.append((time.perf_counter() - t0) * 1e3); dev.append(e0.elapsed_time(e1))
    return dict(device_ms=round(float(np.median(dev)), 3), wall_ms=round(float(np.median(wall)), 3), reps=reps)


def main():
    rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"]); local = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")
    I = int(sys.argv[1]) if len(sys.argv) > 1 else 100_000_000
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 7
    rng = np.random.default_rng(0)
    q1, q1024 = rng.standard_normal((1, D)), rng.standard_normal((1024, D))
    hist = rng.integers(0, min(I, 10_000_000), S).astype(np.int32)[None, :]
    res = dict(rank=rank, world=world, card=card(local), rows=I, D=D, pred_batch=PRED_BATCH)
    for n in sorted({min(I, 10_000_000), I}):
        eng = engine(rank, world, local, n)
        stream = torch.cuda.ExternalStream(eng.stream, device=torch.device("cuda", local))
        W = eng.get_weights()
        eng.set_weights(W[0] * 0.05, W[1] * 0.05, W[2] * 0.3, W[3])
        if n == I:
            res["knn_1q_k10"] = timed(eng, stream, lambda: eng.knn_search(10, queries=q1), reps)
            res["knn_1024q_k10"] = timed(eng, stream, lambda: eng.knn_search(10, queries=q1024), reps)
        res["rec_1u_k100_%dM" % (n // 1_000_000)] = timed(eng, stream, lambda: eng.recommend_topk([17], hist, 100, exclude_history=False), reps)
        eng.close()
    print(json.dumps({"shard_serve_time": res}))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
