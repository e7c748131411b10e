"""Times the full-catalogue rank of held-out items on a row-sharded ITEM_EMB (ctr_rank_items is collective there: each
rank counts its own shard against the targets, whose logits come from their owners, and the ranks' counts are summed).
Table: ctr_table_fill N(0,1), 10 M and 100 M x 64 by default, reserved[1] = 1, pred_batch 65 536, north-star widths.
Calls: one user with 1 and with 16 held-out items (one scoring pass).  Per call: CUDA events on the engine stream and host
wall time around the call, median of several runs after a warm-up, and a profiled pass.  One JSON line per rank, with
the card's name and power limit.  Launch:
    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 --master-port P \\
        tests/tools/shard_rank_time.py [rows ...] [--reps R]"""
import argparse
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
    W = eng.get_weights()
    eng.set_weights(W[0] * 0.05, W[1] * 0.05, W[2] * 0.3, W[3])
    return eng


def timed(stream, f, reps):
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


def profiled(eng, f):
    eng.profile(True); eng.profile_reset()
    f()
    prof = eng.profile_dump(); eng.profile(False)
    return {k: [round(v[0], 3), v[1]] for k, v in sorted(prof.items())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("rows", type=int, nargs="*", default=[10_000_000, 100_000_000])
    ap.add_argument("--reps", type=int, default=7)
    a = ap.parse_args()
    rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"]); local = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")
    res = dict(rank=rank, world=world, card=card(local), D=D, S=S, pred_batch=PRED_BATCH, cases=[])
    for n in a.rows:
        rng = np.random.default_rng(0)
        user, hist = 17, rng.integers(0, n, S).astype(np.int32)
        t16 = rng.integers(0, n, 16).astype(np.int32)
        eng = engine(rank, world, local, n)
        stream = torch.cuda.ExternalStream(eng.stream, device=torch.device("cuda", local))
        r1 = lambda: eng.rank_items([user], hist[None, :], t16[:1], exclude_history=False)                         # noqa: E731
        r16 = lambda: eng.rank_items(np.full(16, user, np.int32), np.tile(hist, (16, 1)), t16, exclude_history=False)  # noqa: E731
        res["cases"].append(dict(rows=n, rank_1=timed(stream, r1, a.reps), rank_16=timed(stream, r16, a.reps), profile_16=profiled(eng, r16)))
        eng.close()
    print(json.dumps({"shard_rank_time": res}))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
