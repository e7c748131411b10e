"""Times the collective live-table calls on a multi-GPU handle: 10^6 new item ids inserted (spread over the ranks, a
tenth of them new on two ranks) and their ITEM_EMB rows written (each rank writes the rows of its own new ids), on a
row-sharded ITEM_EMB (reserved[1] = 1) at W ranks, one process per GPU.  Prints one JSON line per W with the wall time
of each call (host clock around the call, which synchronises the engine stream) on rank 0, the GPU name and its power
limit.

    python tests/tools/shard_live_time.py --worlds 2 4 8 [--n 1000000] [--D 64]

Needs as many GPUs as the largest W; smaller boxes skip the larger W."""
import argparse
import json
import os
import socket
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def _worker(rank, W, port, n, D, out):
    import torch
    import torch.distributed as dist
    import go_ctr_b200 as g
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=W)
    torch.cuda.set_device(rank)
    cfg = g.engine.default_config(g.MODEL_DIN_COS, uP=4, S=5, D=D, cF=4, batch=256, pred_batch=256, device=rank, rank=rank, world=W)
    cfg.reserved[1] = 1
    eng = g.Engine(cfg)
    uid = [eng.comm_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(uid, src=0)
    eng.comm_init(uid[0])
    base = 10**6
    rng = np.random.default_rng(1)
    eng.table_upload(g.TABLE_ITEM_EMB, rng.standard_normal((base, D)).astype(np.float32))
    eng.idmap_build(g.IDMAP_ITEM, np.arange(base, dtype=np.int64))
    ids = 10**9 + np.arange(n, dtype=np.int64)
    mine = ids[rank::W]
    mine = np.concatenate([mine, ids[(rank + 1) % W::W][: mine.size // 10]])          # some ids new on two ranks
    res = {}
    for rep in range(2):                                    # the first pass warms up (publish, allocations)
        dist.barrier()
        t0 = time.perf_counter()
        rows = eng.idmap_insert(g.IDMAP_ITEM, mine + rep * 10**10)
        t1 = time.perf_counter()
        own = np.unique(rows[rows % W == rank])
        data = rng.standard_normal((own.size, D)).astype(np.float32)
        dist.barrier()
        t2 = time.perf_counter()
        eng.table_write_rows(g.TABLE_ITEM_EMB, own.astype(np.int32), data)
        t3 = time.perf_counter()
        res = {"insert_ms": (t1 - t0) * 1e3, "write_ms": (t3 - t2) * 1e3, "rows_written": int(own.size)}
    if rank == 0:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], stdout=subprocess.PIPE, text=True)
        res.update(world=W, new_ids=n, D=D, gpu=q.stdout.strip())
        with open(out, "w") as f:
            json.dump(res, f)
    eng.close()
    dist.barrier(); dist.destroy_process_group()


def main():
    import torch
    import torch.multiprocessing as mp
    ap = argparse.ArgumentParser()
    ap.add_argument("--worlds", type=int, nargs="+", default=[2, 4, 8])
    ap.add_argument("--n", type=int, default=10**6)
    ap.add_argument("--D", type=int, default=64)
    a = ap.parse_args()
    import tempfile
    for W in a.worlds:
        if W > torch.cuda.device_count():
            print(json.dumps({"world": W, "skipped": "needs %d GPUs" % W}))
            continue
        s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
        with tempfile.TemporaryDirectory() as d:
            out = os.path.join(d, "r.json")
            mp.spawn(_worker, args=(W, port, a.n, a.D, out), nprocs=W, join=True)
            with open(out) as f:
                print(json.dumps(json.load(f)))


if __name__ == "__main__":
    main()
