"""ms/step of the row-sharded train step with CTR_TABLE_ADAM against CTR_TABLE_SGD at the benchmark's default workload
(din_100m: 100M-row ITEM_EMB, D 64, S 50, 65536 samples per GPU, uniform ids, hot rows off), same tables, same batches,
the two optimisers alternated twice in one run; prints one JSON line with the card name and power limit beside the
numbers, plus the per-launch device times of one profiled Adam step.  Launch once per world size:
python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 --master-port P tests/tools/shard_adam_time.py [rows] [per_gpu_batch]"""
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import go_ctr_b200 as g          # noqa: E402
from tests.util import make_batch          # noqa: E402


def card(local):
    q = subprocess.run(["nvidia-smi", "-i", str(local), "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(local)


def main():
    rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"]); local = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    I = int(sys.argv[1]) if len(sys.argv) > 1 else 100_000_000
    B = int(sys.argv[2]) if len(sys.argv) > 2 else 65536
    U, uP, S, D, cF = 138_493, 52, 50, 64, 53
    rng = np.random.default_rng(100 + rank)
    batches = [make_batch(rng, U, I, B, S, pad_frac=0.2) for _ in range(4)]
    devb = [tuple(torch.from_numpy(a).to(dev) for a in b) for b in batches]

    def leg(topt, K=20, profile=False):
        cfg = g.engine.default_config(g.MODEL_DIN_COS, uP=uP, S=S, D=D, cF=cF, batch=B, pred_batch=B, table_opt=topt, table_lr=0.05,
                                      device=local, rank=rank, world=world, seed=1)
        cfg.reserved[0] = -1; cfg.reserved[1] = 1
        eng = g.Engine(cfg)
        ids = [eng.comm_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(ids, src=0)
        eng.comm_init(ids[0])
        eng.table_fill(g.TABLE_USER_FEAT, U, uP, 3, 0, 1.0); eng.table_fill(g.TABLE_ITEM_FEAT, I, cF, 4, 0, 1.0)
        eng.table_fill(g.TABLE_ITEM_EMB, I, D, 5, 1, float(1.0 / np.sqrt(D)))
        st = torch.cuda.ExternalStream(eng.stream, device=dev)

        def step(i):
            ur, ir, hist, y = devb[i % 4]
            eng.train_step_idx_dev(ur.data_ptr(), ir.data_ptr(), hist.data_ptr(), y.data_ptr(), B)
        for i in range(5):
            step(i)
        eng.sync(); dist.barrier()
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(st):
            e0.record(st)
            for i in range(K):
                step(i)
            e1.record(st)
        eng.sync(); torch.cuda.synchronize()
        t = torch.tensor([e0.elapsed_time(e1) / K], dtype=torch.float64, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        prof = None
        if profile:
            dist.barrier()
            eng.profile(True); eng.profile_reset()
            for i in range(4):
                step(i)
            eng.sync()
            prof = {k: round(v / n, 4) for k, (v, n) in eng.profile_dump().items()}
            eng.profile(False)
        dist.barrier()
        eng.close()
        torch.cuda.empty_cache()
        return float(t.item()), prof

    runs = {"sgd": [], "adam": []}
    prof = None
    for rep in range(2):
        runs["sgd"].append(leg(g.TABLE_SGD)[0])
        ms, p = leg(g.TABLE_ADAM, profile=rep == 1)
        runs["adam"].append(ms)
        prof = p or prof
    if rank == 0:
        sgd, adam = min(runs["sgd"]), min(runs["adam"])
        print(json.dumps({"world": world, "rows": I, "B_per_gpu": B, "card": card(local), "ms_per_step": runs,
                          "best_sgd_ms": round(sgd, 3), "best_adam_ms": round(adam, 3), "adam_extra_ms": round(adam - sgd, 3),
                          "adam_profile_ms": prof}))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
