"""Times ctr_roc_auc_dist and ctr_group_auc_dist at world 1, 2, 4 and 8 (as many as the machine has GPUs), each rank
holding --n samples (10^8 by default), against the host-gather route a sharded deployment has without them: every
rank's predictions, labels and groups gathered to rank 0's host, concatenated, and ctr_roc_auc / ctr_group_auc run
there on one GPU.  Both routes must give the same bits.  A world the machine cannot run is printed as not measured.

    python tests/tools/auc_dist_time.py [--n 100000000] [--groups 1000000] [--rounds 3]

Prints one JSON line per world: the median wall time of each call over the rounds (every rank synchronised with a
barrier before and after), the GPU's name and power limit."""
import argparse
import json
import os
import socket
import subprocess
import sys
import time

import numpy as np
import torch
import torch.multiprocessing as mp

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import go_ctr_b200 as g  # noqa: E402


def _data(rank, n, groups):
    rng = np.random.default_rng(rank)
    pred = (rng.integers(0, 1 << 20, n) / (1 << 20)).astype(np.float32)
    y = (rng.random(n) < 0.3).astype(np.float32)
    grp = rng.integers(0, groups, n).astype(np.int64)
    return pred, y, grp


def _worker(rank, world, port, a, out):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.cuda.set_device(rank)
    eng = g.Engine(g.engine.default_config(g.MODEL_DIN_COS, batch=1, pred_batch=1, device=rank, rank=rank, world=world))
    if world > 1:
        ids = [eng.comm_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(ids, src=0)
        eng.comm_init(ids[0])
    pred, y, grp = _data(rank, a.n, a.groups)

    def gathered(fn):
        parts = [None] * world if rank == 0 else None
        dist.gather_object((pred, y, grp), parts, dst=0)
        r = [None]
        if rank == 0:
            r = [fn(*(np.concatenate([p[i] for p in parts]) for i in range(3)))]
        dist.broadcast_object_list(r, src=0)
        return r[0]

    routes = {
        "roc_dist": lambda: eng.roc_auc_dist(pred, y),
        "roc_gather": lambda: gathered(lambda p, t, _: eng.roc_auc(p, t)),
        "gauc_dist": lambda: eng.group_auc_dist(pred, y, grp),
        "gauc_gather": lambda: gathered(lambda p, t, q: eng.group_auc(p, t, q)),
    }
    res = {}
    for name, fn in routes.items():
        if world * a.n >= 1 << 31 and name.endswith("gather"):
            res[name] = None                                            # one GPU refuses 2^31 samples or more
            continue
        val, ts = None, []
        for _ in range(a.rounds + 1):
            dist.barrier(); t0 = time.perf_counter()
            val = fn()
            dist.barrier(); ts.append(time.perf_counter() - t0)
        res[name] = dict(ms=1e3 * float(np.median(ts[1:])), value=val)
    if rank == 0:
        out.put(res)
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000_000)
    ap.add_argument("--groups", type=int, default=1_000_000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--worlds", default="1,2,4,8")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("auc_dist_time: no GPU; nothing is measured")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()[0]
    ctx = mp.get_context("spawn")
    for world in (int(w) for w in a.worlds.split(",")):
        if world > torch.cuda.device_count():
            print(json.dumps(dict(world=world, n_per_rank=a.n, measured=False, reason="%d GPUs here" % torch.cuda.device_count())))
            continue
        s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
        q = ctx.Queue()
        mp.start_processes(_worker, args=(world, port, a, q), nprocs=world, join=True, start_method="spawn")
        res = q.get()
        for k in ("roc", "gauc"):
            d, h = res[k + "_dist"], res[k + "_gather"]
            if h is not None:
                assert np.array_equal(np.float64(d["value"][0] if k == "gauc" else d["value"]).view(np.int64),
                                      np.float64(h["value"][0] if k == "gauc" else h["value"]).view(np.int64)), (k, d, h)
        print(json.dumps(dict(world=world, n_per_rank=a.n, groups=a.groups, measured=True, gpu=gpu,
                              **{k: (None if v is None else round(v["ms"], 2)) for k, v in res.items()})), flush=True)


if __name__ == "__main__":
    main()
