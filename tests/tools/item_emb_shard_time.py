"""Times ctr_item_emb_train over a sharded item stream at W ranks, one process per GPU: n tokens of a Zipf stream over
sparse int64 item ids (a few percent of them unmapped), cut into W equal shards, trained into a row-sharded ITEM_EMB
(reserved[1] = 1; W = 1 is the single-GPU call on the whole stream).  Prints one JSON line per W with, on rank 0: the
wall time of the call (host clock around it; the call ends in a device synchronise), global tokens per second, and the
split between the numbering across ranks (profile key i2v_dict_ranks), the rest of the numbering (the other i2v_dict_*
keys), training (the trainer's device time) and the row write (i2v_emb_scatter); plus the GPU name and its power limit.
The first call of each W warms up and is not reported.

    python tests/tools/item_emb_shard_time.py --worlds 1 2 4 8 [--n 100000000] [--items 1000000] [--D 64]

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


def _stream(n, items, seed=0):
    rng = np.random.default_rng(seed)
    cat = rng.permutation(np.unique(rng.integers(-(1 << 62), 1 << 62, int(items * 1.05), dtype=np.int64)))[:items]
    ids = cat[(rng.zipf(1.05, n) - 1) % cat.size]
    imap = cat[np.arange(cat.size) % 32 != 5]                                # about 3 % of the items stay unmapped
    return ids, imap


def _worker(rank, W, port, n, items, D, out):
    import torch
    import go_ctr_b200 as g
    if W > 1:
        import torch.distributed as dist
        os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
        dist.init_process_group("gloo", rank=rank, world_size=W)
    torch.cuda.set_device(rank)
    cfg = g.engine.default_config(g.MODEL_DIN_COS, uP=4, S=5, D=D, cF=4, batch=256, pred_batch=256, device=rank, rank=rank, world=W)
    cfg.reserved[1] = 1
    eng = g.Engine(cfg)
    if W > 1:
        uid = [eng.comm_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(uid, src=0)
        eng.comm_init(uid[0])
    ids, imap = _stream(n, items)
    eng.idmap_build(g.IDMAP_ITEM, imap)
    shard = ids[rank * n // W:(rank + 1) * n // W]
    i2v = g.i2v_default_config(dim=D, window=5, iter=1, seed=3)
    res = {}
    for rep in range(2):                                                      # the first call warms up
        eng.profile(True); eng.profile_reset()
        if W > 1:
            dist.barrier()
        t0 = time.perf_counter()
        vocab, st = eng.item_emb_train(shard, cfg=i2v)
        wall = time.perf_counter() - t0
        prof = eng.profile_dump(); eng.profile(False)
        ms = lambda keys: sum(prof.get(k, (0.0, 0))[0] for k in keys)
        res = dict(world=W, tokens=n, items=items, D=D, V=int(vocab.size), wall_ms=wall * 1e3, tokens_per_s=n / wall,
                   dict_ranks_ms=ms(["i2v_dict_ranks"]), dict_local_ms=ms(["i2v_dict_resolve", "i2v_dict_side", "i2v_dict_rank", "i2v_dict_doc"]),
                   train_ms=st.ms_device, scatter_ms=ms(["i2v_emb_scatter"]))
    if rank == 0:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], stdout=subprocess.PIPE, text=True)
        res["gpu"] = q.stdout.strip()
        with open(out, "w") as f:
            json.dump(res, f)
    eng.close()
    if W > 1:
        dist.barrier(); dist.destroy_process_group()


def main():
    import torch
    import torch.multiprocessing as mp
    ap = argparse.ArgumentParser()
    ap.add_argument("--worlds", type=int, nargs="+", default=[1, 2, 4, 8])
    ap.add_argument("--n", type=int, default=10**8)
    ap.add_argument("--items", type=int, default=10**6)
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
            mp.spawn(_worker, args=(W, port, a.n, a.items, a.D, out), nprocs=W, join=True)
            with open(out) as f:
                print(json.dumps(json.load(f)))


if __name__ == "__main__":
    main()
