"""Times CTR_EXCLUDE_SEEN against CTR_EXCLUDE_WINDOW on a row-sharded ITEM_EMB (each rank marks the rows it owns in a
bitmap of its local rows, from its own behaviour cache, before scoring its shard).  Table: ctr_table_fill N(0,1), 10 M
and 100 M x 64 by default, reserved[1] = 1, pred_batch 65 536, north-star widths.  The same ubcache on every rank: one
user with 10^3, 10^4, 10^5 and 10^6 cached events of distinct items, all before the cut.  Calls: recommend_topk_ex with
k = 100 and rank_items_ex with 16 targets (one scoring pass), the two modes alternated in one process; per call the
median of 5 CUDA-event timings on the engine stream (and host wall time) after a warm-up, and a profiled SEEN call.  One
JSON line per rank, with the card's name and power limit.  Needs 2, 4 or 8 GPUs (a sharded table).  Launch:
    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 --master-port P \\
        tests/tools/shard_seen_time.py [rows ...] [--events E ...] [--reps R]"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import shard_rank_time as srt                    # noqa: E402  (the table, engine and card helpers)

S, K, CUT = srt.S, 100, 10 ** 9


def cache(n_items, n_events, user):
    """user `user` with n_events events of distinct items, time-descending, all at or before CUT"""
    rng = np.random.default_rng(n_events)
    lens = np.zeros(user + 1, np.int64); lens[user] = n_events
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    ts = (CUT - np.arange(n_events, dtype=np.int64))
    items = rng.choice(n_items, n_events, replace=False).astype(np.int32)
    return off, ts, items


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("rows", type=int, nargs="*", default=[10_000_000, 100_000_000])
    ap.add_argument("--events", type=int, nargs="*", default=[1_000, 10_000, 100_000, 1_000_000])
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"]); local = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")
    res = dict(rank=rank, world=world, card=srt.card(local), D=srt.D, S=S, pred_batch=srt.PRED_BATCH, k=K, targets=16, cases=[])
    for n in a.rows:
        rng = np.random.default_rng(0)
        user, hist = 17, rng.integers(0, n, S).astype(np.int32)
        t16 = rng.integers(0, n, 16).astype(np.int32)
        eng = srt.engine(rank, world, local, n)
        stream = torch.cuda.ExternalStream(eng.stream, device=torch.device("cuda", local))
        u16, h16, c16 = np.full(16, user, np.int32), np.tile(hist, (16, 1)), np.full(16, CUT, np.int64)
        calls = {
            "rec_window": lambda: eng.recommend_topk([user], hist[None, :], K, exclude_history=True),
            "rec_seen": lambda: eng.recommend_topk([user], hist[None, :], K, max_ts=[CUT], exclude_seen=True),
            "rank_window": lambda: eng.rank_items(u16, h16, t16, exclude_history=True),
            "rank_seen": lambda: eng.rank_items(u16, h16, t16, max_ts=c16, exclude_seen=True),
        }
        for ne in a.events:
            eng.ubcache_upload(*cache(n, min(ne, n), user))
            for f in calls.values():                     # warm-up
                f()
            times = {name: [] for name in calls}
            for _ in range(a.reps):                      # the modes alternated
                for name, f in calls.items():
                    dist.barrier()
                    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
                    t0 = time.perf_counter()
                    e0.record(stream); f(); e1.record(stream); e1.synchronize()
                    times[name].append((e0.elapsed_time(e1), (time.perf_counter() - t0) * 1e3))
            med = {name: dict(device_ms=round(float(np.median([t[0] for t in v])), 3), wall_ms=round(float(np.median([t[1] for t in v])), 3),
                              spread_ms=round(float(np.ptp([t[0] for t in v])), 3)) for name, v in times.items()}
            res["cases"].append(dict(rows=n, events=ne, reps=a.reps, **med, profile_rank_seen=srt.profiled(eng, calls["rank_seen"]),
                                     profile_rec_seen=srt.profiled(eng, calls["rec_seen"])))
        eng.close()
    print(json.dumps({"shard_seen_time": res}))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
