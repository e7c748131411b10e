"""Times the live id-map and table calls against today's route for admitting new items, and prints one JSON line.

    live route:   ctr_idmap_insert of m ids (half of them new), ctr_table_write_rows of m rows inside ITEM_EMB, and of
                  m rows appended past its end (the table grows in place)
    today's route: ctr_idmap_build of every id plus ctr_table_upload of the whole ITEM_EMB

ITEM_EMB is made by ctr_table_fill at R rows x 64 (default R in {10^7, 10^8}), the item map by ctr_idmap_build of R
sparse int64 ids; m in {1, 10^3, 10^5, 10^7}.  Each call is timed once after a warm-up of the same call at m = 1:
CUDA-event time on the engine stream and host wall time around the call (which ends in a device synchronise).  The
upload route needs a host copy of the whole table; it is skipped (reported null) when the host has less free memory
than twice the table.  Card name and power limit are read in the same run.

    PYTHONPATH=. python tests/tools/live_rows_time.py [--rows 10000000,100000000] [--m 1,1000,100000,10000000] [--out FILE]
"""
import argparse
import json
import os
import time

import numpy as np
import torch

import go_ctr_b200 as g
from tests.tools.item_emb_time import card

D = 64


def timed(eng, f):
    st = torch.cuda.ExternalStream(eng.stream)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(st)
    t0 = time.perf_counter()
    f()
    wall = time.perf_counter() - t0
    b.record(st); b.synchronize()
    return dict(event_ms=a.elapsed_time(b), wall_ms=wall * 1e3)


def free_host_bytes():
    try:
        for line in open("/proc/meminfo"):
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    except OSError:
        pass
    return 0


def run(R, ms, seed=0):
    rng = np.random.default_rng(seed)
    eng = g.Engine(g.engine.default_config(g.MODEL_DIN_COS, uP=4, S=8, D=D, cF=4, batch=512, pred_batch=512))
    ids = rng.choice(1 << 62, R, replace=False).astype(np.int64)
    eng.idmap_build(g.IDMAP_ITEM, ids)
    eng.table_fill(g.TABLE_ITEM_EMB, R, D, seed=5, dist=1, scale=0.125)
    fresh = (1 << 62) + np.arange(max(ms), dtype=np.int64)                   # never among ids
    out = dict(rows=R, live={}, upload_route=None)
    eng.idmap_insert(g.IDMAP_ITEM, ids[:1]); eng.table_write_rows(g.TABLE_ITEM_EMB, [0], np.zeros((1, D), np.float32))
    n_rows = R
    used = 0
    for m in ms:
        half = m // 2
        batch = np.concatenate([ids[rng.integers(0, R, m - half)], fresh[used:used + half]])
        used += half
        r = dict(insert=timed(eng, lambda: eng.idmap_insert(g.IDMAP_ITEM, batch)))
        data = rng.standard_normal((m, D)).astype(np.float32)
        inside = rng.choice(n_rows, m, replace=False).astype(np.int32) if m < n_rows // 4 else rng.permutation(n_rows)[:m].astype(np.int32)
        r["write_inside"] = timed(eng, lambda: eng.table_write_rows(g.TABLE_ITEM_EMB, inside, data))
        app = np.arange(n_rows, n_rows + m, dtype=np.int32)
        r["append"] = timed(eng, lambda: eng.table_write_rows(g.TABLE_ITEM_EMB, app, data))
        n_rows += m
        out["live"][str(m)] = r
    if free_host_bytes() > 2 * R * D * 4:
        table = np.zeros((R, D), np.float32)
        t_build = timed(eng, lambda: eng.idmap_build(g.IDMAP_ITEM, ids))
        t_up = timed(eng, lambda: eng.table_upload(g.TABLE_ITEM_EMB, table))
        out["upload_route"] = dict(idmap_build=t_build, table_upload=t_up)
        del table
    eng.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", default="10000000,100000000")
    ap.add_argument("--m", default="1,1000,100000,10000000")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(card=card(), D=D, runs=[run(int(R), [int(m) for m in a.m.split(",")]) for R in a.rows.split(",")])
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
