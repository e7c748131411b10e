"""Times the full-catalogue rank of held-out items against the route a caller has without it: (a) ctr_rank_items for
one key and for 16 keys of one user (one scoring pass) against (b) ctr_recommend_topk at k = 1024 for the same user, a
list the caller would search for the targets (and which cannot place a target past 1024).  The same for the float64
MLP at configs[0] widths: ctr_mlp_rank_items against ctr_mlp_recommend_topk.  Prints one JSON line: per table size the
CUDA-event medians of the alternated routes, a profiled pass of each, and whether the ranks agree with the lists.  Card
name and power limit are read in the same run.

    PYTHONPATH=. python tests/tools/rank_time.py [--quick]
"""
import argparse
import json
import subprocess

import numpy as np

import go_ctr_b200 as g
from go_ctr_b200 import serving as sv

PRED_BATCH, K = 65_536, 1024
NORTH = dict(uP=52, S=50, D=64, cF=53)           # the north-star widths
CONFIG0 = dict(uP=52, S=10, D=16, cF=53)          # configs[0] (main.go's float64 MLP)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return dict(name=out[0].strip(), power_limit_w=float(out[1]), sm_max_mhz=float(out[2]))
    except Exception as e:          # noqa: BLE001
        return dict(error=str(e))


def engine(torch, I, dims, U=1000):
    cfg = g.engine.default_config(g.MODEL_DIN_COS, pred_batch=PRED_BATCH, seed=3, **dims)
    eng = g.Engine(cfg)
    stream = torch.cuda.Stream()
    eng.set_stream(stream.cuda_stream)              # every route and the events on one stream
    eng.table_fill(g.TABLE_USER_FEAT, U, dims["uP"], seed=1)
    eng.table_fill(g.TABLE_ITEM_FEAT, I, dims["cF"], seed=2)
    eng.table_fill(g.TABLE_ITEM_EMB, I, dims["D"], seed=3, dist=1, scale=0.125)
    W = eng.get_weights()
    eng.set_weights(W[0] * 0.05, W[1] * 0.05, W[2] * 0.3, W[3])
    return eng, stream


def alternate(torch, stream, routes, reps):
    def timed(f):
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(stream); r = f(); e1.record(stream); e1.synchronize()
        return e0.elapsed_time(e1), r
    for _ in range(2):
        for f in routes.values():
            f()
    ms = {k: [] for k in routes}; res = {}
    for _ in range(reps):
        for k, f in routes.items():
            t, res[k] = timed(f); ms[k].append(t)
    return {k: round(float(np.median(v)), 3) for k, v in ms.items()}, {k: round(min(v), 3) for k, v in ms.items()}, res


def profiled(eng, f):
    eng.profile(True); eng.profile_reset()
    f()
    prof = eng.profile_dump(); eng.profile(False)
    return {k: [round(v[0], 3), v[1]] for k, v in sorted(prof.items())}


def din_case(torch, I, reps):
    eng, stream = engine(torch, I, NORTH)
    rng = np.random.default_rng(0)
    user, S = 17, NORTH["S"]
    hist = rng.integers(0, I, S).astype(np.int32)
    t16 = rng.integers(0, I, 16).astype(np.int32)
    routes = {
        "rank_1": lambda: eng.rank_items([user], hist[None, :], t16[:1], exclude_history=False),
        "rank_16": lambda: eng.rank_items(np.full(16, user, np.int32), np.tile(hist, (16, 1)), t16, exclude_history=False),
        "recommend_1024": lambda: eng.recommend_topk([user], hist[None, :], K, exclude_history=False),
    }
    med, mn, res = alternate(torch, stream, routes, reps)
    ranks, _ = res["rank_16"]
    rows, _, _, cnt = res["recommend_1024"]
    lst = rows[0, :cnt[0]].tolist()
    agree = all((0 < r <= K) == (t in lst) and (r > K or lst[r - 1] == t) for t, r in zip(t16.tolist(), ranks.tolist()))
    out = dict(I=I, reps=reps, ms=med, ms_min=mn, ranks_agree_with_list=bool(agree),
               profile={k: profiled(eng, f) for k, f in routes.items() if k != "rank_1"})
    eng.close()
    return out


def mlp_case(torch, I, reps):
    eng, stream = engine(torch, I, CONFIG0, U=1000)
    uid = np.arange(1000, dtype=np.int64) + 10**9
    iid = np.arange(I, dtype=np.int64)
    sv.load_id_maps(eng, uid, iid)
    c = CONFIG0
    nin = c["uP"] + c["S"] * c["D"] + c["D"] + c["cF"]
    m = g.MLPClassifier(nin, hidden=(100,), seed=1)
    rng = np.random.default_rng(1)
    m.set_params(np.concatenate([rng.standard_normal(100) * 0.1, rng.standard_normal(nin * 100) / np.sqrt(nin),
                                 rng.standard_normal(1) * 0.1, rng.standard_normal(100) / 10.0]))
    u = int(uid[17])
    t16 = rng.integers(0, I, 16).astype(np.int64)
    routes = {
        "rank_1": lambda: m.rank_items(eng, [u], t16[:1], [0], exclude_history=False),
        "rank_16": lambda: m.rank_items(eng, np.full(16, u), t16, np.zeros(16, np.int64), exclude_history=False),
        "recommend_1024": lambda: m.recommend_topk(eng, [u], [0], K, exclude_history=False),
    }
    med, mn, res = alternate(torch, stream, routes, reps)
    ranks, _ = res["rank_16"]
    rows, _, _, cnt = res["recommend_1024"]
    lst = rows[0, :cnt[0]].tolist()
    agree = all((0 < r <= K) == (t in lst) and (r > K or lst[r - 1] == t) for t, r in zip(t16.tolist(), ranks.tolist()))
    out = dict(I=I, reps=reps, ms=med, ms_min=mn, ranks_agree_with_list=bool(agree),
               profile={k: profiled(eng, f) for k, f in routes.items() if k != "rank_1"})
    m.close(); eng.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="small tables (a rehearsal of the tool, not a measurement)")
    a = ap.parse_args()
    import torch
    sizes = (100_000, 300_000) if a.quick else (1_000_000, 10_000_000)
    reps = 3 if a.quick else 10
    out = dict(card=card(), pred_batch=PRED_BATCH, k=K, din=dict(dims=NORTH, cases=[din_case(torch, I, reps) for I in sizes]),
               mlp=dict(dims=CONFIG0, hidden=[100], cases=[mlp_case(torch, I, reps) for I in sizes]))
    print(json.dumps({"rank_time": out}))


if __name__ == "__main__":
    main()
