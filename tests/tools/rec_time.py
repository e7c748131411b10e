"""Times ctr_recommend_topk for one user against the whole item table and compares it, in the same process and
alternating, with the route a caller has without it: device index buffers, ctr_predict_idx_dev over every chunk and a
device sort of the scores.  Prints one JSON line: per table size the ms per user and items/s of both routes (CUDA events
on the engine stream, after warm-up), the kernels' split of route (a) from a separate profiled pass, and whether the two
routes return the same top-k rows.  Card name and power limit are read in the same run.

    PYTHONPATH=. python tests/tools/rec_time.py [--quick]
"""
import argparse
import json
import subprocess

import numpy as np

import go_ctr_b200 as g

uP, S, D, cF, PRED_BATCH, K = 52, 50, 64, 53, 65_536, 100


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return dict(name=out[0].strip(), power_limit_w=float(out[1]), sm_max_mhz=float(out[2]))
    except Exception as e:          # noqa: BLE001
        return dict(error=str(e))


def run_case(torch, I, reps):
    cfg = g.engine.default_config(g.MODEL_DIN_COS, uP=uP, S=S, D=D, cF=cF, pred_batch=PRED_BATCH, seed=3)
    eng = g.Engine(cfg)
    stream = torch.cuda.Stream()
    eng.set_stream(stream.cuda_stream)              # both routes and the events on one stream
    U = 1000
    eng.table_fill(g.TABLE_USER_FEAT, U, uP, seed=1)
    eng.table_fill(g.TABLE_ITEM_FEAT, I, cF, seed=2)
    eng.table_fill(g.TABLE_ITEM_EMB, I, D, seed=3, dist=1, scale=0.125)
    W = eng.get_weights()
    eng.set_weights(W[0] * 0.05, W[1] * 0.05, W[2] * 0.3, W[3])
    rng = np.random.default_rng(0)
    user = 17
    hist = rng.integers(0, I, S).astype(np.int32)
    Bc = max(cfg.batch, cfg.pred_batch)
    dev = torch.device("cuda")
    with torch.cuda.stream(stream):
        d_user = torch.full((Bc,), user, dtype=torch.int32, device=dev)
        d_item = torch.arange(I, dtype=torch.int32, device=dev)
        d_hist = torch.from_numpy(np.tile(hist, (Bc, 1))).to(dev)
        d_out = torch.empty(I, dtype=torch.float32, device=dev)
    stream.synchronize()

    def route_a():
        return eng.recommend_topk([user], hist[None, :], K, exclude_history=False)[0][0]

    def route_b():
        for i0 in range(0, I, Bc):
            nb = min(Bc, I - i0)
            eng.predict_idx_dev(d_user.data_ptr(), d_item[i0:].data_ptr(), d_hist.data_ptr(), nb, d_out[i0:].data_ptr())
        with torch.cuda.stream(stream):
            v, idx = torch.sort(d_out, descending=True, stable=True)
            return idx[:K].cpu().numpy().astype(np.int32)

    def timed(f):
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(stream); r = f(); e1.record(stream); e1.synchronize()
        return e0.elapsed_time(e1), r

    for _ in range(3):
        route_a(); route_b()
    ta, tb = [], []
    for _ in range(reps):
        t, ra = timed(route_a); ta.append(t)
        t, rb = timed(route_b); tb.append(t)
    eng.profile(True); eng.profile_reset()
    route_a()
    prof = eng.profile_dump(); eng.profile(False)
    out = dict(I=I, k=K, pred_batch=Bc, reps=reps,
               a_ms=round(float(np.median(ta)), 3), a_ms_min=round(min(ta), 3),
               b_ms=round(float(np.median(tb)), 3), b_ms_min=round(min(tb), 3),
               a_items_per_s=round(I / (np.median(ta) * 1e-3)), b_items_per_s=round(I / (np.median(tb) * 1e-3)),
               a_profile_ms={k: round(v[0], 3) for k, v in sorted(prof.items())},
               a_profile_launches={k: v[1] for k, v in sorted(prof.items())},
               # route (b) sorts saturated scores (many ties at 1.0), so its rows may differ where (a) orders by logit
               same_rows=bool((ra == rb).all()), common_rows=int(np.intersect1d(ra, rb).size))
    eng.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="small tables (a rehearsal of the tool, not a measurement)")
    a = ap.parse_args()
    import torch
    sizes = (100_000, 300_000) if a.quick else (1_000_000, 10_000_000)
    out = dict(card=card(), dims=dict(uP=uP, S=S, D=D, cF=cF), cases=[run_case(torch, I, 10) for I in sizes])
    print(json.dumps({"rec_time": out}))


if __name__ == "__main__":
    main()
