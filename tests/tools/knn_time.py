"""Times ctr_knn_search (knn_scan + knn_merge) on the shapes a 10 M - 100 M item vocabulary gives, and prints one JSON
line: per case the call time (host clock around the synchronous call, after warm-up), the kernels' split (CUDA
events in a separate profiled pass), the algorithmic bytes and DP instructions, and their shares of HBM peak and of
the FP64 issue rate at the SM clock sampled during the timed calls.  Card name and power limit are read in the same run.

    PYTHONPATH=. python tests/tools/knn_time.py [--quick]
"""
import argparse
import json
import subprocess
import time

import numpy as np

import go_ctr_b200 as g
from bench import ClockSampler, load_peaks

D = 64
FP64_LANES_PER_SM = 64          # H100 SXM: 64 FP64 FMA-pipe lanes per SM (one DFMA / DMUL / DADD each per clock)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return dict(name=out[0].strip(), power_limit_w=float(out[1]), sm_max_mhz=float(out[2]))
    except Exception as e:          # noqa: BLE001
        return dict(error=str(e))


def run_case(eng, N, nq, k, mode, reps, rng, sms):
    q = rng.standard_normal((nq, D)) if mode == "vector" else None
    rows = rng.integers(0, N, nq).astype(np.int32) if mode == "row" else None
    call = lambda: eng.knn_search(k, queries=q, rows=rows)      # noqa: E731
    call()                                                        # warm-up: module load, scratch growth
    call()
    sampler = ClockSampler(0)
    time.sleep(0.05)
    t0 = time.time(); ms = []
    for _ in range(reps):
        a = time.perf_counter(); call(); ms.append((time.perf_counter() - a) * 1e3)
    t1 = time.time()
    tail = time.time()
    while time.time() - tail < 0.3:                               # keep the load up while nvidia-smi samples
        call()
    clk = sampler.stop(t0, time.time())
    eng.profile(True); eng.profile_reset()
    for _ in range(max(1, reps // 2)):
        call()
    prof = eng.profile_dump(); eng.profile(False)
    n = max(1, reps // 2)
    scan = prof.get("knn_scan", (0.0, 0))[0] / n; merge = prof.get("knn_merge", (0.0, 0))[0] / n
    t = float(np.median(ms))
    bytes_ = float(N) * D * 4
    dp = float(nq) * N * (D if mode == "row" else 2 * D) + float(N) * D      # dot products + row norms
    hbm_gbs, _ = load_peaks()
    f = clk.get("sm_mhz")
    rate = sms * FP64_LANES_PER_SM * f * 1e6 if f else None
    return dict(N=N, nq=nq, k=k, queries=mode, ms=round(t, 3), ms_min=round(min(ms), 3), reps=reps,
                scan_ms=round(scan, 3), merge_ms=round(merge, 3),
                algorithmic_bytes=bytes_, hbm_frac=round(bytes_ / (scan * 1e-3) / (hbm_gbs * 1e9), 3) if scan else None,
                dp_instr=dp, fp64_frac=round(dp / (scan * 1e-3) / rate, 3) if (rate and scan) else None,
                sm_mhz=f, clock_reasons=clk.get("reasons"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="small tables (a rehearsal of the tool, not a measurement)")
    a = ap.parse_args()
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    big, mid = (1_000_000, 200_000) if a.quick else (100_000_000, 10_000_000)
    rng = np.random.default_rng(0)
    out = dict(card=card(), sms=sms, hbm_peak=load_peaks(), D=D, table="ctr_table_fill N(0,1) float32", cases=[])
    eng = g.Engine(g.engine.default_config(g.MODEL_DIN_COS, uP=0, cF=0, S=1, D=D, batch=1, pred_batch=1))
    eng.table_fill(g.TABLE_ITEM_EMB, big, D, seed=1, dist=1)
    out["cases"].append(run_case(eng, big, 1, 10, "vector", 10, rng, sms))
    eng.table_fill(g.TABLE_ITEM_EMB, mid, D, seed=2, dist=1)
    for nq, k, mode, reps in ((8, 10, "vector", 10), (8, 100, "vector", 10), (1024, 10, "vector", 3), (1024, 100, "vector", 3),
                              (1024, 10, "row", 3), (1024, 100, "row", 3)):
        out["cases"].append(run_case(eng, mid, nq, k, mode, reps, rng, sms))
    eng.close()
    print(json.dumps({"knn_time": out}))


if __name__ == "__main__":
    main()
