"""Times ctr_group_auc (GAUC) against the numpy restatement a caller would otherwise run on the host (tests/gauc_restatement.py
gauc_exact: lexsort, integer areas, math.fsum).  For n samples in {10^6, 10^7, 10^8} and each group layout — one group,
10^3 uniform groups, 10^5 Zipf-sized groups, n singletons — it prints one JSON line: the call's host wall time (median
of consecutive calls after an untimed one; it includes the pageable host-to-device copies of pred, y and group), the
gauc_* kernels' times from a further profiled call, the numpy restatement's time and whether the two GAUCs agree to
1e-12.  The acceptance bar of the design is that, at one n, the call's cost stays within 2x across the layouts.  Card
name and power limit are read in the same run.

    PYTHONPATH=. python tests/tools/gauc_time.py [--quick] [--reps R] [--out FILE]
"""
import argparse
import json
import math
import subprocess
import time

import numpy as np

import go_ctr_b200 as g
from tests.gauc_restatement import gauc_exact


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return dict(name=out[0].strip(), power_limit_w=float(out[1]), sm_max_mhz=float(out[2]))
    except Exception as e:          # noqa: BLE001
        return dict(error=str(e))


def groups(layout, n, rng):
    if layout == "one":
        return np.zeros(n, np.int64)
    if layout == "uniform_1e3":
        return rng.integers(0, 1000, n).astype(np.int64)
    if layout == "zipf_1e5":          # 10^5 users, Zipf-sized: the head user holds a large share of the samples
        return ((rng.zipf(1.2, n) - 1) % 100_000).astype(np.int64) * 7919 - 10**9
    return rng.permutation(n).astype(np.int64)      # singletons


def run(eng, n, layout, reps, with_numpy):
    rng = np.random.default_rng(n % 1000 + len(layout))
    pred = np.round(rng.random(n, np.float32), 4)    # sigmoid outputs with ties
    y = (rng.random(n) < 0.3).astype(np.float32)
    grp = groups(layout, n, rng)
    gauc, ng, nu = eng.group_auc(pred, y, grp)
    times = []
    for _ in range(reps):
        t0 = time.perf_counter(); eng.group_auc(pred, y, grp); times.append((time.perf_counter() - t0) * 1e3)
    eng.profile(True); eng.profile_reset()
    eng.group_auc(pred, y, grp)
    prof = eng.profile_dump(); eng.profile(False)
    rec = dict(n=n, layout=layout, n_groups=ng, n_used=nu, gauc=gauc, call_ms=round(float(np.median(times)), 2),
               call_ms_all=[round(t, 2) for t in times],
               kernels_ms_total=round(sum(v[0] for k, v in prof.items() if k.startswith("gauc_")), 3),
               kernels_ms={k: round(v[0], 3) for k, v in prof.items() if k.startswith("gauc_")})
    if with_numpy:
        t0 = time.perf_counter(); want = gauc_exact(pred, y, grp)[0]; rec["numpy_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
        rec["agrees_1e-12"] = (math.isnan(want) and math.isnan(gauc)) or abs(gauc - want) <= 1e-12 * abs(want)
    print(json.dumps(rec), flush=True)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--numpy-max", type=int, default=10**8, help="time the numpy restatement up to this n")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    info = card()
    print(json.dumps(dict(card=info)), flush=True)
    eng = g.Engine(g.engine.default_config(g.MODEL_YOUTUBE, batch=1, pred_batch=1))
    ns = (10**6,) if a.quick else (10**6, 10**7, 10**8)
    res = [run(eng, n, lay, a.reps, n <= a.numpy_max) for n in ns for lay in ("one", "uniform_1e3", "zipf_1e5", "singletons")]
    eng.close()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(dict(card=info, results=res), f, indent=1)


if __name__ == "__main__":
    main()
