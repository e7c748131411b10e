"""Times the classification and regression metrics on the device: ctr_accuracy_score, ctr_confusion_matrix,
ctr_precision_recall_fscore, ctr_r2_score and ctr_mean_error at n in {10^7, 10^8}, with C in {2, 1024} classes for the
label calls and n_out in {1, 4} columns for the others, unweighted and weighted.  For each call it prints one JSON line:
the host wall time of the call (median of consecutive calls after an untimed one; it includes the pageable host copies
of the inputs) and the time of its kernels from a further profiled call, where the profile brackets every launch with
CUDA events on the engine stream.  Card name and power limit are read in the same run.

    PYTHONPATH=. python tests/tools/metrics_time.py [--quick] [--reps R] [--out FILE]
"""
import argparse
import json
import time

import numpy as np

import go_ctr_b200 as g
from tests.tools.gauc_time import card

PREFIX = {"accuracy": ("acc_",), "confusion_matrix": ("met_",), "precision_recall_fscore": ("met_",),
          "r2": ("r2_",), "mse": ("err_",), "mae": ("err_",)}


def timed(eng, name, call, reps):
    call()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter(); call(); times.append((time.perf_counter() - t0) * 1e3)
    eng.profile(True); eng.profile_reset()
    call()
    prof = eng.profile_dump(); eng.profile(False)
    mine = {k: v[0] for k, v in prof.items() if any(k.startswith(p) for p in PREFIX[name])}
    return dict(call=name, call_ms=round(float(np.median(times)), 2), call_ms_min=round(min(times), 2),
                kernels_ms_total=round(sum(mine.values()), 3) if mine else None,
                kernels_ms={k: round(v, 3) for k, v in mine.items()})


def run(eng, n, reps):
    rng = np.random.default_rng(n % 1000)
    w = rng.random(n) + 0.5
    out = []
    calls = []
    for C in (2, 1024):
        yt = rng.integers(0, C, n).astype(np.float64)
        yp = np.where(rng.random(n) < 0.7, yt, rng.integers(0, C, n).astype(np.float64))
        for wname, ww in (("none", None), ("weighted", w)):
            calls += [("confusion_matrix", lambda yt=yt, yp=yp, ww=ww: eng.confusion_matrix(yt, yp, ww), dict(C=C, weight=wname)),
                      ("precision_recall_fscore", lambda yt=yt, yp=yp, ww=ww: eng.precision_recall_fscore(yt, yp, 1.0, "macro", -1, ww),
                       dict(C=C, weight=wname))]
        del yt, yp
    for k in (1, 4):
        yt = rng.standard_normal((n, k))
        yp = yt + 0.1 * rng.standard_normal((n, k))
        lt = np.round(yt); lp = np.round(yp)
        for wname, ww in (("none", None), ("weighted", w)):
            calls += [("accuracy", lambda lt=lt, lp=lp, ww=ww: eng.accuracy_score(lt, lp, True, ww), dict(n_out=k, weight=wname)),
                      ("r2", lambda yt=yt, yp=yp, ww=ww: eng.r2_score(yt, yp, ww, "uniform_average"), dict(n_out=k, weight=wname))]
        calls += [("mse", lambda yt=yt, yp=yp: eng.mean_error(yt, yp, "squared", "uniform_average"), dict(n_out=k)),
                  ("mae", lambda yt=yt, yp=yp: eng.mean_error(yt, yp, "absolute", "uniform_average"), dict(n_out=k))]
    for name, call, extra in calls:
        rec = dict(n=n, **extra, **timed(eng, name, call, reps))
        print(json.dumps(rec), flush=True)
        out.append(rec)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    info = card()
    print(json.dumps(dict(card=info)), flush=True)
    eng = g.Engine(g.engine.default_config(g.MODEL_YOUTUBE, batch=1, pred_batch=1))
    ns = (10**6,) if a.quick else (10**7, 10**8)
    res = [r for n in ns for r in run(eng, n, a.reps)]
    eng.close()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(dict(card=info, results=res), f, indent=1)


if __name__ == "__main__":
    main()
