"""Times the device curves and average precision against their AUC counterparts: ctr_roc_curve, ctr_pr_curve and
ctr_average_precision against ctr_roc_auc, and ctr_group_average_precision against ctr_group_auc, at n samples in
{10^6, 10^7, 10^8}.  Every call sorts the n scores, so the expectation is that each new call costs about what its AUC
counterpart costs.  For each call it prints one JSON line: the host wall time of the call (median of consecutive calls
after an untimed one; it includes the pageable host copies of the inputs and of the curve arrays) and the time of its
kernels from a further profiled call, where the profile brackets every launch with CUDA events on the engine stream.
The grouped calls run on 10^3 uniform groups and on n singletons.  Card name and power limit are read in the same run.

    PYTHONPATH=. python tests/tools/ap_time.py [--quick] [--reps R] [--out FILE]
"""
import argparse
import json
import time

import numpy as np

import go_ctr_b200 as g
from tests.tools.gauc_time import card

PREFIX = {"roc_auc": (), "roc_curve": ("clf_",), "pr_curve": ("clf_",), "average_precision": ("clf_", "ap_"),
          "group_auc": ("gauc_",), "group_average_precision": ("gap_",)}


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
    pred = np.round(rng.random(n, np.float32), 4)    # sigmoid outputs with ties
    y = (rng.random(n) < 0.05).astype(np.float32)    # a few percent positives, as click data has
    out = []
    calls = [("roc_auc", lambda: eng.roc_auc(pred, y)),
             ("roc_curve", lambda: eng.roc_curve(pred, y, 1.0)),
             ("pr_curve", lambda: eng.precision_recall_curve(pred, y, 1.0)),
             ("average_precision", lambda: eng.average_precision(pred, y))]
    for layout, grp in (("uniform_1e3", rng.integers(0, 1000, n).astype(np.int64)),
                        ("singletons", rng.permutation(n).astype(np.int64))):
        calls += [("group_auc", lambda grp=grp: eng.group_auc(pred, y, grp), layout),
                  ("group_average_precision", lambda grp=grp: eng.group_average_precision(pred, y, grp), layout)]
    for c in calls:
        rec = dict(n=n, **timed(eng, c[0], c[1], reps))
        if len(c) > 2:
            rec["layout"] = c[2]
        print(json.dumps(rec), flush=True)
        out.append(rec)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    info = card()
    print(json.dumps(dict(card=info)), flush=True)
    eng = g.Engine(g.engine.default_config(g.MODEL_YOUTUBE, batch=1, pred_batch=1))
    ns = (10**6,) if a.quick else (10**6, 10**7, 10**8)
    res = [r for n in ns for r in run(eng, n, a.reps)]
    eng.close()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(dict(card=info, results=res), f, indent=1)


if __name__ == "__main__":
    main()
