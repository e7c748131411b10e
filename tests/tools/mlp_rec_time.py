"""Times ctr_mlp_recommend_topk for one user at k = 100 over the whole item table and compares it, in the same process,
with the route a caller has without it: ctr_mlp_predict_keys over every item id, then np.argsort of the scores.  Two
widths: configs[0] (uP 52, S 10, D 16, cF 53) and the north-star widths (S 50, D 64), hidden [100], relu.

Per case it prints the host wall time of both routes (each call ends in a device synchronise), the new route's kernel
times per profile key from a separate profiled call (CUDA events around every launch), the DFMAs the call needs (layer 0
over the item columns, the output layer, the prefix) and their share of the FP64 issue rate at the clock sampled while
the route ran (SMs x 64 lanes x clock), and whether the new scores equal predict_keys' for the same rows.  Card name and
power limit are read in the same run.  One JSON line.

    PYTHONPATH=. python tests/tools/mlp_rec_time.py [--quick] [--out FILE]
"""
import argparse
import json
import subprocess
import threading
import time

import numpy as np

import go_ctr_b200 as g
from go_ctr_b200 import serving as sv

K, H, PRED_BATCH = 100, 100, 65_536
SMS = 132                                            # H100 SXM
WIDTHS = {"configs0": dict(uP=52, S=10, D=16, cF=53), "north_star": dict(uP=52, S=50, D=64, cF=53)}


def smi(q):
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return [x.strip() for x in out]
    except Exception as e:          # noqa: BLE001
        return [str(e)]


class ClockSampler:
    """The SM clock, polled while a route runs; the maximum is reported."""

    def __init__(self):
        self.mhz = []; self.stop = threading.Event()
        self.t = threading.Thread(target=self.run, daemon=True)

    def run(self):
        while not self.stop.is_set():
            v = smi("clocks.sm")
            try:
                self.mhz.append(float(v[0]))
            except ValueError:
                pass
            self.stop.wait(0.2)

    def __enter__(self):
        self.t.start(); return self

    def __exit__(self, *a):
        self.stop.set(); self.t.join()


def run_case(name, w, I, reps_new, reps_old):
    uP, S, D, cF = w["uP"], w["S"], w["D"], w["cF"]
    cfg = g.engine.default_config(g.MODEL_DIN_COS, uP=uP, S=S, D=D, cF=cF, batch=256, pred_batch=PRED_BATCH)
    eng = g.Engine(cfg)
    U = 64
    eng.table_fill(g.TABLE_USER_FEAT, U, uP, seed=1)
    eng.table_fill(g.TABLE_ITEM_FEAT, I, cF, seed=2)
    eng.table_fill(g.TABLE_ITEM_EMB, I, D, seed=3, dist=1, scale=0.125)
    uid = np.arange(U, dtype=np.int64) * 7 + 11
    iid = np.arange(I, dtype=np.int64) * 3 + 5
    sv.load_id_maps(eng, uid, iid)
    rng = np.random.default_rng(0)
    off = np.arange(U + 1, dtype=np.int64) * (2 * S)
    ts = np.tile(np.arange(2 * S, 0, -1, dtype=np.int64) * 10, U)
    eng.ubcache_upload(off, ts, rng.integers(0, I, off[-1]).astype(np.int32))
    nin = uP + S * D + D + cF
    m = g.MLPClassifier(nin, hidden=(H,))
    p = np.concatenate([rng.standard_normal(H) * 0.1, rng.standard_normal(nin * H) / np.sqrt(nin),
                        rng.standard_normal(1) * 0.1, rng.standard_normal(H) / np.sqrt(H)])
    m.set_params(p)
    user, now = int(uid[17]), 0

    def new():
        return m.recommend_topk(eng, [user], [now], K, exclude_history=False)

    def old():
        s = m.predict_keys(eng, np.full(I, user, np.int64), iid, np.full(I, now, np.int64))
        return np.argsort(-s, kind="stable")[:K], s

    new(); old()                                     # warm-up: modules, buffers
    with ClockSampler() as ck:
        t0 = time.perf_counter()
        for _ in range(reps_new):
            rows, sc, lg, cnt = new()
        t_new = (time.perf_counter() - t0) / reps_new * 1e3
    clock = max(ck.mhz) if ck.mhz else float("nan")
    t0 = time.perf_counter()
    for _ in range(reps_old):
        top_old, s = old()
    t_old = (time.perf_counter() - t0) / reps_old * 1e3
    eng.profile(True); eng.profile_reset()
    new()
    prof = {k: v for k, v in eng.profile_dump().items() if k.startswith("mlp_rec") or k == "ubcache_window"}
    eng.profile(False)
    kern = sum(v[0] for v in prof.values())
    dfma = I * ((D + cF) * H + H) + (uP + S * D) * H
    peak = SMS * 64 * clock * 1e6                    # DFMA per second at the sampled clock
    return dict(case=name, items=I, k=K, new_ms=round(t_new, 3), old_ms=round(t_old, 3),
                kernel_ms=round(kern, 3), per_key_ms={k: [round(v[0], 3), v[1]] for k, v in prof.items()},
                dfma=dfma, sampled_sm_mhz=clock, dfma_share_of_issue_rate_kernel=round(dfma / (kern * 1e-3) / peak, 3),
                dfma_share_of_issue_rate_wall=round(dfma / (t_new * 1e-3) / peak, 3),
                scores_equal_predict_keys=bool(np.array_equal(sc[0].view(np.uint32), s[rows[0]].view(np.uint32))),
                same_rows_as_argsort=bool(np.array_equal(rows[0], top_old)), count=int(cnt[0]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    sizes = [10**5] if a.quick else [10**6, 10**7]
    res = dict(card=smi("name,power.limit,clocks.max.sm"), cases=[])
    for wname, w in WIDTHS.items():
        for I in sizes:
            res["cases"].append(run_case(wname, w, I, reps_new=5, reps_old=2 if I <= 10**6 else 1))
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
