"""Times the float64 MLP fed by sample keys (ctr_mlp_fit_keys / ctr_mlp_predict_keys) against the route a caller had
before: Engine.gather_rows to the host, then MLPClassifier.fit / predict on that X.

Two shapes: configs[0] as main.go sets it (uP 52, S 10, D 16, cF 53: nin 281; hidden 100, relu + Adam, max_iter 20;
80 000 samples) and a north-star width (S 50, D 64: nin 3369).  Every epoch runs (tol = 0).  Per shape it prints one
JSON line with the fit's wall time end to end and per epoch for both routes, and predict's median wall time at 1 and
10 000 keys for both.  The two fits are also compared bit for bit.  Card name and power limit are read in the same run.

    PYTHONPATH=. python tests/tools/mlp_keys_time.py [--quick] [--reps R] [--out FILE]
"""
import argparse
import json
import subprocess
import time

import numpy as np

import go_ctr_b200 as g
from go_ctr_b200 import serving as sv


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return dict(name=out[0].strip(), power_limit_w=float(out[1]), sm_max_mhz=float(out[2]))
    except Exception as e:          # noqa: BLE001
        return dict(error=str(e))


def store(rng, U, I, uP, S, D, cF):
    eng = g.Engine(g.engine.default_config(g.MODEL_DIN_COS, uP=uP, S=S, D=D, cF=cF, batch=256, pred_batch=1024))
    eng.table_upload(g.TABLE_USER_FEAT, rng.random((U, uP), np.float32))
    eng.table_upload(g.TABLE_ITEM_FEAT, rng.random((I, cF), np.float32))
    eng.table_upload(g.TABLE_ITEM_EMB, (rng.standard_normal((I, D)) / np.sqrt(D)).astype(np.float32))
    uid = np.arange(U, dtype=np.int64) * 7 + 1; iid = np.arange(I, dtype=np.int64) * 11 + 3
    sv.load_id_maps(eng, uid, iid)
    lens = rng.integers(0, 3 * S, U)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    ts = np.concatenate([1_000_000 - np.sort(rng.integers(0, 500_000, L)) for L in lens]).astype(np.int64)
    eng.ubcache_upload(off, ts, rng.integers(0, I, off[-1]).astype(np.int32))
    return eng, uid, iid


def median_ms(f, reps):
    f()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter(); f(); t.append((time.perf_counter() - t0) * 1e3)
    return round(float(np.median(t)), 3)


def run(name, n, uP, S, D, cF, max_iter, reps):
    rng = np.random.default_rng(7)
    U, I = 6000, 20000
    eng, uid, iid = store(rng, U, I, uP, S, D, cF)
    nin = uP + S * D + D + cF
    ur = rng.integers(0, U, n).astype(np.int32); ir = rng.integers(0, I, n).astype(np.int32)
    u, i = uid[ur], iid[ir]
    t = rng.integers(500_000, 1_000_000, n).astype(np.int64)
    y = (rng.random(n) < 0.3).astype(np.float32)
    kw = dict(hidden=(100,), activation="relu", solver="adam", alpha=1e-4, max_iter=max_iter, tol=0.0, seed=1)
    rec = dict(shape=name, n=n, nin=nin, hidden=100, max_iter=max_iter, dense_x_f64_gb=round(n * nin * 8 / 1e9, 2))

    mk = g.MLPClassifier(nin, **kw)
    t0 = time.perf_counter(); mk.fit_keys(eng, u, i, t, y); keys_s = time.perf_counter() - t0

    md = g.MLPClassifier(nin, **kw)
    t0 = time.perf_counter()
    hist = eng.ubcache_window(ur, t)
    X = eng.gather_rows(ur, ir, hist)
    t1 = time.perf_counter()
    md.fit(X, y)
    t2 = time.perf_counter()
    rec.update(fit_keys_s=round(keys_s, 3), fit_keys_epoch_ms=round(keys_s * 1e3 / mk.n_iter, 2),
               dense_gather_s=round(t1 - t0, 3), dense_fit_s=round(t2 - t1, 3), dense_total_s=round(t2 - t0, 3),
               dense_fit_epoch_ms=round((t2 - t1) * 1e3 / md.n_iter, 2),
               bit_identical=bool(np.array_equal(mk.get_params().view(np.uint64), md.get_params().view(np.uint64))))
    for q in (1, 10_000):
        sel = rng.integers(0, n, q)

        def dense_pred():
            h = eng.ubcache_window(ur[sel], t[sel])
            return md.predict(eng.gather_rows(ur[sel], ir[sel], h))
        rec["predict_keys_ms_%d" % q] = median_ms(lambda: mk.predict_keys(eng, u[sel], i[sel], t[sel]), reps)
        rec["dense_predict_ms_%d" % q] = median_ms(dense_pred, reps)
    print(json.dumps(rec), flush=True)
    eng.close(); mk.close(); md.close()
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    info = card()
    print(json.dumps(dict(card=info)), flush=True)
    res = [run("configs0", 20_000 if a.quick else 80_000, 52, 10, 16, 53, 20, a.reps)]
    res.append(run("north_star_width", 20_000 if a.quick else 80_000, 52, 50, 64, 53, 3, a.reps))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(dict(card=info, results=res), f, indent=1)


if __name__ == "__main__":
    main()
