"""Times the float64 MLP regressor next to the classifier at the same shapes, in one process, the two alternated:

  - one fit epoch over n = 100 000 rows of 281 features, hidden [100], relu, adam, minibatches of 200: the regressor with
    1 and 4 targets (identity output, square_loss) against the classifier with binary labels and with 4 classes
    (logistic / softmax output, log losses);
  - ctr_mlp_score over 1 000 000 rows, 1 and 4 targets, against ctr_mlp_predict_f64 of the same rows (the forward pass
    the score runs first) — the difference is the R² kernels and the targets' upload;
  - ctr_mlp_recommend_topk for one user at k = 100 over 1 000 000 items (configs[0] widths), the regressor against the
    classifier with the same parameters.

Every call ends in a device synchronise; the host wall time per call is the median over the repetitions.  Card name and
power limit are read in the same run.  One JSON line.

    PYTHONPATH=. python tests/tools/mlp_reg_time.py [--quick] [--out FILE]
"""
import argparse
import json
import subprocess
import time

import numpy as np

import go_ctr_b200 as g
from go_ctr_b200 import serving as sv

NF, H = 281, 100


def smi(q):
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return [x.strip() for x in out]
    except Exception as e:          # noqa: BLE001
        return [str(e)]


def alternate(fa, fb, reps):
    """median wall ms of fa and fb, called alternately after one warm-up call each"""
    fa(); fb()
    ta, tb = [], []
    for _ in range(reps):
        t0 = time.perf_counter(); fa(); ta.append(time.perf_counter() - t0)
        t0 = time.perf_counter(); fb(); tb.append(time.perf_counter() - t0)
    return round(float(np.median(ta)) * 1e3, 3), round(float(np.median(tb)) * 1e3, 3)


def fit_epoch(n, reps):
    rng = np.random.default_rng(0)
    X = rng.random((n, NF), np.float32)
    out = []
    for no in (1, 4):
        Y = (X[:, :no] * 3 + 0.5).astype(np.float32)
        labels = (X[:, 0] > 0.5).astype(np.float32) if no == 1 else np.floor(X[:, 0] * 4).astype(np.float32) + 1
        kw = dict(hidden=(H,), max_iter=1, seed=1)
        r = g.MLPRegressor(NF, n_outputs=no, **kw)
        c = g.MLPClassifier(NF, **kw)
        tr, tc = alternate(lambda: r.fit(X, Y), lambda: c.fit(X, labels), reps)
        out.append(dict(targets=no, regressor_ms=tr, classifier_ms=tc, classifier_outputs=no,
                        ratio=round(tr / tc, 3)))
    return out


def score(n, reps):
    rng = np.random.default_rng(1)
    X = rng.random((n, NF), np.float32)
    out = []
    for no in (1, 4):
        Y = (X[:, :no] * 3 + 0.5).astype(np.float32)
        r = g.MLPRegressor(NF, hidden=(H,), max_iter=1, seed=1, n_outputs=no).fit(X[:20_000], Y[:20_000])
        ts, tp = alternate(lambda: r.score(X, Y), lambda: r.predict_f64(X), reps)
        out.append(dict(rows=n, targets=no, score_ms=ts, predict_f64_ms=tp, r2_overhead_ms=round(ts - tp, 3)))
    return out


def recommend(I, reps):
    uP, S, D, cF = 52, 10, 16, 53
    cfg = g.engine.default_config(g.MODEL_DIN_COS, uP=uP, S=S, D=D, cF=cF, batch=256, pred_batch=65_536)
    eng = g.Engine(cfg)
    U = 64
    eng.table_fill(g.TABLE_USER_FEAT, U, uP, seed=1)
    eng.table_fill(g.TABLE_ITEM_FEAT, I, cF, seed=2)
    eng.table_fill(g.TABLE_ITEM_EMB, I, D, seed=3, dist=1, scale=0.125)
    uid = np.arange(U, dtype=np.int64) * 7 + 11
    sv.load_id_maps(eng, uid, np.arange(I, dtype=np.int64) * 3 + 5)
    rng = np.random.default_rng(0)
    off = np.arange(U + 1, dtype=np.int64) * (2 * S)
    eng.ubcache_upload(off, np.tile(np.arange(2 * S, 0, -1, dtype=np.int64) * 10, U), rng.integers(0, I, off[-1]).astype(np.int32))
    nin = uP + S * D + D + cF
    p = np.concatenate([rng.standard_normal(H) * 0.1, rng.standard_normal(nin * H) / np.sqrt(nin),
                        rng.standard_normal(1) * 0.1, rng.standard_normal(H) / np.sqrt(H)])
    r = g.MLPRegressor(nin, hidden=(H,)); r.set_params(p, out_activation="identity")
    c = g.MLPClassifier(nin, hidden=(H,)); c.set_params(p)
    user = int(uid[17])
    tr, tc = alternate(lambda: r.recommend_topk(eng, [user], [0], 100, exclude_history=False),
                       lambda: c.recommend_topk(eng, [user], [0], 100, exclude_history=False), reps)
    a = r.recommend_topk(eng, [user], [0], 100, exclude_history=False)
    b = c.recommend_topk(eng, [user], [0], 100, exclude_history=False)
    return dict(items=I, k=100, regressor_ms=tr, classifier_ms=tc, ratio=round(tr / tc, 3),
                same_rows=bool(np.array_equal(a[0], b[0])), same_logits=bool(np.array_equal(a[2], b[2])))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    n_fit, n_score, n_items, reps = (5_000, 50_000, 50_000, 2) if a.quick else (100_000, 1_000_000, 1_000_000, 5)
    res = dict(card=smi("name,power.limit,clocks.max.sm"), fit_epoch=fit_epoch(n_fit, reps), score=score(n_score, reps),
               recommend=recommend(n_items, reps))
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
