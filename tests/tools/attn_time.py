"""Per-kernel device times of the train step in the HBM regime (12.5 M-row table = one GPU's shard of
BASELINE configs[3], uniform ids, B = 65536).  PYTHONPATH=. python tests/tools/attn_time.py [rows] [zipf]"""
import json
import sys

import numpy as np

import go_ctr_b200 as g


def main():
    import os
    from tests.util import make_batch
    I = int(sys.argv[1]) if len(sys.argv) > 1 else 12_500_000
    zipf = len(sys.argv) > 2
    hot = int(os.environ.get("HOT", "0"))
    U, uP, S, D, cF, B = 138_493, 52, 50, 64, 53, 65_536
    cfg = g.engine.default_config(g.MODEL_DIN_COS, uP=uP, S=S, D=D, cF=cF, batch=B, pred_batch=B, table_opt=g.TABLE_SGD, table_lr=0.01)
    cfg.reserved[0] = hot
    eng = g.Engine(cfg)
    eng.table_fill(g.TABLE_USER_FEAT, U, uP, 1, 0, 1.0); eng.table_fill(g.TABLE_ITEM_FEAT, I, cF, 2, 0, 1.0)
    eng.table_fill(g.TABLE_ITEM_EMB, I, D, 3, 1, 0.125)
    rng = np.random.default_rng(0)
    batches = []
    for _ in range(4):
        batches.append(make_batch(rng, U, I, B, S, pad_frac=0.2, zipf=zipf))
    for b in batches:
        eng.train_step_idx(*b)
    eng.profile(True); eng.profile_reset()
    for _ in range(5):
        for b in batches:
            eng.train_step_idx(*b)
    prof = {k: round(ms / n, 4) for k, (ms, n) in eng.profile_dump().items()}
    rows = sum(int((b[2] >= 0).sum()) + B for b in batches) / len(batches)
    fwd_b = rows * D * 4 + B * ((S + 2) * 4 + (uP + cF) * 4); bwd_b = 2 * rows * D * 4
    # D=64, S=50 from row ids takes the index-route kernels (k_attn_fwd_idx / k_attn_bwd_idx)
    fwd_ms, bwd_ms = prof.get("attn_fwd_idx", 1), prof.get("attn_bwd_idx", 1)
    out = {"rows": I, "zipf": zipf, "hot": hot, "ms": prof, "sum_ms": round(sum(prof.values()), 4),
           "fwd_GBs": round(fwd_b / fwd_ms / 1e6), "bwd_GBs": round(bwd_b / bwd_ms / 1e6),
           # fraction of the H100 SXM data sheet's 3.35 TB/s HBM3 bandwidth
           "pair_frac_of_3350": round((fwd_b + bwd_b) / (fwd_ms + bwd_ms) / 1e6 / 3350.0, 4)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
