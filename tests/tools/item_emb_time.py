"""Times recommend.Train's embedding stage two ways and prints one JSON line.

    host route:   numpy first-appearance numbering of the int64 item stream, ctr_i2v_train (int32 word ids up, the
                  [V, D] table down), numpy remap into item rows (zeros for absent items), ctr_table_upload of [R, D]
    device route: ctr_item_emb_train (int64 item ids up, the vocabulary's item ids down; the table stays in HBM)

Default workload: n = 10^8 tokens of a Zipf stream over ~10^6 sparse int64 item ids, D = 64, every item in the item
map, the trainer's parallel mode.  Both routes are timed once, after an untimed warm-up of both on a small stream; wall
times per stage come from a host clock around calls that end in a device synchronise.  Bytes over PCIe are computed
from the shapes.  The two routes' vocabularies and document statistics are compared (the parallel trainer's vectors
are not deterministic).  Card name and power limit are read in the same run.

    PYTHONPATH=. python tests/tools/item_emb_time.py [--n N] [--items I] [--dim D] [--out FILE]
"""
import argparse
import json
import subprocess
import time

import numpy as np

import go_ctr_b200 as g


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return dict(name=out[0].strip(), power_limit_w=float(out[1]), sm_max_mhz=float(out[2]))
    except Exception as e:          # noqa: BLE001
        return dict(error=str(e))


def workload(n, items, seed=0):
    rng = np.random.default_rng(seed)
    cat = rng.permutation(np.unique(rng.integers(-(1 << 62), 1 << 62, int(items * 1.05), dtype=np.int64)))[:items]
    ids = cat[(rng.zipf(1.05, n) - 1) % cat.size]
    return ids, cat


def host_route(eng, ids, imap, cfg):
    t = {}
    t0 = time.perf_counter()
    uniq, first = np.unique(ids, return_index=True)
    order = np.argsort(first, kind="stable")
    word_of_uniq = np.empty(uniq.size, np.int64); word_of_uniq[order] = np.arange(uniq.size)
    tok = word_of_uniq[np.searchsorted(uniq, ids)].astype(np.int32)
    t["numbering_s"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    emb, st = g.i2v_train_ids(tok, uniq.size, cfg=cfg)
    t["train_s"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    pos = np.minimum(np.searchsorted(uniq, imap), uniq.size - 1)
    hit = uniq[pos] == imap
    table = np.zeros((imap.size, cfg.dim), np.float32)
    table[hit] = emb[word_of_uniq[pos[hit]]]
    t["remap_s"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    eng.table_upload(g.TABLE_ITEM_EMB, table)
    t["upload_s"] = time.perf_counter() - t0
    t["total_s"] = sum(t.values())
    V, D, R = uniq.size, cfg.dim, imap.size
    t["pcie_bytes"] = 4 * ids.size + 4 * V * D + 4 * R * D
    t["trainer_ms_device"] = st.ms_device
    return t, uniq[order], st


def device_route(eng, ids, cfg):
    t0 = time.perf_counter()
    vocab, st = eng.item_emb_train(ids, cfg=cfg)
    eng.sync()
    t = dict(total_s=time.perf_counter() - t0, trainer_ms_device=st.ms_device, pcie_bytes=8 * ids.size + 8 * vocab.size)
    return t, vocab, st


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000_000)
    ap.add_argument("--items", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=64)
    ap.add_argument("--out")
    a = ap.parse_args()
    ids, imap = workload(a.n, a.items)
    cfg = g.i2v_default_config(dim=a.dim, window=5, iter=1, seed=1)
    eng = g.Engine(g.engine.default_config(g.MODEL_DIN_COS, uP=0, cF=0, S=1, D=a.dim, batch=1, pred_batch=1))
    eng.idmap_build(g.IDMAP_ITEM, imap)
    small, _ = workload(200_000, 5_000, seed=1)                    # warm-up: module loads, pinned buffers, cub tuning
    device_route(eng, small, cfg); host_route(eng, small, imap, cfg)
    dev, vocab_d, st_d = device_route(eng, ids, cfg)
    host, vocab_h, st_h = host_route(eng, ids, imap, cfg)
    same = bool(np.array_equal(vocab_d, vocab_h)) and all(getattr(st_d, f) == getattr(st_h, f) for f in ("doc_len", "trained_positions", "pairs"))
    res = dict(tool="item_emb_time", n=a.n, items=int(imap.size), vocab=int(vocab_d.size), dim=a.dim, card=card(),
               device_route=dev, host_route=host, same_vocabulary_and_counts=same,
               speedup=host["total_s"] / dev["total_s"])
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
