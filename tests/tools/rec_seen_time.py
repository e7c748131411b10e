"""Times CTR_EXCLUDE_SEEN against CTR_EXCLUDE_WINDOW for one user at the north-star widths: ctr_recommend_topk_ex at
k = 100 and ctr_rank_items_ex for 16 targets, over ctr_table_fill tables of 10^6 and 10^7 items, with seen sets of 10^2,
10^4 and 10^6 rows (cached events of distinct items, every event before the cut).  Prints one JSON line: per table size
the CUDA-event medians of the alternated routes, a profiled pass of the largest seen set (the seen-list build is
<pre>_seen), and whether every SEEN list and rank left the seen rows out.  Card name and power limit are read in the same
run.

    PYTHONPATH=. python tests/tools/rec_seen_time.py [--quick]
"""
import argparse
import json

import numpy as np

import go_ctr_b200 as g
from tests.tools.rank_time import NORTH, alternate, card, engine, profiled

K = 100
SEEN = (100, 10_000, 1_000_000)


def case(torch, I, reps):
    eng, stream = engine(torch, I, NORTH)
    rng = np.random.default_rng(0)
    S = NORTH["S"]
    users = list(range(17, 17 + len(SEEN)))            # user 17 + j holds SEEN[j] events
    seqs = [rng.permutation(I)[:n].astype(np.int32) if n <= I else rng.integers(0, I, n).astype(np.int32) for n in SEEN]
    lens = np.zeros(users[-1] + 1, np.int64)
    for u, s in zip(users, seqs):
        lens[u] = s.size
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    ts = np.concatenate([np.arange(s.size, 0, -1) for s in seqs]).astype(np.int64)
    eng.ubcache_upload(off, ts, np.concatenate(seqs))
    hist = seqs[0][:S][None, :]
    t16 = rng.integers(0, I, 16).astype(np.int32)
    h16 = np.tile(hist, (16, 1))
    routes = {"recommend_window": lambda: eng.recommend_topk([users[0]], hist, K, exclude_history=True),
              "rank16_window": lambda: eng.rank_items(np.full(16, users[0], np.int32), h16, t16, exclude_history=True)}
    for u, n in zip(users, SEEN):
        routes["recommend_seen_%d" % n] = lambda u=u: eng.recommend_topk([u], hist, K, max_ts=0, exclude_seen=True)
        routes["rank16_seen_%d" % n] = lambda u=u: eng.rank_items(np.full(16, u, np.int32), h16, t16, max_ts=0, exclude_seen=True)
    med, mn, res = alternate(torch, stream, routes, reps)
    excluded = True
    for u, n, s in zip(users, SEEN, seqs):
        seen = np.union1d(s, hist[0])
        rows, _, _, cnt = res["recommend_seen_%d" % n]
        ranks, _ = res["rank16_seen_%d" % n]
        excluded &= not np.isin(rows[0, :cnt[0]], seen).any() and bool((ranks[np.isin(t16, seen)] == -1).all())
    big = "_seen_%d" % SEEN[-1]
    out = dict(I=I, reps=reps, ms=med, ms_min=mn, seen_rows_left_out=bool(excluded),
               profile={k: profiled(eng, routes[k]) for k in ("recommend_window", "recommend" + big, "rank16_window", "rank16" + big)})
    eng.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="small tables (a rehearsal of the tool, not a measurement)")
    a = ap.parse_args()
    import torch
    sizes = (100_000, 300_000) if a.quick else (1_000_000, 10_000_000)
    reps = 3 if a.quick else 10
    out = dict(card=card(), k=K, dims=NORTH, cases=[case(torch, I, reps) for I in sizes])
    print(json.dumps({"rec_seen_time": out}))


if __name__ == "__main__":
    main()
