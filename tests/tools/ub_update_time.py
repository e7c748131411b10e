"""Times ctr_ubcache_append against the route a caller has without it: merge the events into a host copy of the CSR
with numpy, then ctr_ubcache_upload the whole CSR.  For every (stored events n, users U, appended events m) it uploads
the same base cache, appends the same batch both ways, asserts the two downloads are the same CSR, and prints one JSON
line: the append's CUDA-event time on the engine stream (median of consecutive appends after two untimed ones, as
online appends run, the cache growing by m each), the kernels' split from a further profiled call, the host route's merge and upload times, and
the bytes the rewrite moves (24 B per stored and per new event: ts + item row read and written, 16 B per user: old and
new offset) over the call time and over the rewrite kernels' time, as a share of the H100 SXM's 3.35 TB/s.  Card name
and power limit are read in the same run.

    PYTHONPATH=. python tests/tools/ub_update_time.py [--quick] [--out FILE]
"""
import argparse
import json
import subprocess
import time

import numpy as np

import go_ctr_b200 as g

PEAK = 3.35e12                    # H100 SXM5 HBM3 data-sheet bandwidth, bytes/s
T0 = 1_600_000_000
REWRITE = ("ubcache_offsets", "ubcache_move_stored", "ubcache_place_new")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return dict(name=out[0].strip(), power_limit_w=float(out[1]), sm_max_mhz=float(out[2]))
    except Exception as e:          # noqa: BLE001
        return dict(error=str(e))


def base_cache(rng, n, U):
    """n events over U users (uniform), time-descending per user in runs of three equal timestamps."""
    lens = np.bincount(rng.integers(0, U, n), minlength=U).astype(np.int64)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    pos = np.arange(n, dtype=np.int64) - np.repeat(off[:-1], lens)
    ts = T0 - (pos // 3) * 7
    return off, ts, rng.integers(0, 1 << 20, n).astype(np.int32)


def batch(rng, m, U):
    """m events: random users, timestamps among and newer than the stored ones (ties included)."""
    return rng.integers(0, U, m).astype(np.int32), T0 - 7 * rng.integers(-50, 500, m), rng.integers(0, 1 << 20, m).astype(np.int32)


def host_merge(off, ts, items, rows, t, it):
    """Today's route: the append merged into the host CSR in numpy (same order rule as the device)."""
    U, n, m = off.size - 1, ts.size, rows.size
    Un = max(U, int(rows.max()) + 1)
    assert Un < 1 << 31 and (T0 + 4096 - ts).max() < 1 << 32 and (T0 + 4096 - t).max() < 1 << 32
    skey = (np.repeat(np.arange(U, dtype=np.int64), np.diff(off)) << 32) | (T0 + 4096 - ts)
    nkey = (rows.astype(np.int64) << 32) | (T0 + 4096 - t)
    order = (m - 1 - np.argsort(nkey[::-1], kind="stable"))        # key ascending, later arrival first among ties
    pos = np.searchsorted(skey, nkey[order], side="left")          # before the stored events with an equal key
    ts_new = np.insert(ts, pos, t[order]); it_new = np.insert(items, pos, it[order])
    off_ext = np.concatenate([off, np.full(Un - U, n, np.int64)])
    off_new = off_ext + np.searchsorted(np.sort(rows), np.arange(Un + 1), side="left")
    return off_new, ts_new, it_new


def run(torch, n, U, ms, reps):
    rng = np.random.default_rng(n + U)
    base = base_cache(rng, n, U)
    eng = g.Engine(g.engine.default_config(g.MODEL_DIN_COS, S=50, batch=8, pred_batch=8))
    eng.table_upload(g.TABLE_USER_FEAT, np.zeros((U, eng.cfg.uP), np.float32))
    stream = torch.cuda.Stream()
    eng.set_stream(stream.cuda_stream)
    out = []
    for m in ms:
        ev = batch(rng, m, U)
        # the host route, and the device route's first append on the same uploaded base: the same CSR
        eng.ubcache_upload(*base)
        t0 = time.perf_counter(); ref = host_merge(*base, *ev); t1 = time.perf_counter()
        eng.ubcache_upload(*ref); t2 = time.perf_counter()
        eng.ubcache_upload(*base)
        eng.ubcache_append(*ev)
        dev = eng.ubcache_download()
        same = all(x.shape == y.shape and (x == y).all() for x, y in zip(dev, ref))
        assert same, (n, U, m)
        del dev, ref
        # steady state, as online appends run: consecutive appends (one more untimed, so both CSR buffers have been
        # grown once), each moving the cache as it then stands
        eng.ubcache_append(*ev)
        times, shares = [], []
        for r in range(reps):
            n_at = n + (2 + r) * m
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            eng.ubcache_append(*ev)
            b.record(stream)
            b.synchronize()
            times.append(a.elapsed_time(b))
            shares.append((24 * (n_at + m) + 16 * (U + 1)) / (times[-1] * 1e-3) / PEAK)
        n_at = n + (2 + reps) * m
        eng.profile(True); eng.profile_reset()
        eng.ubcache_append(*ev)
        prof = eng.profile_dump(); eng.profile(False)
        ms_call = float(np.median(times))
        ms_rw = sum(prof.get(k, (0.0, 0))[0] for k in REWRITE)
        nbytes = 24 * (n_at + m) + 16 * (U + 1)
        rec = dict(n=n, U=U, m=m, append_ms=round(ms_call, 4), append_ms_all=[round(x, 4) for x in times],
                   share_of_peak_call=round(float(np.median(shares)), 3),
                   profiled_at_n=n_at, rewrite_kernels_ms=round(ms_rw, 4), kernels_ms={k: round(v[0], 4) for k, v in prof.items()},
                   rewrite_bytes=nbytes, share_of_peak_rewrite=round(nbytes / (ms_rw * 1e-3) / PEAK, 3) if ms_rw else None,
                   host_merge_ms=round((t1 - t0) * 1e3, 1), host_upload_ms=round((t2 - t1) * 1e3, 1), same_csr=same)
        print(json.dumps(rec), flush=True)
        out.append(rec)
    eng.close()
    return out


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    info = card()
    print(json.dumps(dict(card=info)), flush=True)
    ns, Us, ms = ((10_000_000,), (138_493,), (1, 1000)) if a.quick else ((10_000_000, 100_000_000), (138_493, 10_000_000), (1, 1000, 100_000, 10_000_000))
    res = [r for n in ns for U in Us for r in run(torch, n, U, ms, a.reps)]
    if a.out:
        with open(a.out, "w") as f:
            json.dump(dict(card=info, results=res), f, indent=1)


if __name__ == "__main__":
    main()
