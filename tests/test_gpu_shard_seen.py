"""CTR_EXCLUDE_SEEN on a row-sharded ITEM_EMB (needs >= 2 GPUs): the owner of a row decides whether it is seen.  Each
rank builds the seen bitmap of its own rows from its own behaviour cache; a target's verdict travels with its logit.

With the same ubcache on every rank, recommend_topk_ex and rank_items_ex under SEEN must equal, bit for bit, a
single-GPU handle holding the assembled table, the same weights and that cache: rows, score and logit bits, counts,
ranks and logits.  With caches that differ, both ranks return the owner-rule result, which equals a single GPU whose
cache holds each row's events from its owner's cache (the seen set of a cut is a union over events, so the events can
be regrouped).  Cases: the placements of test_gpu_shard_rank.py, k in {1, 100, 1024}, the rank/list invariant, a call
queued right behind sharded train steps with no host sync, an append applied on every rank between calls, a max_ts
disagreement (CTR_EINVAL on both ranks), serving.Recommend / Evaluate(exclude_seen=True) and the profile keys."""
import os

import numpy as np
import pytest
import torch

import go_ctr_b200 as g
from go_ctr_b200 import serving
from tests import test_gpu_shard_rank as sr

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200)]

WORLD = sr.WORLD
U = sr.U
CASES = sr.CASES
I64_MIN, I64_MAX = -2 ** 63, 2 ** 63 - 1


def _cache(name, salt=0, users=U):
    """time-descending sequences with tied runs; items include -1, repeats and rows past the table"""
    N = CASES[name]["N"]
    rng = np.random.default_rng(sum(name.encode()) + 77 + salt)
    seqs = []
    for u in range(users):
        n = int(rng.integers(0, 40)) if u != 3 else 3000          # one long history
        ts = np.sort(rng.integers(1, 30, n))[::-1].astype(np.int64)
        items = rng.integers(-1, N + 3, n).astype(np.int64)
        seqs.append(list(zip(ts.tolist(), items.tolist())))
    seqs[5] = []                                                   # a user with no events
    return seqs


def _csr(seqs):
    off = np.concatenate([[0], np.cumsum([len(s) for s in seqs])]).astype(np.int64)
    ts = np.array([t for s in seqs for t, _ in s], np.int64)
    it = np.array([i for s in seqs for _, i in s], np.int32)
    return off, ts, it


def _owner_merge(caches, N):
    """one cache whose events of item g come from rank g % WORLD's cache (events of rows outside [0, N) dropped)"""
    users = max(len(c) for c in caches)
    out = []
    for u in range(users):
        ev = [(t, i) for r, c in enumerate(caches) if u < len(c) for t, i in c[u] if 0 <= i < N and i % WORLD == r]
        out.append(sorted(ev, key=lambda e: -e[0]))
    return out


def _keys(name):
    c = CASES[name]
    N, S = c["N"], c["S"]
    rng = np.random.default_rng(3000 + len(name))
    users = np.array([0, 3, 5, U + 5, 7, 3], np.int32)               # a long history, no events, outside the cache
    hist = rng.integers(-1, N + 40, (6, S)).astype(np.int32)
    hist[2] = -1
    cuts = np.array([0, 15, I64_MAX, 9, I64_MIN, 14], np.int64)      # every event, inside tied runs, the extremes
    n = 60
    ku = rng.integers(0, 6, n)
    items = rng.integers(0, max(N, 1), n).astype(np.int32)
    items[:8] = [0, 1 % max(N, 1), 4 % max(N, 1), 10 % max(N, 1), N - 1, -1, N, N + 7]
    big = rng.integers(-2, N + 2, 1100).astype(np.int32)            # one (user, window, cut) of 1100 targets: two passes
    return dict(users=users, hist=hist, cuts=cuts, rank=dict(user_rows=users[ku], hist=hist[ku], item_rows=items, max_ts=cuts[ku]),
                big=dict(user_rows=np.full(big.size, 3, np.int32), hist=np.tile(hist[1], (big.size, 1)), item_rows=big,
                         max_ts=np.full(big.size, 20, np.int64)))


def _calls(eng, keys, res, tag):
    for k in (1, 100, 1024):
        r, s, l, n = eng.recommend_topk(keys["users"], keys["hist"], k, max_ts=keys["cuts"], exclude_seen=True)
        res["%s.rec%d.rows" % (tag, k)], res["%s.rec%d.scores" % (tag, k)] = r, s
        res["%s.rec%d.logits" % (tag, k)], res["%s.rec%d.count" % (tag, k)] = l, n
    for key in ("rank", "big"):
        r, l = eng.rank_items(exclude_seen=True, **keys[key])
        res["%s.%s.rank" % (tag, key)], res["%s.%s.logit" % (tag, key)] = r, l


def _append(eng, name):
    """the same events on every rank: new users' items and a repeat of an existing row, before and inside old runs"""
    N = CASES[name]["N"]
    rng = np.random.default_rng(91)
    u = np.array([0, 0, 3, 7, 7, 7], np.int32)
    ts = np.array([31, 15, 9, 2, 29, 29], np.int64)
    it = (rng.integers(0, N, 6) % max(N, 1)).astype(np.int32)
    eng.ubcache_append(u, ts, it)
    return u, ts, it


def _worker(rank, port, out_dir, names):
    import torch.distributed as dist
    sr._init(rank, port)
    for name in names:
        eng = sr._engine(rank, sr._sharded_cfg(name))
        sr._upload(eng, name)
        eng.ubcache_upload(*_csr(_cache(name)))
        keys = _keys(name)
        res = {}
        _calls(eng, keys, res, "a")
        eng.profile(True); eng.profile_reset()
        eng.recommend_topk(keys["users"], keys["hist"], 10, max_ts=keys["cuts"], exclude_seen=True)
        eng.rank_items(exclude_seen=True, **keys["rank"])
        prof = eng.profile_dump()
        eng.profile(False)
        res["prof.rec_seen"] = np.array(prof.get("rec_seen", (0, 0))[1]); res["prof.rank_seen"] = np.array(prof.get("rank_seen", (0, 0))[1])
        _append(eng, name)
        _calls(eng, keys, res, "b")
        sr._snapshot(eng, name, res)
        np.savez(os.path.join(out_dir, "%s_%d.npz" % (name, rank)), **res)
        eng.close()
    dist.barrier(); dist.destroy_process_group()


def _reference(name, emb, weights, seqs):
    ref = sr._reference(name, emb, weights)
    ref.ubcache_upload(*_csr(seqs))
    return ref


def _same(r0, r1, want, prefix):
    keys = [k for k in want if k.startswith(prefix)]
    assert keys
    for key in keys:
        sr._assert_same(r0[key], r1[key], key + " (rank 0 vs rank 1)")
        sr._assert_same(r0[key], want[key], key)


def _invariant(res, tag, keys):
    """a target ranked r <= 1024 sits at place r - 1 of its user's k = 1024 list; an unranked one is not listed"""
    rows, cnt = res[tag + ".rec1024.rows"], res[tag + ".rec1024.count"]
    kr = keys["rank"]
    j_of = {}
    for j, (u, h, c) in enumerate(zip(keys["users"], keys["hist"], keys["cuts"])):
        j_of.setdefault((int(u), h.tobytes(), int(c)), j)
    for u, h, c, t, r in zip(kr["user_rows"], kr["hist"], kr["max_ts"], kr["item_rows"], res[tag + ".rank.rank"]):
        j = j_of[(int(u), h.tobytes(), int(c))]
        if 0 < r <= cnt[j]:
            assert rows[j, r - 1] == t
        else:
            assert t not in rows[j, :cnt[j]].tolist()


def test_sharded_seen_equals_single_gpu(tmp_path):
    sr._needs_two()
    import torch.multiprocessing as mp
    names = list(CASES)
    mp.spawn(_worker, args=(sr._free_port(), str(tmp_path), names), nprocs=WORLD, join=True)
    for name in names:
        r0, r1, emb = sr._load(tmp_path, name, CASES[name]["N"])
        keys = _keys(name)
        ref = _reference(name, emb, [r0["w%d" % i] for i in range(4)], _cache(name))
        want = {}
        _calls(ref, keys, want, "a")
        _append(ref, name)
        _calls(ref, keys, want, "b")
        _same(r0, r1, want, "a.")
        _same(r0, r1, want, "b.")
        if CASES[name]["N"] > 1:
            assert (want["a.rank.rank"] > 0).any() and (want["a.rank.rank"] == -1).any()
        _invariant(r0, "a", keys)
        _invariant(r0, "b", keys)
        # one bitmap per user on every rank; one per pass
        npass = len({(int(u), h.tobytes(), int(c)) for u, h, c in zip(keys["rank"]["user_rows"], keys["rank"]["hist"], keys["rank"]["max_ts"])})
        for res in (r0, r1):
            assert int(res["prof.rec_seen"]) == keys["users"].size, name
            assert int(res["prof.rank_seen"]) == npass, name


# ---- divergent caches, a cut disagreement, serving, a call queued behind train steps
NAME = "din_cos_d16"


def _misc_worker(rank, port, out_dir):
    import torch.distributed as dist
    sr._init(rank, port)
    c = CASES[NAME]
    keys = _keys(NAME)
    res = {}
    eng = sr._engine(rank, sr._sharded_cfg(NAME, hot=64))
    sr._upload(eng, NAME)
    for i, w in enumerate(eng.get_weights()):
        res["w0_%d" % i] = w
    # divergent caches: rank 1's has fewer users
    eng.ubcache_upload(*_csr(_cache(NAME, salt=rank, users=U - 20 * rank)))
    _calls(eng, keys, res, "div")
    # a cut that differs on the two ranks: EINVAL on both, and a matching call afterwards
    bad = dict(keys["rank"]); bad["max_ts"] = keys["rank"]["max_ts"] + rank
    res["bad_rank_code"] = np.array(sr._err(lambda: eng.rank_items(exclude_seen=True, **bad))[0])
    res["bad_rec_code"] = np.array(sr._err(lambda: eng.recommend_topk(keys["users"], keys["hist"], 5, max_ts=keys["cuts"] + rank,
                                                                       exclude_seen=True))[0])
    r, l = eng.rank_items(exclude_seen=True, **keys["rank"])
    res["after.rank"], res["after.logit"] = r, l
    # train steps queued right before the calls, no host sync
    rng = np.random.default_rng(31)
    for step in range(3):
        ur = rng.integers(0, U, 128).astype(np.int32); ir = rng.integers(0, c["N"], 128).astype(np.int32)
        ir[:8] = np.arange(8)
        hist = rng.integers(-1, c["N"], (128, c["S"])).astype(np.int32); y = (rng.random(128) > 0.5).astype(np.float32)
        sl = slice(rank * 64, (rank + 1) * 64)
        if step < 2:
            eng.train_step_idx(ur[sl], ir[sl], hist[sl], y[sl])
        else:
            d = "cuda:%d" % rank
            t = [torch.from_numpy(np.ascontiguousarray(a[sl])).to(d) for a in (ur, ir, hist, y)]
            torch.cuda.synchronize(d)
            eng.train_step_idx_dev(t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), t[3].data_ptr(), 64)   # asynchronous
    _calls(eng, keys, res, "live")
    sr._snapshot(eng, NAME, res)
    eng.close()
    # serving on the same cache everywhere (test_gpu_shard_rank's setup)
    srv = sr._engine(rank, sr._sharded_cfg(NAME))
    sr._upload(srv, NAME)
    held = sr._serving_setup(srv, NAME)
    res["eval"] = np.array(sorted(serving.Evaluate(srv, held, ks=(1, 10, 100), exclude_seen=True).items()), dtype=object).astype(str)
    recs = [serving.Recommend(srv, s.UserId, 50, now=s.Timestamp, exclude_seen=True) for s in held[:5]]
    res["recommend"] = np.array([[x.ItemId for x in r] + [-1] * (50 - len(r)) for r in recs], np.int64)
    for i, w in enumerate(srv.get_weights()):
        res["srv_w%d" % i] = w
    srv.close()
    np.savez(os.path.join(out_dir, "misc_%d.npz" % rank), **res)
    dist.barrier(); dist.destroy_process_group()


def test_sharded_seen_divergent_caches_disagreement_serving_and_live(tmp_path):
    sr._needs_two()
    import torch.multiprocessing as mp
    mp.spawn(_misc_worker, args=(sr._free_port(), str(tmp_path)), nprocs=WORLD, join=True)
    N = CASES[NAME]["N"]
    r0, r1, emb = sr._load(tmp_path, "misc", N)
    keys = _keys(NAME)
    for r in (r0, r1):
        assert int(r["bad_rank_code"]) == g.EINVAL and int(r["bad_rec_code"]) == g.EINVAL
    _, _, emb0 = sr._tables(NAME)
    merged = _owner_merge([_cache(NAME, salt=r, users=U - 20 * r) for r in range(WORLD)], N)
    # the divergent calls and the one after the disagreement ran on the uploaded table and the initial weights
    ref0 = _reference(NAME, emb0, [r0["w0_%d" % i] for i in range(4)], merged)
    want = {}
    _calls(ref0, keys, want, "div")
    _same(r0, r1, want, "div.")
    rr, ll = ref0.rank_items(exclude_seen=True, **keys["rank"])
    for key, w in (("after.rank", rr), ("after.logit", ll)):
        sr._assert_same(r0[key], r1[key], key); sr._assert_same(r0[key], w, key)
    # after the train steps: the trained table and weights, the same divergent caches
    assert np.abs(emb - emb0).max() > 1e-6
    ref = _reference(NAME, emb, [r0["w%d" % i] for i in range(4)], merged)
    want = {}
    _calls(ref, keys, want, "live")
    _same(r0, r1, want, "live.")
    # serving: one GPU with the same id maps and cache
    srv = sr._reference(NAME, sr._tables(NAME)[2], [r0["srv_w%d" % i] for i in range(4)])
    held = sr._serving_setup(srv, NAME)
    ev = np.array(sorted(serving.Evaluate(srv, held, ks=(1, 10, 100), exclude_seen=True).items()), dtype=object).astype(str)
    assert np.array_equal(r0["eval"], ev) and np.array_equal(r1["eval"], ev), (r0["eval"], ev)
    recs = [serving.Recommend(srv, s.UserId, 50, now=s.Timestamp, exclude_seen=True) for s in held[:5]]
    want_rec = np.array([[x.ItemId for x in r] + [-1] * (50 - len(r)) for r in recs], np.int64)
    assert np.array_equal(r0["recommend"], want_rec) and np.array_equal(r1["recommend"], want_rec)
