"""ctr_roc_auc_dist and ctr_group_auc_dist restated in numpy, step by step as auc.cuh runs them on each rank: runs,
regular samples, splitters, range partition, routes in rank order, merge and integer area (ROC AUC); records sorted by
group, the same partition, and the grouped terms of each rank's groups (GAUC).  Shared by test_auc_dist_cpu.py and the
GPU tests, which compare the device's per-rank counts with it."""
import math

import numpy as np

from tests.gauc_restatement import auc_score_keys, gauc_exact

SAMPLES = 31                                                    # auc.cuh kDistSamples


def runs(keys, cnt):
    """equal keys summed: (sorted unique keys, their summed uint64 counts)"""
    if keys.size == 0:
        return keys.copy(), cnt.copy()
    u, inv = np.unique(keys, return_inverse=True)
    out = np.zeros(u.size, np.uint64)
    np.add.at(out, inv, cnt)
    return u, out


def samples(keys):
    """k_dist_samples: [u, key (i u) / 31 for i < 31] (zeros when u = 0), as uint64"""
    u = keys.size
    s = [keys[(i * u) // SAMPLES] if u else 0 for i in range(SAMPLES)]
    return [u] + [int(x) for x in s]


def splitters(all_samples, W):
    """dist_splitters: weighted quantiles of every rank's samples, each sample of rank r weighing u_r"""
    s = []
    total = 0
    for a in all_samples:
        if a[0] <= 0:
            continue
        s += [(k, a[0]) for k in a[1:]]
        total += a[0] * SAMPLES
    s.sort()
    out, i, cum = [], 0, 0
    for d in range(1, W):
        while i < len(s) and cum * W < d * total:
            cum += s[i][1]
            i += 1
        out.append(s[i - 1][0] if i > 0 else 0)
    return out


def part(keys, spl, W):
    """k_dist_part: off[0] = 0, off[d] = #keys <= spl[d - 1], off[W] = u"""
    return [0] + [int(np.searchsorted(keys, np.uint64(s), side="right")) for s in spl] + [keys.size]


def route(W, offs, arrays):
    """what each rank receives: the ranks' parts for it concatenated in rank order"""
    return [np.concatenate([arrays[r][offs[r][d]:offs[r][d + 1]] for r in range(W)]) for d in range(W)]


def roc_dist(pred, y, cuts):
    """(auc, area2, P, N, sent runs per rank, owned runs per rank) over the ranks [cuts[r], cuts[r + 1])"""
    W = len(cuts) - 1
    key = auc_score_keys(pred).astype(np.uint64)
    cnt = np.where(np.asarray(y, np.float32) > np.float32(0.5), np.uint64(1) << np.uint64(32), np.uint64(1)).astype(np.uint64)
    local = [runs(key[cuts[r]:cuts[r + 1]], cnt[cuts[r]:cuts[r + 1]]) for r in range(W)]
    spl = splitters([samples(k) for k, _ in local], W)
    offs = [part(k, spl, W) for k, _ in local]
    rk = route(W, offs, [k for k, _ in local])
    rc = route(W, offs, [c for _, c in local])
    merged = [runs(rk[d], rc[d]) for d in range(W)]
    area2, base, P, N = 0, 0, 0, 0
    for k, c in merged:
        pos = (c >> np.uint64(32)).astype(object)
        neg = (c & np.uint64(0xffffffff)).astype(object)
        before = base + np.concatenate([[0], np.cumsum(pos)[:-1]]) if pos.size else pos
        area2 += int(np.sum(neg * (2 * before + pos))) if pos.size else 0
        base += int(pos.sum()); P += int(pos.sum()); N += int(neg.sum())
    auc = (area2 * 0.5) / (float(P) * float(N)) if P > 0 and N > 0 else float("nan")
    return auc, area2, P, N, [k.size for k, _ in local], [k.size for k, _ in merged]


def roc_exact(pred, y):
    """(auc, area2, P, N) of ctr_roc_auc over one set, the area as an exact integer"""
    key = auc_score_keys(pred)
    pos = np.asarray(y, np.float32) > np.float32(0.5)
    u, inv = np.unique(key, return_inverse=True)
    p = np.bincount(inv, weights=pos, minlength=u.size).astype(np.int64)
    ng = np.bincount(inv, minlength=u.size).astype(np.int64) - p
    tp = np.cumsum(p)
    tpp = np.r_[0, tp[:-1]]
    area2 = int(np.sum(ng.astype(object) * (tp + tpp).astype(object)))
    P, N = int(p.sum()), int(ng.sum())
    return ((area2 * 0.5) / (float(P) * float(N)) if P > 0 and N > 0 else float("nan")), area2, P, N


def gauc_dist(pred, y, group, cuts):
    """(gauc, groups, n, pos, auc, received samples per rank): each rank's records sorted by group key, partitioned,
    routed, gauc_exact on each rank's records, the groups' arrays concatenated in rank order and the weighted mean
    taken over the concatenation"""
    W = len(cuts) - 1
    g = np.asarray(group, np.int64)
    gkey = g.view(np.uint64) ^ np.uint64(0x8000000000000000)
    idx = np.arange(g.size)
    srt = [idx[cuts[r]:cuts[r + 1]][np.argsort(gkey[cuts[r]:cuts[r + 1]], kind="stable")] for r in range(W)]
    spl = splitters([samples(gkey[s]) for s in srt], W)
    offs = [part(gkey[s], spl, W) for s in srt]
    mine = route(W, offs, srt)
    per = [gauc_exact(pred[m], y[m], g[m]) for m in mine if m.size]
    groups = np.concatenate([p[1] for p in per]); n = np.concatenate([p[2] for p in per])
    pos = np.concatenate([p[3] for p in per]); auc = np.concatenate([p[4] for p in per])
    used = (pos > 0) & (n - pos > 0)
    gauc = math.fsum(n[used] * auc[used]) / float(n[used].sum()) if used.any() else float("nan")
    return gauc, groups, n, pos, auc, [m.size for m in mine]
