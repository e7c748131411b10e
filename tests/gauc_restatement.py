"""The grouped AUC of ctr_group_auc restated in numpy, shared by test_gauc_cpu.py, test_gpu_gauc.py and
tools/gauc_time.py."""
import math

import numpy as np


def auc_score_keys(pred):
    """ctr_roc_auc's sort key on the float32 bits (auc.cuh auc_score_key): -0 read as +0, the order-preserving flip of
    the sign-magnitude bits, complemented so that ascending keys are descending scores.  Equal keys form one threshold
    group; NaNs keep their sign and payload, so they order as the device orders them."""
    u = np.ascontiguousarray(pred, np.float32).view(np.uint32).copy()
    u[u == np.uint32(0x80000000)] = 0
    u = np.where(u & np.uint32(0x80000000), ~u, u | np.uint32(0x80000000))
    return ~u


def gauc_exact(pred, y, group):
    """Samples ordered by (group, score key), tp / fp counted from each group's start, the integer trapezoid
    area2 = sum (fp_i - fp_{i-1}) (tp_i + tp_{i-1}) over the threshold-group ends of each group, AUC_g = area2 / (2.0 P N)
    (NaN with one class), and the mean of AUC_g weighted by n_g over the groups with both classes, summed by math.fsum.
    Returns (gauc, groups, n, pos, auc)."""
    key = auc_score_keys(pred)
    pos = np.asarray(y, np.float32) > np.float32(0.5)
    g = np.asarray(group, np.int64)
    n = key.size
    order = np.lexsort((key, g))
    gs, ks, ps = g[order], key[order], pos[order].astype(np.int64)
    new_group = np.r_[True, gs[1:] != gs[:-1]]
    starts = np.flatnonzero(new_group)
    gid = np.cumsum(new_group) - 1
    tp = np.cumsum(ps)
    tp_in = tp - np.r_[0, tp][starts][gid]
    fp_in = np.arange(1, n + 1, dtype=np.int64) - starts[gid] - tp_in
    ends = np.flatnonzero(np.r_[(gs[1:] != gs[:-1]) | (ks[1:] != ks[:-1]), True])
    tpe, fpe, ge = tp_in[ends], fp_in[ends], gid[ends]
    first = np.r_[True, ge[1:] != ge[:-1]]               # each group's first threshold-group end
    tpp = np.where(first, 0, np.r_[0, tpe[:-1]]); fpp = np.where(first, 0, np.r_[0, fpe[:-1]])
    area2 = np.add.reduceat((fpe - fpp) * (tpe + tpp), np.flatnonzero(first))
    cnt = np.diff(np.r_[starts, n]).astype(np.int64)
    P = np.add.reduceat(ps, starts)
    N = cnt - P
    used = (P > 0) & (N > 0)
    auc = np.full(starts.size, np.nan)
    auc[used] = area2[used].astype(np.float64) / (2.0 * P[used].astype(np.float64) * N[used].astype(np.float64))
    gauc = math.fsum(cnt[used] * auc[used]) / float(cnt[used].sum()) if used.any() else float("nan")
    return gauc, gs[starts], cnt, P, auc
