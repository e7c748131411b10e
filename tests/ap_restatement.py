"""The curves and average precision of nn/metrics/ranking.go restated twice, shared by test_ap_cpu.py,
test_gpu_ap.py and tools/ap_time.py.

* The literal restatement (`literal_*`) transliterates binaryClfCurve, ROCCurve, PrecisionRecallCurve,
  AveragePrecisionScore and typeOfTarget (ranking.go:13-222, base.go:12-22 and 89-119): the same loops over Python
  floats, which are float64, in the same order.  The reference's sort.Slice leaves the order of equal scores open;
  here they keep their input order, except that +0 comes before -0, so the ±0 group's threshold is +0.0 as on the
  device.  With NaN scores the reference's order is undefined, so this restatement is meant for NaN-free scores.
* The vectorised restatement (`clf_curve`, `roc_curve`, `pr_curve`, `average_precision`, `group_average_precision`)
  orders scores by ctr_roc_auc's key (`auc_score_keys`), counts with np.unique / cumsum and sums AP and MAP with
  math.fsum.  It covers NaN scores as the device orders them, and writes every NaN it computes as float("nan")
  (0x7ff8000000000000), as the device does.
"""
import math

import numpy as np

from tests.gauc_restatement import auc_score_keys

QNAN = float("nan")


# ---- literal transliteration ----------------------------------------------------------------------------------------

def literal_binary_clf_curve(y_true, y_score, pos_label):
    """binaryClfCurve (ranking.go:13-57) without sample weights: (fps, tps, thresholds) as lists of floats."""
    m = len(y_score)
    idx = sorted(range(m), key=lambda i: (-y_score[i], math.copysign(1.0, y_score[i]) < 0))
    distinct = []
    for ii in range(len(idx)):
        if ii == 0 or y_score[idx[ii]] < y_score[idx[ii - 1]]:
            distinct.append([idx[ii]])
        else:
            distinct[-1].append(idx[ii])
    tpw, fpw, w = 0.0, 0.0, 1.0
    fps, tps, thresholds = [], [], []
    for group in distinct:
        for i3 in group:
            if y_true[i3] == pos_label:
                tpw += w
            else:
                fpw += w
        tps.append(tpw)
        fps.append(fpw)
        thresholds.append(y_score[group[0]])
    return fps, tps, thresholds


def literal_roc_curve(y_true, y_score, pos_label):
    """ROCCurve (ranking.go:71-103): (fpr, tpr, thresholds)."""
    fps, tps, thresholds = literal_binary_clf_curve(y_true, y_score, pos_label)
    if len(tps) == 0 or fps[0] != 0.0:
        fps = [0.0] + fps
        tps = [0.0] + tps
        thresholds = [thresholds[0] + 1.0] + thresholds
    fpr, tpr = fps, tps
    fpmax = fps[-1]
    if fpmax <= 0.0:
        fpr = [QNAN] * len(fpr)
    else:
        c = 1.0 / fpmax
        fpr = [v * c for v in fpr]                     # floats.Scale multiplies by the reciprocal
    tpmax = tps[-1]
    if tpmax <= 0:
        tpr = [QNAN] * len(tpr)
    else:
        c = 1.0 / tpmax
        tpr = [v * c for v in tpr]
    return fpr, tpr, thresholds


def _search_float64s(a, x):
    """sort.SearchFloat64s: the first index i with a[i] >= x."""
    lo, hi = 0, len(a)
    while lo < hi:
        h = (lo + hi) // 2
        if a[h] < x:
            lo = h + 1
        else:
            hi = h
    return lo


def _div(a, b):
    """float64 division as Go does it at run time: 0 / 0 is NaN rather than an exception."""
    return a / b if b != 0.0 else (QNAN if a == 0.0 or a != a else math.copysign(math.inf, a) * math.copysign(1.0, b))


def literal_pr_curve(y_true, probas_pred, pos_label):
    """PrecisionRecallCurve (ranking.go:183-209): (precision, recall, thresholds)."""
    fps, tps, thresholds = literal_binary_clf_curve(y_true, probas_pred, pos_label)
    lentps = len(tps)
    precision = [0.0] * lentps
    recall = [0.0] * lentps
    for i in range(lentps):
        precision[i] = _div(tps[i], tps[i] + fps[i])
        recall[i] = _div(tps[i], tps[lentps - 1])
    last_ind = _search_float64s(tps, tps[lentps - 1])

    def reverse_and_append(a, l, *v):
        a = list(a)
        for i in range(l // 2):
            j = l - 1 - i
            a[i], a[j] = a[j], a[i]
        return a[:l] + list(v)

    return (reverse_and_append(precision, last_ind + 1, 1.0), reverse_and_append(recall, last_ind + 1, 0.0),
            reverse_and_append(thresholds, last_ind + 1))


def literal_type_of_target(y_true):
    """typeOfTarget (base.go:89-119) of one column: "binary" or "unknown"."""
    lo = hi = y_true[0]
    for v in y_true:
        if v < lo:
            lo = v
        if v > hi:
            hi = v
    for v in y_true:
        if v != lo and v != hi:
            return "unknown"
    return "binary"


def literal_ap_terms(y_true, y_score):
    """The terms of binaryUninterpolatedAveragePrecision (ranking.go:214-220) in the reference's summation order."""
    precision, recall, _ = literal_pr_curve(y_true, y_score, 1.0)
    return [(recall[i] - recall[i + 1]) * precision[i] for i in range(len(precision) - 1)]


def literal_average_precision(y_true, y_score):
    """AveragePrecisionScore (ranking.go:212-222) of one column: 0 for labels that are not binary (averageBinaryScore
    prints "unsupported"), else the terms summed one by one from the high-recall end."""
    if literal_type_of_target(y_true) != "binary":
        return 0.0
    score = 0.0
    for t in literal_ap_terms(y_true, y_score):
        score += t
    return score


def literal_auc(fpr, tpr):
    """AUC (ranking.go:106-118): the trapezoid rule over the curve."""
    auc, xp, yp = 0.0, 0.0, 0.0
    for x, y in zip(fpr, tpr):
        auc += (x - xp) * (y + yp) / 2.0
        xp, yp = x, y
    return auc


# ---- vectorised restatement -----------------------------------------------------------------------------------------

def key_thresholds(keys):
    """The inverse of auc_score_keys widened to float64 exactly; NaNs keep sign and payload (no quieting)."""
    v = ~np.asarray(keys, np.uint32)
    u = np.where(v & np.uint32(0x80000000), v & np.uint32(0x7fffffff), ~v).astype(np.uint32)
    with np.errstate(invalid="ignore"):
        out = u.view(np.float32).astype(np.float64)
    nan = (u & np.uint32(0x7f800000)) == np.uint32(0x7f800000)
    nan &= (u & np.uint32(0x7fffff)) != 0
    if nan.any():
        un = u[nan].astype(np.uint64)
        bits = (un >> np.uint64(31)) << np.uint64(63) | np.uint64(0x7ff0000000000000) | (un & np.uint64(0x7fffff)) << np.uint64(29)
        out[nan] = bits.view(np.float64)
    return out


def clf_curve(pred, y, pos_label):
    """binaryClfCurve: int64 (tps, fps) and float64 thresholds, one point per threshold group from the highest score
    down, a sample positive when (double)y == pos_label."""
    keys = auc_score_keys(pred)
    pos = np.asarray(y, np.float32).astype(np.float64) == pos_label
    uk, inv, cnt = np.unique(keys, return_inverse=True, return_counts=True)
    tps = np.cumsum(np.bincount(inv.ravel(), weights=pos, minlength=uk.size)).astype(np.int64)
    fps = np.cumsum(cnt).astype(np.int64) - tps
    return tps, fps, key_thresholds(uk)


def _scale(counts, top):
    return counts.astype(np.float64) * (1.0 / float(top)) if top > 0 else np.full(counts.size, QNAN)


def roc_curve(pred, y, pos_label):
    """ROCCurve: (fpr, tpr, thresholds)."""
    tps, fps, thr = clf_curve(pred, y, pos_label)
    if fps[0] != 0:
        t0 = thr[0]
        tps, fps = np.r_[0, tps], np.r_[0, fps]
        thr = np.r_[t0 if np.isnan(t0) else t0 + 1.0, thr]
    return _scale(fps, fps[-1]), _scale(tps, tps[-1]), thr


def _pr_points(tps, fps):
    """precision and recall at every point, and last_ind"""
    precision = tps.astype(np.float64) / (tps + fps).astype(np.float64)
    recall = tps.astype(np.float64) / float(tps[-1]) if tps[-1] > 0 else np.full(tps.size, QNAN)
    return precision, recall, int(np.searchsorted(tps, tps[-1], side="left"))


def pr_curve(pred, y, pos_label):
    """PrecisionRecallCurve: (precision, recall, thresholds)."""
    tps, fps, thr = clf_curve(pred, y, pos_label)
    precision, recall, last = _pr_points(tps, fps)
    return np.r_[precision[last::-1], 1.0], np.r_[recall[last::-1], 0.0], thr[last::-1].copy()


def ap_terms(tps, fps):
    """The AP terms (recall_j - recall_{j-1}) * precision_j for j = 0 … last_ind, recall_{-1} = 0."""
    precision, recall, last = _pr_points(tps, fps)
    return (recall[:last + 1] - np.r_[0.0, recall[:last]]) * precision[:last + 1]


def is_binary(y):
    """typeOfTarget(y) == "binary": every label the lowest or the highest, and no NaN."""
    v = np.asarray(y, np.float32)
    if np.isnan(v).any():
        return False
    return bool(((v == v.min()) | (v == v.max())).all())


def average_precision(pred, y):
    """AveragePrecisionScore of a binary target, pos_label = 1, summed by math.fsum; NaN with no positives.  Raises
    ValueError for labels that are not binary, which the device refuses."""
    if not is_binary(y):
        raise ValueError("labels are not binary")
    tps, fps, _ = clf_curve(pred, y, 1.0)
    return math.fsum(ap_terms(tps, fps)) if tps[-1] > 0 else QNAN


def group_average_precision(pred, y, group):
    """Samples ordered by (group, score key), counts from each group's start, AP_g = math.fsum of the group's terms
    (recall over the group's own positives; NaN with none), MAP = math.fsum of AP_g over the groups with a positive
    divided by their number.  Returns (map, groups, n, pos, ap)."""
    if not is_binary(y):
        raise ValueError("labels are not binary")
    key = auc_score_keys(pred)
    pos = np.asarray(y, np.float32) == np.float32(1.0)
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
    cnt = np.diff(np.r_[starts, n]).astype(np.int64)
    P = np.add.reduceat(ps, starts)
    first = np.r_[True, ge[1:] != ge[:-1]]
    Pe = P[ge].astype(np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        rec = tpe / Pe
        prev = np.where(first, 0.0, np.r_[0.0, rec[:-1]])
        terms = (rec - prev) * (tpe / (tpe + fpe).astype(np.float64))
    ap = np.full(starts.size, QNAN)
    bounds = np.r_[np.flatnonzero(first), ends.size]
    for k in np.flatnonzero(P > 0):
        s, e = bounds[k], bounds[k + 1]
        ap[k] = terms[s] if e - s == 1 else math.fsum(terms[s:e])
    used = P > 0
    m = math.fsum(ap[used]) / float(used.sum()) if used.any() else QNAN
    return m, gs[starts], cnt, P, ap
