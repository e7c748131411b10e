"""Python restatement of the reference's nn/metrics/classification.go and regression.go (with LabelEncoder,
feature/preprocessing/label.go:273-340, and AccuracyScore64, nn/neural_network/basemlp64.go:1143-1155), line by line
and quirks included, for the tests of ctr_accuracy_score, ctr_confusion_matrix, ctr_precision_recall_fscore,
ctr_r2_score, ctr_mean_error and ctr_mlp_accuracy.

The literal functions take lists of rows (lists of floats) as the reference's mat.Dense and loop as the Go does.  The
vectorised helpers below them give the same quantities with numpy for the large GPU cases: exact integer counts, and
weighted sums by math.fsum."""
import bisect
import math

import numpy as np


# ---- classification.go -------------------------------------------------------------------------------------------
def accuracy_score(Ytrue, Ypred, normalize, sampleWeight):
    """AccuracyScore (classification.go:12-34)"""
    N, D = 0.0, 0.0
    w = 1.0
    for i in range(len(Ytrue)):
        if sampleWeight is not None:
            w = sampleWeight[i]
        eq = True
        for j in range(len(Ytrue[i])):
            eq = eq and Ytrue[i][j] == Ypred[i][j]
        if eq:
            N += w
        D += w
    if normalize:
        return N / D if D != 0 else (math.nan if N == 0 else math.copysign(math.inf, N) * math.copysign(1.0, D))
    return N


def accuracy_score64(Y, H):
    """AccuracyScore64 (basemlp64.go:1143-1155): unweighted, normalised by the rows"""
    N = 0
    for i in range(len(Y)):
        if all(H[i][c] == Y[i][c] for c in range(len(Y[i]))):
            N += 1
    return float(N) / float(len(Y))


def search_float64s(a, x):
    """sort.SearchFloat64s: the first i with a[i] >= x (len(a) when none)"""
    return bisect.bisect_left(a, x)


def label_encoder_fit(y):
    """LabelEncoder.Fit / PartialFit (label.go:288-321) of one column: (classes, support)"""
    classes, support = [], []
    for v in y:
        pos = search_float64s(classes, v)
        if pos < len(classes) and classes[pos] == v:
            support[pos] += 1
            continue
        classes.insert(pos, v)
        support.insert(pos, 1.0)
    return classes, support


def label_encoder_transform(classes, y):
    """LabelEncoder.Transform (:324-339) of one column: the class index, -1 above the largest class"""
    out = []
    for v in y:
        pos = search_float64s(classes, v)
        if pos < 0 or pos >= len(classes):
            pos = -1
        out.append(pos)
    return out


def internal_confusion_matrix(YTrue, YPred, sampleWeight):
    """internalConfusionMatrix (classification.go:154-178) of 1-D labels: (cm as a list of rows, classes, support).
    The flat write cmmat.Data[r*C + c] of the Go: a prediction above the largest class (c = -1) lands in the cell
    before (r, 0), and at r = 0 the index -1 panics (IndexError here)."""
    classes, support = label_encoder_fit(YTrue)
    yt = label_encoder_transform(classes, YTrue)
    yp = label_encoder_transform(classes, YPred)
    C = len(classes)
    data = [0.0] * (C * C)
    for sample, (r, c) in enumerate(zip(yt, yp)):
        w = 1.0
        if sampleWeight is not None:
            w = sampleWeight[sample]
        idx = r * C + c
        if idx < 0:
            raise IndexError("index out of range [-1]")
        data[idx] += w
    return [data[r * C:(r + 1) * C] for r in range(C)], classes, support


def confusion_matrix(YTrue, YPred, sampleWeight):
    return internal_confusion_matrix(YTrue, YPred, sampleWeight)[0]


def prfs(tpsum, truesum, predsum, beta):
    """the prfs closure (:83-101) without support"""
    precision = recall = fscore = 0.0
    if predsum > 0.0:
        precision = tpsum / predsum
    if truesum > 0.0:
        recall = tpsum / truesum
    beta2 = beta * beta
    if beta2 * precision + recall > 0.0:
        fscore = (1 + beta2) * precision * recall / (beta2 * precision + recall)
    return precision, recall, fscore


def precision_recall_fscore_support(YTrue, YPred, beta, posLabel, average, sampleWeight, per_class=False):
    """PrecisionRecallFScoreSupport (:74-148).  Where the Go panics (posLabel >= NClasses) this raises IndexError; an
    unknown average returns zeros as the Go does.  per_class=True also returns the (p, r, f, support) of every class."""
    cm, classes, support = internal_confusion_matrix(YTrue, YPred, sampleWeight)
    C = len(classes)
    sums = []
    rows = []
    for c in range(C):
        g = (cm[c][c], sum(cm[c]), sum(cm[r][c] for r in range(C)))
        sums.append(g)
        p, r, f = prfs(*g, beta)
        rows.append((p, r, f, float(support[c])))
    if posLabel >= 0:
        if posLabel >= C:
            raise IndexError("posLabel>=NClasses %d,%d" % (posLabel, C))
        res = rows[posLabel]
    else:
        res = (0.0, 0.0, 0.0, 0.0)
        if average in ("macro", "weighted"):
            # the support weights are built and then stat.Mean(p, nil) ignores them (:116-131)
            res = (sum(x[0] for x in rows) / C, sum(x[1] for x in rows) / C, sum(x[2] for x in rows) / C, 0.0)
        if average == "micro":
            g = [0.0, 0.0, 0.0]
            for g1 in sums:
                g = [g[0] + g1[0], g[1] + g1[1], g[2] + g1[2]]
            res = prfs(*g, beta) + (0.0,)
    return (res, rows) if per_class else res


# ---- regression.go -----------------------------------------------------------------------------------------------
def r2_score(yTrue, yPred, sampleWeight, multioutput):
    """R2Score (regression.go:83-128): a list of n_out floats for "raw_values", else one float"""
    n, k = len(yTrue), len(yTrue[0])
    w = [1.0] * n if sampleWeight is None else list(sampleWeight)
    num = [sum(w[i] * ((yPred[i][j] - yTrue[i][j]) * (yPred[i][j] - yTrue[i][j])) for i in range(n)) for j in range(k)]
    wsum = sum(w)
    avg = [sum(w[i] * yTrue[i][j] for i in range(n)) * (1.0 / wsum) for j in range(k)]
    den = [sum(w[i] * ((yTrue[i][j] - avg[j]) * (yTrue[i][j] - avg[j])) for i in range(n)) for j in range(k)]
    r2 = [1.0 - num[j] / go_max(den[j], 1e-20) for j in range(k)]
    if multioutput == "raw_values":
        return r2
    if multioutput == "variance_weighted":
        dot = sum(den[j] * r2[j] for j in range(k))
        sumden = sum(den)
        return dot * (1.0 / sumden) if sumden != 0 else (math.nan if dot == 0 or math.isnan(dot) else dot * math.inf)
    return sum(r2) / float(k)


def go_max(a, b):
    """math.Max: NaN wins"""
    if math.isnan(a) or math.isnan(b):
        return math.nan
    return max(a, b)


def _mean_error(yTrue, yPred, multioutput, f):
    n, k = len(yTrue), len(yTrue[0])
    tmp = []
    for j in range(k):
        N, D = 0.0, 0.0
        for i in range(n):
            N += 1.0 * f(yPred[i][j] - yTrue[i][j])
            D += 1.0
        tmp.append(N / D)
    if multioutput == "raw_values":
        return tmp
    return sum(tmp) / float(k)


def mean_squared_error(yTrue, yPred, multioutput):
    """MeanSquaredError (regression.go:153-176) without sample weights"""
    return _mean_error(yTrue, yPred, multioutput, lambda d: d * d)


def mean_absolute_error(yTrue, yPred, multioutput):
    """MeanAbsoluteError (regression.go:220-244) without sample weights"""
    return _mean_error(yTrue, yPred, multioutput, abs)


# ---- vectorised, for large n -------------------------------------------------------------------------------------
def classes_of(y_true):
    """LabelEncoder.Fit's classes with numpy: distinct values ascending, ±0 one class with the sign of its first
    occurrence"""
    y = np.asarray(y_true, np.float64)
    key = np.where(y == 0, 0.0, y)
    u, first = np.unique(key, return_index=True)
    return y[first]


def encode(classes, y):
    return np.searchsorted(np.where(classes == 0, 0.0, classes), np.where(np.asarray(y) == 0, 0.0, y), side="left")


def counts(y_true, y_pred):
    """(classes, cm int64 [C, C]) unweighted"""
    cl = classes_of(y_true)
    C = cl.size
    t, p = encode(cl, y_true), encode(cl, y_pred)
    cm = np.bincount(t.astype(np.int64) * C + p, minlength=C * C).reshape(C, C) if C * C <= 1 << 26 else None
    return cl, t, p, cm


def fsum_by(keys, w, size):
    """out[k] = math.fsum of w over the samples with key k (0 where none)"""
    out = np.zeros(size, np.float64)
    order = np.argsort(keys, kind="stable")
    ks, ws = keys[order], w[order]
    if ks.size == 0:
        return out
    starts = np.flatnonzero(np.r_[True, ks[1:] != ks[:-1]])
    ends = np.r_[starts[1:], ks.size]
    for s, e in zip(starts, ends):
        out[ks[s]] = math.fsum(ws[s:e])
    return out


def prf_exact(y_true, y_pred, weight, beta):
    """per class (tp, truesum, predsum, support) with exact counts or fsum-weighted sums, and the per-class rows (p, r,
    f, support) by prfs"""
    cl, t, p, _ = counts(y_true, y_pred)
    C = cl.size
    support = np.bincount(t, minlength=C).astype(np.float64)
    if weight is None:
        tp = np.bincount(t[t == p], minlength=C).astype(np.float64)
        ts = support.copy()
        ps = np.bincount(p, minlength=C).astype(np.float64)
    else:
        w = np.asarray(weight, np.float64)
        tp = fsum_by(t[t == p], w[t == p], C)
        ts = fsum_by(t, w, C)
        ps = fsum_by(p, w, C)
    rows = np.array([prfs(tp[c], ts[c], ps[c], beta) + (support[c],) for c in range(C)], np.float64).reshape(C, 4)
    return cl, tp, ts, ps, rows
