"""ctr_accuracy_score, ctr_confusion_matrix, ctr_precision_recall_fscore, ctr_r2_score, ctr_mean_error and
ctr_mlp_accuracy on one H100 against the restatement (tests/metrics_restatement.py).  Unweighted counts and matrix
cells must be exactly equal; weighted sums within 1e-12 relative of math.fsum (exactly equal where the weights are
dyadic, so every order sums them exactly); a second call gives the same bits.  The grid-stride loops run several passes
at n = 300 001 and 5 000 003."""
import ctypes as C
import math

import numpy as np
import pytest

import go_ctr_b200 as g
from tests import metrics_restatement as R

pytestmark = pytest.mark.gpu
_dp = C.POINTER(C.c_double)
SIZES = [1, 2, 33, 257, 300_001, 5_000_003]


@pytest.fixture(scope="module")
def eng():
    return g.Engine(g.engine.default_config(g.MODEL_YOUTUBE, batch=1, pred_batch=1))


def _bits(a):
    return np.asarray(a, np.float64).view(np.uint64)


def _same(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(_bits(a), _bits(b))


def _close(a, b, rel=1e-12):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    both_nan = np.isnan(a) & np.isnan(b)
    return a.shape == b.shape and bool(np.all(both_nan | (np.abs(a - b) <= rel * np.maximum(1.0, np.abs(b)))))


def _labels(n, C, rng):
    """y_true with min(n, C) classes (sparse, negative, ±0 in both signs), y_pred on classes, between two classes,
    below the smallest and equal to the largest"""
    vals = np.unique(rng.integers(-4 * C - 8, 4 * C + 8, 4 * C + 16)).astype(np.float64) * 0.5
    vals = np.unique(np.r_[vals[rng.permutation(vals.size)[:C - 1]], 0.0])
    vals = vals[:C]
    k = min(n, vals.size)
    idx = rng.integers(0, k, n)
    idx[rng.permutation(n)[:k]] = np.arange(k)               # every class present
    yt = vals[:k][idx]
    z = yt == 0
    yt[z & (rng.random(n) < 0.5)] = -0.0
    cl = np.unique(np.where(yt == 0, 0.0, yt))
    r = rng.random(n)
    pi = rng.integers(0, cl.size, n)
    yp = cl[pi].copy()
    mid = (r < 0.2) & (pi + 1 < cl.size)
    yp[mid] = (cl[pi[mid]] + cl[pi[mid] + 1]) / 2                 # between two classes: the higher one
    yp[(r >= 0.2) & (r < 0.25)] = cl[0] - 3.0                     # below the smallest: class 0
    yp[(r >= 0.25) & (r < 0.3)] = cl[-1]                          # the largest
    yp[(r >= 0.3) & (r < 0.35) & (yp == 0)] = -0.0
    return yt, yp


def _weights(kind, n, rng):
    if kind == "none":
        return None
    if kind == "positive":
        return rng.integers(1, 33, n) / 8.0
    if kind == "zero":
        w = rng.integers(0, 9, n) / 4.0
        w[rng.random(n) < 0.5] = 0.0
        return w
    if kind == "negative":
        return rng.integers(-16, 17, n) / 4.0
    if kind == "float":
        return rng.random(n) * 3.0 - 1.0
    raise ValueError(kind)


def _prf(eng, yt, yp, w, beta, average, pos_label=-1, per_class=True, cap=None):
    n = yt.size
    nc = C.c_int32(-1)
    o = [C.c_double(0) for _ in range(4)]
    pc = np.full((n if cap is None else max(cap, 1), 4), -7.0)
    wp = None if w is None else w.ctypes.data_as(_dp)
    rc = eng.L.ctr_precision_recall_fscore(eng.h, yt.ctypes.data_as(_dp), yp.ctypes.data_as(_dp), C.c_int64(n), wp, C.c_double(beta),
                                           C.c_int32(average), C.c_int32(pos_label), *[C.byref(x) for x in o],
                                           pc.ctypes.data_as(_dp) if per_class else None, C.c_int64(n if cap is None else cap), C.byref(nc))
    return rc, np.array([x.value for x in o]), pc, nc.value


CASES = [(n, c) for n in SIZES for c in (1, 2, 3, 1024, 70_000) if c <= max(n, 3) and not (c == 70_000 and n < 300_001)]


@pytest.mark.parametrize("n,ncls", CASES)
@pytest.mark.parametrize("wkind", ["none", "positive", "zero", "negative"])
def test_classes_matrix_and_scores_equal_the_restatement(eng, n, ncls, wkind):
    if wkind != "none" and n == 5_000_003 and ncls == 70_000:
        pytest.skip("covered by the unweighted case and the smaller weighted ones")
    rng = np.random.default_rng(n * 7 + ncls + len(wkind))
    yt, yp = _labels(n, ncls, rng)
    w = _weights(wkind, n, rng)
    cl, t, p, _ = R.counts(yt, yp)
    Cn = cl.size
    # classes and matrix (cm NULL when C² does not fit)
    classes = np.full(n, -9.0)
    want_cm = Cn * Cn <= 1 << 21
    cm = np.full(Cn * Cn if want_cm else 1, -9.0)
    nc = C.c_int32(-1)
    rc = eng.L.ctr_confusion_matrix(eng.h, yt.ctypes.data_as(_dp), yp.ctypes.data_as(_dp), C.c_int64(n),
                                    None if w is None else w.ctypes.data_as(_dp), classes.ctypes.data_as(_dp),
                                    cm.ctypes.data_as(_dp) if want_cm else None, C.c_int64(Cn * Cn), C.byref(nc))
    assert rc == 0, eng.L.ctr_last_error(eng.h)
    assert nc.value == Cn and _same(classes[:Cn], cl)                    # ±0 keeps the sign of its first occurrence
    if want_cm:
        key = t.astype(np.int64) * Cn + p
        expect = np.bincount(key, weights=w, minlength=Cn * Cn) if w is not None else np.bincount(key, minlength=Cn * Cn)
        assert np.array_equal(cm, expect.astype(np.float64))              # dyadic weights sum exactly in any order
    # per-class rows, every average, pos_label
    beta = 0.5 if ncls == 3 else 1.0
    _, tp, ts, ps, rows = R.prf_exact(yt, yp, w, beta)
    for avg in (g.AVERAGE["macro"], g.AVERAGE["micro"], g.AVERAGE["weighted"]):
        rc, out, pc, ncl = _prf(eng, yt, yp, w, beta, avg)
        assert rc == 0, eng.L.ctr_last_error(eng.h)
        assert ncl == Cn and _same(pc[:Cn], rows)
        if avg == g.AVERAGE["micro"]:
            want = R.prfs(math.fsum(tp), math.fsum(ts), math.fsum(ps), beta)
            assert _same(out[:3], want) and out[3] == 0.0
        else:
            want = [math.fsum(rows[:, k]) / Cn for k in range(3)]
            assert _close(out[:3], want) and out[3] == 0.0
        rc2, out2, pc2, _ = _prf(eng, yt, yp, w, beta, avg)
        assert rc2 == 0 and _same(out2, out) and _same(pc2, pc)
    for pos in {0, Cn // 2, Cn - 1}:
        rc, out, _, _ = _prf(eng, yt, yp, w, beta, 0, pos_label=pos, per_class=False)
        assert rc == 0 and _same(out, rows[pos])


@pytest.mark.parametrize("n,ncls", [(300_001, 3), (300_001, 1024), (5_000_003, 2)])
def test_float_weights_within_1e12_of_fsum(eng, n, ncls):
    rng = np.random.default_rng(n + ncls)
    yt, yp = _labels(n, ncls, rng)
    w = _weights("float", n, rng)
    _, tp, ts, ps, rows = R.prf_exact(yt, yp, w, 1.0)
    rc, out, pc, Cn = _prf(eng, yt, yp, w, 1.0, g.AVERAGE["micro"])
    assert rc == 0
    assert _close(out[:3], R.prfs(math.fsum(tp), math.fsum(ts), math.fsum(ps), 1.0))
    assert _same(pc[:Cn, 3], rows[:, 3]) and _close(pc[:Cn, :3], rows[:, :3])
    if ncls <= 3:
        cl, cm = eng.confusion_matrix(yt, yp, w)
        _, t, p, _ = R.counts(yt, yp)
        assert _close(cm.ravel(), R.fsum_by(t.astype(np.int64) * cl.size + p, w, cl.size ** 2))
        cl2, cm2 = eng.confusion_matrix(yt, yp, w)
        assert _same(cm2, cm)


def test_between_classes_counts_as_the_higher_one(eng):
    yt = np.array([0.0, 1.0, 3.0, 3.0]); yp = np.array([0.5, 2.0, -7.0, 3.0])
    cl, cm = eng.confusion_matrix(yt, yp)
    assert cl.tolist() == [0.0, 1.0, 3.0]
    assert cm.tolist() == [[0, 1, 0], [0, 0, 1], [1, 0, 1]]


def test_classification_refusals_write_nothing_but_n_classes(eng):
    yt = np.array([0.0, 1.0, 2.0, 1.0]); n = 4
    cases = [(yt, np.array([0.0, 1.0, 2.5, 1.0]), None, b"y_pred[2] = 2.5 is above the largest class", 3),
             (np.array([0.0, np.nan, 2.0, np.nan]), yt, None, b"y_true[1] is NaN", -1),
             (yt, np.array([0.0, 1.0, np.nan, np.nan]), None, b"y_pred[2] is NaN", 3),
             (yt, yt, np.array([1.0, 1.0, np.inf, 1.0]), b"weight[2]", 3),
             (yt, yt, np.array([1.0, np.nan, 1.0, 1.0]), b"weight[1]", 3)]
    for a, b, w, msg, want_nc in cases:
        classes = np.full(n, -9.0); cm = np.full(16, -9.0); nc = C.c_int32(-1)
        rc = eng.L.ctr_confusion_matrix(eng.h, a.ctypes.data_as(_dp), b.ctypes.data_as(_dp), C.c_int64(n),
                                        None if w is None else w.ctypes.data_as(_dp), classes.ctypes.data_as(_dp),
                                        cm.ctypes.data_as(_dp), C.c_int64(16), C.byref(nc))
        assert rc == g.EINVAL and msg in eng.L.ctr_last_error(eng.h), eng.L.ctr_last_error(eng.h)
        assert nc.value == want_nc and np.all(classes == -9.0) and np.all(cm == -9.0)
        rc, out, pc, ncl = _prf(eng, a, b, w, 1.0, 0)
        assert rc == g.EINVAL and ncl == want_nc and np.all(out == 0) and np.all(pc == -7.0)
    # capacity: C² > cap, C > cap for the per-class rows, pos_label >= C
    classes = np.full(n, -9.0); cm = np.full(16, -9.0); nc = C.c_int32(-1)
    rc = eng.L.ctr_confusion_matrix(eng.h, yt.ctypes.data_as(_dp), yt.ctypes.data_as(_dp), C.c_int64(n), None,
                                    classes.ctypes.data_as(_dp), cm.ctypes.data_as(_dp), C.c_int64(8), C.byref(nc))
    assert rc == g.EINVAL and nc.value == 3 and np.all(classes == -9.0) and np.all(cm == -9.0)
    rc, out, pc, ncl = _prf(eng, yt, yt, None, 1.0, 0, cap=2)
    assert rc == g.EINVAL and ncl == 3 and np.all(out == 0) and np.all(pc == -7.0)
    rc, out, pc, ncl = _prf(eng, yt, yt, None, 1.0, 0, pos_label=3)
    assert rc == g.EINVAL and b"pos_label 3" in eng.L.ctr_last_error(eng.h) and np.all(out == 0) and np.all(pc == -7.0)
    # every output NULL but n_classes
    rc = eng.L.ctr_confusion_matrix(eng.h, yt.ctypes.data_as(_dp), yt.ctypes.data_as(_dp), C.c_int64(n), None, None, None,
                                    C.c_int64(9), C.byref(nc))
    assert rc == 0 and nc.value == 3


ACC_SIZES = [(n, k) for n in SIZES for k in (1, 3, 1024) if n * k <= 20_000_000]


@pytest.mark.parametrize("n,n_out", ACC_SIZES)
@pytest.mark.parametrize("wkind", ["none", "negative", "float"])
def test_accuracy_equals_the_restatement(eng, n, n_out, wkind):
    rng = np.random.default_rng(n + n_out)
    yt = rng.integers(-2, 3, (n, n_out)).astype(np.float64)
    yp = yt.copy()
    flip = rng.random((n, n_out)) < 0.5 / n_out
    yp[flip] += 1.0
    yt[(yt == 0) & (rng.random((n, n_out)) < 0.5)] = -0.0           # -0 == +0
    nan_rows = rng.random(n) < 0.01
    yt[nan_rows, 0] = np.nan; yp[nan_rows, 0] = np.nan               # a NaN never equals
    w = _weights(wkind, n, rng)
    ok = np.all(yt == yp, axis=1)
    for normalize in (1, 0):
        got = eng.accuracy_score(yt, yp, normalize=bool(normalize), weight=w)
        if w is None:
            want = ok.sum() / n if normalize else float(ok.sum())
            assert _same(got, want)
        else:
            N, D = math.fsum(w[ok]), math.fsum(w)
            with np.errstate(divide="ignore", invalid="ignore"):
                want = float(np.float64(N) / np.float64(D)) if normalize else N
            assert _close(got, want) or got == want, (got, want)
        assert _same(eng.accuracy_score(yt, yp, normalize=bool(normalize), weight=w), got)


def test_accuracy_weights_and_refusals(eng):
    yt = np.array([1.0, 2.0]); yp = np.array([0.0, 0.0])
    assert math.isnan(eng.accuracy_score(yt, yp, weight=np.array([0.0, 0.0])))
    assert eng.accuracy_score(yt, yt, weight=np.array([2.0, -0.5])) == 1.0
    assert eng.accuracy_score(yt, yt, normalize=False, weight=np.array([2.0, -0.5])) == 1.5
    out = C.c_double(-3.0)
    for bad in (np.inf, -np.inf, np.nan):
        w = np.array([1.0, bad])
        rc = eng.L.ctr_accuracy_score(eng.h, yt.ctypes.data_as(_dp), yp.ctypes.data_as(_dp), C.c_int64(2), C.c_int32(1),
                                      w.ctypes.data_as(_dp), C.c_int32(1), C.byref(out))
        assert rc == g.EINVAL and out.value == -3.0


REG = [(n, k) for n in SIZES for k in (1, 3, 1024) if n * k <= 20_000_000]


def _reg_expect(yt, yp, w):
    n, k = yt.shape
    ww = np.ones(n) if w is None else w
    num = np.array([math.fsum(ww * ((yp[:, j] - yt[:, j]) * (yp[:, j] - yt[:, j]))) for j in range(k)])
    avg = np.array([math.fsum(ww * yt[:, j]) / math.fsum(ww) for j in range(k)])
    den = np.array([math.fsum(ww * ((yt[:, j] - avg[j]) * (yt[:, j] - avg[j]))) for j in range(k)])
    r2 = 1.0 - num / np.maximum(den, 1e-20)
    return num, den, r2


@pytest.mark.parametrize("n,n_out", REG)
@pytest.mark.parametrize("wkind", ["none", "positive", "zero"])
def test_regression_equals_the_restatement(eng, n, n_out, wkind):
    if n < 2 and wkind == "zero":
        pytest.skip("every weight zero: 0/0 in the mean")
    rng = np.random.default_rng(n * 3 + n_out)
    yt = rng.standard_normal((n, n_out)) * 3.0 + 1.0
    yp = yt + rng.standard_normal((n, n_out)) * 0.5
    if n_out > 1:
        yt[:, 1] = 2.5                                                 # a constant column is not refused
    w = _weights(wkind, n, rng)
    if w is not None and not np.any(w):
        w[0] = 1.0
    num, den, r2 = _reg_expect(yt, yp, w)
    tol = 1e-12 * (1.0 + np.abs(num / np.maximum(den, 1e-20)))
    raw = eng.r2_score(yt, yp, w, "raw_values")
    assert np.all(np.abs(raw - r2) <= tol), (raw, r2)
    uni = eng.r2_score(yt, yp, w, "uniform_average")
    assert abs(uni - math.fsum(raw) / n_out) <= 1e-12 * (1.0 + np.max(tol) * 1e12)
    vw = eng.r2_score(yt, yp, w, "variance_weighted")
    sd = math.fsum(den)
    if sd == 0:
        assert math.isnan(vw)
    else:
        want = math.fsum(den * r2) / sd
        assert abs(vw - want) <= 1e-12 * (1.0 + math.fsum(np.abs(den * r2)) / abs(sd)), (vw, want)
    assert _same(eng.r2_score(yt, yp, w, "raw_values"), raw)
    if w is None:
        for kind, f in (("squared", lambda d: d * d), ("absolute", np.abs)):
            e = np.array([math.fsum(f(yp[:, j] - yt[:, j])) / n for j in range(n_out)])
            got = eng.mean_error(yt, yp, kind, "raw_values")
            assert _close(got, e), (kind, got, e)
            assert _close(eng.mean_error(yt, yp, kind, "uniform_average"), math.fsum(got) / n_out)
            assert _same(eng.mean_error(yt, yp, kind, "raw_values"), got)


def test_regression_edges(eng):
    # every column constant: den 0 everywhere, the 1e-20 floor, variance weighted NaN
    yt = np.full((5, 2), 3.0); yp = yt.copy(); yp[0, 0] = 4.0
    raw = eng.r2_score(yt, yp, None, "raw_values")
    assert raw[0] == 1.0 - 1.0 / 1e-20 and raw[1] == 1.0
    assert math.isnan(eng.r2_score(yt, yp, None, "variance_weighted"))
    # NaN and inf propagate
    yt = np.array([[1.0, 1.0], [2.0, np.nan], [3.0, 2.0]]); yp = np.array([[1.0, 1.0], [np.inf, 1.0], [3.0, 2.0]])
    raw = eng.r2_score(yt, yp, None, "raw_values")
    assert math.isnan(raw[0]) or raw[0] == -math.inf
    assert math.isnan(raw[1])
    assert math.isnan(eng.mean_error(yt, yp, "squared", "raw_values")[1])
    assert eng.mean_error(yt, yp, "absolute", "raw_values")[0] == math.inf
    # the reference's known answers through the mirrors
    assert abs(g.R2Score([[3], [-0.5], [2], [7]], [[2.5], [0.0], [2], [8]], None, "", engine=eng) - 0.948) <= 1e-3
    assert abs(g.R2Score([[0.5, 1], [-1, 1], [7, -6]], [[0, 2], [-1, 2], [8, -5]], None, "variance_weighted", engine=eng) - 0.938) <= 1e-3
    assert g.R2Score([[1], [2], [3]], [[3], [2], [1]], np.ones((3, 1)), "", engine=eng) == -3.0
    assert g.MeanSquaredError([[3, -0.5, 2, 7]], [[2.5, 0.0, 2, 8]], None, "", engine=eng) == 0.375
    assert g.MeanAbsoluteError([[3, -0.5, 2, 7]], [[2.5, 0.0, 2, 8]], None, "", engine=eng) == 0.5
    np.testing.assert_allclose(g.MeanSquaredError([[0.5, 1], [-1, 1], [7, -6]], [[0, 2], [-1, 2], [8, -5]], None, "raw_values", engine=eng),
                               [0.416, 1.0], atol=1e-3)
    with pytest.raises(g.CtrError) as e:
        g.MeanSquaredError([[1.0]], [[1.0]], None, "variance_weighted", engine=eng)
    assert e.value.code == g.EINVAL


def test_classification_mirrors_give_the_known_answers(eng):
    assert g.AccuracyScore([[0], [1], [2], [3]], [[0], [2], [1], [3]], True, None, engine=eng) == 0.5
    assert g.AccuracyScore([[0, 1], [1, 1]], [[1, 1], [1, 1]], True, None, engine=eng) == 0.5
    assert g.ConfusionMatrix([[2], [0], [2], [2], [0], [1]], [[0], [0], [2], [2], [0], [2]], None, engine=eng).tolist() == \
        [[2, 0, 0], [0, 0, 1], [1, 0, 2]]
    yt, yp = [0, 1, 2, 0, 1, 2], [0, 2, 1, 0, 0, 1]
    got = [("%.2f" % f(yt, yp, a, None, engine=eng)) for f in (g.PrecisionScore, g.RecallScore, g.F1Score) for a in ("macro", "micro", "weighted")]
    assert got == ["0.22", "0.33", "0.22", "0.33", "0.33", "0.33", "0.27", "0.33", "0.27"]
    assert ["%.2f" % g.FBetaScore(yt, yp, 0.5, a, None, engine=eng) for a in ("macro", "micro", "weighted")] == ["0.24", "0.33", "0.24"]
    assert ["%.2f" % v for v in g.PrecisionRecallFScoreSupport(yt, yp, 1, None, -1, "macro", None, None, engine=eng)] == ["0.22", "0.33", "0.27", "0.00"]
    assert g.PrecisionRecallFScoreSupport(yt, yp, 1, [], -1, "weighted", [], [1, 2, 3, 4, 5, 6], engine=eng) == \
        g.PrecisionRecallFScoreSupport(yt, yp, 1, [], -1, "macro", [], [1, 2, 3, 4, 5, 6], engine=eng)


def test_profile_names_the_metric_kernels(eng):
    rng = np.random.default_rng(0)
    yt, yp = _labels(1000, 5, rng)
    w = _weights("positive", 1000, rng)
    eng.profile(True)
    try:
        eng.profile_reset()
        eng.accuracy_score(yt, yp); eng.precision_recall_fscore(yt, yp, weight=w); eng.confusion_matrix(yt, yp)
        eng.r2_score(yt[:, None], yp[:, None], w); eng.mean_error(yt[:, None], yp[:, None])
        keys = set(eng.profile_dump())
    finally:
        eng.profile(False)
    assert {"acc_part", "acc_final", "met_keys", "met_classes", "met_class_values", "met_encode", "met_sort_cells", "met_sort_cols",
            "met_seg_piece", "met_seg_heads", "met_seg_total", "met_cm", "met_prf", "r2_mean", "r2_mean_fold", "r2_sums", "r2_fold",
            "err_sums", "err_fold"} <= keys, keys


# ---- MLPClassifier.Score ------------------------------------------------------------------------------------------
def _predict_f64(m, X, width):
    out = np.empty((X.shape[0], width), np.float64)
    Xa = np.ascontiguousarray(X, np.float32)
    assert m.L.ctr_mlp_predict_f64(m.h, Xa.ctypes.data_as(C.POINTER(C.c_float)), C.c_int64(Xa.shape[0]), C.c_int32(Xa.shape[1]),
                                   out.ctypes.data_as(_dp)) == 0
    return out


def test_binary_score_compares_the_float64_probability(eng):
    m = g.MLPClassifier(2, hidden=(), max_iter=1)
    m.set_params(np.array([0.0, 60.0, -900.0]))                     # logistic(60 x0 − 900 x1): 1.0 or 0.0 at the extremes
    rng = np.random.default_rng(1)
    n = 20_011                                                       # three forward chunks
    X = np.c_[rng.choice([0.0, 1.0, 0.01, 0.5], n), rng.choice([0.0, 1.0, 0.001], n)].astype(np.float32)
    Y = rng.choice(np.array([0.0, 1.0], np.float32), n)
    prob = _predict_f64(m, X, 1)
    assert np.any(prob == 1.0) and np.any(prob == 0.0) and np.any((prob > 0) & (prob < 1))
    acc = m.score(X, Y)
    want = np.sum(prob[:, 0] == Y.astype(np.float64)) / n
    assert _same(acc, want)
    assert _same(acc, eng.accuracy_score(Y.astype(np.float64), prob[:, 0]))
    assert _same(m.score(X, Y), acc)


def test_multiclass_score_equals_accuracy_of_predict(eng):
    rng = np.random.default_rng(2)
    n, nf = 20_000, 6
    X = rng.standard_normal((n, nf)).astype(np.float32)
    cls = np.array([-1.0, 2.5, 7.0], np.float32)
    Y = cls[np.argmax(X[:, :3] + 0.5 * rng.standard_normal((n, 3)), axis=1)]
    m = g.MLPClassifier(nf, hidden=(16,), max_iter=3, seed=3).fit(X, Y)
    assert m.classes_.size == 3
    acc = m.score(X, Y)
    pred = m.predict(X)
    assert _same(acc, eng.accuracy_score(Y.astype(np.float64), pred.astype(np.float64)))
    assert 0.3 < acc <= 1.0


def test_one_class_score_is_label_equals_the_class(eng):
    m = g.MLPClassifier(2, hidden=(), max_iter=1)
    m.set_params(np.array([0.1, 0.2, -0.3]), classes=[5.0])
    rng = np.random.default_rng(4)
    X = rng.standard_normal((999, 2)).astype(np.float32)
    Y = rng.choice(np.array([5.0, 4.0, 6.0], np.float32), 999)
    assert _same(m.score(X, Y), np.sum(Y == 5.0) / 999)


def test_score_refusals(eng):
    X = np.zeros((4, 3), np.float32); Y = np.zeros(4, np.float32)
    m = g.MLPClassifier(3, hidden=(4,))
    with pytest.raises(g.CtrError) as e:
        m.score(X, Y)                                               # not fitted
    assert e.value.code == g.ESTATE
    r = g.MLPRegressor(3, hidden=(4,), max_iter=1).fit(X, Y)
    acc = C.c_double(-1)
    Xa = np.ascontiguousarray(X)
    assert r.L.ctr_mlp_accuracy(r.h, Xa.ctypes.data_as(C.POINTER(C.c_float)), Y.ctypes.data_as(C.POINTER(C.c_float)), C.c_int64(4),
                                C.c_int32(3), C.byref(acc)) == g.ESTATE and acc.value == -1
    assert b"ctr_mlp_score" in r.L.ctr_mlp_last_error(r.h)
    m.set_params(np.zeros(m.get_params().size))
    assert m.L.ctr_mlp_accuracy(m.h, Xa.ctypes.data_as(C.POINTER(C.c_float)), Y.ctypes.data_as(C.POINTER(C.c_float)), C.c_int64(4),
                                C.c_int32(2), C.byref(acc)) == g.EINVAL and acc.value == -1
    rc = m.L.ctr_mlp_score(m.h, Xa.ctypes.data_as(C.POINTER(C.c_float)), Y.ctypes.data_as(C.POINTER(C.c_float)), C.c_int64(4),
                           C.c_int32(3), C.byref(acc))
    assert rc == g.ESTATE and b"ctr_mlp_accuracy" in m.L.ctr_mlp_last_error(m.h)
