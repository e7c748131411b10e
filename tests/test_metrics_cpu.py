"""The classification and regression metrics without a device: the restatement (tests/metrics_restatement.py) against
the reference's known answers (tests/golden/metrics_kat.json) and its own quirks, every argument refusal of the C calls
that comes before any device work (read through ctr_last_error(NULL)), and the ValueErrors of the model.py mirrors."""
import ctypes as C
import json
import math
import os

import numpy as np
import pytest

import go_ctr_b200 as g
from tests import metrics_restatement as R

KAT = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "metrics_kat.json")))
_dp = C.POINTER(C.c_double)


def test_accuracy_known_answers():
    for c in KAT["accuracy"]:
        assert R.accuracy_score(c["y_true"], c["y_pred"], c["normalize"], c["weight"]) == c["expect"]


def test_confusion_matrix_known_answer():
    c = KAT["confusion_matrix"]
    assert R.confusion_matrix([float(v) for v in c["y_true"]], [float(v) for v in c["y_pred"]], None) == c["expect"]


@pytest.mark.parametrize("metric,beta,index", [("precision", 1.0, 0), ("recall", 1.0, 1), ("f1", 1.0, 2), ("fbeta_0.5", 0.5, 2),
                                               ("support", 1.0, 3)])
def test_precision_recall_fscore_known_answers(metric, beta, index):
    c = KAT["prf"]
    yt, yp = [float(v) for v in c["y_true"]], [float(v) for v in c["y_pred"]]
    for avg, want in c[metric].items():
        got = R.precision_recall_fscore_support(yt, yp, beta, -1, avg, None)[index]
        assert "%.*f" % (c["digits"], got) == "%.*f" % (c["digits"], want), (metric, avg, got)


def test_r2_known_answers():
    for c in KAT["r2"]:
        got = R.r2_score(c["y_true"], c["y_pred"], c["weight"], c["multioutput"])
        assert abs(got - c["expect"]) <= c["tol"], (c, got)
        fmt = "%g" if c["printed"] in ("0", "-3") else "%.3f"
        assert fmt % got == c["printed"]


@pytest.mark.parametrize("kind", ["mse", "mae"])
def test_mean_error_known_answers(kind):
    f = R.mean_squared_error if kind == "mse" else R.mean_absolute_error
    for c in KAT[kind]:
        got = f(c["y_true"], c["y_pred"], c["multioutput"])
        got = got if isinstance(got, list) else [got]
        for a, b in zip(got, c["expect"]):
            assert abs(a - b) <= c["tol"], (c, got)


def test_restatement_quirks():
    # a prediction between two classes counts as the higher one (sort.SearchFloat64s)
    assert R.confusion_matrix([0.0, 1.0, 3.0], [0.5, 2.0, -7.0], None) == [[0, 1, 0], [0, 0, 1], [1, 0, 0]]
    # above the largest class: the Go writes the cell before (r, 0), and panics at r = 0
    assert R.confusion_matrix([0.0, 1.0], [0.0, 5.0], None) == [[1, 1], [0, 0]]
    with pytest.raises(IndexError):
        R.confusion_matrix([0.0, 1.0], [5.0, 0.0], None)
    # ±0 are one class, keeping the sign of the first occurrence
    cl, sup = R.label_encoder_fit([-0.0, 0.0, 1.0])
    assert len(cl) == 2 and math.copysign(1.0, cl[0]) == -1.0 and sup == [2.0, 1.0]
    assert np.array_equal(np.signbit(R.classes_of([-0.0, 0.0, 1.0])), [True, False])
    # weighted equals macro; support comes from the unweighted counts
    yt, yp = [0.0, 1.0, 2.0, 0.0, 1.0, 2.0], [0.0, 2.0, 1.0, 0.0, 0.0, 1.0]
    w = [1.0, 2.0, 0.5, 3.0, 0.25, 1.0]
    assert R.precision_recall_fscore_support(yt, yp, 1.0, -1, "weighted", w) == R.precision_recall_fscore_support(yt, yp, 1.0, -1, "macro", w)
    assert R.precision_recall_fscore_support(yt, yp, 1.0, 0, "macro", w)[3] == 2.0
    assert R.precision_recall_fscore_support(yt, yp, 1.0, -1, "other", None) == (0.0, 0.0, 0.0, 0.0)
    # R² never divides by zero; variance_weighted with every den 0 is NaN
    assert R.r2_score([[1.0], [1.0]], [[1.0], [2.0]], None, "") == 1.0 - 1.0 / 1e-20
    assert math.isnan(R.r2_score([[1.0], [1.0]], [[1.0], [2.0]], None, "variance_weighted"))
    # accuracy: -0 == +0, NaN never equal; weights summing to zero with nothing correct give 0/0 = NaN
    assert R.accuracy_score([[-0.0], [math.nan]], [[0.0], [math.nan]], True, None) == 0.5
    assert math.isnan(R.accuracy_score([[1.0], [2.0]], [[0.0], [0.0]], True, [1.0, -1.0]))


def test_vectorised_restatement_equals_the_literal_one():
    rng = np.random.default_rng(3)
    for _ in range(20):
        n = int(rng.integers(1, 300))
        vals = np.array([-3.0, -0.0, 0.0, 1.5, 2.0, 7.0])
        yt = rng.choice(vals, n)
        yp = rng.choice(np.r_[vals, -5.0, 0.75, 1.6], n)
        cl = R.classes_of(yt)
        yp = np.minimum(yp, cl.max())                           # no prediction above the largest class
        w = rng.integers(-8, 9, n) / 4.0
        cm, classes, support = R.internal_confusion_matrix(list(yt), list(yp), list(w))
        assert np.array_equal(cl.view(np.uint64), np.array(classes).view(np.uint64))
        (_, rows) = R.precision_recall_fscore_support(list(yt), list(yp), 0.7, -1, "macro", list(w), per_class=True)
        _, tp, ts, ps, vrows = R.prf_exact(yt, yp, w, 0.7)
        assert np.array_equal(tp, np.diag(cm)) and np.array_equal(ts, np.sum(cm, axis=1))
        assert np.array_equal(vrows, np.array(rows))


def _lib():
    return g.load_library()


def _err():
    return _lib().ctr_last_error(None)


def _dd(*a):
    x = np.ascontiguousarray(a, np.float64)
    return x, x.ctypes.data_as(_dp)


def test_abi_refusals_before_device_work():
    L = _lib()
    yt, ytp = _dd(0, 1, 2)
    out, outp = _dd(0, 0, 0, 0)
    nc = C.c_int32(-7)
    i64, i32, dbl = C.c_int64, C.c_int32, C.c_double
    # accuracy: null pointers, n, n_out
    for args in [(None, ytp, i64(3), i32(1), None, i32(1), outp), (ytp, None, i64(3), i32(1), None, i32(1), outp),
                 (ytp, ytp, i64(3), i32(1), None, i32(1), None), (ytp, ytp, i64(0), i32(1), None, i32(1), outp),
                 (ytp, ytp, i64(1 << 31), i32(1), None, i32(1), outp), (ytp, ytp, i64(3), i32(0), None, i32(1), outp),
                 (ytp, ytp, i64(3), i32(1025), None, i32(1), outp)]:
        assert L.ctr_accuracy_score(None, *args) == g.EINVAL
        assert b"bad accuracy arguments" in _err()
    assert L.ctr_accuracy_score(None, ytp, ytp, i64(3), i32(1), None, i32(1), outp) == g.EINVAL and b"null handle" in _err()
    # confusion matrix
    for args in [(None, ytp, i64(3), None, None, None, i64(9), C.byref(nc)), (ytp, None, i64(3), None, None, None, i64(9), C.byref(nc)),
                 (ytp, ytp, i64(3), None, None, None, i64(9), None), (ytp, ytp, i64(0), None, None, None, i64(9), C.byref(nc))]:
        assert L.ctr_confusion_matrix(None, *args) == g.EINVAL
        assert b"bad confusion matrix arguments" in _err()
    assert nc.value == -7
    # precision / recall / F: nulls, n, average, beta
    base = [ytp, ytp, i64(3), None, dbl(1.0), i32(0), i32(-1), None, None, None, None, None, i64(3), C.byref(nc)]

    def prf(**kw):
        a = list(base)
        for k, v in kw.items():
            a[int(k[1:])] = v
        return L.ctr_precision_recall_fscore(None, *a)
    assert prf(a0=None) == g.EINVAL and b"bad precision/recall arguments" in _err()
    assert prf(a13=None) == g.EINVAL and b"bad precision/recall arguments" in _err()
    assert prf(a2=i64(0)) == g.EINVAL and b"bad precision/recall arguments" in _err()
    for avg in (-1, 3, 7):
        assert prf(a5=i32(avg)) == g.EINVAL and (b"average %d" % avg) in _err()
    for beta in (math.nan, math.inf, -math.inf):
        assert prf(a4=dbl(beta)) == g.EINVAL and b"beta" in _err() and b"finite" in _err()
    assert prf() == g.EINVAL and b"null handle" in _err()
    assert nc.value == -7
    # R²
    for args in [(None, ytp, i64(3), i32(1), None, i32(1), outp), (ytp, ytp, i64(3), i32(1), None, i32(1), None),
                 (ytp, ytp, i64(-1), i32(1), None, i32(1), outp), (ytp, ytp, i64(3), i32(0), None, i32(1), outp),
                 (ytp, ytp, i64(3), i32(2000), None, i32(1), outp)]:
        assert L.ctr_r2_score(None, *args) == g.EINVAL and b"bad r2 arguments" in _err()
    for mo in (-1, 3):
        assert L.ctr_r2_score(None, ytp, ytp, i64(3), i32(1), None, i32(mo), outp) == g.EINVAL and b"multioutput" in _err()
    # MSE / MAE
    for args in [(None, ytp, i64(3), i32(1), i32(0), i32(1), outp), (ytp, ytp, i64(3), i32(1), i32(0), i32(1), None),
                 (ytp, ytp, i64(0), i32(1), i32(0), i32(1), outp), (ytp, ytp, i64(3), i32(1025), i32(0), i32(1), outp)]:
        assert L.ctr_mean_error(None, *args) == g.EINVAL and b"bad mean error arguments" in _err()
    for k in (-1, 2):
        assert L.ctr_mean_error(None, ytp, ytp, i64(3), i32(1), i32(k), i32(1), outp) == g.EINVAL and b"kind" in _err()
    for mo in (2, 3, -1):
        assert L.ctr_mean_error(None, ytp, ytp, i64(3), i32(1), i32(0), i32(mo), outp) == g.EINVAL and b"multioutput" in _err()
    assert np.all(out == 0)
    # the classifier's accuracy
    acc = C.c_double(-1)
    assert L.ctr_mlp_accuracy(None, None, None, i64(3), i32(2), C.byref(acc)) == g.EINVAL and acc.value == -1


def test_mirror_value_errors():
    yt = [0.0, 1.0, 2.0]
    with pytest.raises(ValueError, match="average"):
        g.PrecisionScore(yt, yt, "samples", None)
    with pytest.raises(ValueError, match="average"):
        g.PrecisionRecallFScoreSupport(yt, yt, 1.0, None, -1, "binary", None, None)
    with pytest.raises(ValueError, match="labels"):
        g.PrecisionRecallFScoreSupport(yt, yt, 1.0, [0.0, 1.0], -1, "macro", None, None)
    with pytest.raises(ValueError, match="warnFor"):
        g.PrecisionRecallFScoreSupport(yt, yt, 1.0, [], -1, "macro", ["precision"], None)
    with pytest.raises(ValueError, match="multioutput"):
        g.R2Score([[1.0]], [[1.0]], None, "uniform")
    with pytest.raises(ValueError, match="multioutput"):
        g.MeanSquaredError([[1.0]], [[1.0]], None, "raw")
    with pytest.raises(ValueError, match="multioutput"):
        g.MeanAbsoluteError([[1.0]], [[1.0]], None, "weighted")
    with pytest.raises(ValueError, match="sampleWeight"):
        g.MeanSquaredError([[1.0]], [[1.0]], np.ones((1, 1)), "")
    with pytest.raises(ValueError, match="sampleWeight"):
        g.MeanAbsoluteError([[1.0]], [[1.0]], [1.0], "raw_values")


def test_kernels_have_no_stack_frame_or_spills():
    import subprocess
    so = g.build.SO
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-res-usage", so], capture_output=True, text=True).stdout
    lines = out.splitlines()
    names = ("k_met_", "k_class_values", "k_mlp64_acc_count", "k_mlp64_r2_part")
    seen = 0
    for i, line in enumerate(lines):
        if "Function" in line and any(k in line for k in names):
            seen += 1
            assert "STACK:0" in lines[i + 1] and "LOCAL:0" in lines[i + 1], line
    assert seen >= 12
