"""The two restatements of tests/ap_restatement.py against each other and against the reference's example outputs
(tests/golden/ranking_kat.json): the vectorised one, which the GPU tests use at large n, must equal the literal
transliteration bit for bit on every curve array for NaN-free scores; its AP must be math.fsum of the literal
terms, and within 1e-12 of the literal sequential sum."""
import json
import math
import os

import numpy as np
import pytest

from tests import ap_restatement as R

KAT = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "ranking_kat.json")))


def _w(a):
    """float32 values widened to float64, as the device widens scores"""
    return np.asarray(a, np.float32).astype(np.float64)


def _nan(a):
    return np.array([np.nan if v is None else v for v in a], np.float64)


def _bits(a):
    return np.asarray(a, np.float64).view(np.uint64)


def _same(a, b):
    """bit-equal float64 arrays"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(_bits(a), _bits(b))


def _literal(pred, y):
    """the literal restatement's inputs: float32 values widened to Python floats"""
    return [float(v) for v in _w(y)], [float(v) for v in _w(pred)]


def _pos_zero(a):
    """-0.0 read as +0.0: the device's threshold of the ±0 group is +0.0 whichever zero the reference's sort puts first"""
    a = np.asarray(a, np.float64).copy()
    a[a == 0] = 0.0
    return a


def _inputs(kind, n, rng):
    f = np.float32
    if kind == "random":
        return rng.random(n).astype(f), rng.choice(np.array([0, 1], f), n)
    if kind == "ties":
        return np.round(rng.random(n), 1).astype(f), rng.choice(np.array([0, 1, 2], f), n)
    if kind == "signed_zero_inf":
        return rng.choice(np.array([-0.0, 0.0, np.inf, -np.inf, 1.0, -1.0, 0.5, 1e-45], f), n), rng.choice(np.array([0, 1], f), n)
    if kind == "one_class_neg":
        return np.round(rng.random(n), 2).astype(f), np.zeros(n, f)
    if kind == "one_class_pos":
        return np.round(rng.random(n), 2).astype(f), np.ones(n, f)
    if kind == "all_equal":
        return np.full(n, 0.25, f), rng.choice(np.array([0, 1], f), n)
    raise ValueError(kind)


KINDS = ["random", "ties", "signed_zero_inf", "one_class_neg", "one_class_pos", "all_equal"]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", [1, 2, 3, 17, 200, 2000])
def test_vectorised_restatement_equals_the_literal_one(kind, n):
    rng = np.random.default_rng(n * 31 + KINDS.index(kind))
    pred, y = _inputs(kind, n, rng)
    yl, pl = _literal(pred, y)
    for pos_label in (1.0, 2.0, 0.5, 0.0):
        fpr, tpr, thr = R.roc_curve(pred, y, pos_label)
        lf, lt, lth = R.literal_roc_curve(yl, pl, pos_label)
        assert _same(fpr, lf) and _same(tpr, lt), (kind, n, pos_label)
        assert _same(thr, _pos_zero(lth)), (kind, n, pos_label)
        p, r, th = R.pr_curve(pred, y, pos_label)
        lp, lr, lth = R.literal_pr_curve(yl, pl, pos_label)
        assert _same(p, lp) and _same(r, lr) and _same(th, _pos_zero(lth)), (kind, n, pos_label)
        assert len(th) == len(p) - 1
    if R.is_binary(y):
        assert R.literal_type_of_target(yl) == "binary"
        ap = R.average_precision(pred, y)
        lit = R.literal_average_precision(yl, pl)
        terms = R.literal_ap_terms(yl, pl)
        assert _same(R.ap_terms(*R.clf_curve(pred, y, 1.0)[:2]), terms[::-1])
        if np.isnan(ap):
            assert np.isnan(lit) and not (y == 1).any()
        else:
            assert ap == math.fsum(terms)                          # the literal terms, exactly rounded
            assert abs(ap - lit) <= 1e-12, (kind, n, ap, lit)        # their sequential sum drifts by a few ulps
    else:
        assert R.literal_type_of_target(yl) == "unknown" and R.literal_average_precision(yl, pl) == 0.0
        with pytest.raises(ValueError):
            R.average_precision(pred, y)


def test_known_answers_of_the_reference_examples():
    s = KAT["scores"]
    k = KAT["roc"]
    for fpr, tpr, thr in (R.roc_curve(s, k["y"], k["pos_label"]), R.literal_roc_curve(*_literal(s, k["y"]), k["pos_label"])):
        assert list(fpr) == k["fpr"] and list(tpr) == k["tpr"] and _same(thr, _w(k["thresholds"]))
        assert R.literal_auc(fpr, tpr) == KAT["auc"]["auc"]
    k = KAT["pr"]
    for p, r, th in (R.pr_curve(s, k["y"], k["pos_label"]), R.literal_pr_curve(*_literal(s, k["y"]), k["pos_label"])):
        assert list(p) == k["precision"] and list(r) == k["recall"] and _same(th, _w(k["thresholds"]))
        assert "[%s]" % " ".join("%.3g" % v for v in p) == k["precision_printed"]
    k = KAT["ap"]
    assert R.average_precision(s, k["y"]) == k["ap"] == R.literal_average_precision(*_literal(s, k["y"]))
    assert "%.2f" % k["ap"] == k["ap_printed"]
    fpr, tpr, _ = R.roc_curve(s, KAT["roc_auc_score"]["y"], 1.0)
    assert R.literal_auc(fpr, tpr) == KAT["roc_auc_score"]["auc"]

    k = KAT["no_positives"]
    assert np.isnan(R.average_precision(s, k["y"])) and np.isnan(R.literal_average_precision(*_literal(s, k["y"])))
    for p, r, th in (R.pr_curve(s, k["y"], 1.0), R.literal_pr_curve(*_literal(s, k["y"]), 1.0)):
        assert _same(p, k["precision"]) and _same(r, _nan(k["recall"])) and _same(th, _w(k["pr_thresholds"]))
    for fpr, tpr, th in (R.roc_curve(s, k["y"], 1.0), R.literal_roc_curve(*_literal(s, k["y"]), 1.0)):
        assert _same(fpr, k["fpr"]) and _same(tpr, _nan(k["tpr"]))
        assert _same(th, np.r_[_w(0.8) + 1.0, _w(k["roc_thresholds"][1:])]) and abs(th[0] - k["roc_thresholds"][0]) < 1e-6
    k = KAT["no_negatives"]
    for fpr, tpr, th in (R.roc_curve(s, k["y"], 1.0), R.literal_roc_curve(*_literal(s, k["y"]), 1.0)):
        assert _same(fpr, _nan(k["fpr"])) and _same(tpr, k["tpr"]) and _same(th, _w(k["roc_thresholds"]))
    assert R.average_precision(s, k["y"]) == k["ap"] == R.literal_average_precision(*_literal(s, k["y"]))


def test_nan_scores_order_as_the_device_orders_them():
    """positive NaNs above +inf, negative NaNs below -inf, each bit pattern its own threshold group, thresholds keep
    their bits; the ±0 group's threshold is +0.0"""
    nan = np.array([0x7fc00000, 0xffc00000, 0x7f800001, 0xffc00001], np.uint32).view(np.float32)
    pred = np.r_[np.array([np.inf, -np.inf, -0.0, 0.0, 1.0], np.float32), nan, nan[:1]]
    y = np.array([1, 0, 1, 0, 1, 0, 1, 0, 1, 1], np.float32)
    tps, fps, thr = R.clf_curve(pred, y, 1.0)
    want_bits = [0x7ff8000000000000, 0x7ff0000020000000, 0x7ff0000000000000, 0x3ff0000000000000, 0,
                 0xfff0000000000000, 0xfff8000000000000, 0xfff8000020000000]
    assert thr.view(np.uint64).tolist() == want_bits
    assert tps.tolist() == [1, 1, 2, 3, 4, 4, 5, 6] and fps.tolist() == [1, 2, 2, 2, 3, 4, 4, 4]


def test_group_restatement_against_per_group_calls():
    rng = np.random.default_rng(3)
    n = 3000
    pred = np.round(rng.random(n), 2).astype(np.float32)
    y = rng.choice(np.array([0, 1], np.float32), n, p=[0.8, 0.2])
    grp = rng.integers(-20, 20, n)
    y[grp == 5] = 0
    m, groups, cnt, P, ap = R.group_average_precision(pred, y, grp)
    ug, c = np.unique(grp, return_counts=True)
    assert np.array_equal(groups, ug) and np.array_equal(cnt, c)
    for k, gid in enumerate(ug):
        sel = grp == gid
        assert P[k] == int((y[sel] == 1).sum())
        one = R.average_precision(pred[sel], y[sel])
        assert (np.isnan(one) and np.isnan(ap[k])) or one == ap[k], gid
    used = P > 0
    assert not used[np.searchsorted(ug, 5)]
    assert m == math.fsum(ap[used]) / used.sum()
    with pytest.raises(ValueError):
        R.group_average_precision(pred, np.r_[y[:-1], np.float32(0.5)], grp)
