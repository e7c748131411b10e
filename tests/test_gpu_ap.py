"""ctr_roc_curve, ctr_pr_curve, ctr_average_precision and ctr_group_average_precision on the device against the
vectorised restatement of tests/ap_restatement.py: every curve array bit for bit (NaN bits included), AP within 1 ulp
of math.fsum of the reference's terms, identical bits on a repeated call, and the refusals.  The score kinds, group
layouts and sizes are those of test_gpu_gauc.py; sizes up to 5 000 003 make the capped grids stride."""
import ctypes as C
import math

import numpy as np
import pytest

import go_ctr_b200 as g
from tests import ap_restatement as R
from tests.test_gpu_gauc import KINDS, LAYOUTS, SIZES, groups_for, scores

pytestmark = pytest.mark.gpu

LABELS = np.array([0, 1, 0.5, 0.5000001, 2, -1], np.float32)
CLF_KEYS = ["clf_keys", "clf_sort", "clf_scan", "clf_ends", "clf_points"]
GAP_KEYS = ["gap_label_range", "gap_label_check", "gap_keys", "gap_sort_score", "gap_gather", "gap_sort_group",
            "gap_heads", "gap_scan", "gap_pos", "gap_terms", "gap_reduce", "gap_groups", "gap_final"]
_dp = C.POINTER(C.c_double)


@pytest.fixture(scope="module")
def eng():
    return g.Engine(g.engine.default_config(g.MODEL_YOUTUBE, batch=1, pred_batch=1))


def _bits(a):
    return np.asarray(a, np.float64).view(np.uint64)


def _same(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(_bits(a), _bits(b))


def _ulps(a, b):
    """|a - b| in units of the last place of b (0 for two NaNs)"""
    if np.isnan(a) or np.isnan(b):
        return 0 if np.isnan(a) and np.isnan(b) else math.inf
    return abs(a - b) / math.ulp(b) if b != 0 else abs(a) / math.ulp(0.0)


def _binary_labels(n, rng, case):
    """0/1 labels with about 5 % positives, as click data has, or -1/1 in every third case (binary too; the positive
    label stays 1).  Returns the labels and the negative label."""
    neg = np.float32(-1 if case % 3 == 2 else 0)
    return np.where(rng.random(n) < 0.05, np.float32(1), neg).astype(np.float32), neg


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", SIZES)
def test_curves_against_the_restatement(eng, n, kind):
    rng = np.random.default_rng(100 + SIZES.index(n) * len(KINDS) + KINDS.index(kind))
    s = scores(kind, n, rng)
    y = rng.choice(LABELS, n)
    case = (n, kind)
    for pos_label in (1.0, 2.0, 0.5):
        fpr, tpr, thr = eng.roc_curve(s, y, pos_label)
        wf, wt, wth = R.roc_curve(s, y, pos_label)
        assert _same(fpr, wf) and _same(tpr, wt) and _same(thr, wth), (case, pos_label)
        p, r, th = eng.precision_recall_curve(s, y, pos_label)
        wp, wr, wth = R.pr_curve(s, y, pos_label)
        assert _same(p, wp) and _same(r, wr) and _same(th, wth), (case, pos_label)
        # the integer counts come back from the scaled curve
        tps, fps, _ = R.clf_curve(s, y, pos_label)
        P, N = int(tps[-1]), int(fps[-1])
        pre = int(fps[0] != 0)
        if P > 0:
            assert np.array_equal(np.rint(tpr * P).astype(np.int64), np.r_[[0] * pre, tps]), (case, pos_label)
        if N > 0:
            assert np.array_equal(np.rint(fpr * N).astype(np.int64), np.r_[[0] * pre, fps]), (case, pos_label)

    # on 0/1 labels AUC() of the ROC curve is ctr_roc_auc
    y01 = (rng.random(n) < 0.3).astype(np.float32)
    fpr, tpr, _ = eng.roc_curve(s, y01, 1.0)
    auc = eng.roc_auc(s, y01)
    if np.isnan(auc):
        assert np.isnan(fpr).all() or np.isnan(tpr).all(), case
    else:
        trap = math.fsum((fpr - np.r_[0.0, fpr[:-1]]) * (tpr + np.r_[0.0, tpr[:-1]]) / 2.0)
        assert abs(trap - auc) <= 1e-12, (case, trap, auc)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", SIZES)
def test_average_precision_against_fsum_of_the_terms(eng, n, kind):
    i = SIZES.index(n) * len(KINDS) + KINDS.index(kind)
    rng = np.random.default_rng(300 + i)
    s = scores(kind, n, rng)
    y, _ = _binary_labels(n, rng, i)
    case = (n, kind)
    ap = eng.average_precision(s, y)
    tps, fps, _ = R.clf_curve(s, y, 1.0)
    if tps[-1] == 0:
        assert np.isnan(ap), case
    else:
        terms = R.ap_terms(tps, fps)
        want = math.fsum(terms)
        assert _ulps(ap, want) <= 1, (case, ap, want)
        if n <= 300_001:                                         # the reference's own order: from the high-recall end
            seq = float(np.cumsum(terms[::-1])[-1])
            assert abs(ap - seq) <= 1e-12, (case, ap, seq)
    assert _bits(eng.average_precision(s, y)) == _bits(ap), case
    assert np.isnan(eng.average_precision(s, np.zeros(n, np.float32))), case


def test_average_precision_refuses_labels_that_are_not_binary(eng):
    rng = np.random.default_rng(8)
    n = 5000
    s = np.round(rng.random(n), 2).astype(np.float32)
    for labels in ([0, 1, 2], [0, 0.5, 1]):
        y = rng.choice(np.array(labels, np.float32), n)
        y[:3] = labels
        assert _raw_ap(eng, s, y, n) == (g.EINVAL, -7.0)
    y = (rng.random(n) < 0.5).astype(np.float32)
    y[4321] = np.nan
    assert _raw_ap(eng, s, y, n) == (g.EINVAL, -7.0)
    y[4321] = 1.0
    rc, ap = _raw_ap(eng, s, y, n)
    assert rc == 0 and ap == R.average_precision(s, y)
    y0 = np.full(n, np.nan, np.float32)
    assert _raw_ap(eng, s, y0, n)[0] == g.EINVAL
    with pytest.raises(g.CtrError) as e:
        eng.average_precision(s, y0)
    assert e.value.code == g.EINVAL and "binary" in str(e.value)
    grp = rng.integers(0, 10, n)
    y[7] = 2.0
    with pytest.raises(g.CtrError) as e:
        eng.group_average_precision(s, y, grp)
    assert e.value.code == g.EINVAL


def _raw_ap(eng, pred, y, n, ap=True, pred_ok=True, y_ok=True):
    p = np.ascontiguousarray(pred, np.float32); t = np.ascontiguousarray(y, np.float32)
    out = C.c_double(-7.0)
    rc = eng.L.ctr_average_precision(eng.h, p.ctypes.data_as(C.POINTER(C.c_float)) if pred_ok else None,
                                     t.ctypes.data_as(C.POINTER(C.c_float)) if y_ok else None, C.c_int64(n),
                                     C.byref(out) if ap else None)
    return rc, out.value


def _raw_curve(eng, fn, pred, y, n, cap, pos_label=1.0, arrays=(True, True, True), npoints=True, pred_ok=True, y_ok=True):
    p = np.ascontiguousarray(pred, np.float32); t = np.ascontiguousarray(y, np.float32)
    m = max(cap, 1)
    outs = [np.full(m, -7.0) for _ in range(3)]
    npts = C.c_int64(-7)
    rc = fn(eng.h, p.ctypes.data_as(C.POINTER(C.c_float)) if pred_ok else None,
            t.ctypes.data_as(C.POINTER(C.c_float)) if y_ok else None, C.c_int64(n), C.c_double(pos_label),
            *[o.ctypes.data_as(_dp) if on else None for o, on in zip(outs, arrays)], C.c_int64(cap),
            C.byref(npts) if npoints else None)
    return rc, npts.value, outs


def test_curve_refusals_write_nothing_but_the_size_needed(eng):
    rng = np.random.default_rng(6)
    n = 1000
    s = np.round(rng.random(n), 2).astype(np.float32)
    y = (rng.random(n) < 0.3).astype(np.float32)
    for fn, want in ((eng.L.ctr_roc_curve, R.roc_curve(s, y, 1.0)), (eng.L.ctr_pr_curve, R.pr_curve(s, y, 1.0))):
        need = want[0].size
        for bad in (dict(n=0), dict(n=2**31), dict(n=-1), dict(pred_ok=False), dict(y_ok=False), dict(npoints=False)):
            kw = dict(n=n); kw.update(bad)
            rc, npts, outs = _raw_curve(eng, fn, s, y, kw.pop("n"), n + 1, **kw)
            assert rc == g.EINVAL and npts == -7 and all((o == -7.0).all() for o in outs), bad
        rc, npts, outs = _raw_curve(eng, fn, s, y, n, need - 1)
        assert rc == g.EINVAL and npts == need and all((o == -7.0).all() for o in outs)
        rc, npts, outs = _raw_curve(eng, fn, s, y, n, need)
        assert rc == 0 and npts == need
        nthr = want[2].size
        assert _same(outs[0], want[0]) and _same(outs[1], want[1]) and _same(outs[2][:nthr], want[2])
        assert (outs[2][nthr:] == -7.0).all()
        # each array may be NULL
        rc, npts, outs = _raw_curve(eng, fn, s, y, n, need, arrays=(False, True, False))
        assert rc == 0 and npts == need and (outs[0] == -7.0).all() and (outs[2] == -7.0).all() and _same(outs[1], want[1])
    for bad in (dict(n=0), dict(n=2**31), dict(pred_ok=False), dict(y_ok=False), dict(ap=False)):
        kw = dict(n=n); kw.update(bad)
        assert _raw_ap(eng, s, y, kw.pop("n"), **kw) == (g.EINVAL, -7.0), bad


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("n", SIZES)
def test_group_average_precision_against_the_restatement(eng, n, layout):
    i = SIZES.index(n) * len(LAYOUTS) + LAYOUTS.index(layout)
    kind = KINDS[i % len(KINDS)]
    rng = np.random.default_rng(2000 + i)
    s = scores(kind, n, rng)
    y, neg = _binary_labels(n, rng, i)
    grp = groups_for(layout, n, rng)
    if layout == "single_class_group":
        y[grp == grp[0]] = neg
        y[grp == grp[-1]] = 1.0 if grp[-1] != grp[0] else neg
    case = (n, layout, kind)

    m, ng, nu, pg = eng.group_average_precision(s, y, grp, per_group=True)
    want, wg, wn, wp, wa = R.group_average_precision(s, y, grp)
    ug, inv, cnt = np.unique(grp, return_inverse=True, return_counts=True)
    inv = inv.ravel()
    pos = np.bincount(inv, weights=(y == 1).astype(np.float64), minlength=ug.size).astype(np.int64)
    assert ng == ug.size and np.array_equal(pg["group"], ug), case
    assert np.array_equal(pg["n"], cnt) and np.array_equal(pg["pos"], pos), case
    assert np.array_equal(wg, ug) and np.array_equal(wn, cnt) and np.array_equal(wp, pos), case
    assert np.array_equal(np.isnan(pg["ap"]), pos == 0), case
    worst = max((_ulps(a, b) for a, b in zip(pg["ap"], wa)), default=0)
    assert worst <= 1, (case, worst)
    assert nu == int((pos > 0).sum()), case
    if np.isnan(want):
        assert np.isnan(m) and nu == 0, case
    else:
        assert abs(m - want) <= 1e-12 * abs(want), (case, m, want)

    # ctr_average_precision on the group's own samples; normally the same bits
    pick = rng.choice(ug.size, min(50, ug.size), replace=False)
    pick = np.unique(np.r_[pick, np.argmax(cnt)])
    differ = []
    for k in pick:
        sel = inv == k
        one = eng.average_precision(s[sel], y[sel])
        a = pg["ap"][k]
        assert _ulps(a, one) <= 1, (case, int(ug[k]), one, a)
        if not (np.isnan(one) and np.isnan(a)) and _bits(one) != _bits(a):
            differ.append((int(ug[k]), one, a))
    if differ:
        print("AP_g and ctr_average_precision differ in the last bit:", case, differ)

    again = eng.group_average_precision(s, y, grp, per_group=True)
    assert _bits(again[0]) == _bits(m) and again[1:3] == (ng, nu), case
    for key in pg:
        assert pg[key].tobytes() == again[3][key].tobytes(), (case, key)


def _raw_gap(eng, pred, y, grp, n, out=True, outs=(True, True, True, True), counts=True):
    def ptr(a, dt, ct):
        if a is None:
            return None, None
        a = np.ascontiguousarray(a, dt)
        return a, a.ctypes.data_as(C.POINTER(ct))
    (p, pp), (t, tp), (gr, gp) = ptr(pred, np.float32, C.c_float), ptr(y, np.float32, C.c_float), ptr(grp, np.int64, C.c_int64)
    m = max(n, 1) if 0 < n < 2**31 else 1
    res = C.c_double(-7.0); ng = C.c_int64(-7); nu = C.c_int64(-7)
    o = [np.full(m, -7, np.int64), np.full(m, -7, np.int32), np.full(m, -7, np.int32), np.full(m, -7.0)]
    ty = [C.c_int64, C.c_int32, C.c_int32, C.c_double]
    ptrs = [a.ctypes.data_as(C.POINTER(t_)) if on else None for a, t_, on in zip(o, ty, outs)]
    rc = eng.L.ctr_group_average_precision(eng.h, pp, tp, gp, C.c_int64(n), C.byref(res) if out else None,
                                           C.byref(ng) if counts else None, C.byref(nu) if counts else None, *ptrs)
    return rc, res.value, ng.value, nu.value, o


def test_group_refusals_and_null_optional_outputs(eng):
    rng = np.random.default_rng(5)
    n = 1000
    s = np.round(rng.random(n), 2).astype(np.float32); y = (rng.random(n) < 0.2).astype(np.float32)
    grp = rng.integers(-5, 5, n)
    untouched = lambda r: r[1] == -7.0 and r[2] == -7 and r[3] == -7 and all((a == -7).all() for a in r[4])
    for bad in (dict(n=0), dict(n=2**31), dict(n=-1), dict(pred=None), dict(y=None), dict(grp=None), dict(out=False)):
        kw = dict(pred=s, y=y, grp=grp, n=n); kw.update(bad)
        r = _raw_gap(eng, kw.pop("pred"), kw.pop("y"), kw.pop("grp"), **kw)
        assert r[0] == g.EINVAL and untouched(r), bad
    for yb in (np.r_[y[:-1], np.float32(2)], np.r_[y[:-1], np.float32(0.5)], np.r_[y[:-1], np.float32(np.nan)]):
        r = _raw_gap(eng, s, yb, grp, n)
        assert r[0] == g.EINVAL and untouched(r)
    want, wg, wn, wp, wa = R.group_average_precision(s, y, grp)
    rc, m, _, _, o = _raw_gap(eng, s, y, grp, n, outs=(False, False, False, False), counts=False)
    assert rc == 0 and abs(m - want) <= 1e-12 * want
    rc, m2, ng, nu, o = _raw_gap(eng, s, y, grp, n, outs=(False, True, False, True))
    assert rc == 0 and m2 == m and ng == wg.size and nu == int((wp > 0).sum())
    assert np.array_equal(o[1][:ng], wn) and all(_ulps(a, b) <= 1 for a, b in zip(o[3][:ng], wa))
    assert (o[1][ng:] == -7).all() and (o[0] == -7).all() and (o[2] == -7).all()


def test_profile_names_the_new_kernels(eng):
    rng = np.random.default_rng(9)
    n = 20_000
    s = rng.random(n).astype(np.float32); y = (rng.random(n) < 0.1).astype(np.float32)
    eng.profile(True)
    try:
        keys = {}
        for name, call in (("roc", lambda: eng.roc_curve(s, y, 1.0)), ("pr", lambda: eng.precision_recall_curve(s, y, 1.0)),
                           ("ap", lambda: eng.average_precision(s, y)),
                           ("gap", lambda: eng.group_average_precision(s, y, rng.integers(0, 300, n)))):
            eng.profile_reset()
            call()
            keys[name] = set(eng.profile_dump())
    finally:
        eng.profile(False)
    assert set(CLF_KEYS) | {"clf_roc"} <= keys["roc"] and set(CLF_KEYS) | {"clf_pr"} <= keys["pr"], keys
    assert set(CLF_KEYS) | {"ap_label_range", "ap_label_check", "ap_terms", "ap_final"} <= keys["ap"], keys
    assert set(GAP_KEYS) <= keys["gap"], keys
    for name in ("roc", "pr", "ap"):
        assert not any(k.startswith("gauc_") or k.startswith("gap_") for k in keys[name]), (name, keys[name])
    assert not any(k.startswith("gauc_") for k in keys["gap"]), keys["gap"]


def test_python_and_model_mirrors_return_the_c_arrays(eng):
    s = np.array([0.1, 0.4, 0.35, 0.8], np.float32)
    fpr, tpr, thr = g.ROCCurve(np.array([[1], [1], [2], [2]], np.float32), s.reshape(4, 1), 2.0, engine=eng)
    assert fpr.tolist() == [0, 0.5, 0.5, 1] and tpr.tolist() == [0.5, 0.5, 1, 1]      # ranking_test.go:9-21
    assert _same(thr, s[[3, 1, 2, 0]].astype(np.float64))
    p, r, th = g.PrecisionRecallCurve([0, 0, 1, 1], s, 1.0, engine=eng)
    assert p.tolist() == [2 / 3, 0.5, 1, 1] and r.tolist() == [1, 0.5, 0.5, 0]          # ranking_test.go:45-58
    assert _same(th, s[[2, 1, 3]].astype(np.float64))
    assert g.AveragePrecisionScore([0, 0, 1, 1], s, engine=eng) == 0.8333333333333333  # ranking_test.go:60-62
    assert np.isnan(g.AveragePrecisionScore([0, 0, 0, 0], s, engine=eng))

    rng = np.random.default_rng(11)
    n = 10_000
    s = np.round(rng.random(n), 3).astype(np.float32); y = (rng.random(n) < 0.1).astype(np.float32)
    grp = rng.integers(0, 100, n)
    for mirror, fn in ((lambda: g.ROCCurve(y, s, 1.0, engine=eng), eng.L.ctr_roc_curve),
                       (lambda: g.PrecisionRecallCurve(y, s, 1.0, engine=eng), eng.L.ctr_pr_curve)):
        a, b, t = mirror()
        rc, npts, outs = _raw_curve(eng, fn, s, y, n, n + 1)
        assert rc == 0 and npts == a.size
        assert _same(a, outs[0][:npts]) and _same(b, outs[1][:npts]) and _same(t, outs[2][:t.size])
    assert _bits(g.AveragePrecisionScore(y, s, engine=eng)) == _bits(_raw_ap(eng, s, y, n)[1])
    assert _bits(g.GroupAveragePrecision32(s, y, grp, engine=eng)) == _bits(_raw_gap(eng, s, y, grp, n)[1])


def test_average_precision_of_a_trained_din_model():
    """AveragePrecisionScore on the held-out predictions of a small DIN trained through the mirrored API (the set-up of
    test_gpu_parity's end-to-end test at a smaller size) equals the restatement."""
    rng = np.random.default_rng(42)
    uP, S, D, cF, N, B = 5, 3, 7, 5, 6000, 200
    xu = rng.random((N, uP), np.float32); cx = rng.random((N, cF), np.float32)
    ub = np.zeros((N, S, D), np.float32); ub[:, 1] = rng.random((N, D), np.float32)
    it = rng.random((N, D), np.float32)
    lab = np.round((np.abs(xu - cx).mean(1) + np.abs(ub[:, 1] - it).mean(1)) * 0.6).astype(np.float32)
    X = np.concatenate([xu, ub.reshape(N, -1), it, cx], 1)
    si = g.SampleInfo((0, uP), (uP, uP + S * D), (uP + S * D, uP + S * D + D), (uP + S * D + D, uP + S * D + D + cF))
    ntrain = 5000
    impl = g.DinImpl(S, D, PredBatchSize=20, BatchSize=B, epochs=2, earlyStop=0, seed=7)
    impl.Fit(g.TrainSample(X[:ntrain], lab[:ntrain], ntrain, X.shape[1], si))
    pred = impl.Predict(X[ntrain:]).ravel().astype(np.float32)
    y = lab[ntrain:]
    assert R.is_binary(y) and (y == 1).any() and (y == 0).any()
    ap = g.AveragePrecisionScore(y, pred)
    want = R.average_precision(pred, y)
    assert _ulps(ap, want) <= 1, (ap, want)
    yl, pl = [float(v) for v in y], [float(v) for v in pred.astype(np.float64)]
    assert abs(ap - R.literal_average_precision(yl, pl)) <= 1e-12
