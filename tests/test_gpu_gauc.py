"""ctr_group_auc (GAUC) on the device against the numpy restatement gauc_exact (tests/gauc_restatement.py) and against ctr_roc_auc
on each group's samples: per-group counts exactly, every group's AUC bit for bit, the weighted mean within 1e-12 of
math.fsum, and identical bits on a repeated call.  Sizes up to 5 000 003 make the capped grids stride; the group
layouts run from one group to all singletons, sparse int64 ids at the extremes, unsorted input and one group holding
half the samples."""
import ctypes as C

import numpy as np
import pytest

import go_ctr_b200 as g
from tests.gauc_restatement import gauc_exact
from tests.util import INT64_MAX, INT64_MIN

pytestmark = pytest.mark.gpu

LABELS = np.array([0, 1, 0.5, 0.5000001, 2, -1], np.float32)
KINDS = ["all_equal", "distinct", "two_decimal_ties", "signed_zero_inf", "denormals", "nans"]
LAYOUTS = ["one_group", "singletons", "dense", "sparse_extremes", "interleaved", "zipf_half", "single_class_group"]
SIZES = [1, 2, 33, 257, 300_001, 5_000_003]
GAUC_KEYS = ["gauc_keys", "gauc_sort_score", "gauc_gather", "gauc_sort_group", "gauc_heads", "gauc_scan", "gauc_terms",
             "gauc_reduce", "gauc_groups", "gauc_final"]


def scores(kind, n, rng):
    f = np.float32
    if kind == "all_equal":
        return np.full(n, 0.37, f)
    if kind == "distinct":
        return (rng.permutation(n) - n // 2).astype(f)
    if kind == "two_decimal_ties":
        return np.round(rng.random(n), 2).astype(f)
    if kind == "signed_zero_inf":
        return rng.choice(np.array([-0.0, 0.0, np.inf, -np.inf, 1.0, -1.0, 0.5], f), n)
    if kind == "denormals":
        return rng.choice(np.array([0.0, -0.0, 1e-45, -1e-45, 3e-45, 1e-40, -1e-40, 6e-39, np.finfo(f).tiny, 1e-3], f), n)
    # NaNs of both signs and several payloads among tied finite scores
    nan = np.array([0x7fc00000, 0xffc00000, 0x7f800001, 0xff800001, 0x7fffffff], np.uint32).view(f)
    s = np.round(rng.random(n), 1).astype(f)
    m = rng.random(n) < 0.2
    s[m] = rng.choice(nan, int(m.sum()))
    return s


def groups_for(layout, n, rng):
    if layout == "one_group":
        return np.full(n, 42, np.int64)
    if layout == "singletons":
        return rng.permutation(n).astype(np.int64) * 3 - n
    if layout == "dense":
        return rng.integers(0, max(1, n // 20), n).astype(np.int64)
    if layout == "sparse_extremes":
        pool = np.r_[np.array([INT64_MIN, INT64_MAX, -1, 0], np.int64),
                     rng.integers(INT64_MIN, INT64_MAX, max(4, n // 50), dtype=np.int64, endpoint=True)]
        return rng.choice(pool, n)
    if layout == "interleaved":                                  # consecutive samples in different groups
        return (np.arange(n, dtype=np.int64) % max(1, n // 7)) * -1_000_003
    if layout == "zipf_half":                                    # one group holds half the samples, the rest Zipf
        return np.where(rng.random(n) < 0.5, 7, rng.zipf(1.3, n) % 1_000_000_007).astype(np.int64)
    return rng.integers(0, max(1, n // 30), n).astype(np.int64)  # dense; the test makes two of its groups one-class


@pytest.fixture(scope="module")
def eng():
    return g.Engine(g.engine.default_config(g.MODEL_YOUTUBE, batch=1, pred_batch=1))


def _bits(a):
    return np.asarray(a, np.float64).view(np.uint64)


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("n", SIZES)
def test_group_auc_against_the_restatement(eng, n, layout):
    i = SIZES.index(n) * len(LAYOUTS) + LAYOUTS.index(layout)
    kind = KINDS[i % len(KINDS)]
    rng = np.random.default_rng(1000 + i)
    s = scores(kind, n, rng)
    y = rng.choice(LABELS, n)
    grp = groups_for(layout, n, rng)
    if layout == "single_class_group":
        y[grp == grp[0]] = 0.0
        y[grp == grp[-1]] = 1.0 if grp[-1] != grp[0] else 0.0
    case = (n, layout, kind)

    gauc, ng, nu, pg = eng.group_auc(s, y, grp, per_group=True)
    want, wg, wn, wp, wa = gauc_exact(s, y, grp)

    ug, inv, cnt = np.unique(grp, return_inverse=True, return_counts=True)
    pos = np.bincount(inv.ravel(), weights=(y > 0.5).astype(np.float64), minlength=ug.size).astype(np.int64)
    assert ng == ug.size, case
    assert np.array_equal(pg["group"], ug), case
    assert np.array_equal(pg["n"], cnt) and np.array_equal(pg["pos"], pos), case
    assert np.array_equal(wg, ug) and np.array_equal(wn, cnt) and np.array_equal(wp, pos), case
    assert np.array_equal(_bits(pg["auc"]), _bits(wa)) or (
        np.array_equal(np.isnan(pg["auc"]), np.isnan(wa))
        and np.array_equal(_bits(pg["auc"][~np.isnan(wa)]), _bits(wa[~np.isnan(wa)]))), case
    used = (pos > 0) & (pos < cnt)
    assert nu == int(used.sum()), case
    if layout == "single_class_group" and n > 1:
        assert not used[np.searchsorted(ug, grp[0])], case
    if np.isnan(want):
        assert np.isnan(gauc) and nu == 0, case
    else:
        assert abs(gauc - want) <= 1e-12 * abs(want), (case, gauc, want)

    # ctr_roc_auc on the group's own samples, bit for bit (2 P N < 2^53 at these sizes)
    pick = rng.choice(ug.size, min(50, ug.size), replace=False)
    pick = np.unique(np.r_[pick, np.argmax(cnt)])
    for k in pick:
        m = inv.ravel() == k
        one = eng.roc_auc(s[m], y[m])
        a = pg["auc"][k]
        assert (np.isnan(one) and np.isnan(a)) or _bits(one) == _bits(a), (case, int(ug[k]), one, a)

    again = eng.group_auc(s, y, grp, per_group=True)
    assert _bits(again[0]) == _bits(gauc) and again[1:3] == (ng, nu), case
    for key in pg:
        assert pg[key].tobytes() == again[3][key].tobytes(), (case, key)


def test_known_answer_and_the_model_wrapper(eng):
    """ranking_test.go's {.1, .4, .35, .8} / {0, 0, 1, 1} (0.75), a one-class group left out, {.2, .9} / {0, 1} (1.0):
    GAUC = (4 * 0.75 + 2 * 1) / 6."""
    pred = [0.1, 0.7, 0.4, 0.2, 0.35, 0.3, 0.9, 0.8]
    y = [0, 1, 0, 0, 1, 1, 1, 1]
    grp = [7, -3, 7, 11, 7, -3, 11, 7]
    gauc, ng, nu, pg = eng.group_auc(pred, y, grp, per_group=True)
    assert (ng, nu) == (3, 2) and gauc == 5 / 6
    assert pg["group"].tolist() == [-3, 7, 11] and pg["n"].tolist() == [2, 4, 2] and pg["pos"].tolist() == [2, 2, 1]
    assert np.isnan(pg["auc"][0]) and pg["auc"][1:].tolist() == [0.75, 1.0]
    assert g.GroupAuc32(pred, y, grp, engine=eng) == 5 / 6
    assert eng.group_auc(pred, y, grp) == (5 / 6, 3, 2)


def _raw(eng, pred, y, grp, n, gauc=True, outs=(True, True, True, True), counts=True):
    def ptr(a, dt, ct):
        if a is None:
            return None, None
        a = np.ascontiguousarray(a, dt)
        return a, a.ctypes.data_as(C.POINTER(ct))
    (p, pp), (t, tp), (gr, gp) = ptr(pred, np.float32, C.c_float), ptr(y, np.float32, C.c_float), ptr(grp, np.int64, C.c_int64)
    m = max(n, 1) if 0 < n < 2**31 else 1
    res = C.c_double(-1.0); ng = C.c_int64(-1); nu = C.c_int64(-1)
    o = [np.full(m, -7, np.int64), np.full(m, -7, np.int32), np.full(m, -7, np.int32), np.full(m, -7.0)]
    ty = [C.c_int64, C.c_int32, C.c_int32, C.c_double]
    ptrs = [a.ctypes.data_as(C.POINTER(t_)) if on else None for a, t_, on in zip(o, ty, outs)]
    rc = eng.L.ctr_group_auc(eng.h, pp, tp, gp, C.c_int64(n),
                             C.byref(res) if gauc else None, C.byref(ng) if counts else None, C.byref(nu) if counts else None,
                             *ptrs)
    return rc, res.value, ng.value, nu.value, o


def test_bad_arguments_are_einval_and_optional_outputs_may_be_null(eng):
    rng = np.random.default_rng(5)
    n = 1000
    s = np.round(rng.random(n), 2).astype(np.float32); y = rng.choice(LABELS, n); grp = rng.integers(-5, 5, n)
    for bad in (dict(n=0), dict(n=2**31), dict(n=-1), dict(pred=None), dict(y=None), dict(grp=None), dict(gauc=False)):
        kw = dict(pred=s, y=y, grp=grp, n=n); kw.update(bad)
        rc = _raw(eng, kw.pop("pred"), kw.pop("y"), kw.pop("grp"), **kw)[0]
        assert rc == g.EINVAL, bad
    want, wg, wn, wp, wa = gauc_exact(s, y, grp)
    rc, gauc, _, _, o = _raw(eng, s, y, grp, n, outs=(False, False, False, False), counts=False)
    assert rc == 0 and abs(gauc - want) <= 1e-12 * want
    rc, gauc2, ng, nu, o = _raw(eng, s, y, grp, n, outs=(False, True, False, True))
    assert rc == 0 and gauc2 == gauc and ng == wg.size
    assert np.array_equal(o[1][:ng], wn) and np.array_equal(_bits(o[3][:ng]), _bits(wa))
    assert (o[1][ng:] == -7).all() and (o[0] == -7).all() and (o[2] == -7).all()


def test_profile_names_the_gauc_kernels(eng):
    rng = np.random.default_rng(9)
    n = 20_000
    eng.profile(True)
    try:
        eng.profile_reset()
        eng.group_auc(rng.random(n).astype(np.float32), rng.choice(LABELS, n), rng.integers(0, 300, n))
        prof = eng.profile_dump()
    finally:
        eng.profile(False)
    assert set(GAUC_KEYS) <= set(prof), sorted(prof)
