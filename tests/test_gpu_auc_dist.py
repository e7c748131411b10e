"""ctr_roc_auc_dist and ctr_group_auc_dist on a single-GPU handle are ctr_roc_auc and ctr_group_auc: the same bits, the
per-group arrays included, the same refusals and messages, and cap bounding the per-group arrays (a cap below the group
count is CTR_EINVAL with nothing written).  The new calls' profile keys are the single-GPU calls' keys."""
import ctypes as C

import numpy as np
import pytest

import go_ctr_b200 as g

pytestmark = pytest.mark.gpu


def _bits(x):
    return np.asarray(x, np.float64).view(np.int64)


@pytest.fixture(scope="module")
def eng():
    return g.Engine(g.engine.default_config(g.MODEL_DIN_COS, batch=1, pred_batch=1))


@pytest.mark.parametrize("n", [1, 2, 257, 300_001])
def test_world_one_is_the_single_gpu_call(eng, n):
    rng = np.random.default_rng(n)
    pred = (rng.integers(0, 30, n) / 29).astype(np.float32)
    pred[rng.integers(0, n, max(1, n // 50))] = np.nan
    y = (rng.random(n) < 0.3).astype(np.float32)
    grp = rng.integers(-5, max(6, n // 40), n).astype(np.int64)
    assert _bits(eng.roc_auc_dist(pred, y)) == _bits(eng.roc_auc(pred, y))
    a = eng.group_auc_dist(pred, y, grp, per_group=True)
    b = eng.group_auc(pred, y, grp, per_group=True)
    assert _bits(a[0]) == _bits(b[0]) and a[1:3] == b[1:3]
    for k in ("group", "n", "pos"):
        assert np.array_equal(a[3][k], b[3][k]), k
    assert np.array_equal(_bits(a[3]["auc"]), _bits(b[3]["auc"]))
    assert eng.group_auc_dist(pred, y, grp)[:3] == b[:3] or np.isnan(b[0])


def test_cap_and_refusals(eng):
    L, h = eng.L, eng.h
    pred = np.array([0.1, 0.9, 0.4, 0.6], np.float32); y = np.array([0, 1, 1, 0], np.float32)
    grp = np.array([3, 1, 3, 1], np.int64)
    fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    gp = grp.ctypes.data_as(C.POINTER(C.c_int64))
    gauc = C.c_double(-7.0); ng = C.c_int64(-7); nu = C.c_int64(-7)
    og = np.full(2, -9, np.int64)
    # two groups, cap 1: refused, nothing written
    rc = L.ctr_group_auc_dist(h, fp(pred), fp(y), gp, C.c_int64(4), C.byref(gauc), C.byref(ng), C.byref(nu), C.c_int64(1),
                              og.ctypes.data_as(C.POINTER(C.c_int64)), None, None, None)
    assert rc == g.EINVAL and b"do not fit" in L.ctr_last_error(h)
    assert gauc.value == -7.0 and ng.value == -7 and nu.value == -7 and (og == -9).all()
    rc = L.ctr_group_auc_dist(h, fp(pred), fp(y), gp, C.c_int64(4), C.byref(gauc), C.byref(ng), C.byref(nu), C.c_int64(2),
                              og.ctypes.data_as(C.POINTER(C.c_int64)), None, None, None)
    assert rc == 0 and ng.value == 2 and list(og) == [1, 3]
    # no per-group array: cap is not read
    assert L.ctr_group_auc_dist(h, fp(pred), fp(y), gp, C.c_int64(4), C.byref(gauc), None, None, C.c_int64(0), None, None, None, None) == 0
    # the single-GPU refusals and messages
    for args in [(None, fp(y), 4), (fp(pred), None, 4), (fp(pred), fp(y), 0), (fp(pred), fp(y), 2 ** 31)]:
        auc = C.c_double(-7.0)
        assert L.ctr_roc_auc_dist(h, args[0], args[1], C.c_int64(args[2]), C.byref(auc)) == g.EINVAL
        m1 = L.ctr_last_error(h)
        assert L.ctr_roc_auc(h, args[0], args[1], C.c_int64(args[2]), C.byref(auc)) == g.EINVAL
        assert L.ctr_last_error(h) == m1 and auc.value == -7.0
        assert L.ctr_group_auc_dist(h, args[0], args[1], gp, C.c_int64(args[2]), C.byref(gauc), None, None, C.c_int64(0),
                                    None, None, None, None) == g.EINVAL
        m2 = L.ctr_last_error(h)
        assert L.ctr_group_auc(h, args[0], args[1], gp, C.c_int64(args[2]), C.byref(gauc), None, None, None, None, None, None) == g.EINVAL
        assert L.ctr_last_error(h) == m2


def test_profile_keys(eng):
    rng = np.random.default_rng(3)
    pred = rng.random(1000).astype(np.float32); y = (rng.random(1000) < 0.5).astype(np.float32)
    grp = rng.integers(0, 30, 1000)
    eng.profile(True); eng.profile_reset()
    eng.group_auc_dist(pred, y, grp)
    keys = set(eng.profile_dump())
    eng.profile(False)
    assert keys == {"gauc_keys", "gauc_sort_score", "gauc_gather", "gauc_sort_group", "gauc_heads", "gauc_scan", "gauc_terms",
                    "gauc_reduce", "gauc_groups", "gauc_final"}, keys
