"""The grouped-AUC restatement (tests/gauc_restatement.py gauc_exact) that the device's ctr_group_auc is held to, checked without a
GPU: against a per-group loop over the oracle's reference-semantics AUC, a hand-computed answer and the all-unused case."""
import math

import numpy as np
import pytest

from oracle import oracle as orc
from tests.gauc_restatement import auc_score_keys, gauc_exact


def _per_group_loop(pred, y, group):
    pred = np.asarray(pred, np.float32); y = np.asarray(y, np.float32); group = np.asarray(group, np.int64)
    gs = np.unique(group)
    aucs, ns = [], []
    for g in gs:
        m = group == g
        aucs.append(orc.roc_auc(pred[m], y[m])); ns.append(int(m.sum()))
    aucs = np.array(aucs); ns = np.array(ns)
    used = ~np.isnan(aucs)
    gauc = math.fsum(ns[used] * aucs[used]) / ns[used].sum() if used.any() else float("nan")
    return gauc, gs, ns, aucs


@pytest.mark.parametrize("seed", range(6))
def test_restatement_equals_a_per_group_loop_over_the_oracle(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(50, 4000))
    pred = np.round(rng.random(n), 2).astype(np.float32)              # many ties inside a group
    pred[rng.random(n) < 0.05] = -0.0
    pred[rng.random(n) < 0.05] = 0.0
    y = rng.choice(np.array([0, 1, 0.5, 0.5000001, 2, -1], np.float32), n)
    ids = np.array([-5, 0, 3, 2**40, -2**62, 17], np.int64)
    group = ids[np.minimum(rng.zipf(1.6, n) - 1, ids.size - 1)] if seed % 2 else rng.integers(-20, 20, n)
    gauc, groups, cnt, pos, auc = gauc_exact(pred, y, group)
    want, wg, wn, wa = _per_group_loop(pred, y, group)
    assert np.array_equal(groups, wg) and np.array_equal(cnt, wn)
    assert np.array_equal(np.isnan(auc), np.isnan(wa))
    np.testing.assert_allclose(auc[~np.isnan(auc)], wa[~np.isnan(wa)], rtol=1e-12, atol=0)
    assert abs(gauc - want) <= 1e-12 * abs(want)
    assert np.array_equal(pos, [int((np.asarray(y)[group == g] > 0.5).sum()) for g in groups])


def test_known_answer():
    """Group A is ranking_test.go's {.1, .4, .35, .8} / {0, 0, 1, 1} (AUC 0.75), group B has one class and is left
    out, group C is {.2, .9} / {0, 1} (AUC 1).  GAUC = (4 * 0.75 + 2 * 1) / 6 = 5/6."""
    pred = [0.1, 0.7, 0.4, 0.2, 0.35, 0.3, 0.9, 0.8]
    y = [0, 1, 0, 0, 1, 1, 1, 1]
    group = [7, -3, 7, 11, 7, -3, 11, 7]                    # A = 7, B = -3, C = 11, interleaved
    gauc, groups, cnt, pos, auc = gauc_exact(pred, y, group)
    assert groups.tolist() == [-3, 7, 11] and cnt.tolist() == [2, 4, 2] and pos.tolist() == [2, 2, 1]
    assert np.isnan(auc[0]) and auc[1] == 0.75 and auc[2] == 1.0
    assert gauc == 5 / 6


def test_nan_when_no_group_holds_both_classes():
    gauc, groups, cnt, pos, auc = gauc_exact([0.3, 0.1, 0.9, 0.5], [1, 1, 0, 0.5], [1, 1, 2, 2])
    assert math.isnan(gauc) and np.isnan(auc).all() and pos.tolist() == [2, 0]


def test_score_keys_order_like_the_float_order():
    """Ascending keys are descending scores; -0 and +0 share a key; NaNs of either sign sort outside the finite range."""
    s = np.array([-np.inf, -1.0, -1e-45, -0.0, 0.0, 1e-45, 0.5, np.inf], np.float32)
    k = auc_score_keys(s)
    assert (np.diff(k.astype(np.int64)) <= 0).all() and k[3] == k[4] and len(set(k.tolist())) == s.size - 1
    nan = np.array([0x7fc00000, 0xffc00000, 0x7f800001], np.uint32).view(np.float32)
    kn = auc_score_keys(nan)
    assert kn[0] < k.min() and kn[1] > k.max() and kn[2] < k.min()
