"""ctr_roc_auc_dist and ctr_group_auc_dist without a GPU.

The refusals that need no device: a null handle is CTR_EINVAL with its message in ctr_last_error(NULL) and nothing
written.  The Python methods, through a fake library that answers as one GPU would: the arguments they pass (lengths,
cap, NULL per-group arrays without per_group, the second call sized by the first's group count) and the shapes they
return, which are those of roc_auc and group_auc.  And the numpy model of the collective algorithm
(tests/auc_dist_model.py): runs, splitters, partition, routes in rank order, merge and integer area, for random cuts into
2, 4 and 8 ranks (empty ranks included), equal to the single-set AUC and GAUC exactly."""
import ctypes as C

import numpy as np
import pytest

import go_ctr_b200 as g
from tests import auc_dist_model as model
from tests.gauc_restatement import gauc_exact


def test_null_handle_is_refused_first():
    L = g.load_library()
    pred = np.array([0.2, 0.7], np.float32); y = np.array([0, 1], np.float32); grp = np.array([1, 1], np.int64)
    fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    auc = C.c_double(-7.0)
    assert L.ctr_roc_auc_dist(None, fp(pred), fp(y), C.c_int64(2), C.byref(auc)) == g.EINVAL
    assert b"null handle" in L.ctr_last_error(None) and auc.value == -7.0
    gauc = C.c_double(-7.0); ng = C.c_int64(-7)
    assert L.ctr_group_auc_dist(None, fp(pred), fp(y), grp.ctypes.data_as(C.POINTER(C.c_int64)), C.c_int64(2), C.byref(gauc), C.byref(ng),
                                None, C.c_int64(0), None, None, None, None) == g.EINVAL
    assert b"null handle" in L.ctr_last_error(None) and gauc.value == -7.0 and ng.value == -7
    assert {"ctr_roc_auc_dist", "ctr_group_auc_dist"} <= set(g.EXPORTS)


class FakeLib:
    """answers ctr_roc_auc_dist / ctr_group_auc_dist with fixed results; a cap below the group count is refused"""
    GROUPS = [-3, 5, 9]

    def __init__(self):
        self.calls = []

    def ctr_roc_auc_dist(self, h, pp, tp, n, auc):
        self.calls.append(("roc", n.value))
        C.cast(auc, C.POINTER(C.c_double))[0] = 0.75 if n.value else 0.5
        return 0

    def ctr_group_auc_dist(self, h, pp, tp, gp, n, gauc, ng, nu, cap, og, on, opos, oauc):
        self.calls.append(("gauc", n.value, cap.value, og is None))
        R = len(self.GROUPS)
        if og is not None and cap.value < R:
            return g.EINVAL
        C.cast(gauc, C.POINTER(C.c_double))[0] = 0.625
        C.cast(ng, C.POINTER(C.c_int64))[0] = R
        C.cast(nu, C.POINTER(C.c_int64))[0] = 2
        if og is not None:
            for i, v in enumerate(self.GROUPS):
                og[i] = v; on[i] = 10 + i; opos[i] = i; oauc[i] = 0.5 + i
        return 0

    def ctr_last_error(self, h):
        return b"fake refusal"


def _engine(L):
    e = g.Engine.__new__(g.Engine)
    e.L, e.h = L, C.c_void_p(8)
    return e


def test_python_methods_pass_the_arguments_and_return_the_single_gpu_shapes():
    L = FakeLib()
    e = _engine(L)
    assert e.roc_auc_dist(np.zeros(4), np.ones(4)) == 0.75
    assert e.roc_auc_dist([], []) == 0.5                                     # an empty rank takes part
    assert e.group_auc_dist(np.zeros(4), np.ones(4), np.arange(4)) == (0.625, 3, 2)
    got = e.group_auc_dist(np.zeros(4), np.ones(4), np.arange(4), per_group=True)
    assert got[:3] == (0.625, 3, 2)
    assert list(got[3]["group"]) == FakeLib.GROUPS and list(got[3]["n"]) == [10, 11, 12]
    assert list(got[3]["pos"]) == [0, 1, 2] and list(got[3]["auc"]) == [0.5, 1.5, 2.5]
    assert got[3]["group"].dtype == np.int64 and got[3]["n"].dtype == np.int32 and got[3]["auc"].dtype == np.float64
    assert L.calls == [("roc", 4), ("roc", 0), ("gauc", 4, 0, True), ("gauc", 4, 0, True), ("gauc", 4, 3, False)]
    with pytest.raises(ValueError):
        e.roc_auc_dist(np.zeros(3), np.ones(4))
    with pytest.raises(ValueError):
        e.group_auc_dist(np.zeros(4), np.ones(4), np.arange(3))


def _cuts(rng, n, W):
    c = [0] + sorted(int(x) for x in rng.integers(0, n + 1, W - 1)) + [n]
    if rng.random() < 0.5:
        k = int(rng.integers(1, W))
        c[k] = c[k - 1]                                                       # an empty rank
    return c


SCORE_KINDS = ["random", "ties", "equal", "special"]


def _scores(kind, rng, n):
    if kind == "equal":
        return np.full(n, 1.0, np.float32)
    if kind == "ties":
        return (rng.integers(0, 12, n) / 11).astype(np.float32)
    if kind == "special":
        pool = np.r_[np.array([0.0, -0.0, np.inf, -np.inf, 1e-45], np.float32), np.array([0x7fc00000, 0xffc00000, 0x7f800001], np.uint32).view(np.float32)]
        return pool[rng.integers(0, pool.size, n)]
    return rng.random(n).astype(np.float32)


@pytest.mark.parametrize("W", [2, 4, 8])
@pytest.mark.parametrize("kind", SCORE_KINDS)
def test_model_equals_the_single_set(W, kind):
    rng = np.random.default_rng(W * 10 + SCORE_KINDS.index(kind))
    for t in range(6):
        n = int(rng.integers(1, 4000))
        pred = _scores(kind, rng, n)
        y = (rng.random(n) < rng.random()).astype(np.float32)
        if t == 0:
            y[:] = 1.0                                                        # one class absent: NaN on both sides
        cuts = _cuts(rng, n, W)
        got = model.roc_dist(pred, y, cuts)
        want = model.roc_exact(pred, y)
        assert got[1:4] == want[1:4]
        assert np.array_equal(np.float64(got[0]).view(np.int64), np.float64(want[0]).view(np.int64))
        assert sum(got[5]) >= len(np.unique(pred.view(np.uint32)[pred.view(np.uint32) != 0x80000000]))
        if kind == "equal":
            assert sum(got[5]) == 1                                           # one tie group stays one run on one rank
        grp = rng.choice(np.array([np.iinfo(np.int64).min, np.iinfo(np.int64).max, -1, 0, 3, 77], np.int64), n) if t == 1 else \
            rng.integers(-30, 30, n).astype(np.int64)
        ga = model.gauc_dist(pred, y, grp, cuts)
        gb = gauc_exact(pred, y, grp)
        assert np.array_equal(np.float64(ga[0]).view(np.int64), np.float64(gb[0]).view(np.int64))
        for a, b in zip(ga[1:4], gb[1:4]):
            assert np.array_equal(a, b)
        assert np.array_equal(ga[4].view(np.int64), gb[4].view(np.int64))
        assert sum(ga[5]) == n


def test_splitters_keep_equal_keys_together_and_balance():
    rng = np.random.default_rng(5)
    keys = [np.sort(rng.integers(0, 1 << 20, int(rng.integers(0, 5000)))).astype(np.uint64) for _ in range(8)]
    spl = model.splitters([model.samples(k) for k in keys], 8)
    assert spl == sorted(spl)
    offs = [model.part(k, spl, 8) for k in keys]
    recv = [sum(o[d + 1] - o[d] for o in offs) for d in range(8)]
    assert sum(recv) == sum(k.size for k in keys)
    assert max(recv) < 2 * sum(recv) / 8                                      # regular sampling: no rank twice its share
    for d in range(8):                                                        # a key lands on one rank only
        for k, o in zip(keys, offs):
            part = k[o[d]:o[d + 1]]
            if part.size:
                assert d == 0 or part[0] > spl[d - 1]
                assert d == 7 or part[-1] <= spl[d]
