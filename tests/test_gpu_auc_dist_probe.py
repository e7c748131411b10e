"""The per-rank steps of ctr_roc_auc_dist and ctr_group_auc_dist on one GPU: W = 2, 4 and 8 ranks emulated as W shards
of one device through the kernel-level probe tests/cuda/auc_dist_probe.cu (auc.cuh itself, not a copy), the exchanges
done by device copies in rank order.  Every case must equal ctr_roc_auc and ctr_group_auc on the concatenation at 0 ulp
(the per-group arrays included), and the per-rank run and record counts must equal the numpy model
(tests/auc_dist_model.py).  Cases: all scores equal; ±0, ±inf, denormals and several NaN bit patterns; one class absent
(NaN); one rank all positives and another all negatives; a group on every rank; group ids INT64_MIN and INT64_MAX; one
giant group; n = 1 on a rank; empty ranks."""
import numpy as np
import pytest
import torch

import go_ctr_b200 as g
from tests import auc_dist_model as model
from tests import auc_dist_probe as ap

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

DEV = "cuda"
WS = [2, 4, 8]
NAN_BITS = [0x7fc00000, 0xffc00000, 0x7f800001, 0xff812345, 0x7fffffff]


def _scores(kind, rng, n):
    if kind == "equal":
        return np.full(n, 0.625, np.float32)
    if kind == "special":
        pool = np.r_[np.array([0.0, -0.0, np.inf, -np.inf, 1e-45, -1e-45, 0.5, 1.0], np.float32),
                     np.array(NAN_BITS, np.uint32).view(np.float32)]
        return pool[rng.integers(0, pool.size, n)]
    if kind == "ties":
        return (rng.integers(0, 20, n) / 19).astype(np.float32)
    return rng.random(n).astype(np.float32)


def _cuts(rng, n, W, empty=False, one=False):
    c = np.sort(rng.integers(0, n + 1, W - 1))
    c = [0] + [int(x) for x in c] + [n]
    if empty:
        c[1] = 0                                                         # rank 0 passes no samples
    if one and W > 2:
        c[2] = c[1] + 1                                                  # rank 1 passes one
        c[2:] = [max(x, c[2]) for x in c[2:]]
    return c


CASES = ["random", "ties", "equal", "special", "one_class", "split_classes", "empty_and_one"]


def _case(name, rng, W):
    n = 20_000
    pred = _scores({"ties": "ties", "equal": "equal", "special": "special"}.get(name, "random"), rng, n)
    y = (rng.random(n) < 0.4).astype(np.float32)
    y[rng.integers(0, n, 50)] = 0.5                                     # binarised at 0.5: negative
    cuts = _cuts(rng, n, W, empty=name == "empty_and_one", one=name == "empty_and_one")
    if name == "one_class":
        y[:] = 1.0
    if name == "split_classes":                                          # rank 0 all positives, the last rank all negatives
        y[cuts[0]:cuts[1]] = 1.0
        y[cuts[W - 1]:cuts[W]] = 0.0
    return pred, y, cuts


def _bits(x):
    return np.array([x], np.float64).view(np.int64)[0]


@pytest.fixture(scope="module")
def eng():
    return g.Engine(g.engine.default_config(g.MODEL_DIN_COS, batch=1, pred_batch=1))


@pytest.mark.parametrize("W", WS)
@pytest.mark.parametrize("name", CASES)
def test_roc_auc_ranks_equal_one_gpu(eng, W, name):
    rng = np.random.default_rng(W * 100 + CASES.index(name))
    pred, y, cuts = _case(name, rng, W)
    got, stats = ap.roc(torch.from_numpy(pred).to(DEV), torch.from_numpy(y).to(DEV), cuts)
    want = eng.roc_auc(pred, y)
    assert _bits(got) == _bits(want), (got, want)
    m = model.roc_dist(pred, y, cuts)
    assert [int(x) for x in stats[:W]] == m[4] and [int(x) for x in stats[W:2 * W]] == m[5]
    assert [int(x) for x in stats[2 * W:]] == [m[1], m[2], m[3]]
    if name == "equal":
        assert int(stats[W:2 * W].sum()) == 1                            # one tie group, one run, on one rank


def _groups(name, rng, n, W, cuts):
    if name == "every_rank":
        g_ = rng.integers(0, 50, n)
        for r in range(W):                                               # group 7 holds samples on every non-empty rank
            if cuts[r + 1] > cuts[r]:
                g_[cuts[r]] = 7
        return g_
    if name == "extremes":
        return rng.choice(np.array([np.iinfo(np.int64).min, np.iinfo(np.int64).max, -1, 0, 1], np.int64), n)
    if name == "giant":
        g_ = np.full(n, 42, np.int64)
        g_[rng.integers(0, n, n // 20)] = rng.integers(-1000, 1000, n // 20)
        return g_
    return rng.integers(-(1 << 40), 1 << 40, n) // (1 << 30)            # about 2000 groups


GCASES = ["spread", "every_rank", "extremes", "giant", "special", "empty_and_one"]


@pytest.mark.parametrize("W", WS)
@pytest.mark.parametrize("name", GCASES)
def test_group_auc_ranks_equal_one_gpu(eng, W, name):
    rng = np.random.default_rng(W * 1000 + GCASES.index(name))
    n = 20_000
    pred = _scores("special" if name == "special" else "ties", rng, n)
    y = (rng.random(n) < 0.4).astype(np.float32)
    cuts = _cuts(rng, n, W, empty=name == "empty_and_one", one=name == "empty_and_one")
    grp = _groups(name, rng, n, W, cuts).astype(np.int64)
    want = eng.group_auc(pred, y, grp, per_group=True)
    R = want[1]
    outs = dict(group=torch.empty(R, dtype=torch.int64, device=DEV), n=torch.empty(R, dtype=torch.int32, device=DEV),
                pos=torch.empty(R, dtype=torch.int32, device=DEV), auc=torch.empty(R, dtype=torch.float64, device=DEV))
    got = ap.gauc(torch.from_numpy(pred).to(DEV), torch.from_numpy(y).to(DEV), torch.from_numpy(grp).to(DEV), cuts, outs)
    assert _bits(got[0]) == _bits(want[0]) and got[1:3] == want[1:3], (got, want[:3])
    for k in ("group", "n", "pos"):
        assert np.array_equal(outs[k].cpu().numpy(), want[3][k]), k
    assert np.array_equal(outs["auc"].cpu().numpy().view(np.int64), want[3]["auc"].view(np.int64))
    m = model.gauc_dist(pred, y, grp, cuts)
    assert [int(x) for x in got[3]] == m[5]
    if name == "giant":
        assert max(m[5]) >= n * 0.9                                      # the giant group lands whole on one rank
