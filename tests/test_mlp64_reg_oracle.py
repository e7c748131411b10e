"""The CPU restatement of the float64 MLP regressor (tests/mlp64_reg_oracle.c) checked on its own: its gradients
against finite differences (multilayer_perceptron_test.go:118-130 restated), its losses and R² against numpy
transcriptions of basemlp64.go, the output kind a cold fit takes from the targets, bit-identity with the classifier
restatements where the reference runs the same code, and the shape of the reference's TestMLPRegressor."""
import numpy as np
import pytest

from oracle import oracle as orc
from tests import mlp64_class_oracle as co
from tests import mlp64_reg_oracle as ro
from tests import mlp64_solver_oracle as so


def _cfg(nf, hidden, no, activation="relu", **kw):
    c = orc.mlp64_cfg(nf, hidden=hidden, activation="relu" if activation == "tanh" else activation, n_outputs=no, **kw)
    if activation == "tanh":
        c.hidden_act = so.ACT_TANH
    return c


def _fd(cfg, kind, p, X, Y, h=1e-6):
    g = np.empty_like(p)
    for i in range(p.size):
        a = p.copy(); a[i] += h
        b = p.copy(); b[i] -= h
        g[i] = (ro.loss_grad(cfg, kind, a, X, Y)[0] - ro.loss_grad(cfg, kind, b, X, Y)[0]) / (2 * h)
    return g


@pytest.mark.parametrize("kind,hidden,activation,no,signs", [
    ("identity", (), "relu", 1, [+1]),
    ("identity", (6,), "tanh", 3, [-1, +1]),
    ("identity", (5, 4), "logistic", 2, [+1, +1, +1]),
    ("softmax", (), "relu", 3, [+1]),
    ("softmax", (6,), "tanh", 4, [-1, +1]),
])
def test_gradients_match_finite_differences(kind, hidden, activation, no, signs):
    """Layer by layer; tanh's reference backprop negates the data gradient below an odd number of tanh layers (the
    forward pass computes tanh(−z), the derivative is tanh's), so those cases run with alpha = 0.  The softmax delta
    h − y is log_loss's gradient only on rows that sum to 1, so its targets here are one-hot; the dense 0/1 rows the
    reference also trains on are checked through the loss transcription and the device comparison."""
    rng = np.random.default_rng(len(hidden) * 10 + no)
    nf, n = 4, 9
    cfg = _cfg(nf, hidden, no, activation, alpha=0.0 if activation == "tanh" else 0.3)
    p = rng.standard_normal(ro.nparams(cfg)) * 0.5
    X = rng.standard_normal((n, nf))
    if kind == "identity":
        Y = rng.standard_normal((n, no)) * 2
    else:
        Y = np.eye(no)[rng.integers(0, no, n)]
    _, g = ro.loss_grad(cfg, kind, p, X, Y)
    fd = _fd(cfg, kind, p, X, Y)
    off = 0
    for l, s in enumerate(signs):
        m = (1 + cfg.units[l]) * cfg.units[l + 1]
        np.testing.assert_allclose(g[off:off + m], s * fd[off:off + m], rtol=1e-5, atol=1e-7)
        off += m
    assert off == g.size


def test_losses_are_the_reference_transcriptions():
    rng = np.random.default_rng(1)
    nf, no, n = 3, 2, 7
    cfg = _cfg(nf, (4,), no, alpha=0.2)
    p = rng.standard_normal(ro.nparams(cfg))
    X = rng.standard_normal((n, nf))
    sq = 0.0
    off = 0
    for fi, fo in ((nf, 4), (4, no)):
        W = p[off + fo:off + fo + fi * fo]
        sq += float(W @ W); off += (1 + fi) * fo
    l2 = 0.5 * 0.2 * sq / n
    Y = rng.standard_normal((n, no))
    h = ro.predict(cfg, "identity", p, X)
    loss, _ = ro.loss_grad(cfg, "identity", p, X, Y)
    assert loss == pytest.approx(((h - Y) ** 2).sum() / 2 / n + l2, rel=1e-13)       # square_loss :152-161
    Yb = (rng.random((n, no)) < 0.5).astype(np.float64)
    h = ro.predict(cfg, "softmax", p, X)
    np.testing.assert_allclose(h.sum(axis=1), 1.0, rtol=1e-14)
    loss, _ = ro.loss_grad(cfg, "softmax", p, X, Yb)
    assert loss == pytest.approx(-(Yb * np.log(h)).sum() / n + l2, rel=1e-13)         # log_loss :162-178


def test_r2_by_hand_and_the_mean_over_columns():
    yt = np.array([1.0, 2.0, 3.0, 4.0])
    yp = np.array([1.1, 1.9, 3.2, 3.8])
    s, bad = ro.r2(yt.reshape(-1, 1), yp.reshape(-1, 1))
    assert bad == -1 and s == pytest.approx(1 - 0.1 / 5.0, abs=1e-15)          # mean 2.5, den 5, num .1
    yt2 = np.stack([yt, [0.0, 2.0, 0.0, 2.0]], axis=1)
    yp2 = np.stack([yp, [1.0, 1.0, 1.0, 1.0]], axis=1)                         # column 2: num = den = 4 → r2 0
    s, bad = ro.r2(yt2, yp2)
    assert bad == -1 and s == pytest.approx((0.98 + 0.0) / 2, abs=1e-15)
    s, bad = ro.r2(np.stack([yt, np.full(4, 3.0)], axis=1), yp2)
    assert bad == 1                                                            # a constant column: the reference panics


def test_out_kind_follows_all_targets():
    assert ro.out_kind(np.array([[0.0], [1.0], [-0.0]], np.float32)) == "logistic"
    assert ro.out_kind(np.array([[0.0, 1.0], [1.0, 1.0]], np.float32)) == "softmax"
    assert ro.out_kind(np.array([[0.0, 1.0], [1.0, 0.5]], np.float32)) == "identity"
    assert ro.out_kind(np.array([[2.0]], np.float32)) == "identity"


def test_zero_one_targets_are_the_classifier_restatements_bit_for_bit():
    """One 0/1 column is the binary classifier (mlp64_solver_oracle.c); one-hot rows are the multi-class one
    (mlp64_class_oracle.c): the reference runs the same code for both."""
    rng = np.random.default_rng(3)
    X = rng.random((450, 6))
    o = so.opts("sgd", nesterov=True, learning_rate="invscaling")
    y = (rng.random(450) < 0.5).astype(np.float64).reshape(-1, 1)
    cfg = _cfg(6, (5,), 1, max_iter=4, seed=2, tol=0.0)
    pr, ps = ro.init(cfg), so.init(cfg)
    a = ro.fit(cfg, "logistic", o, pr, X, y)
    b = so.fit(cfg, o, ps, X, y)
    assert pr.tobytes() == ps.tobytes() and a[0] == b[0] and a[1].tobytes() == b[1].tobytes()
    Y = np.eye(3)[rng.integers(0, 3, 450)]
    cfg = _cfg(6, (5,), 3, max_iter=4, seed=2, tol=0.0)
    pr, pc = ro.init(cfg), co.init(cfg)
    a = ro.fit(cfg, "softmax", o, pr, X, Y)
    b = co.fit(cfg, o, pc, X, Y)
    assert pr.tobytes() == pc.tobytes() and a[1].tobytes() == b[1].tobytes()


def test_reference_regressor_test_shape_scores_at_least_095():
    """TestMLPRegressor (multilayer_perceptron_test.go:426-437): no hidden layer, relu, adam, alpha 0, lr .1, 100
    samples of 2 features with a linear target.  MakeRegression is not in the reference tree: the data is synthesised."""
    rng = np.random.default_rng(4)
    X = rng.standard_normal((100, 2))
    y = (X @ np.array([3.0, -2.0]) + 0.5).astype(np.float32)
    cfg = _cfg(2, (), 1, alpha=0.0, lr_init=0.1, seed=1)
    kind, p, it, curve = ro.cold_fit(cfg, so.opts("adam"), X.astype(np.float32).astype(np.float64), y)
    assert kind == "identity" and curve[-1] < curve[0]
    s, bad = ro.r2(y.astype(np.float64).reshape(-1, 1), ro.predict(cfg, kind, p, X.astype(np.float32).astype(np.float64)))
    assert bad == -1 and s >= 0.95
