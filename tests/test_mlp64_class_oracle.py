"""The multi-class restatement of the float64 MLP classifier (tests/mlp64_class_oracle.c) against numpy transcripts of
basemlp64.go, against tests/mlp64_solver_oracle.c on binary labels, and against finite differences; and the refusals
of ctr_mlp_set_classes that need no device.  CPU only."""
import ctypes as C

import numpy as np
import pytest

import go_ctr_b200 as g
from oracle import oracle as orc
from tests import mlp64_class_oracle as co
from tests import mlp64_solver_oracle as so


# ---- numpy transcripts of basemlp64.go ------------------------------------------------------------------------------
def np_is_binarized(y):                              # isBinarized64 :1378-1388
    return all(v == 0 or v == 1 for v in np.asarray(y, np.float64))


def np_binarizer_fit(y):                             # LabelBinarizer64.Fit :1294-1313 (a map keyed by float64, then sort)
    seen = []
    for v in np.asarray(y, np.float32).astype(np.float64):
        if not any(s == v for s in seen):
            seen.append(v)
    return np.array(sorted(seen), np.float64)


def np_transform(y, classes):                        # :1324-1351
    out = np.zeros((len(y), len(classes)))
    for i, v in enumerate(np.asarray(y, np.float32).astype(np.float64)):
        for c, cv in enumerate(classes):
            if cv == v:
                out[i, c] = 1
    return out


def np_max_idx(a):                                   # MaxIdx64, mathCompat.go:93-101
    mi = 0
    for i in range(len(a)):
        if a[i] > a[mi]:
            mi = i
    return mi


def np_inverse(h, classes):                          # InverseTransform :1360-1376
    return np.array([classes[np_max_idx(row)] for row in h], np.float64).astype(np.float32)


def np_softmax(z):                                   # Activations64["softmax"] :104-117
    z = z.copy()
    for r in range(z.shape[0]):
        s = 0.0
        for c in range(z.shape[1]):
            z[r, c] = np.exp(z[r, c])
            s += z[r, c]
        for c in range(z.shape[1]):
            z[r, c] /= s
    return z


def np_log_loss(y, h):                               # LossFunctions64["log_loss"] :162-178
    hmin, hmax = np.nextafter(0, 1), np.nextafter(1, 0)
    s = 0.0
    for r in range(y.shape[0]):
        for c in range(y.shape[1]):
            hv = min(max(h[r, c], hmin), hmax) if not np.isnan(h[r, c]) else h[r, c]
            if y[r, c] != 0:
                s += -y[r, c] * np.log(hv)
    return s / y.shape[0]


def _data(n, nf, seed, labels):
    rng = np.random.default_rng(seed)
    X = rng.random((n, nf))
    score = (X - 0.5) @ rng.standard_normal(nf) + 0.3 * rng.standard_normal(n)
    q = np.quantile(score, np.linspace(0, 1, len(labels) + 1)[1:-1])
    return X, np.asarray(labels, np.float32)[np.searchsorted(q, score)]


LABEL_SETS = [
    [0.0, 1.0, 0.0, 1.0],
    [0.0, 0.0],
    [-0.0, 1.0, 0.0],
    [2.0, 2.0, 2.0],
    [5.0, 1.0, 5.0],
    [3.5, 0.5, 5.0, 0.5, 1.0, 4.0],
    [-0.0, 2.0, 0.0, 1.0],
    [0.0, -0.0, 2.0],
    [np.inf, -np.inf, 1.0, 0.0],
    [1e-45, 0.0, 1.0],
]


@pytest.mark.parametrize("y", LABEL_SETS)
def test_binarizer_matches_the_transcripts(y):
    y = np.asarray(y, np.float32)
    cls = co.classes(y)
    if np_is_binarized(y):
        assert cls.size == 0
        assert co.transform(y, cls).tobytes() == y.astype(np.float64).reshape(-1, 1).tobytes()
        return
    ref = np_binarizer_fit(y)
    assert cls.tobytes() == ref.tobytes()            # sign of ±0 included: the first occurrence's
    Y = co.transform(y, cls)
    assert np.array_equal(Y, np_transform(y, ref) if ref.size > 1 else np.ones((y.size, 1)))


def test_a_class_keeps_the_sign_of_its_first_occurrence():
    assert np.signbit(co.classes([-0.0, 2.0, 0.0])[0]) and not np.signbit(co.classes([0.0, 2.0, -0.0])[0])


def test_nan_labels_are_refused():
    assert co.classes([1.0, np.nan, 2.0]) is None


def test_max_idx_and_inverse_transform_match_the_transcripts():
    rng = np.random.default_rng(1)
    h = rng.random((200, 5))
    h[:20, 0] = np.nan; h[20:40, 3] = np.nan; h[40:60] = h[40:60, :1]     # NaN in column 0 / elsewhere, exact ties
    cls = np.array([-2.0, 0.5, 1.0, 3.0, 7.25])
    assert co.labels_of(h, cls).tobytes() == np_inverse(h, cls).tobytes()
    assert np.all(co.labels_of(h[:20], cls) == -2.0) and not np.any(co.labels_of(h[20:40], cls) == 3.0)
    assert np.all(co.labels_of(h[:, :1], np.array([4.0])) == 4.0)


@pytest.mark.parametrize("hidden", [(), (6,)])
def test_softmax_and_log_loss_match_the_transcripts(hidden):
    X, y = _data(60, 7, 2, [0.5, 2.0, 3.0, 4.5])
    cfg = co.widen(orc.mlp64_cfg(7, hidden=hidden, alpha=0.0, seed=2), co.classes(y))
    rng = np.random.default_rng(2)
    p = rng.standard_normal(co.nparams(cfg))
    h = co.predict_proba(cfg, p, X)
    a, off = X, 0
    for l in range(cfg.n_layers - 1):
        fi, fo = cfg.units[l], cfg.units[l + 1]
        b, W = p[off:off + fo], p[off + fo:off + fo + fi * fo].reshape(fi, fo)
        off += (1 + fi) * fo
        z = np.array([[sum(a[r, k] * W[k, j] for k in range(fi)) + b[j] for j in range(fo)] for r in range(a.shape[0])])
        a = np_softmax(z) if l == cfg.n_layers - 2 else np.maximum(z, 0)
    np.testing.assert_allclose(h, a, rtol=1e-14, atol=0)
    Y = co.transform(y, co.classes(y))
    loss, _ = co.loss_grad(cfg, p, X, Y)
    assert loss == pytest.approx(np_log_loss(Y, h), rel=1e-14)


def test_softmax_overflow_is_nan_without_max_subtraction():
    cfg = co.widen(orc.mlp64_cfg(1, hidden=(), alpha=0.0), [1.0, 2.0, 3.0])
    p = np.array([800.0, 0.0, 0.0, 0.0, 0.0, 0.0])              # intercepts [800, 0, 0], W = 0: exp(800) = inf
    h = co.predict_proba(cfg, p, np.zeros((1, 1)))
    assert np.isnan(h[0, 0]) and h[0, 1] == 0.0
    assert co.labels_of(h, np.array([1.0, 2.0, 3.0]))[0] == 1.0    # MaxIdx64: a NaN in column 0 wins


@pytest.mark.parametrize("act,hidden,signs", [
    ("relu", (), [+1]),
    ("relu", (5,), [+1, +1]),
    ("tanh", (5,), [-1, +1]),
    ("tanh", (5, 4), [+1, -1, +1]),
])
def test_softmax_log_loss_gradient_against_finite_differences(act, hidden, signs):
    """alpha = 0; tanh's reference backprop negates the gradient below an odd number of tanh layers (as in the binary
    restatement)."""
    X, y = _data(30, 6, 4, [1.0, 2.0, 3.0, 4.0])
    cfg = co.widen(orc.mlp64_cfg(6, hidden=hidden, activation="relu", alpha=0.0, seed=4), co.classes(y))
    if act == "tanh":
        cfg.hidden_act = so.ACT_TANH
    Y = co.transform(y, co.classes(y))
    p = np.random.default_rng(4).standard_normal(co.nparams(cfg)) * 0.5
    _, gr = co.loss_grad(cfg, p, X, Y)
    fd = np.empty_like(p)
    for i in range(p.size):
        e = np.zeros_like(p); e[i] = 1e-6
        fd[i] = (co.loss_grad(cfg, p + e, X, Y)[0] - co.loss_grad(cfg, p - e, X, Y)[0]) / 2e-6
    off = 0
    for l, s in enumerate(signs):
        n = (1 + cfg.units[l]) * cfg.units[l + 1]
        np.testing.assert_allclose(gr[off:off + n], s * fd[off:off + n], rtol=1e-5, atol=1e-8)
        off += n


@pytest.mark.parametrize("solver,schedule,act,wd", [
    ("adam", "constant", "relu", 0.0),
    ("adam", "adaptive", "logistic", 0.0),
    ("sgd", "constant", "relu", 0.0),
    ("sgd", "invscaling", "identity", 1e-3),
    ("sgd", "adaptive", "relu", 0.0),
    ("adam", "constant", "tanh", 1e-3),
])
def test_binary_labels_are_the_solver_restatement_bit_for_bit(solver, schedule, act, wd):
    X, y = _data(300, 12, 5, [0.0, 1.0])
    cfg = orc.mlp64_cfg(12, hidden=(8, 5), activation="relu" if act == "tanh" else act, batch=64, max_iter=8, seed=6,
                        tol=1e-2, n_iter_no_change=1, lr_init=1e-2, adaptive=schedule == "adaptive")
    if act == "tanh":
        cfg.hidden_act = so.ACT_TANH
    o = so.opts(solver, schedule, weight_decay=wd)
    cls, wc, p, it, curve = co.cold_fit(cfg, o, X, y)
    ps = so.init(cfg)
    its, curves, _, _ = so.fit(cfg, o, ps, X, y.astype(np.float64).reshape(-1, 1))
    assert cls.size == 0 and wc.units[wc.n_layers - 1] == 1
    assert it == its and curve.tobytes() == curves.tobytes() and p.tobytes() == ps.tobytes()


def test_single_class_is_a_logistic_unit_on_an_all_ones_target():
    X, _ = _data(120, 5, 7, [0.0, 1.0])
    cfg = orc.mlp64_cfg(5, hidden=(4,), batch=50, max_iter=4, seed=7)
    o = so.opts()
    cls, wc, p, it, curve = co.cold_fit(cfg, o, X, np.full(120, 3.0, np.float32))
    ps = so.init(cfg)
    its, curves, _, _ = so.fit(cfg, o, ps, X, np.ones((120, 1)))
    assert cls.tolist() == [3.0] and curve.tobytes() == curves.tobytes() and p.tobytes() == ps.tobytes()
    assert np.all(co.predict(wc, p, cls, X) == 3.0)


def test_multiclass_init_uses_the_wide_output_layer():
    """initialize :458-476 over the longer packed vector: the layers below the output are the binary model's, the
    output layer's bound uses fo = C."""
    cfg = orc.mlp64_cfg(9, hidden=(7,), seed=9)
    wc = co.widen(cfg, [1.0, 2.0, 3.0])
    pw, pb = co.init(wc), so.init(cfg)
    n0 = (1 + 9) * 7
    assert pw.size == n0 + (1 + 7) * 3 and pw[:n0].tobytes() == pb[:n0].tobytes()
    assert np.all(pw[n0:] < np.sqrt(6 / (7 + 3))) and not np.array_equal(pw[n0:n0 + 8], pb[n0:n0 + 8])


# ---- refusals of ctr_mlp_set_classes that need no device --------------------------------------------------------------
@pytest.mark.parametrize("classes,msg", [
    ([1.0, np.nan], b"NaN"),
    ([2.0, 1.0], b"ascending"),
    ([1.0, 1.0], b"ascending"),
    (list(range(1025)), b"1024"),
])
def test_set_classes_refuses_bad_classes(classes, msg):
    L = g.load_library()
    c = np.ascontiguousarray(classes, np.float64)
    assert L.ctr_mlp_set_classes(None, c.ctypes.data_as(C.POINTER(C.c_double)), C.c_int32(c.size)) == g.EINVAL
    assert msg in L.ctr_mlp_last_error(None)


def test_set_classes_refuses_a_null_buffer_and_a_negative_count():
    L = g.load_library()
    assert L.ctr_mlp_set_classes(None, None, C.c_int32(2)) == g.EINVAL
    assert L.ctr_mlp_set_classes(None, None, C.c_int32(-1)) == g.EINVAL
    assert L.ctr_mlp_set_classes(None, None, C.c_int32(0)) == g.EINVAL and b"null classifier" in L.ctr_mlp_last_error(None)
    assert L.ctr_mlp_get_classes(None, None, C.c_int32(0), None) == g.EINVAL


def test_abi_exports_the_class_calls():
    assert {"ctr_mlp_get_classes", "ctr_mlp_set_classes"} <= set(g.engine.EXPORTS)
