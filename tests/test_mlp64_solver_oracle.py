"""The float64 MLP solver restatement (tests/mlp64_solver_oracle.c) against independent numpy transcripts of
basemlp64.go, against oracle/mlp64_oracle.c where the two overlap, and against finite differences.  CPU only."""
import numpy as np
import pytest

from oracle import oracle as orc
from tests import mlp64_solver_oracle as so


def _data(n, nf, seed):
    rng = np.random.default_rng(seed)
    X = rng.random((n, nf))
    y = ((X - 0.5) @ rng.standard_normal(nf) + 0.3 * rng.standard_normal(n) > 0).astype(np.float64).reshape(-1, 1)
    return X, y


def _layers(cfg, p):
    """packed vector → [(b, W)] views (basemlp64.go:459-463)"""
    out, off = [], 0
    for l in range(cfg.n_layers - 1):
        fi, fo = cfg.units[l], cfg.units[l + 1]
        out.append((p[off:off + fo], p[off + fo:off + fo + fi * fo].reshape(fi, fo)))
        off += (1 + fi) * fo
    return out


# ---- an independent numpy restatement of fitStochastic (basemlp64.go:729-857) -----------------------------------
def _act(name, z):
    return {0: lambda v: np.maximum(v, 0), 1: lambda v: 1 / (1 + np.exp(-v)), 2: lambda v: v, 3: lambda v: np.tanh(-v)}[name](z)


def _deriv(name, a):
    return {0: lambda v: (v != 0).astype(np.float64), 1: lambda v: v * (1 - v), 2: lambda v: np.ones_like(v),
            3: lambda v: 1 - v * v}[name](a)


def _np_backprop(cfg, p, X, y):
    L, layers, m = cfg.n_layers, _layers(cfg, p), X.shape[0]
    acts = [X]
    for l, (b, W) in enumerate(layers):
        z = acts[-1] @ W + b
        acts.append(1 / (1 + np.exp(-z)) if l == L - 2 else _act(cfg.hidden_act, z))
    h = np.clip(acts[-1], np.nextafter(0, 1), np.nextafter(1, 0))
    loss = np.sum(-y * np.log(h) - (1 - y) * np.log1p(-h)) / m
    loss += 0.5 * cfg.alpha * sum(np.sum(W * W) for _, W in layers) / m
    g = np.empty_like(p)
    gl = _layers(cfg, g)
    D = acts[-1] - y
    for l in range(L - 2, -1, -1):
        b, W = layers[l]
        gl[l][1][:] = acts[l].T @ D / m + cfg.alpha / m * W
        gl[l][0][:] = D.sum(0) / m
        if l >= 1:
            D = (D @ W.T) * _deriv(cfg.hidden_act, acts[l])
    return loss, g


def _perm(seed, it, idx):
    for i in range(idx.size - 1, 0, -1):
        j = int(orc.lib().orc_mix64(seed, 100 + it, i) % (i + 1))
        idx[i], idx[j] = idx[j], idx[i]


def _np_fit(cfg, solver, schedule, p, X, y, t=0.0, power_t=0.5, momentum=0.9, nesterov=True, wd=0.0):
    n, bs = X.shape[0], min(cfg.batch, X.shape[0])
    idx = np.arange(n)
    vel, ms, vs = np.zeros_like(p), np.zeros_like(p), np.zeros_like(p)
    lr, lr_init, best, noimp, curve, lrs, b1t, b2t = cfg.lr_init, cfg.lr_init, np.inf, 0, [], [], 1.0, 1.0
    for it in range(cfg.max_iter):
        if cfg.shuffle:
            _perm(cfg.seed, it, idx)
        acc = 0.0
        for b0 in range(0, n, bs):
            rows = idx[b0:b0 + bs]
            if wd > 0:
                p *= 1 - wd
            loss, g = _np_backprop(cfg, p, X[rows], y[rows])
            acc += loss * rows.size
            if solver == "sgd":
                u = momentum * vel - lr * g
                vel = u
                p += momentum * vel - lr * g if nesterov else u
            else:
                for i in range(p.size):
                    ms[i] = cfg.beta1 * ms[i] + (1 - cfg.beta1) * g[i]
                    vs[i] = cfg.beta2 * vs[i] + (1 - cfg.beta2) * g[i] * g[i]
                    b1t *= cfg.beta1; b2t *= cfg.beta2
                    lr = lr_init * np.sqrt(1 - b2t) / (1 - b1t)
                    p[i] += -lr * ms[i] / (np.sqrt(vs[i]) + cfg.eps)
        curve.append(acc / n)
        t += n
        noimp = noimp + 1 if curve[-1] > best - cfg.tol else 0
        best = min(best, curve[-1])
        if solver == "sgd" and schedule == "invscaling":
            lr = cfg.lr_init / (t + 1) ** power_t
        stop = False
        if noimp > cfg.n_iter_no_change:
            if schedule != "adaptive" or lr <= 1e-6:
                stop = True
            else:
                if solver == "sgd":
                    lr *= .8
                else:
                    lr_init *= .8
                noimp = 0
        lrs.append(lr if solver == "sgd" else lr_init)
        if stop:
            break
    return len(curve), np.array(curve), np.array(lrs), t


# ---- the pieces ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("momentum", [0.0, 0.9])
@pytest.mark.parametrize("nesterov", [False, True])
def test_sgd_update_is_the_reference_transcript_bit_for_bit(momentum, nesterov):
    """SGDOptimizer64.updateParams (basemlp64.go:1024-1039), two consecutive calls so the velocity is live."""
    rng = np.random.default_rng(1)
    p = rng.standard_normal(1000); v = np.zeros(1000); o = so.opts("sgd", momentum=momentum, nesterov=nesterov)
    pn, vn = p.copy(), v.copy()
    for lr in (0.01, 0.003):
        g = rng.standard_normal(1000)
        so.sgd(o, lr, p, g, v)
        update = momentum * vn - lr * g
        vn = update
        pn = pn + (momentum * vn - lr * g if nesterov else update)
        assert p.tobytes() == pn.tobytes() and v.tobytes() == vn.tobytes()


def test_weight_decay_step_is_the_reference_transcript_bit_for_bit():
    """backprop :342-346: every packed element, intercepts included, times (1 - wd); wd = 0 leaves them untouched."""
    rng = np.random.default_rng(2)
    p0 = rng.standard_normal(777)
    for wd in (0.0, 1e-4, 0.3):
        p = p0.copy(); so.decay(wd, p)
        assert p.tobytes() == (p0 * (1 - wd) if wd > 0 else p0).tobytes()


def test_tanh_forward_is_tanh_of_minus_z():
    """Activations64["tanh"] (basemlp64.go:88-94) evaluates tanh(-z); the output stays logistic."""
    cfg = orc.mlp64_cfg(7, hidden=(5, 4), activation="relu", seed=3)
    cfg.hidden_act = so.ACT_TANH
    rng = np.random.default_rng(3)
    p = rng.standard_normal(so.nparams(cfg)) * 0.7
    X = rng.random((40, 7))
    (b0, W0), (b1, W1), (b2, W2) = _layers(cfg, p)
    h = np.tanh(-(np.tanh(-(X @ W0 + b0)) @ W1 + b1))
    np.testing.assert_allclose(so.predict(cfg, p, X).ravel(), (1 / (1 + np.exp(-(h @ W2 + b2)))).ravel(), rtol=1e-13)
    assert so.init(cfg).tobytes() == so.init(orc.mlp64_cfg(7, hidden=(5, 4), activation="relu", seed=3)).tobytes()  # Glorot factor 6 (:466-470)


@pytest.mark.parametrize("act,hidden,signs", [
    ("tanh", (5,), [-1, +1]),
    ("tanh", (5, 4), [+1, -1, +1]),
    ("relu", (5, 4), [+1, +1, +1]),
    ("logistic", (5, 4), [+1, +1, +1]),
])
def test_gradient_against_finite_differences(act, hidden, signs):
    """alpha = 0.  With tanh the reference's backprop multiplies by 1 - a² where the forward pass's derivative is
    -(1 - a²) (:91 vs :135): every layer below an odd number of tanh layers gets the negated gradient."""
    cfg = orc.mlp64_cfg(6, hidden=hidden, activation="relu" if act == "tanh" else act, alpha=0.0, seed=4)
    if act == "tanh":
        cfg.hidden_act = so.ACT_TANH
    rng = np.random.default_rng(4)
    p = rng.standard_normal(so.nparams(cfg)) * 0.5
    X, y = _data(30, 6, 4)
    _, g = so.loss_grad(cfg, p, X, y)
    fd = np.empty_like(p)
    for i in range(p.size):
        e = np.zeros_like(p); e[i] = 1e-6
        fd[i] = (so.loss_grad(cfg, p + e, X, y)[0] - so.loss_grad(cfg, p - e, X, y)[0]) / 2e-6
    for (gb, gW), (fb, fW), s in zip(_layers(cfg, g), _layers(cfg, fd), signs):
        np.testing.assert_allclose(np.concatenate([gb, gW.ravel()]), s * np.concatenate([fb, fW.ravel()]), rtol=1e-5, atol=1e-8)


# ---- against the existing oracle where they overlap ---------------------------------------------------------------
@pytest.mark.parametrize("act", ["relu", "logistic", "identity"])
@pytest.mark.parametrize("adaptive", [False, True])
def test_default_options_reproduce_the_adam_oracle_bit_for_bit(act, adaptive):
    """adam + constant / adaptive and no weight decay is what oracle/mlp64_oracle.c restates: same init, same
    loss curve, same parameters, to the bit (adaptive with a stopping rule that triggers)."""
    X, y = _data(300, 20, 5)
    cfg = orc.mlp64_cfg(20, hidden=(8, 6), activation=act, batch=64, max_iter=12, seed=6, adaptive=adaptive,
                        tol=1e-2, n_iter_no_change=1, lr_init=1e-2)
    p = so.init(cfg)
    assert p.tobytes() == orc.mlp64_init(cfg).tobytes()
    po = p.copy()
    it, curve, lrs, t = so.fit(cfg, so.opts("adam", "adaptive" if adaptive else "constant"), p, X, y)
    ito, curveo, lr_init = orc.mlp64_fit(cfg, po, X, y)
    assert it == ito and curve.tobytes() == curveo.tobytes() and p.tobytes() == po.tobytes()
    assert lrs[-1] == lr_init and t == 300.0 * it


def test_adam_invscaling_is_adam_constant():
    """AdamOptimizer64.iterationEnds is a no-op (:1053) and triggerStopping stops for any non-adaptive schedule."""
    X, y = _data(300, 20, 7)
    cfg = orc.mlp64_cfg(20, hidden=(8,), batch=64, max_iter=30, seed=8, tol=1e-2, n_iter_no_change=1)
    pa, pb = so.init(cfg), so.init(cfg)
    ra = so.fit(cfg, so.opts("adam", "constant"), pa, X, y)
    rb = so.fit(cfg, so.opts("adam", "invscaling", power_t=0.25), pb, X, y)
    assert ra[0] == rb[0] < 30 and ra[1].tobytes() == rb[1].tobytes() and pa.tobytes() == pb.tobytes()


# ---- whole fits against the numpy restatement ---------------------------------------------------------------------
@pytest.mark.parametrize("solver,schedule,act,wd", [
    ("sgd", "constant", "relu", 0.0),
    ("sgd", "invscaling", "relu", 0.0),
    ("sgd", "constant", "tanh", 0.0),
    ("sgd", "constant", "logistic", 1e-3),
    ("adam", "constant", "tanh", 1e-3),
])
def test_fit_matches_the_numpy_restatement(solver, schedule, act, wd):
    X, y = _data(150, 12, 9)
    cfg = orc.mlp64_cfg(12, hidden=(7, 5), activation="relu" if act == "tanh" else act, batch=40, max_iter=4, seed=10,
                        lr_init=0.05 if solver == "sgd" else 1e-2, alpha=1e-3)
    if act == "tanh":
        cfg.hidden_act = so.ACT_TANH
    p = so.init(cfg); pn = p.copy()
    it, curve, lrs, t = so.fit(cfg, so.opts(solver, schedule, weight_decay=wd), p, X, y)
    itn, curven, lrsn, tn = _np_fit(cfg, solver, schedule, pn, X, y, wd=wd)
    assert it == itn == 4 and t == tn
    np.testing.assert_allclose(curve, curven, rtol=1e-12)
    np.testing.assert_allclose(lrs, lrsn, rtol=1e-15)
    np.testing.assert_allclose(p, pn, rtol=1e-10, atol=1e-13)


def test_invscaling_schedule_and_warm_start_continue_t():
    """lr = lr_init / (t+1)^power_t at every epoch end (:999-1003) with t the samples seen since the cold initialise
    (:814); a warm-start fit skips initialize (:502-512), so t continues, while its optimizer starts again from
    lr_init (:731-752)."""
    n = 120
    X, y = _data(n, 10, 11)
    cfg = orc.mlp64_cfg(10, hidden=(6,), batch=50, max_iter=3, seed=12, lr_init=0.1, n_iter_no_change=100)
    o = so.opts("sgd", "invscaling", power_t=0.3)
    p = so.init(cfg); pn = p.copy()
    it, curve, lrs, t = so.fit(cfg, o, p, X, y)
    assert t == 3 * n
    assert lrs.tolist() == [0.1 / (n * (e + 1) + 1) ** 0.3 for e in range(3)]
    it2, curve2, lrs2, t2 = so.fit(cfg, o, p, X, y, t=t)
    assert t2 == 6 * n
    assert lrs2.tolist() == [0.1 / (n * (e + 4) + 1) ** 0.3 for e in range(3)]
    _np_fit(cfg, "sgd", "invscaling", pn, X, y, power_t=0.3)
    _, curven2, _, _ = _np_fit(cfg, "sgd", "invscaling", pn, X, y, t=3.0 * n, power_t=0.3)
    np.testing.assert_allclose(curve2, curven2, rtol=1e-12)
    np.testing.assert_allclose(p, pn, rtol=1e-10, atol=1e-13)
    pc = so.init(cfg)                                            # a cold second fit restarts t: a different trajectory
    so.fit(cfg, o, pc, X, y)
    _, curvec, _, _ = so.fit(cfg, o, pc, X, y, t=0.0)
    assert curvec.tobytes() != curve2.tobytes()


def test_adaptive_sgd_shrinks_the_current_rate_until_it_is_tiny():
    """SGDOptimizer64.triggerStopping (:1005-1023): each trigger multiplies the CURRENT rate by .8 and resets the
    count; once the rate is <= 1e-6 the next trigger stops."""
    X, y = _data(100, 8, 13)
    cfg = orc.mlp64_cfg(8, hidden=(4,), batch=50, max_iter=200, seed=14, lr_init=1e-5, tol=1e9, n_iter_no_change=1)
    p = so.init(cfg)
    it, curve, lrs, _ = so.fit(cfg, so.opts("sgd", "adaptive"), p, X, y)
    lr, best, noimp, want = 1e-5, np.inf, 0, []                  # the rule, replayed on the oracle's own loss curve
    for e, loss in enumerate(curve):
        noimp = noimp + 1 if loss > best - 1e9 else 0
        best = min(best, loss)
        stop = False
        if noimp > 1:
            if lr <= 1e-6:
                stop = True
            else:
                lr *= .8; noimp = 0
        want.append(lr)
        if stop:
            break
    assert lrs.tolist() == want and len(want) == it < 200
    rates = [1e-5]
    while rates[-1] > 1e-6:
        rates.append(rates[-1] * .8)
    assert len(rates) == 12 and sorted(set(lrs.tolist()), reverse=True) == rates and lrs[-1] == rates[-1]
