"""Plain numpy references for the row-sharded kernel checks (tests/test_gpu_shard_probe.py): the float32 summation bound
of an atomically accumulated gradient row, the float64 row-Adam update with its float32 rounding budget, and the
top-k order of search and recommendation.  tests/test_shard_probe_cpu.py checks these helpers themselves."""
import numpy as np

U32 = 2.0 ** -24            # unit roundoff of float32


def sum_bound(n_terms, abs_sum):
    """Largest error of any float32 summation order of n_terms terms whose magnitudes add up to abs_sum: each of the at
    most n_terms - 1 additions rounds by at most 2^-24 of a partial sum, and every partial sum is at most abs_sum.  The
    bar is twice that, n·2^-23·Σ|t|; a sum of one term is exact."""
    n = np.asarray(n_terms, np.float64)
    return np.where(n > 1, n * 2.0 ** -23 * np.asarray(abs_sum, np.float64), 0.0)


def within_sum_bound(got, exact, n_terms, abs_sum):
    """elementwise: |got - exact| <= sum_bound(n_terms, abs_sum)"""
    return np.abs(np.asarray(got, np.float64) - exact) <= sum_bound(n_terms, abs_sum)


def row_adam64(w, m, v, g, lr, b1, b2, eps, c1, c2, inv_batch):
    """row_adam_elem (attn.cuh) in float64 from float32 inputs and float32 constants.  Returns (w, m, v, tol_m, tol_v):
    the moments with the bound of their float32 evaluation (a few roundings of the terms' magnitudes)."""
    f = lambda x: np.float64(np.float32(x))
    w, m, v, g = (np.asarray(a, np.float32).astype(np.float64) for a in (w, m, v, g))
    b1, b2, lr, eps, c1, c2, ib = f(b1), f(b2), f(lr), f(eps), f(c1), f(c2), f(inv_batch)
    gs = np.float32(g * ib).astype(np.float64)          # g *= inv_batch is one float32 product
    m1 = b1 * m + (1.0 - b1) * gs                        # 1 - b1 and 1 - b2 are exact in float32 (Sterbenz)
    v1 = b2 * v + (1.0 - b2) * gs * gs
    tol_m = 4 * U32 * (np.abs(b1 * m) + np.abs((1.0 - b1) * gs))
    tol_v = 6 * U32 * (b2 * v + (1.0 - b2) * gs * gs)
    w1 = w - lr * (m1 / c1) / (np.sqrt(v1 / c2) + eps)
    return w1, m1, v1, tol_m, tol_v


def adam_weight_from(w0, m, v, lr, eps, c1, c2):
    """The weight row_adam_elem leaves given the float32 moments it computed, in float64, with the bound of its float32
    evaluation: six roundings of the step (two quotients, a square root, a sum, a product, a quotient) and the final
    rounding of the weight."""
    f = lambda x: np.float64(np.float32(x))
    w0, m, v = (np.asarray(a, np.float32).astype(np.float64) for a in (w0, m, v))
    step = f(lr) * (m / f(c1)) / (np.sqrt(v / f(c2)) + f(eps))
    w = w0 - step
    return w, 8 * U32 * np.abs(step) + U32 * np.abs(w)


def topk(scores, rows, k, qualifies):
    """The first k (score, row) pairs under (score descending, row ascending) among those whose score qualifies.
    Returns (rows, scores, count) padded to k with row -1 and score 0."""
    scores = np.asarray(scores); rows = np.asarray(rows)
    keep = np.array([bool(qualifies(s)) for s in scores], bool) if scores.size else np.zeros(0, bool)
    s, r = scores[keep], rows[keep]
    order = np.lexsort((r, -s.astype(np.float64)))[:k]
    n = order.size
    out_r = np.full(k, -1, np.int32); out_s = np.zeros(k, scores.dtype)
    out_r[:n] = r[order]; out_s[:n] = s[order]
    return out_r, out_s, n
