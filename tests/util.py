import numpy as np


def close_frac(a, b, rtol, atol):
    a = np.asarray(a, np.float64).ravel(); b = np.asarray(b, np.float64).ravel()
    return float(np.mean(np.abs(a - b) <= atol + rtol * np.abs(b)))


def assert_mostly_close(a, b, rtol, atol, frac=0.999, what=""):
    """Adam turns a gradient whose sign flips inside fp32 rounding noise into a ±lr weight step, so a
    handful of elements may legitimately differ after optimiser steps; everything else must agree."""
    f = close_frac(a, b, rtol, atol)
    assert f >= frac, "%s: only %.5f of elements within rtol=%g atol=%g" % (what, f, rtol, atol)


def make_tables(rng, U, I, uP, cF, D):
    uf = rng.random((U, uP), np.float32)
    itf = rng.random((I, cF), np.float32)
    emb = (rng.standard_normal((I, D)) / np.sqrt(D)).astype(np.float32)
    return uf, itf, emb


def make_batch(rng, U, I, B, S, pad_frac=0.2, zipf=False):
    ur = rng.integers(0, U, B).astype(np.int32)
    if zipf:
        ir = (rng.zipf(1.05, B) - 1) % I
        hist = (rng.zipf(1.05, (B, S)) - 1) % I
    else:
        ir = rng.integers(0, I, B)
        hist = rng.integers(0, I, (B, S))
    hist = hist.astype(np.int32); ir = ir.astype(np.int32)
    # most-recent-first with a -1 padded tail (prepare.go:49-51, rcmd.go:517-522)
    lens = np.where(rng.random(B) < pad_frac, rng.integers(0, S + 1, B), S)
    hist[np.arange(S)[None, :] >= lens[:, None]] = -1
    y = (rng.random(B) > 0.5).astype(np.float32)
    return ur, ir, hist, y


INT64_MIN, INT64_MAX = int(np.iinfo(np.int64).min), int(np.iinfo(np.int64).max)

# idmap.cuh starts an id's linear probe at idmap_hash(id) & (cap - 1); idmap_hash is MurmurHash3's fmix64, a bijection
# on 64-bit words, so inverting it yields ids that start at any chosen slot (collisions made to order)
_C1, _C2 = 0xff51afd7ed558ccd, 0xc4ceb9fe1a85ec53
_C1_INV, _C2_INV = (np.uint64(pow(c, -1, 1 << 64)) for c in (_C1, _C2))
_C1, _C2, _S33 = np.uint64(_C1), np.uint64(_C2), np.uint64(33)


def idmap_hash(ids):
    """idmap_hash of int64 ids, in wrapping uint64 arithmetic."""
    k = np.array(ids, np.int64).view(np.uint64)
    k ^= k >> _S33; k *= _C1; k ^= k >> _S33; k *= _C2; k ^= k >> _S33
    return k


def idmap_unhash(h):
    """The int64 ids whose idmap_hash is h: fmix64's steps undone in reverse order (x ^= x >> 33 is its own inverse)."""
    k = np.array(h, np.uint64)
    k ^= k >> _S33; k *= _C2_INV; k ^= k >> _S33; k *= _C1_INV; k ^= k >> _S33
    return k.view(np.int64)


def idmap_capacity(n):
    """Slots of a map of n ids: the smallest power of two >= 2n, at least 64 (load factor <= 0.5)."""
    cap = 64
    while cap < 2 * n:
        cap <<= 1
    return cap


def ids_probing_from(rng, slots, cap, avoid=()):
    """Distinct ids whose probe starts at slots[i] in a map of cap slots: random high hash bits over the slot, inverted.
    INT64_MIN (the empty-slot marker) and the ids in `avoid` are never returned."""
    seen = {int(v) for v in avoid}
    out = np.empty(len(slots), np.int64)
    for j, s in enumerate(slots):
        while True:
            h = (rng.integers(0, 2**64, dtype=np.uint64) & ~np.uint64(cap - 1)) | np.uint64(s)
            v = int(idmap_unhash([h])[0])
            if v != INT64_MIN and v not in seen:
                break
        seen.add(v); out[j] = v
    return out


def scaled_init(orc, ocfg, seed, s0=0.05, s1=0.05, s2=0.3):
    """N(0,1) init (din.go:187-191) scaled so sigmoids are not saturated and parity is informative."""
    W0, W1, W2, att = orc.init_weights(ocfg, seed)
    rng = np.random.default_rng(seed)
    return [np.ascontiguousarray(W0 * s0), np.ascontiguousarray(W1 * s1), np.ascontiguousarray(W2 * s2),
            (att + 0.2 * rng.standard_normal(att.shape)).astype(np.float32)]
