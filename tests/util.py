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


_M0, _M1, _M2 = 0x9E3779B97F4A7C15, 0xD1B54A32D192ED03, 0x632BE59BD9B4E019
_M3, _M4 = np.uint64(0xBF58476D1CE4E5B9), np.uint64(0x94D049BB133111EB)


def mix64(seed, stream, ctr):
    """The engine's counter RNG (common.cuh mix64, oracle orc_mix64) over an array of uint64 counters."""
    z = np.asarray(ctr, np.uint64) * np.uint64(_M1) + np.uint64((((seed << 32) | stream) * _M0 + _M2) % (1 << 64))
    z ^= z >> np.uint64(30); z *= _M3
    z ^= z >> np.uint64(27); z *= _M4
    z ^= z >> np.uint64(31)
    return z


def fill_rows(rows, width, seed, stream, dist, scale):
    """Rows of a table made by ctr_table_fill on one GPU (attn.cuh k_table_fill): element (row, c) draws
    mix64(seed, stream = table index, row * width + c).  dist 0: U[0, 1) * scale as float32, bit for bit.  dist 1:
    Box-Muller N(0, 1) * scale in float64 from the device's float32 u1, u2, with r = sqrt(-2 ln u1), which bounds the
    error of the device's __logf (see fill_normal_tol)."""
    ctr = np.asarray(rows, np.uint64)[:, None] * np.uint64(width) + np.arange(width, dtype=np.uint64)
    z = mix64(seed, stream, ctr)
    if dist == 0:
        return (z >> np.uint64(40)).astype(np.float32) * np.float32(1.0 / 16777216.0) * np.float32(scale)
    # the float32 arithmetic of the kernel: 16777217.0f rounds to 2^24, so u1 lies in (0, 1]
    u1 = ((z >> np.uint64(40)).astype(np.float32) + np.float32(1.0)) * (np.float32(1.0) / np.float32(16777217.0))
    u2 = ((z >> np.uint64(8)) & np.uint64(0xFFFFFF)).astype(np.float32) * np.float32(1.0 / 16777216.0)
    r = np.sqrt(-2.0 * np.log(u1.astype(np.float64)))
    return r * np.cos((np.float32(6.2831853) * u2).astype(np.float64)) * scale, r


def fill_normal_tol(r, scale):
    """Bound on |device - fill_rows| for dist 1: 1e-5 * scale for the float32 rounding and __cosf, plus __logf's absolute
    error (2^-21.41 on [0.5, 2]) carried through the square root, which grows as r -> 0 (u1 -> 1) and is at most
    sqrt(2 * 2^-21.41)."""
    return scale * (1e-5 + 4e-7 / np.maximum(r, 4e-4))


def scaled_init(orc, ocfg, seed, s0=0.05, s1=0.05, s2=0.3):
    """N(0,1) init (din.go:187-191) scaled so sigmoids are not saturated and parity is informative."""
    W0, W1, W2, att = orc.init_weights(ocfg, seed)
    rng = np.random.default_rng(seed)
    return [np.ascontiguousarray(W0 * s0), np.ascontiguousarray(W1 * s1), np.ascontiguousarray(W2 * s2),
            (att + 0.2 * rng.standard_normal(att.shape)).astype(np.float32)]
