"""The parallel item2vec kernel k_i2v_skipgram_hs<LPR> against the float64 model of tests/i2v_pair_model.py, at every
vector width, launched through the kernel-level probe tests/cuda/i2v_probe.cu (the production header, not a copy).

The trainer is Hogwild: what two warps do to one vector at the same time is not defined.  Each tier is built so that
its verdict does not depend on that.
  A  isolated updates: every vector is written for one centre only, so the result is defined up to the order of two
     addends; every float of both tables within 2 ulp (float32) of the model, untouched floats bit for bit.
     Cannot see: anything that needs two centres on one vector.
  B  window enumeration: which rows move is exact, by how much to 1e-3 (both model orders lie inside that).
     Cannot see: an error of the arithmetic below 1e-3.
  C  a full grid on a Zipf document in the linear regime (tiny lr): the summed update of every row against the model's
     stale sum, under real contention on the top of the tree.  Cannot see: errors below 2 % of a row's increment."""
import numpy as np
import pytest

import go_ctr_b200 as g
from oracle import oracle as orc
from tests import i2v_pair_model as pm
from tests import i2v_probe as probe

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

DIMS = [4, 8, 16, 32, 64, 128]
K_HOT, K_FLUSH = 64, 8                       # kI2vHot, kI2vFlush of item2vec.cuh (asserted against the probe below)
f32, f64, u32 = np.float32, np.float64, np.uint32


def test_probe_reports_the_kernels_constants():
    assert probe.lib().i2v_probe_hot_max() == K_HOT and probe.lib().i2v_probe_flush_every() == K_FLUSH


# ---- comparison ---------------------------------------------------------------------------------------------------
def assert_tables(a, out0, out1, want, ulps=2):
    """Every float of both tables: bit-equal where the model adds nothing, else within `ulps` float32 ulps (taken at the
    larger of the initial and the final magnitude: the addends are rounded there) of the model's float64 sum."""
    for name, out, init, w in (("syn0", out0, a.syn0, want.syn0), ("syn1", out1, a.syn1, want.syn1)):
        moved = w != init.astype(f64)
        still = out.view(u32)[~moved] == init.view(u32)[~moved]
        assert still.all(), "%s: %d floats moved that the model leaves alone, first rows %s" % (name, (~still).sum(), np.unique(np.nonzero(~moved)[0][~still])[:5])
        tol = ulps * np.spacing(np.maximum(np.abs(init), np.abs(w)).astype(f32)).astype(f64)
        err = np.abs(out.astype(f64) - w)
        bad = err > tol
        assert not bad.any(), "%s: %d floats off, worst %.1f ulp, first rows %s" % (name, bad.sum(), (err / tol * ulps).max(), np.unique(np.nonzero(bad)[0])[:5])
        assert moved.any() or name == "syn1"


def run_isolated(a, D, grid, block, exact_f=False):
    want = pm.launch_model(a, "passes", rpw=32 // (D // 4))
    assert exact_f or want.margin > 0, "an f of this input is too close to a table-bin edge for a float32 dot product"
    out0, out1, ctr = probe.skipgram(a, grid, block)
    assert ctr == want.counters, (ctr, want.counters)
    assert_tables(a, out0, out1, want)
    return out0, out1, want


# ---- tier A: isolated updates -------------------------------------------------------------------------------------
def centre_positions(n):
    """n >= 2 centres, W = 1: 'c x | x c x | ... | x c'.  The first centre has no left context, the last no right one
    (cpos < 0 and cpos >= nd), no token is context to two centres."""
    return [0] + [3 * j for j in range(1, n - 1)] + [3 * n - 3], 3 * n - 2


def magnitude(D):
    return np.sqrt(1.5 / (0.58 * np.sqrt(D)))               # f = c . nv gets a standard deviation of ~1.5: many table bins


def rand_table(rng, rows, D, scale=1.0):
    m = magnitude(D) * scale
    return (rng.uniform(0.5 * m, m, (rows, D)) * rng.choice([-1.0, 1.0], (rows, D))).astype(f32)


def isolated(D, path_lens, rng, hot="none", lr=0.025, scales=False, upd=None, spare=0):
    """All words distinct (word id = position); z = 1 at the centres, 0 elsewhere; every centre owns a private chain of
    nodes, numbered by a random permutation so that a hot range cuts through every path."""
    n = len(path_lens)
    cpos, nd = centre_positions(n)
    used = int(sum(path_lens)); nn = max(used + spare, 1)
    ids = rng.permutation(used)
    poff = np.zeros(nd + 1, np.int64); ln = np.zeros(nd, np.int64); ln[cpos] = path_lens
    poff[1:] = np.cumsum(ln)
    pnode = ids.astype(np.int32)                             # centres are in position order, and so is the CSR
    pcode = rng.integers(0, 2, used).astype(np.uint8)
    z = np.zeros(nd); z[cpos] = 1.0
    hot_n = {"none": 0, "split": min(K_HOT, used // 2), "all": nn, "max": K_HOT, "spare": min(K_HOT, used // 2 + spare)}[hot]
    assert hot_n <= K_HOT and hot_n <= nn
    pick = [1.0, 0.5, 1.0 / 3.0, 1e-3]
    return pm.Launch(doc=np.arange(nd, dtype=np.int32), z=z, poff=poff, pnode=pnode, pcode=pcode, syn0=rand_table(rng, nd, D), syn1=rand_table(rng, nn, D),
                     W=1, lr_tab=np.full(1, lr, f32) if upd is None else rng.uniform(0.4 * lr, lr, nd // upd + 1).astype(f32), upd=nd + 1 if upd is None else upd,
                     seed=int(rng.integers(1, 1 << 31)), iter=int(rng.integers(0, 5)),
                     node_scale=rng.choice(pick, nn).astype(f32) if scales else np.ones(nn, f32), word_scale=rng.choice(pick, nd).astype(f32) if scales else np.ones(nd, f32),
                     hot_base=nn - hot_n, hot_n=hot_n)


def safe(make, D):
    """The first seeded instance of a random case in which no f lies within float32 summation error of a bin edge."""
    for s in range(50):
        a = make(np.random.default_rng(1000 * D + s))
        if pm.launch_model(a, "passes", rpw=32 // (D // 4)).margin > 0:
            return a
    raise AssertionError("no safe instance in 50 seeds")


@pytest.mark.parametrize("block", [32, 256])
@pytest.mark.parametrize("D", DIMS)
def test_isolated_path_lengths(D, block):
    """Paths of 0 (a word without a path), 1, 7 and 40 nodes with mixed codes; one block of 256 or of 32 threads."""
    a = safe(lambda rng: isolated(D, [7, 0, 1, 40, 7, 1, 0, 40], rng), D)
    _, _, want = run_isolated(a, D, 1, block)
    assert want.counters[0] == 8 and want.counters[1] == 14 and set(a.pcode.tolist()) == {0, 1}


@pytest.mark.parametrize("D", DIMS)
def test_isolated_scales_go_to_their_own_table_and_index(D):
    """node_scale and word_scale drawn from {1, 1/2, 1/3, 1e-3} per node and per word."""
    a = safe(lambda rng: isolated(D, [3, 5, 2, 7, 4, 6], rng, scales=True), D)
    assert len(set(a.node_scale.tolist())) == 4 and len(set(a.word_scale.tolist())) == 4
    run_isolated(a, D, 2, 64)


@pytest.mark.parametrize("hot", ["none", "split", "all", "max", "spare"])
@pytest.mark.parametrize("D", DIMS)
def test_isolated_hot_ranges(D, hot):
    """No hot node; a hot_base that splits every path between the shared-memory route and the red route; every node
    hot; hot_n = kI2vHot; hot nodes nobody touches (the flush skips zeros)."""
    lens = [40, 30, 7, 1, 0, 5] if hot == "max" else [3, 7, 0, 1, 12, 5, 9, 2]
    a = safe(lambda rng: isolated(D, lens, rng, hot=hot, scales=True, spare=3 if hot == "spare" else 0), D)
    if hot in ("split", "spare", "max"):                     # some centre's path really uses both routes
        assert any(len({bool(n >= a.hot_base) for n in a.pnode[a.poff[w]:a.poff[w + 1]]}) == 2 for w in range(a.doc.size))
    out0, out1, want = run_isolated(a, D, 1, 128)
    if hot == "spare":
        assert out1[-3:].tobytes() == a.syn1[-3:].tobytes()


@pytest.mark.parametrize("niter", [1, 7, 8, 9, 17])
@pytest.mark.parametrize("D", DIMS)
def test_isolated_flush_schedule(D, niter):
    """4 warps in 2 blocks, every node hot, documents of 1, 7, 8, 9 and 17 positions per warp: the shared-memory sums are
    flushed every kI2vFlush iterations and at the last one, whichever comes first, and the last iteration leaves some
    warps without a position."""
    n = next(n for n in range(2, 40) if -(-(3 * n - 2) // 4) == niter)
    a = safe(lambda rng: isolated(D, [2] * n, rng, hot="all"), D)
    assert -(-a.doc.size // 4) == niter and (a.doc.size % 4 != 0 or niter == 1)
    run_isolated(a, D, 2, 64)


@pytest.mark.parametrize("D", DIMS)
def test_isolated_position_range_and_lr_table(D):
    """pos_begin > 0 and pos_end < nd, as ctr_i2v_train_dist segments the document: centres outside the range stay
    untouched, a context outside the range of a centre inside it is updated.  lr_tab has one distinct value per
    4 positions and every centre uses its own."""
    a = safe(lambda rng: isolated(D, [3] * 10, rng, upd=4, hot="split"), D)
    cpos, nd = centre_positions(10)
    a.pos_begin, a.pos_end = cpos[2], cpos[6] + 1            # left context of centre 2 and right context of centre 6 lie outside
    assert len(set(a.lr_tab[[p // 4 for p in cpos[2:7]]].tolist())) >= 4
    out0, out1, want = run_isolated(a, D, 1, 64)
    assert want.counters[0] == 5 and want.counters[1] == 10
    assert cpos[2] - 1 in want.rows and cpos[6] + 1 in want.rows and cpos[1] + 1 not in want.rows
    assert out0[cpos[2] - 1].tobytes() != a.syn0[cpos[2] - 1].tobytes() and out0[cpos[7] - 1].tobytes() == a.syn0[cpos[7] - 1].tobytes()


@pytest.mark.parametrize("D", DIMS)
def test_isolated_subsampling_thresholds_straddle_each_draw(D):
    """z one part in 10^12 above or below the position's own U[0,1) draw, besides z = 0 and z = 1: the three counters
    are exact and only the kept centres train."""
    a = safe(lambda rng: isolated(D, [4] * 12, rng), D)
    cpos, nd = centre_positions(12)
    keep = []
    for j, p in enumerate(cpos):
        u = pm.draw_u(a.seed, a.iter, p)
        a.z[p] = [u + 1e-12, u - 1e-12, 1.0, 0.0][j % 4]
        keep.append(j % 4 in (0, 2))
    want = pm.launch_model(a, "passes", rpw=32 // (D // 4))
    assert want.counters[0] == sum(keep) == 6
    run_isolated(a, D, 1, 256)


def designed(D, targets, rng, hot="none", lr=2.0 ** -5):
    """Inputs whose every f is exact in float32 in any summation order: a left context is 2*e_0, a right context
    2*e_{D-1}, and component 0 (D-1) of the centre's i-th node is half the f wanted there.  targets[j] = (f of the left
    context per node, f of the right context per node)."""
    a = isolated(D, [max(len(l), len(r)) for l, r in targets], rng, hot=hot, lr=lr)
    cpos, nd = centre_positions(len(targets))
    for p, (fl, fr) in zip(cpos, targets):
        for side, col, fs in ((-1, 0, fl), (1, D - 1, fr)):
            if 0 <= p + side < nd:
                a.syn0[p + side] = 0.0; a.syn0[p + side, col] = 2.0
            for i, f in enumerate(fs):
                assert f32(f) == f
                a.syn1[a.pnode[a.poff[p] + i], col] = f32(f) / f32(2.0)
    return a


@pytest.mark.parametrize("hot", ["none", "all"])
@pytest.mark.parametrize("D", DIMS)
def test_isolated_cut_off_at_exactly_six(D, hot):
    """f exactly -6, 6, their float32 neighbours towards zero, and a path that crosses the cut-off half way.  A context
    that is cut stops there (later nodes untouched, node_visits counts only the visited ones) but keeps the tmp it has
    gathered; the other context of the same warp pass carries on.  f = nextafterf(6, 0) is NOT cut and its float32
    table index is 1000: it must read the last entry (the clamp)."""
    up, dn = float(np.nextafter(f32(6), f32(0))), float(np.nextafter(f32(-6), f32(0)))
    targets = [((), (1.0, 6.0, 0.5, 0.5, 0.5)),                                   # right context only: cut at node 1 after one visit
               ((0.5, -6.0, 1.0, 1.0, 1.0), (0.25, 1.5, -2.0, 3.0, 0.75)),        # left cut at node 1, right walks all five
               ((-1.0, 2.0, 0.125, -3.0, 4.0), (up, dn, 6.0, 1.0, 1.0)),          # right: bins 999 and 0, then cut at node 2
               ((1.0, 1.0, 7.5, 1.0, 1.0), (1.0, 1.0, 1.0, -8.0, 1.0)),           # cut at nodes 2 and 3: nodes 3 and 4 take no update
               ((6.0, 1.0, 1.0, 1.0, 1.0), ())]                                   # left context only: cut at the first node, tmp = 0
    a = designed(D, targets, np.random.default_rng(D), hot=hot)
    cpos, nd = centre_positions(5)
    out0, out1, want = run_isolated(a, D, 1, 256, exact_f=True)
    assert want.counters == [5, 8, 1 + (1 + 5) + (5 + 2) + (2 + 3) + 0]
    nodes = lambda j: a.pnode[a.poff[cpos[j]]:a.poff[cpos[j] + 1]]
    assert out1[nodes(3)[3:]].tobytes() == a.syn1[nodes(3)[3:]].tobytes() and out1[nodes(4)].tobytes() == a.syn1[nodes(4)].tobytes()
    assert out0[cpos[4] - 1].tobytes() == a.syn0[cpos[4] - 1].tobytes()            # cut at once: tmp = 0
    assert np.abs(out0[cpos[0] + 1] - a.syn0[cpos[0] + 1]).max() > 1e-3            # cut later: the tmp gathered so far arrives
    lut = pm.sigmoid_lut(True)
    assert pm.lut_bin(up, True) == 999 and int((f32(up) + f32(6.0)) * pm._K32) == 1000 and pm.lut_bin(dn, True) == 0
    # the update the clamp decides: node 0 of centre 2 from its right context, g = (1 - code - lut[999]) * lr
    n0 = nodes(2)[0]; code = a.pcode[a.poff[cpos[2]]]
    g = (f32(1.0) - f32(code) - lut[999]) * f32(2.0 ** -5)
    assert abs(float(out1[n0, D - 1]) - (float(a.syn1[n0, D - 1]) + float(g) * 2.0)) <= 2 * np.spacing(f32(3.0))


@pytest.mark.parametrize("D", DIMS)
def test_isolated_table_bins_at_their_edges(D):
    """f two float32 steps below to two above the edges of bins 1, 2, 250, 500, 501, 750, 998 and 999, and inside bins 0
    and 999.  One bin off is 3e-3 of the gradient, a thousand times the tolerance."""
    fs = [float(np.nextafter(f32(-6), f32(0))), float(np.nextafter(f32(6), f32(0)))]
    for b in (1, 2, 250, 500, 501, 750, 998, 999):
        x, hi = f32(-6.0 + 0.012 * b - 1e-3), f32(-6.0 + 0.012 * b + 1e-3)   # bisect to the float32 edge of the kernel's own index expression
        while np.nextafter(x, f32(7)) < hi:
            mid = f32((float(x) + float(hi)) / 2)
            mid = np.nextafter(x, f32(7)) if mid <= x or mid >= hi else mid
            x, hi = (x, mid) if pm.lut_bin(float(mid), True) >= b else (mid, hi)
        lo2 = np.nextafter(x, f32(-7)); hi1 = np.nextafter(x, f32(7)); hi2 = np.nextafter(hi1, f32(7))
        five = [lo2, x, hi1, hi2, np.nextafter(hi2, f32(7))]
        assert [pm.lut_bin(float(v), True) for v in five] == [b - 1, b - 1, b, b, b]
        fs += [float(v) for v in five]
    fs += [0.0] * (48 - len(fs))
    sides = [fs[6 * i:6 * i + 6] for i in range(8)]
    targets = [((), sides[0]), (sides[1], sides[2]), (sides[3], sides[4]), (sides[5], sides[6]), (sides[7], ())]
    a = designed(D, targets, np.random.default_rng(100 + D), lr=2.0 ** -6)
    _, _, want = run_isolated(a, D, 1, 256, exact_f=True)
    assert want.counters == [5, 8, 48]


# ---- tier B: window enumeration and ragged passes ------------------------------------------------------------------
@pytest.mark.parametrize("W", [1, 2, 5, 8, 20])
@pytest.mark.parametrize("D", DIMS)
def test_window_rows_are_exactly_the_models(D, W):
    """del comes from the kernel's own draw (the model repeats it with mix64).  The rows whose bits change are exactly
    [del, 2W+1-del) \\ {W} around each centre, clipped at the ends of the document — with nctx below, at and above a
    multiple of the 32/LPR contexts of a pass.  A centre's nodes take several adds and whether one sees another is not
    specified, so the amounts are compared with both model orders at 1e-3 plus the distance two legal orders can be apart, which is
    second order: at most lr * nctx of the largest increment, plus one step of the sigmoid table (3e-3) where the two
    orders' f fall on either side of a bin edge (lr = 2^-10 keeps float32 rounding of the adds below the 1e-3)."""
    rng = np.random.default_rng(10 * D + W)
    n, gap = 9, 2 * W + 2
    cpos = [2 + gap * j for j in range(n)]
    nd = cpos[-1] + 3                                           # the first and the last window are clipped for W > 2
    ln = np.zeros(nd, np.int64); ln[cpos] = 3
    poff = np.zeros(nd + 1, np.int64); poff[1:] = np.cumsum(ln)
    z = np.zeros(nd); z[cpos] = 1.0
    a = pm.Launch(doc=np.arange(nd, dtype=np.int32), z=z, poff=poff, pnode=rng.permutation(3 * n).astype(np.int32), pcode=rng.integers(0, 2, 3 * n).astype(np.uint8),
                  syn0=rand_table(rng, nd, D, 0.5), syn1=rand_table(rng, 3 * n, D, 0.5), W=W, lr_tab=np.full(1, 2.0 ** -10, f32), upd=nd + 1,
                  seed=int(rng.integers(1, 1 << 31)), iter=int(rng.integers(0, 5)), node_scale=np.ones(3 * n, f32), word_scale=np.ones(nd, f32), hot_base=3 * n, hot_n=0)
    seq, stale = pm.launch_model(a, "sequential"), pm.launch_model(a, "stale")
    dels = {pm.draw_del(a.seed, a.iter, p, W) for p in cpos}
    assert W == 1 or len(dels) > 1
    out0, out1, ctr = probe.skipgram(a, 2, 128)
    assert ctr == seq.counters == stale.counters and ctr[2] == 3 * ctr[1]
    changed = set(np.nonzero((out0.view(u32) != a.syn0.view(u32)).any(axis=1))[0].tolist())
    assert changed == seq.rows, (sorted(changed - seq.rows), sorted(seq.rows - changed))
    assert set(np.nonzero((out1.view(u32) != a.syn1.view(u32)).any(axis=1))[0].tolist()) == seq.nodes
    for out, init, m1, m2 in ((out0, a.syn0, seq.syn0, stale.syn0), (out1, a.syn1, seq.syn1, stale.syn1)):
        inc = out.astype(f64) - init
        i1, i2 = m1 - init, m2 - init
        norm = np.linalg.norm(i1, axis=1)
        between = np.linalg.norm(i1 - i2, axis=1)
        apart = (2.0 ** -10 * 2 * W + 4e-3) * norm.max()
        assert (between <= apart).all()
        assert (np.linalg.norm(inc - i1, axis=1) <= 1e-3 * norm + apart).all() and (np.linalg.norm(inc - i2, axis=1) <= 1e-3 * norm + apart).all()


# ---- tier C: a full grid in the linear regime ----------------------------------------------------------------------
def huffman_node_values(cnt):
    V = cnt.size
    parent, code = orc.i2v_huffman(cnt, True)
    val = np.concatenate([cnt.astype(np.int64), np.zeros(V - 1, np.int64)])
    for i in range(2 * V - 2):                               # children are created before their parent
        val[parent[i]] += val[i]
    return parent, code, val[V:]


def zipf_launch(D, lr, sms=132):
    rng = np.random.default_rng(77)
    V, n = 2000, 200000
    p = 1.0 / np.arange(1, V + 1); p /= p.sum()
    doc = rng.choice(V, n, p=p).astype(np.int32)
    doc[:V] = np.arange(V)                                   # every word occurs
    cnt = np.bincount(doc, minlength=V)
    poff, pnode, pcode = g.i2v_paths(cnt, 100)
    parent, code, node_val = huffman_node_values(cnt)
    rp = pm.paths_from_parent(parent, code, cnt, V, 100)
    assert np.array_equal(rp[0], poff) and np.array_equal(rp[1], pnode) and np.array_equal(rp[2], pcode)
    rpw = 32 // (D // 4)                                     # i2v_train_impl's launch geometry
    warps = max(1, min(sms * 64, (n + 63) // 64, max(1, V // 4 // rpw)))
    grid = (warps + 7) // 8
    zz, ws, ns = probe.tables(cnt, 5.0, float(grid * 8 * rpw), float(n), node_val)
    hot_n = min(K_HOT, V - 1)
    a = pm.Launch(doc=doc, z=zz, poff=poff, pnode=pnode, pcode=pcode, syn0=rng.uniform(-0.5, 0.5, (V, D)).astype(f32),
                  syn1=(0.25 * rng.uniform(-1, 1, (V - 1, D))).astype(f32), W=5, lr_tab=np.linspace(lr, 0.5 * lr, n // 10000 + 2).astype(f32), upd=10000,
                  seed=9, iter=1, node_scale=ns, word_scale=ws, hot_base=V - 1 - hot_n, hot_n=hot_n)
    return a, grid


def linear_gap(a, grid):
    d0, d1, want_ctr = pm.stale_sum(a)
    out0, out1, ctr = probe.skipgram(a, grid, 256)
    assert ctr == want_ctr, (ctr, want_ctr)
    rel, agg = [], []
    for out, init, d in ((out0, a.syn0, d0), (out1, a.syn1, d1)):
        inc = out.astype(f64) - init
        rel.append(float(((np.linalg.norm(inc - d, axis=1) - 1e-7) / np.linalg.norm(d, axis=1).clip(1e-30)).max()))
        agg.append(float(np.linalg.norm(inc - d) / np.linalg.norm(d)))
    return rel, agg, ctr


@pytest.mark.parametrize("D", [4, 16, 128])
def test_full_grid_sums_to_the_stale_model_in_the_linear_regime(D):
    """2*10^5 Zipf tokens over 2000 words, real Huffman paths and staleness scales, 64 hot nodes, the trainer's grid:
    thousands of adds collide on the top of the tree.  At lr = 2^-14 the total increment of both tables equals the sum
    of the updates computed from the initial tables.  Two things keep the two apart and pull in opposite directions: the
    second-order term (updates that did see each other), which shrinks with lr, and the float32 rounding of every
    red.add of a scaled-down step into a table value, which grows as lr shrinks.  Measured on an H100 80GB HBM3 at
    D = 4 / 16 / 128: whole-table gap 0.7 / 0.9 / 2.4 % (syn0) and 0.7 / 0.8 / 1.4 % (syn1), worst single row 6.9 / 3.9 /
    4.8 %; at lr / 4 syn1's gap falls to 0.63 / 0.56 / 0.44 of that (second order dominates there), syn0's rises
    (rounding dominates).  A hot-node flush lost or doubled for good, or a wrong hot_base, is a first-order error on the
    top nodes; the last flush alone is too small a share to show here (test_isolated_flush_schedule pins it)."""
    a, grid = zipf_launch(D, 2.0 ** -14)
    rel, agg, ctr = linear_gap(a, grid)
    a4, _ = zipf_launch(D, 2.0 ** -16)
    rel4, agg4, _ = linear_gap(a4, grid)
    print("D=%d grid=%d counters=%s worst row gap syn0 %.2e syn1 %.2e, whole-table gap %.2e %.2e; at lr/4 %.2e %.2e"
          % (D, grid, ctr, rel[0], rel[1], agg[0], agg[1], agg4[0], agg4[1]))
    assert ctr[0] > 100000 and ctr[1] > 4 * ctr[0] and ctr[2] > 5 * ctr[1]
    assert max(agg) < 0.04 and max(rel) < 0.12, (agg, rel)
    assert agg4[1] < 0.8 * agg[1], (agg, agg4)


# ---- the smaller kernels --------------------------------------------------------------------------------------------
def test_word_tables_and_node_scales_follow_their_formulas():
    cnt = np.array([0, 1, 2, 3, 5, 50, 1000, 10 ** 6, 7], np.uint64)
    node_val = np.array([1, 3, 99, 100, 101, 10 ** 7], np.int64)
    for subsample, ceff, total in ((1e-3, 100.0, 10000.0), (4.0, 2048.0, 1.0e6), (0.5, 1.0, 3.0)):
        z, ws, ns = probe.tables(cnt, subsample, ceff, total, node_val)
        c = cnt.astype(f64)
        with np.errstate(divide="ignore"):
            want_z = np.where(c > 0, np.maximum(0.0, 1.0 - np.sqrt(subsample / c)), 0.0)    # subsample.go:34-38
        assert np.array_equal(z, want_z) and z[0] == 0.0
        assert np.array_equal(ws, (1.0 / np.maximum(1.0, ceff * c / total)).astype(f32))
        assert np.array_equal(ns, (1.0 / np.maximum(1.0, ceff * node_val / total)).astype(f32))
    z, ws, ns = probe.tables(cnt, 4.0, 100.0, 10000.0, node_val)
    assert (z[1:4] == 0.0).all() and z[4] > 0                                     # clamped at 0 up to count 4
    assert ws[5] == 1.0 and ws[6] == f32(0.1) and ns[2] == 1.0 and ns[3] == 1.0 and ns[4] < 1.0   # both sides of ceff*c/total = 1


@pytest.mark.parametrize("max_depth", [2, 5, 100])
def test_paths_kernel_on_combs_zero_counts_and_two_words(max_depth):
    # a comb of 300 leaves, deeper than every max_depth: leaf i hangs off inner node i - 1, which hangs off inner node i
    V = 300
    parent = np.full(2 * V - 1, -1, np.int32); code = np.zeros(2 * V - 1, np.uint8)
    parent[0] = parent[1] = V; code[1] = 1
    for i in range(2, V):
        parent[i] = V + i - 1; parent[V + i - 2] = V + i - 1; code[i] = i % 2; code[V + i - 2] = 1 - i % 2
    cnt = np.ones(V, np.uint64); cnt[[5, 17, 299]] = 0                            # words that never occur have no path
    got = probe.paths(parent, code, cnt, max_depth)
    want = pm.paths_from_parent(parent, code, cnt, V, max_depth)
    assert all(np.array_equal(x, y) for x, y in zip(got, want))
    assert np.diff(got[0]).max() == min(max_depth, V) - 1 and got[0][6] == got[0][5]
    # Huffman trees from counts: the device paths equal the host plan's (ctr_i2v_paths)
    rng = np.random.default_rng(max_depth)
    for cnt in (np.array([3, 9]), 2 ** np.arange(40), np.concatenate([rng.integers(1, 50, 200), np.zeros(7, np.int64)])):
        cnt = cnt.astype(np.int64)
        parent, code = orc.i2v_huffman(cnt, True)
        got = probe.paths(parent, code, cnt.astype(np.uint64), max_depth)
        host = g.i2v_paths(cnt, max_depth)
        assert all(np.array_equal(x, y) for x, y in zip(got, host)), cnt.size
        assert all(np.array_equal(x, y) for x, y in zip(got, pm.paths_from_parent(parent, code, cnt, cnt.size, max_depth)))


# ---- through the public ABI -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("W", [1, 5, 8])
@pytest.mark.parametrize("D", DIMS)
def test_public_trainer_counts_every_pair_and_node_visit(D, W):
    """ctr_i2v_train's own dispatch on D / 4 and launch geometry.  At lr = 1e-6 no f reaches the cut-off, so the three
    counters are determined by the draws: pairs = the model's window count, node visits = the path length of every
    pair's centre, trained positions = the oracle's.  Documents of 1 token and of grid*8 - 1, grid*8 and grid*8 + 1
    (one position per warp, one warp short and one over; the grid is one block for documents this small)."""
    V = 12
    for nd in (1, 7, 8, 9):
        rng = np.random.default_rng(100 * D + 10 * W + nd)
        toks = rng.integers(0, V, nd).astype(np.int32)
        cfg = g.i2v_default_config(dim=D, window=W, iter=1, min_count=0, init_lr=1e-6, min_lr=1e-6, seed=nd + W)
        emb, st = g.i2v_train_ids(toks, V, cfg=cfg)
        cnt = np.bincount(toks, minlength=V)
        poff, pnode, pcode = g.i2v_paths(cnt, cfg.max_depth)
        sub = float(f32(cfg.subsample))
        with np.errstate(divide="ignore"):
            z = np.where(cnt > 0, np.maximum(0.0, 1.0 - np.sqrt(sub / cnt)), 0.0)
        a = pm.Launch(doc=toks, z=z, poff=poff, pnode=pnode, pcode=pcode, syn0=np.zeros((V, D), f32), syn1=np.zeros((V - 1, D), f32), W=W,
                      lr_tab=np.zeros(1, f32), upd=nd + 1, seed=cfg.seed, iter=0)
        P, Cp, trained = pm.launch_pairs(a)
        ocfg = orc.i2v_cfg(dim=D, window=W, iters=1, min_count=0, init_lr=1e-6, subsample=sub, seed=cfg.seed, rng_mode=1)
        assert st.doc_len == nd and st.trained_positions == trained == orc.i2v_train(ocfg, toks, V)[1]
        assert st.pairs == P.size and st.node_visits == int((poff[toks[P] + 1] - poff[toks[P]]).sum())
        assert np.isfinite(emb).all()
