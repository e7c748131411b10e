"""Plain reference of the item2vec update (SkipGram + hierarchical softmax) that judges the parallel kernel
k_i2v_skipgram_hs (go-ctr_b200/csrc/item2vec.cuh): float64 numpy and Python integers, no device code.

Cites are relative to the reference's feature/embedding directory, as in oracle/i2v_oracle.c:
    skipGram.trainOne          model/word2vec/model.go:48-78      the window [del, 2W+1-del) \\ {W} around a centre
    hierarchicalSoftmax.optim  model/word2vec/optimizer.go:107-129 the walk down the centre's Huffman path
    sigmoid table              model/word2vec/sigmoid_table.go:28-45
    Subsampler.Trial           subsample.go:45-52
With both scales absent and float64 f the sequential order reproduces oracle/i2v_oracle.c bit for bit
(tests/test_i2v_pair_model_cpu.py); that is what entitles it to judge the kernel."""
from dataclasses import dataclass
from typing import Optional

import numpy as np

from oracle import oracle as orc

_M = (1 << 64) - 1
_K32 = np.float32(1000.0) / np.float32(6.0) / np.float32(2.0)          # the kernel's 1000.0f / 6.0f / 2.0f


def mix64(seed, stream, ctr):
    """The counter RNG of common.cuh / ctr_oracle.c on Python integers."""
    z = ((((seed & 0xFFFFFFFF) << 32) | (stream & 0xFFFFFFFF)) * 0x9E3779B97F4A7C15 + ctr * 0xD1B54A32D192ED03 + 0x632BE59BD9B4E019) & _M
    z ^= z >> 30; z = (z * 0xBF58476D1CE4E5B9) & _M
    z ^= z >> 27; z = (z * 0x94D049BB133111EB) & _M
    return z ^ (z >> 31)


def draw_u(seed, it, pos):
    """Subsampler.Trial's U[0,1): the position trains when z[word] > u."""
    return (mix64(seed, 200 + it, pos) >> 11) * (1.0 / 9007199254740992.0)


def draw_del(seed, it, pos, W):
    """modelutil.NextRandom(window): the window shrinks by del on both sides."""
    return mix64(seed, 300 + it, pos) % W


def sigmoid_lut(f32=False):
    """The 1000-entry table: orc_i2v_sigmoid_lut read at every bin's centre; float32-rounded for the parallel kernel."""
    L = orc.lib()
    t = np.array([L.orc_i2v_sigmoid_lut((i + 0.5) * 0.012 - 6.0) for i in range(1000)], np.float64)
    return t.astype(np.float32) if f32 else t


def lut_bin(f, f32):
    """optimizer.go:121's table index.  f32: the kernel's float32 expression, clamped to the last entry (in float32
    f = nextafterf(6, 0) gives (f + 6) * (1000 / 12) == 1000.0f)."""
    if f32:
        return min(int((np.float32(f) + np.float32(6.0)) * _K32), 999)
    return int((f + 6.0) * (1000.0 / 6.0 / 2.0))


def _edge_margin(f, c, nv):
    """Distance from f to the nearest table-bin edge (the +-6 cut-off is edge 0 and edge 1000), less a bound on what a
    float32 dot product in any summation order can differ from f.  Positive: every order lands in the same bin."""
    t = (f + 6.0) * (1000.0 / 12.0)
    d = abs(f) - 6.0 if abs(f) >= 6.0 else min(t - np.floor(t), np.ceil(t) - t) * 0.012
    return d - 2.0 ** -21 * float(np.abs(c * nv).sum())


def pair_update(c, path_nodes, path_codes, syn1, lr, lut, read=None, node_scale=None, f32=False):
    """optimizer.go:113-128 for one (centre, context) pair.  c: the context row as read; syn1 takes nv += g*c (times
    node_scale[node] when given); read: where nv is read from (default syn1 itself: every node sees all earlier
    updates).  f32=True is the parallel kernel's specification: f rounded to float32 before the cut-off and the table
    index, g, the step g*nv and the addends rounded as float32 operations; the tables stay float64 sums of them.
    Returns (tmp, nodes visited, the smallest bin-edge margin of any f on the path)."""
    src = syn1 if read is None else read
    margin = np.inf
    visits = 0
    if f32:
        c32 = c.astype(np.float32); tmp = np.zeros(c.size, np.float32)
    else:
        tmp = np.zeros(c.size, np.float64)
    cl = c.tolist()
    for node, code in zip(path_nodes, path_codes):
        node = int(node)
        nv = np.array(src[node], np.float64)
        f = 0.0
        for x, y in zip(cl, nv.tolist()):                   # element order, products and sums rounded separately
            f += x * y
        margin = min(margin, _edge_margin(f, c, nv))
        if f32:
            f = float(np.float32(f))
        if f <= -6.0 or f >= 6.0:                            # `return`: the rest of the path is abandoned
            break
        if f32:
            g = (np.float32(1.0) - np.float32(code) - lut[lut_bin(f, True)]) * np.float32(lr)
            tmp = (float(g) * nv + tmp.astype(np.float64)).astype(np.float32)             # fmaf(g, nv, tmp)
            gs = g * np.float32(node_scale[node]) if node_scale is not None else g
            syn1[node] += (gs * c32).astype(np.float64)
        else:
            g = (1.0 - float(code) - lut[lut_bin(f, False)]) * lr
            tmp += g * nv
            syn1[node] += (g * float(node_scale[node]) if node_scale is not None else g) * c
        visits += 1
    return tmp, visits, margin


@dataclass
class Launch:
    """Every field of the kernel's I2vArgs, as host arrays."""
    doc: np.ndarray
    z: np.ndarray
    poff: np.ndarray
    pnode: np.ndarray
    pcode: np.ndarray
    syn0: np.ndarray
    syn1: np.ndarray
    W: int
    lr_tab: np.ndarray
    upd: int
    seed: int = 0
    iter: int = 0
    node_scale: Optional[np.ndarray] = None
    word_scale: Optional[np.ndarray] = None
    hot_base: int = 1 << 30
    hot_n: int = 0
    pos_begin: int = 0
    pos_end: int = -1

    def __post_init__(self):
        if self.pos_end < 0:
            self.pos_end = len(self.doc)


@dataclass
class Result:
    syn0: np.ndarray          # float64
    syn1: np.ndarray
    rows: set                 # context rows that took an add
    nodes: set                # inner nodes that took an add
    counters: list            # trained positions, (centre, context) pairs, node visits
    margin: float             # smallest bin-edge margin of any f (see _edge_margin)


def contexts(pos, dl, W, nd):
    """model.go:59-77: [(k, cpos)] of a centre; k counts the slots of [del, 2W+1-del) \\ {W}, inside the document or not,
    which is the kernel's context index (32/LPR of them per pass)."""
    out = []; k = 0
    for aa in range(dl, 2 * W + 1 - dl):
        if aa == W:
            continue
        cpos = pos - W + aa
        if 0 <= cpos < nd:
            out.append((k, cpos))
        k += 1
    return out


def launch_model(a, order, f32=True, rpw=1):
    """Every trained position of [pos_begin, pos_end), in position order.
        "sequential"  each pair sees all earlier updates (the reference as one goroutine runs it)
        "stale"       every pair reads the launch's initial tables, the updates are summed (the linear regime)
        "passes"      the kernel's own schedule for inputs where centres share no vector: the rpw contexts of one warp
                      pass read the same node vectors, the next pass of that centre reads them updated; nodes at or
                      above hot_base are read as the launch found them (their updates wait in shared memory)"""
    assert order in ("sequential", "stale", "passes")
    doc = np.asarray(a.doc); nd = doc.size
    syn0 = np.array(a.syn0, np.float64); syn1 = np.array(a.syn1, np.float64)
    init0, init1 = syn0.copy(), syn1.copy()
    lut = sigmoid_lut(f32)
    rows, nodes, counters, margin = set(), set(), [0, 0, 0], np.inf
    for pos in range(a.pos_begin, a.pos_end):
        wid = int(doc[pos])
        if not a.z[wid] > draw_u(a.seed, a.iter, pos):
            continue
        counters[0] += 1
        dl = draw_del(a.seed, a.iter, pos, a.W)
        lr = a.lr_tab[pos // a.upd]
        lr = float(lr) if not f32 else np.float32(lr)
        pn = a.pnode[a.poff[wid]:a.poff[wid + 1]]; pc = a.pcode[a.poff[wid]:a.poff[wid + 1]]
        ctx = contexts(pos, dl, a.W, nd)
        groups = {}
        for k, cpos in ctx:
            groups.setdefault(k // rpw if order == "passes" else k, []).append(cpos)
        for _, cps in sorted(groups.items()):
            if order == "stale":
                read = init1
            elif order == "passes":
                read = {int(n): (init1[n] if n >= a.hot_base else syn1[n].copy()) for n in pn}
            else:
                read = None
            cs = [(init0 if order == "stale" else syn0)[doc[cp]].copy() for cp in cps]
            for cp, c in zip(cps, cs):
                cid = int(doc[cp])
                if order == "sequential":
                    c = syn0[cid].copy()
                tmp, visits, m = pair_update(c, pn, pc, syn1, lr, lut, read=read, node_scale=a.node_scale, f32=f32)
                if f32:
                    add = tmp * np.float32(a.word_scale[cid]) if a.word_scale is not None else tmp
                    syn0[cid] += add.astype(np.float64)
                elif order == "sequential" and a.word_scale is None:
                    syn0[cid] = c + tmp                                           # ctx[k] += tmp[k], model.go:74-76
                else:
                    syn0[cid] += tmp * (float(a.word_scale[cid]) if a.word_scale is not None else 1.0)
                counters[1] += 1; counters[2] += visits; margin = min(margin, m)
                rows.add(cid); nodes.update(int(n) for n in pn[:visits])
    return Result(syn0, syn1, rows, nodes, counters, margin)


def _mix64_np(seed, stream, ctr):
    with np.errstate(over="ignore"):
        z = np.uint64((((seed & 0xFFFFFFFF) << 32) | (stream & 0xFFFFFFFF)) * 0x9E3779B97F4A7C15 & _M) + ctr.astype(np.uint64) * np.uint64(0xD1B54A32D192ED03) \
            + np.uint64(0x632BE59BD9B4E019)
        z ^= z >> np.uint64(30); z *= np.uint64(0xBF58476D1CE4E5B9)
        z ^= z >> np.uint64(27); z *= np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def launch_pairs(a):
    """The (centre position, context position) pairs of a launch as arrays, and the number of trained positions."""
    doc = np.asarray(a.doc); nd = doc.size
    pos = np.arange(a.pos_begin, a.pos_end, dtype=np.int64)
    u = (_mix64_np(a.seed, 200 + a.iter, pos) >> np.uint64(11)).astype(np.float64) * (1.0 / 9007199254740992.0)
    train = np.asarray(a.z)[doc[pos]] > u
    dl = (_mix64_np(a.seed, 300 + a.iter, pos) % np.uint64(a.W)).astype(np.int64)
    P, Cp = [], []
    for aa in range(2 * a.W + 1):
        if aa == a.W:
            continue
        cpos = pos - a.W + aa
        m = train & (aa >= dl) & (aa < 2 * a.W + 1 - dl) & (cpos >= 0) & (cpos < nd)
        P.append(pos[m]); Cp.append(cpos[m])
    return np.concatenate(P), np.concatenate(Cp), int(train.sum())


def stale_sum(a):
    """launch_model(a, "stale", f32=False) without the Python loop, for documents of 10^5 tokens: every f comes from
    one matrix product of the initial tables.  Refuses a launch in which any pair would be cut off.
    Returns (syn0 increment, syn1 increment, counters)."""
    doc = np.asarray(a.doc); poff = np.asarray(a.poff, np.int64); pnode = np.asarray(a.pnode); pcode = np.asarray(a.pcode)
    s0 = np.array(a.syn0, np.float64); s1 = np.array(a.syn1, np.float64)
    V, nn = s0.shape[0], s1.shape[0]
    F = s0 @ s1.T
    lut = sigmoid_lut(True).astype(np.float64)
    P, Cp, trained = launch_pairs(a)
    wid = doc[P]; cid = doc[Cp].astype(np.int64)
    ln = poff[wid + 1] - poff[wid]
    lr = np.asarray(a.lr_tab, np.float64)[P // a.upd]
    M = np.zeros(nn * V, np.float64)
    visits = 0
    for i in range(int(ln.max()) if ln.size else 0):
        sel = ln > i
        node = pnode[poff[wid[sel]] + i].astype(np.int64); code = pcode[poff[wid[sel]] + i].astype(np.float64)
        f = F[cid[sel], node]
        if np.any(np.abs(f) >= 5.99):
            raise ValueError("a pair reaches the cut-off: not the linear regime")
        b = np.minimum(((f.astype(np.float32) + np.float32(6.0)) * _K32).astype(np.int64), 999)
        M += np.bincount(node * V + cid[sel], weights=(1.0 - code - lut[b]) * lr[sel], minlength=nn * V)
        visits += int(sel.sum())
    M = M.reshape(nn, V)
    ns = np.ones(nn) if a.node_scale is None else np.asarray(a.node_scale, np.float64)
    ws = np.ones(V) if a.word_scale is None else np.asarray(a.word_scale, np.float64)
    return ws[:, None] * (M.T @ s1), ns[:, None] * (M @ s0), [trained, int(P.size), visits]


def paths_from_parent(parent, code, cnt, V, max_depth):
    """Node.GetPath(maxDepth) (node.go:26-43) as optimizer.go:113-115 walks it: the first min(maxDepth, len) - 1 inner
    nodes from the root, each with the code of the child the path takes.  Words that never occur have no path."""
    poff = [0]; pn = []; pc = []
    for w in range(V):
        if cnt[w] > 0:
            chain = []
            p = w
            while p != -1:
                chain.append(p); p = int(parent[p])
            chain = chain[::-1]                              # root .. leaf
            for i in range(min(max_depth, len(chain)) - 1):
                pn.append(chain[i] - V); pc.append(int(code[chain[i + 1]]))
        poff.append(len(pn))
    return np.array(poff, np.int64), np.array(pn, np.int32), np.array(pc, np.uint8)
