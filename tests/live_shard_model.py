"""A numpy restatement of the live id maps and table writes on a multi-GPU handle (ctr_idmap_insert and
ctr_table_write_rows with world > 1).  The rule: after a call, every rank holds what one GPU would hold after the same call
on the concatenation of the ranks' arguments in rank order.

SingleMap / SingleTable restate the single-GPU semantics test_gpu_live_tables.py pins (first-occurrence numbering, the
rehash capacity, growth with zero gaps, row-Adam moments zeroed only for written rows).  insert_ranks and ShardedTable
restate how the ranks get there: each rank numbers its own missing ids, the lists are merged by (rank, position); each
written row goes to its owner row % world, a hot row (below hot_k) to every rank's replica as well, and a shard that
outgrows its allocation is reallocated at max(new local rows, 2 x old local rows)."""
import numpy as np

INT64_MIN = -2**63
INT32_MAX = 2**31 - 1


class Refused(Exception):
    """the call is CTR_EINVAL on every rank and changes nothing"""


def idmap_capacity(n):
    cap = 64
    while cap < 2 * n:
        cap <<= 1
    return cap


class SingleMap:
    """ctr_idmap_insert on one GPU: ids the map lacks get rows n, n + 1, ... by first occurrence."""

    def __init__(self):
        self.row = {}
        self.cap = 0                                   # slots of the device table (0: no map)

    def insert(self, ids):
        ids = [int(v) for v in np.asarray(ids, np.int64)]
        if INT64_MIN in ids:
            raise Refused("INT64_MIN")
        fresh = list(dict.fromkeys(v for v in ids if v not in self.row))
        if len(self.row) + len(fresh) > INT32_MAX:
            raise Refused("rows")
        for v in fresh:
            self.row[v] = len(self.row)
        if fresh:
            self.cap = max(self.cap, idmap_capacity(len(self.row)))
        return np.array([self.row[v] for v in ids], np.int32)

    def ids(self):
        out = np.empty(len(self.row), np.int64)
        for v, r in self.row.items():
            out[r] = v
        return out


def number(row, ids):
    """One rank's numbering: its distinct missing ids ascending as uint64, with the first position of each."""
    first = {}
    for p, v in enumerate(np.asarray(ids, np.int64).tolist()):
        if v not in row and v not in first:
            first[v] = p
    keys = sorted(first, key=lambda v: v & (2**64 - 1))
    return np.array(keys, np.int64), np.array([first[v] for v in keys], np.int32)


def merge(lists):
    """The rank merge: every (id, rank, position), the smallest (rank, position) per id, ordered by it."""
    best = {}
    for j, (ids, pos) in enumerate(lists):
        for v, p in zip(ids.tolist(), pos.tolist()):
            best[v] = min(best.get(v, (j, p)), (j, p))
    return np.array(sorted(best, key=lambda v: best[v]), np.int64)


def insert_ranks(m, per_rank):
    """The collective insert on rank maps that all equal m (a SingleMap, updated): each rank's rows of its own ids."""
    per_rank = [np.asarray(a, np.int64) for a in per_rank]
    if any(INT64_MIN in a.tolist() for a in per_rank):
        raise Refused("INT64_MIN")
    fresh = merge([number(m.row, a) for a in per_rank])
    if len(m.row) + fresh.size > INT32_MAX:
        raise Refused("rows")
    for v in fresh.tolist():
        m.row[v] = len(m.row)
    if fresh.size:
        m.cap = max(m.cap, idmap_capacity(len(m.row)))
    return [np.array([m.row[v] for v in a.tolist()], np.int32) for a in per_rank]


def check_rows(rows):
    rows = np.asarray(rows, np.int64)
    if rows.size and (rows.min() < 0 or rows.max() >= INT32_MAX):
        raise Refused("range")
    if np.unique(rows).size != rows.size:
        raise Refused("duplicate")


class SingleTable:
    """ctr_table_write_rows on one GPU: rows written bit for bit, a row past the end grows the table with zero rows in
    between, written rows' row-Adam moments zeroed (adam: the table is ITEM_EMB with moments)."""

    def __init__(self, tab, adam=False):
        self.t = np.array(tab, np.float32)
        self.m = np.ones_like(self.t) if adam else None          # stand-ins for moments the solver has filled
        self.v = np.ones_like(self.t) if adam else None

    def write(self, rows, data):
        rows = np.asarray(rows, np.int64)
        check_rows(rows)
        top = int(rows.max()) + 1 if rows.size else 0
        if top > self.t.shape[0]:
            pad = np.zeros((top - self.t.shape[0], self.t.shape[1]), np.float32)
            self.t = np.concatenate([self.t, pad])
            if self.m is not None:
                self.m = np.concatenate([self.m, pad]); self.v = np.concatenate([self.v, pad])
        self.t[rows] = data
        if self.m is not None:
            self.m[rows] = 0; self.v[rows] = 0


def local_rows(nrows, world, rank):
    return (nrows - rank + world - 1) // world


def shard_capacity(cap, old, want):
    """rows a shard holds after growing from `old` live rows (allocation of `cap` rows) to `want` (before the allocation
    granule rounds it up)"""
    return cap if want <= cap else max(want, 2 * old)


class ShardedTable:
    """The same table row-sharded over `world` ranks: shard r holds rows r, r + W, ...; rows [0, hot_k) also live in every
    rank's replica (hot = None: no live replica)."""

    def __init__(self, tab, world, hot_k=0, adam=False):
        tab = np.array(tab, np.float32)
        self.W, self.n = world, tab.shape[0]
        self.shard = [tab[r::world].copy() for r in range(world)]
        self.cap = [s.shape[0] for s in self.shard]
        self.m = [np.ones_like(s) for s in self.shard] if adam else None
        self.v = [np.ones_like(s) for s in self.shard] if adam else None
        self.hot_k = hot_k
        self.hot = [tab[:hot_k].copy() for _ in range(world)] if hot_k else None
        self.hm = [np.ones_like(tab[:hot_k]) for _ in range(world)] if hot_k and adam else None
        self.hv = [np.ones_like(tab[:hot_k]) for _ in range(world)] if hot_k and adam else None
        self.reallocs = 0

    def route(self, per_rank):
        """what each rank receives: its own rows, and every hot row"""
        got = [([], []) for _ in range(self.W)]
        for rows, data in per_rank:
            for r, d in zip(np.asarray(rows, np.int64).tolist(), np.asarray(data, np.float32)):
                for k in range(self.W):
                    if r % self.W == k or r < self.hot_k:
                        got[k][0].append(r); got[k][1].append(d)
        return got

    def write(self, per_rank):
        check_rows(np.concatenate([np.asarray(r, np.int64) for r, _ in per_rank]))
        top = max([int(np.max(r)) + 1 for r, _ in per_rank if len(r)] + [0])
        if top > self.n:
            # the hot rows return to their shards, the shards grow, and the replica is rebuilt on the next republish
            if self.hot is not None:
                for h in range(self.hot_k):
                    self.shard[h % self.W][h // self.W] = self.hot[0][h]
                    if self.m is not None:
                        self.m[h % self.W][h // self.W] = self.hm[0][h]; self.v[h % self.W][h // self.W] = self.hv[0][h]
                self.hot = self.hm = self.hv = None
            for r in range(self.W):
                old, want = self.shard[r].shape[0], local_rows(top, self.W, r)
                cap = shard_capacity(self.cap[r], old, want)
                self.reallocs += cap != self.cap[r]
                self.cap[r] = cap
                pad = np.zeros((want - old, self.shard[r].shape[1]), np.float32)
                self.shard[r] = np.concatenate([self.shard[r], pad])
                if self.m is not None:
                    self.m[r] = np.concatenate([self.m[r], pad]); self.v[r] = np.concatenate([self.v[r], pad])
            self.n = top
        for k, (rows, data) in enumerate(self.route(per_rank)):
            for r, d in zip(rows, data):
                if r % self.W == k:
                    self.shard[k][r // self.W] = d
                    if self.m is not None:
                        self.m[k][r // self.W] = 0; self.v[k][r // self.W] = 0
                if self.hot is not None and r < self.hot_k:
                    self.hot[k][r] = d
                    if self.hm is not None:
                        self.hm[k][r] = 0; self.hv[k][r] = 0

    def assembled(self, which="t"):
        """the logical table (hot rows from the replica while it is live), or its moments"""
        src = {"t": self.shard, "m": self.m, "v": self.v}[which]
        out = np.zeros((self.n, self.shard[0].shape[1]), np.float32)
        for r in range(self.W):
            out[r::self.W] = src[r]
        rep = {"t": self.hot, "m": self.hm, "v": self.hv}[which]
        if rep is not None:
            out[:self.hot_k] = rep[0]
        return out
