"""Semantic model of CTR_TABLE_ADAM on the row-sharded placement (test infrastructure; go-ctr_b200/csrc/comm_impl.cuh,
attn.cuh k_shard_adam / k_hot_adam), built on the data movement of tests/shard_model.py.  Every lookup's gradient
(scaled by 1/world) goes home to the owner's fp32 gradient shard and marks its row touched by occurrence; after a barrier
each owner applies one row-Adam update per touched row and clears the shard.  Rows [0, hot_k) are replicated: their
gradient sums and touch marks are all-reduced, every rank updates its replica and the replicated moments identically.
On the GPUs the gradient return is a red.add over NVLink and the touch an atomic on the owner's flag; here both are
all-to-alls over gloo (tests/test_shard_adam_gloo.py)."""
import numpy as np

from tests.shard_model import _all_to_all, plan_exchange


def valid_lookups(hist, item_row, n_rows, nvalid):
    """[B, S+1] global row of each lookup, -1 where the slot is not valid (id -1, id past the table, sample >= nvalid)."""
    rows = np.concatenate([np.asarray(hist), np.asarray(item_row)[:, None]], axis=1).astype(np.int64)
    rows = np.where((rows >= 0) & (rows < n_rows), rows, -1)
    rows[nvalid:] = -1
    return rows


def row_adam(w, m, v, g, t, lr, b1, b2, eps, inv_batch):
    """row_adam_elem (attn.cuh) in float32, in place on the rows given: the dense solver's step with counter t."""
    f = np.float32
    c1, c2 = f(1.0 - b1 ** t), f(1.0 - b2 ** t)
    g = g.astype(f) * f(inv_batch)
    m[...] = f(b1) * m + (f(1.0) - f(b1)) * g
    v[...] = f(b2) * v + (f(1.0) - f(b2)) * g * g
    w[...] = w - f(lr) * (m / c1) / (np.sqrt(v / c2) + f(eps))


def adam_step_sharded(dist, torch, st, rank, world, lookups, grads, hot_k, t, lr, b1, b2, eps, inv_batch):
    """One sharded row-Adam step of this rank.  st: dict with the owner's 'shard', 'm', 'v' (local rows) and the
    replicas 'hot', 'hot_m', 'hot_v' ([hot_k, D]); lookups [B, S+1] from valid_lookups; grads [B, S+1, D] the per-lookup
    row gradients of this rank (unscaled)."""
    D = st["shard"].shape[1]
    flat = lookups.reshape(-1); g = grads.reshape(-1, D).astype(np.float32) * np.float32(1.0 / world)
    cold = flat >= hot_k
    # owner leg: ids of cold lookups and their gradients go home; the owner sums them into its gradient shard
    hist_like = np.where(cold, flat, -1).reshape(1, -1)
    send_rows, scnt, slot = plan_exchange(hist_like[:, :-1], hist_like[:, -1], world)
    slot = slot.reshape(-1)
    send_g = np.zeros((send_rows.size, D), np.float32)
    send_g[slot[slot >= 0]] = g[slot >= 0]
    rcnt_t = torch.empty(world, dtype=torch.int64)
    dist.all_to_all_single(rcnt_t, torch.from_numpy(scnt))
    rcnt = rcnt_t.numpy()
    recv_rows = _all_to_all(dist, torch, send_rows, scnt, rcnt)
    recv_g = _all_to_all(dist, torch, send_g, scnt, rcnt)
    gshard = np.zeros_like(st["shard"]); touched = np.zeros(st["shard"].shape[0], bool)
    np.add.at(gshard, recv_rows, recv_g)
    touched[recv_rows] = True                              # by occurrence: a zero gradient sum still counts
    tr = np.nonzero(touched)[0]
    w, m, v = st["shard"][tr], st["m"][tr], st["v"][tr]
    row_adam(w, m, v, gshard[tr], t, lr, b1, b2, eps, inv_batch)
    st["shard"][tr], st["m"][tr], st["v"][tr] = w, m, v
    # hot leg: local sums and touch marks, all-reduced; the identical update on every replica
    if hot_k > 0:
        hsum = np.zeros((hot_k, D + 1), np.float32)
        hot = (flat >= 0) & ~cold
        np.add.at(hsum[:, :D], flat[hot], g[hot])
        hsum[flat[hot], D] = 1.0
        ht = torch.from_numpy(hsum)
        dist.all_reduce(ht)
        hsum = ht.numpy()
        hr = np.nonzero(hsum[:, D] > 0)[0]
        w, m, v = st["hot"][hr], st["hot_m"][hr], st["hot_v"][hr]
        row_adam(w, m, v, hsum[hr, :D], t, lr, b1, b2, eps, inv_batch)
        st["hot"][hr], st["hot_m"][hr], st["hot_v"][hr] = w, m, v
    return st


def assemble_sharded(st_by_rank, world, hot_k):
    """The table and both moments as one GPU would hold them: shards interleaved, the hot rows from a replica
    (comm_hot_writeback)."""
    n = sum(s["shard"].shape[0] for s in st_by_rank)
    out = {}
    for k, hk in (("shard", "hot"), ("m", "hot_m"), ("v", "hot_v")):
        a = np.zeros((n, st_by_rank[0][k].shape[1]), np.float32)
        for r in range(world):
            a[r::world] = st_by_rank[r][k]
        if hot_k > 0:
            a[:hot_k] = st_by_rank[0][hk]
        out[k] = a
    return out
