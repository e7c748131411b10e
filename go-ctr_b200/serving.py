"""Host mirror of the serving side of the boundary (SURVEY.md §8f rows f3/f4): recommend.Rank /
recommend.BatchPredict (rcmd.go:248-337) over sample keys, with the id→row maps, the ubcache window and
the forward pass all on the device (ctr_batch_predict_keys).  Names and argument order follow the
reference; `recSys` is an Engine that already holds the tables, both id maps and (optionally) the ubcache.
"""
import time
from dataclasses import dataclass

import numpy as np

from . import engine as _e
from . import model as _m


@dataclass
class Sample:                      # rcmd.go:189-194
    UserId: int
    ItemId: int
    Timestamp: int = 0
    Label: float = 0.0


@dataclass
class ItemScore:                   # rcmd.go:184-187
    ItemId: int
    Score: float


def BatchPredict(recSys, sampleKeys):
    """rcmd.go:277-337.  Returns float32 [n, 1] like the tensor the reference hands back.  An unknown
    user/item in key 0 raises (CtrError code ENOTFOUND), in later keys it scores as a zero X row.  Over an MLP fitted
    on labels other than 0 / 1 the scores are predicted labels."""
    if len(sampleKeys) == 0:
        raise ValueError("no sample keys")
    u = np.fromiter((s.UserId for s in sampleKeys), np.int64, len(sampleKeys))
    i = np.fromiter((s.ItemId for s in sampleKeys), np.int64, len(sampleKeys))
    t = np.fromiter((s.Timestamp for s in sampleKeys), np.int64, len(sampleKeys))
    return recSys.batch_predict_keys(u, i, t).reshape(-1, 1)


def Rank(recSys, userId, itemIds, now=None):
    """rcmd.go:248-275: score `itemIds` for one user at the current time; order is the caller's."""
    ts = int(time.time()) if now is None else int(now)
    y = BatchPredict(recSys, [Sample(userId, it, ts) for it in itemIds])
    return [ItemScore(int(it), float(y[k, 0])) for k, it in enumerate(itemIds)]


def Recommend(recSys, userId, k, now=None, exclude_history=True, exclude_seen=False):
    """What recommend/api.go's empty-itemIdList branch would return (api.go:115-118, "todo: some default recall
    algorithm"): the k best items of the whole table for one user at the current time, best first, as [ItemScore].
    Every ITEM_EMB row is scored with the trained model (ctr_recommend_topk); the user's history is windowed from the
    device ubcache at `now` (empty without one, as in BatchPredict); exclude_history drops the items of that window, and
    exclude_seen (implies exclude_history) every item of the user's ubcache events up to `now`: nothing the user has
    already consumed is recommended.  On a row-sharded ITEM_EMB each row's seen verdict comes from the cache of the rank
    that owns it, so keep the same behaviour cache on every rank (Engine.recommend_topk).
    An unknown user raises CtrError with code ENOTFOUND, as BatchPredict does for an unresolvable first key.
    On an engine whose ITEM_EMB is row-sharded over several GPUs the call is collective: every rank's process makes
    the same call (same user, k, now and history) and receives the same complete result (Engine.recommend_topk).
    A sharded deployment must pass `now` explicitly, the value broadcast with the request: the default reads each
    process's own clock, so ranks can window different histories and then all fail with CTR_EINVAL.
    recSys may also be the SimpleMlpPredWrap that SimpleMlpFitWrap.FitKeys returns, main.go's model: its MLP scores
    every ITEM_EMB row of the feature store it is bound to (ctr_mlp_recommend_topk), under the same rules.  An MLP
    fitted on labels other than 0 / 1 predicts labels, not click probabilities, and raises CtrError with code ESTATE."""
    ts = int(time.time()) if now is None else int(now)
    if isinstance(recSys, _m.SimpleMlpPredWrap):
        rows, scores, _ = recSys.recommend(userId, k, now=ts, exclude_history=exclude_history, exclude_seen=exclude_seen)
        item_ids = recSys.engine.item_ids
        return [ItemScore(int(item_ids[r]), float(s)) for r, s in zip(rows, scores)]
    row = int(recSys.idmap_lookup(_e.IDMAP_USER, [int(userId)])[0])
    if row < 0:
        raise _e.CtrError(_e.ENOTFOUND, "user %d is not found" % int(userId))
    try:
        hist = recSys.ubcache_window([row], [ts])
    except _e.CtrError as err:          # ESTATE: no ubcache uploaded
        if err.code != _e.ESTATE:
            raise
        hist = np.full((1, recSys.cfg.S), -1, np.int32)
    rows, scores, _, cnt = recSys.recommend_topk([row], hist, k, exclude_history=exclude_history, max_ts=ts, exclude_seen=exclude_seen)
    item_ids = recSys.item_ids
    return [ItemScore(int(item_ids[rows[0, i]]), float(scores[0, i])) for i in range(int(cnt[0]))]


def Evaluate(recSys, heldOut, ks=(10,), exclude_history=True, exclude_seen=False):
    """Offline full-catalogue evaluation of Recommend: each held-out Sample's ItemId is ranked against every ITEM_EMB row
    for its UserId, with the history windowed at its Timestamp (the window cut), exactly as Recommend(userId, k,
    now=Timestamp, exclude_history) would list it (Engine.rank_items / _Mlp64.rank_items).  Samples are grouped by
    (UserId, Timestamp).  Returns {"HR@k", "Recall@k", "NDCG@k" for every k in ks, "MRR"} (engine.rank_metrics); an
    item the model can never list — unknown to the item map, in an excluded window, a NaN logit — is a miss.
    recSys is an Engine or a SimpleMlpPredWrap, as for Recommend.  An unknown user raises CtrError with code ENOTFOUND.
    On an Engine with a row-sharded ITEM_EMB, Evaluate is collective (Engine.rank_items): every rank passes the same
    held-out samples and returns the same metrics.  The ranks' windows and item rows must agree too, so every rank needs
    the same id maps and behaviour cache; a rank whose rows differ makes the call raise CtrError EINVAL on every rank.
    exclude_seen (implies exclude_history) is the filtered protocol: every item of the user's ubcache events with ts <=
    the sample's Timestamp is removed from the catalogue it is ranked against (and ranks -1 itself), so no event after
    the cut is excluded.  On a row-sharded ITEM_EMB it follows the owner rule (Engine.recommend_topk): with the same
    behaviour cache on every rank, the metrics equal one GPU's."""
    if len(heldOut) == 0:
        raise ValueError("no held-out samples")
    u = np.fromiter((s.UserId for s in heldOut), np.int64, len(heldOut))
    i = np.fromiter((s.ItemId for s in heldOut), np.int64, len(heldOut))
    t = np.fromiter((s.Timestamp for s in heldOut), np.int64, len(heldOut))
    if isinstance(recSys, _m.SimpleMlpPredWrap):
        recSys._bound()
        ranks, _ = recSys.pred.rank_items(recSys.engine, u, i, t, exclude_history=exclude_history, exclude_seen=exclude_seen)
    else:
        rows = recSys.idmap_lookup(_e.IDMAP_USER, u)
        if (rows < 0).any():
            raise _e.CtrError(_e.ENOTFOUND, "user %d is not found" % int(u[int(np.flatnonzero(rows < 0)[0])]))
        try:
            hist = recSys.ubcache_window(rows, t)
        except _e.CtrError as err:          # ESTATE: no ubcache uploaded
            if err.code != _e.ESTATE:
                raise
            hist = np.full((u.size, recSys.cfg.S), -1, np.int32)
        items = recSys.idmap_lookup(_e.IDMAP_ITEM, i)
        ranks, _ = recSys.rank_items(rows, hist, items, exclude_history=exclude_history, max_ts=t, exclude_seen=exclude_seen)
    _, groups = np.unique(np.stack([u, t], axis=1), axis=0, return_inverse=True)
    ks = [int(k) for k in ks]
    hit, recall, ndcg, mrr = _e.rank_metrics(ranks, groups.ravel(), ks)
    out = {}
    for a, k in enumerate(ks):
        out["HR@%d" % k] = float(hit[a]); out["Recall@%d" % k] = float(recall[a]); out["NDCG@%d" % k] = float(ndcg[a])
    out["MRR"] = float(mrr)
    return out


class UserBehaviorCache:
    """feature/ubcache's UserBehaviorCache (cache.go:16-55) over the engine's device ubcache, keyed by external ids
    through the engine's id maps (load_id_maps).  Every change is applied in HBM, so the next Rank / BatchPredict /
    Recommend / train_keys sees it.  An item id the item map does not hold is stored as row -1 and reads as a zero row
    in its history slot, as in the reference.  Sequences are TimeSeq's: timestamps descending."""

    def __init__(self, engine):
        self.e = engine

    def _user_rows(self, user_ids):
        return self.e.idmap_lookup(_e.IDMAP_USER, np.asarray(user_ids, np.int64))

    def _item_rows(self, item_ids):
        item_ids = np.asarray(item_ids, np.int64)
        return self.e.idmap_lookup(_e.IDMAP_ITEM, item_ids) if item_ids.size else np.zeros(0, np.int32)

    def Set(self, userId, ts, itemIds):
        """cache.go:28-33: replace one user's whole sequence."""
        self.BatchSet({userId: (ts, itemIds)})

    def BatchSet(self, ub):
        """cache.go:36-41: replace the sequences of every user in {userId: (ts, itemIds)}.  A user id the user map does
        not hold raises CtrError(ENOTFOUND) before anything changes."""
        if not ub:
            return
        users = list(ub)
        rows = self._user_rows(users)
        if (rows < 0).any():
            raise _e.CtrError(_e.ENOTFOUND, "user %d is not found" % int(users[int(np.flatnonzero(rows < 0)[0])]))
        ts = [np.asarray(ub[u][0], np.int64).ravel() for u in users]
        items = [np.asarray(ub[u][1], np.int64).ravel() for u in users]
        if any(t.size != i.size for t, i in zip(ts, items)):
            raise ValueError("every sequence needs one timestamp per item")
        off = np.concatenate([[0], np.cumsum([t.size for t in ts])]).astype(np.int64)
        all_ts = np.concatenate(ts) if ts else np.zeros(0, np.int64)
        self.e.ubcache_set(rows, off, all_ts, self._item_rows(np.concatenate(items)))

    def Delete(self, userId):
        """cache.go:44-48: the user's history becomes empty.  Like Go's delete, an unknown user is a no-op."""
        row = int(self._user_rows([userId])[0])
        if row >= 0:
            self.e.ubcache_set([row], [0, 0], np.zeros(0, np.int64), np.zeros(0, np.int32))

    def Clear(self):
        """cache.go:51-55: every user's history becomes empty (an upload of an empty cache)."""
        self.e.ubcache_upload([0, 0], np.zeros(0, np.int64), np.zeros(0, np.int32))

    def Append(self, userIds, itemIds, ts):
        """Online learning's write path: append events (userIds[i] clicked itemIds[i] at ts[i]) to their users'
        sequences.  Among equal timestamps the latest arrival comes first.  Events of user ids the user map does not
        hold are dropped; returns how many."""
        u = np.asarray(userIds, np.int64).ravel(); it = np.asarray(itemIds, np.int64).ravel(); t = np.asarray(ts, np.int64).ravel()
        if not u.size == it.size == t.size:
            raise ValueError("userIds, itemIds and ts must have one entry per event")
        if u.size == 0:
            return 0
        rows = self._user_rows(u)
        keep = rows >= 0
        if keep.any():
            self.e.ubcache_append(rows[keep], t[keep], self._item_rows(it[keep]))
        return int((~keep).sum())


class FeatureCache:
    """The Set of UserFeatureCache / ItemFeatureCache (rcmd.go:25-26, 34-35) over the engine's live id maps and tables: a
    user or item that was not there when the engine was set up gets a row and its features in HBM, so the next Rank /
    BatchPredict / Recommend / train_keys sees it.  Setting a known id overwrites its row."""

    def __init__(self, engine):
        self.e = engine

    def SetUser(self, userId, feature):
        """The user's USER_FEAT row (uP floats); returns its row."""
        row = self.e.idmap_insert(_e.IDMAP_USER, [int(userId)])
        self.e.table_write_rows(_e.TABLE_USER_FEAT, row, np.asarray(feature, np.float32).reshape(1, -1))
        return int(row[0])

    def SetItem(self, itemId, feature, embedding=None):
        """The item's ITEM_FEAT row (cF floats) and, when given, its ITEM_EMB row (D floats).  Without one a new item's
        embedding reads as zeros until the next item2vec run, the reference's "embedding not found" (rcmd.go:501-505).
        Returns its row."""
        row = self.e.idmap_insert(_e.IDMAP_ITEM, [int(itemId)])
        if self.e.cfg.cF > 0:
            self.e.table_write_rows(_e.TABLE_ITEM_FEAT, row, np.asarray(feature, np.float32).reshape(1, -1))
        if embedding is not None:
            self.e.table_write_rows(_e.TABLE_ITEM_EMB, row, np.asarray(embedding, np.float32).reshape(1, -1))
        return int(row[0])


def load_id_maps(recSys, user_ids, item_ids):
    """user_ids[r] / item_ids[r] = external id of table row r (what the Go side's string-keyed caches hold,
    rcmd.go:472-505).  The item ids stay on the engine (item_ids) to map Recommend's rows back to ids."""
    recSys.idmap_build(_e.IDMAP_USER, user_ids)
    recSys.idmap_build(_e.IDMAP_ITEM, item_ids)
    recSys.item_ids = np.array(item_ids, np.int64)
