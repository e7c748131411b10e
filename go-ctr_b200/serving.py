"""Host mirror of the serving side of the boundary (SURVEY.md §8f rows f3/f4): recommend.Rank /
recommend.BatchPredict (rcmd.go:248-337) over sample keys, with the id→row maps, the ubcache window and
the forward pass all on the device (ctr_batch_predict_keys).  Names and argument order follow the
reference; `recSys` is an Engine that already holds the tables, both id maps and (optionally) the ubcache.
"""
import time
from dataclasses import dataclass

import numpy as np

from . import engine as _e


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
    user/item in key 0 raises (CtrError code ENOTFOUND), in later keys it scores as a zero X row."""
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


def Recommend(recSys, userId, k, now=None, exclude_history=True):
    """What recommend/api.go's empty-itemIdList branch would return (api.go:115-118, "todo: some default recall
    algorithm"): the k best items of the whole table for one user at the current time, best first, as [ItemScore].
    Every ITEM_EMB row is scored with the trained model (ctr_recommend_topk); the user's history is windowed from the
    device ubcache at `now` (empty without one, as in BatchPredict); exclude_history drops the items of that window.
    An unknown user raises CtrError with code ENOTFOUND, as BatchPredict does for an unresolvable first key."""
    ts = int(time.time()) if now is None else int(now)
    row = int(recSys.idmap_lookup(_e.IDMAP_USER, [int(userId)])[0])
    if row < 0:
        raise _e.CtrError(_e.ENOTFOUND, "user %d is not found" % int(userId))
    try:
        hist = recSys.ubcache_window([row], [ts])
    except _e.CtrError as err:          # ESTATE: no ubcache uploaded
        if err.code != _e.ESTATE:
            raise
        hist = np.full((1, recSys.cfg.S), -1, np.int32)
    rows, scores, _, cnt = recSys.recommend_topk([row], hist, k, exclude_history=exclude_history)
    item_ids = recSys.item_ids
    return [ItemScore(int(item_ids[rows[0, i]]), float(scores[0, i])) for i in range(int(cnt[0]))]


def load_id_maps(recSys, user_ids, item_ids):
    """user_ids[r] / item_ids[r] = external id of table row r (what the Go side's string-keyed caches hold,
    rcmd.go:472-505).  The item ids stay on the engine (item_ids) to map Recommend's rows back to ids."""
    recSys.idmap_build(_e.IDMAP_USER, user_ids)
    recSys.idmap_build(_e.IDMAP_ITEM, item_ids)
    recSys.item_ids = np.array(item_ids, np.int64)
