"""A numpy model of ctr_item_emb_train's numbering over the ranks' streams (world > 1), step for step as the device runs
it, and the rule it must meet: dictionary.Add (dictionary.go:70-81) over the ranks' streams concatenated in rank order.

  1. every rank resolves its own stream through the (shared) item map and tags each row's first position in it as
     (rank << 32) | position, NEVER when its stream lacks the row's id; the tags meet in a min all-reduce;
  2. every rank lists its distinct unmapped ("side") ids with their first positions; the lists are all-gathered, and
     every rank keeps the smallest tag of each id;
  3. rows and side words sorted by tag: the rank in that order is the word id;
  4. each rank's document takes the word of each of its tokens."""
import numpy as np

NEVER = np.uint64(0xFFFFFFFFFFFFFFFF)


def tag(rank, pos):
    return (np.uint64(rank) << np.uint64(32)) | np.asarray(pos, np.uint64)


def rows_of(stream, imap):
    """the map's row of every token, -1 without an entry (INT64_MIN is never a key)"""
    row = {int(v): r for r, v in enumerate(imap)}
    return np.array([row.get(int(v), -1) for v in stream], np.int64)


def rank_local(stream, rank, imap):
    """steps 1 and 2 on one rank: (row tags [R], side ids ascending, their first positions)"""
    R = len(imap)
    rows = rows_of(stream, imap)
    first = np.full(R, -1, np.int64)
    for p in range(len(stream) - 1, -1, -1):
        if rows[p] >= 0:
            first[rows[p]] = p
    tags = np.where(first >= 0, tag(rank, np.maximum(first, 0)), NEVER)
    side = np.asarray(stream, np.int64)[rows < 0]
    pos = np.nonzero(rows < 0)[0]
    ids, at = np.unique(side.view(np.uint64), return_index=True)   # ascending as uint64, the first position of each
    return tags.astype(np.uint64), ids, pos[at]


def numbering(streams, imap):
    """The whole rule over the ranks' streams: (vocab_ids, word_of_row, side_ids, word_of_side, docs)."""
    W = len(streams)
    loc = [rank_local(s, r, imap) for r, s in enumerate(streams)]
    row_tag = np.minimum.reduce([l[0] for l in loc]) if len(imap) else np.zeros(0, np.uint64)
    g_ids = np.concatenate([l[1] for l in loc])
    g_tag = np.concatenate([tag(r, loc[r][2]) for r in range(W)])
    side_ids = np.unique(g_ids)
    side_tag = np.array([g_tag[g_ids == v].min() for v in side_ids], np.uint64)
    key = np.concatenate([row_tag, side_tag])
    val = np.concatenate([np.arange(len(imap)), -1 - np.arange(side_ids.size)])
    order = np.argsort(key, kind="stable")
    V = int((key != NEVER).sum())
    word_of_row = np.full(len(imap), -1, np.int64)
    word_of_side = np.empty(side_ids.size, np.int64)
    vocab = np.empty(V, np.int64)
    for w in range(V):
        v = val[order[w]]
        if v >= 0:
            word_of_row[v] = w; vocab[w] = imap[v]
        else:
            word_of_side[-v - 1] = w; vocab[w] = side_ids[-v - 1].view(np.int64)
    docs = []
    for s in streams:
        rows = rows_of(s, imap)
        d = np.empty(len(s), np.int64)
        for p, v in enumerate(s):
            d[p] = word_of_row[rows[p]] if rows[p] >= 0 else word_of_side[np.searchsorted(side_ids, np.int64(v).view(np.uint64))]
        docs.append(d)
    return vocab, word_of_row, side_ids.view(np.int64), word_of_side, docs


def dictionary_add(stream):
    """dictionary.Add over one stream: (vocab_ids in word order, the word of every token)"""
    word, vocab, doc = {}, [], []
    for v in stream:
        v = int(v)
        if v not in word:
            word[v] = len(vocab); vocab.append(v)
        doc.append(word[v])
    return np.array(vocab, np.int64), np.array(doc, np.int64)


def split(stream, cuts):
    """the stream cut at the sorted positions cuts into len(cuts) + 1 shards (empty shards where cuts repeat)"""
    b = [0] + list(cuts) + [len(stream)]
    return [np.asarray(stream[b[i]:b[i + 1]], np.int64) for i in range(len(b) - 1)]
