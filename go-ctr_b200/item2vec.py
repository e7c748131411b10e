"""Host-side mirror of feature/embedding for the device trainer (include/ctr_b200.h ctr_i2v_train).

    embedding.TrainEmbedding(inputCh, window, dim, iter)        wordemb.go:9-32
    model.GenEmbeddingMap32() map[string][]float32              word2vec.go:298-324

    vector.Save(f, dic, mat, ...)  word2vec text format           model/modelutil/vector/vector.go:40-67
    emb.Load(r) / parse / parseLine → []Embedding{Word,Dim,Vector,Norm}   emb/embedding.go:73-131

    search.New(embs...) / SearchInternal / SearchVector → Neighbors        search/search.go:53-134

The channel carries one WORD per message (cpsutil.ReadWord, cpsutil.go:46-53); ids are assigned by first
appearance (dictionary.Add, dictionary.go:70-81)."""
import ctypes as C

import numpy as np

from . import engine as _e

__all__ = ["i2v_paths", "I2vConfig", "I2vStats", "i2v_default_config", "i2v_train_ids", "i2v_train_dist", "TrainEmbedding", "EmbeddingModel",
           "item_ids_from_seq", "TrainItemEmbedding",
           "Embedding", "SaveVectors", "LoadVectors", "ParseLine", "Neighbor", "Searcher", "neighbors_from_result"]


class I2vConfig(C.Structure):
    _fields_ = [("dim", C.c_int32), ("window", C.c_int32), ("iter", C.c_int32), ("min_count", C.c_int32), ("max_depth", C.c_int32),
                ("init_lr", C.c_float), ("min_lr", C.c_float), ("subsample", C.c_float), ("update_lr_batch", C.c_int32),
                ("seed", C.c_uint32), ("device", C.c_int32), ("reserved", C.c_int32 * 8)]


class I2vStats(C.Structure):
    _fields_ = [("doc_len", C.c_int64), ("trained_positions", C.c_int64), ("pairs", C.c_int64), ("node_visits", C.c_int64),
                ("algorithmic_bytes", C.c_double), ("ms_device", C.c_float), ("launches", C.c_int32)]


def i2v_default_config(**kw):
    cfg = I2vConfig()
    _e.load_library().ctr_i2v_config_default(C.byref(cfg))
    for k, v in kw.items():
        if not hasattr(cfg, k):
            raise AttributeError(k)
        setattr(cfg, k, v)
    return cfg


def i2v_paths(count, max_depth=100):
    """Host-side Huffman paths of the trainer (no GPU needed): returns (path_off [V+1], nodes, codes)."""
    L = _e.load_library()
    cnt = np.ascontiguousarray(count, np.int64); V = cnt.size
    cap = V * min(max_depth, 64) + 64
    off = np.empty(V + 1, np.int64); nodes = np.empty(cap, np.int32); codes = np.empty(cap, np.uint8)
    rc = L.ctr_i2v_paths(cnt.ctypes.data_as(C.POINTER(C.c_int64)), C.c_int32(V), C.c_int32(max_depth), off.ctypes.data_as(C.POINTER(C.c_int64)),
                         nodes.ctypes.data_as(C.POINTER(C.c_int32)), codes.ctypes.data_as(C.POINTER(C.c_uint8)), C.c_int64(cap))
    if rc != 0:
        raise _e.CtrError(rc, L.ctr_last_error(None).decode())
    return off, nodes[:off[-1]], codes[:off[-1]]


def i2v_train_ids(tokens, vocab, cfg=None, **kw):
    """tokens: int32 word ids in corpus order.  Returns (emb [vocab, dim] float32, I2vStats)."""
    L = _e.load_library()
    cfg = cfg or i2v_default_config(**kw)
    tok = np.ascontiguousarray(tokens, np.int32)
    emb = np.empty((vocab, cfg.dim), np.float32)
    st = I2vStats()
    rc = L.ctr_i2v_train(C.byref(cfg), tok.ctypes.data_as(C.POINTER(C.c_int32)), C.c_int64(tok.size), C.c_int32(vocab),
                         emb.ctypes.data_as(C.POINTER(C.c_float)), C.byref(st))
    if rc != 0:
        raise _e.CtrError(rc, L.ctr_last_error(None).decode())
    return emb, st


def i2v_train_dist(tokens_shard, vocab, rank, world, nccl_id, sync_every=0, cfg=None, want_table=True, **kw):
    """One rank of the multi-GPU trainer (ctr_i2v_train_dist): this rank's shard of the stream in, the averaged table out
    (want_table=False: this rank skips the copy of the table to the host and returns None for it)."""
    L = _e.load_library()
    cfg = cfg or i2v_default_config(**kw)
    tok = np.ascontiguousarray(tokens_shard, np.int32)
    emb = np.empty((vocab, cfg.dim), np.float32) if want_table else None
    st = I2vStats()
    rc = L.ctr_i2v_train_dist(C.byref(cfg), tok.ctypes.data_as(C.POINTER(C.c_int32)), C.c_int64(tok.size), C.c_int32(vocab),
                              emb.ctypes.data_as(C.POINTER(C.c_float)) if want_table else None, C.byref(st), C.c_int32(rank), C.c_int32(world),
                              C.c_char_p(nccl_id), C.c_int32(len(nccl_id)), C.c_int64(sync_every))
    if rc != 0:
        raise _e.CtrError(rc, L.ctr_last_error(None).decode())
    return emb, st


class EmbeddingModel:
    def __init__(self, id2word, emb, stats):
        self.id2word, self.emb, self.stats = id2word, emb, stats

    def GenEmbeddingMap32(self):
        if len(self.id2word) == 0:
            raise ValueError("dictionary is empty")                          # word2vec.go:305-308
        return {w: self.emb[i] for i, w in enumerate(self.id2word)}


def TrainEmbedding(inputCh, window, dim, iter, **kw):
    """inputCh: iterable of words (item ids as strings)."""
    word2id, id2word, toks = {}, [], []
    for w in inputCh:
        i = word2id.get(w)
        if i is None:
            i = word2id[w] = len(id2word); id2word.append(w)
        toks.append(i)
    emb, st = i2v_train_ids(np.asarray(toks, np.int32), len(id2word), window=window, dim=dim, iter=iter, **kw)
    return EmbeddingModel(id2word, emb, st)


_I64_MIN, _I64_MAX = -(1 << 63), (1 << 63) - 1


def item_ids_from_seq(itemSeq):
    """The int64 item stream of ItemSeqGenerator's messages: ints, or the decimal strings it sends (fmt.Sprintf("%d")).
    A string that is not the canonical decimal of its value ("007", "+7", " 7") is another word in the reference and
    raises ValueError rather than merging with the int's word; so does a value outside int64."""
    out = []
    for w in itemSeq:
        if isinstance(w, str):
            try:
                v = int(w)
            except ValueError:
                raise ValueError("item %r is not a decimal item id" % (w,)) from None
            if str(v) != w:
                raise ValueError("item %r is not the canonical decimal of %d: it would be a different word" % (w, v))
        elif isinstance(w, (int, np.integer)) and not isinstance(w, (bool, np.bool_)):
            v = int(w)
        else:
            raise ValueError("item %r is neither an int nor a decimal string" % (w,))
        if not _I64_MIN <= v <= _I64_MAX:
            raise ValueError("item id %d is outside int64" % v)
        out.append(v)
    return np.asarray(out, np.int64)


def TrainItemEmbedding(engine, itemSeq, window=5, iter=1, **kw):
    """GetItemEmbeddingModelFromUb (rcmd.go:538-545) + GenEmbeddingMap32 into engine's ITEM_EMB (ctr_item_emb_train):
    embedding.TrainEmbedding(itemSeq, window, D, iter) with dim = the engine's D.  Row r of ITEM_EMB becomes the vector
    of the item the engine's item map sends to r, zeros for an item the stream never holds.  Returns (vocab_ids, I2vStats):
    the item id of every word in word-id order (first appearance).  On a multi-GPU engine (world > 1) every rank's
    process calls it with its own part of the item sequence, possibly empty: words are numbered over the ranks' parts
    concatenated in rank order, so vocab_ids is the same on every rank, each rank trains its part with the replicas
    averaged (sync_every=, Engine.item_emb_train), and each rank writes the ITEM_EMB rows it holds."""
    return engine.item_emb_train(item_ids_from_seq(itemSeq), window=window, iter=iter, **kw)


# ---- the word2vec text format the reference saves / loads its vectors in -------------------------------------
class Embedding:
    """emb.Embedding (emb/embedding.go:27-32): Word, Dim, Vector (float64), Norm = sqrt(sum v^2) (embutil.Norm)."""

    def __init__(self, Word, Vector):
        self.Word = Word
        self.Vector = np.asarray(Vector, np.float64)
        self.Dim = int(self.Vector.size)
        n = 0.0
        for v in self.Vector:                      # embutil/embutil.go: sequential float64 sum
            n += float(v) * float(v)
        self.Norm = float(np.sqrt(n))

    def Validate(self):                            # embedding.go:34-43
        if self.Word == "":
            raise ValueError("word must not be empty")
        if self.Dim == 0:
            raise ValueError("Dim of %s is zero" % self.Word)

    def __eq__(self, o):
        return (self.Word, self.Dim, self.Norm) == (o.Word, o.Dim, o.Norm) and np.array_equal(self.Vector, o.Vector)


def ParseLine(line):
    """emb.parseLine (embedding.go:107-131): whitespace-separated fields, the first is the word."""
    fields = line.split()
    if len(fields) < 2:
        raise ValueError("Must be over 2 lenghth for word and vector elems")
    return Embedding(fields[0], [float(x) for x in fields[1:]])


def LoadVectors(r):
    """emb.Load (embedding.go:73-105): one embedding per line; lines that START WITH A SPACE are skipped; every vector
    must be non-empty.  r: iterable of lines, a file object, or one string."""
    lines = r.splitlines() if isinstance(r, str) else r
    out = []
    for line in lines:
        line = line.rstrip("\r\n")
        if line.startswith(" "):
            continue
        e = ParseLine(line)
        e.Validate()
        out.append(e)
    if out and any(e.Dim != out[0].Dim for e in out):      # Embeddings.Validate, :61-71
        raise ValueError("dimension for all vectors must be the same")
    return out


def SaveVectors(f, words, mat):
    """vector.Save (vector.go:40-67): per word `word ` then every element as `%f ` (six decimals, trailing space), newline."""
    mat = np.asarray(mat)
    if len(words) != mat.shape[0]:
        raise ValueError("different for length of dic and row of matrix: %d, %d" % (len(words), mat.shape[0]))
    for w, row in zip(words, mat):
        f.write("%s " % w + "".join("%f " % float(v) for v in row) + "\n")


# ---- search.Searcher: top-k cosine neighbours, scanned on the device (ctr_knn_search) ---------------------------
class Neighbor:
    """search.Neighbor (search.go:27-32); compares by value like the reference's reflect.DeepEqual."""
    __slots__ = ("Word", "Rank", "Similarity")

    def __init__(self, Word, Rank, Similarity):
        self.Word, self.Rank, self.Similarity = Word, int(Rank), float(Similarity)

    def __eq__(self, o):
        return isinstance(o, Neighbor) and (self.Word, self.Rank, self.Similarity) == (o.Word, o.Rank, o.Similarity)

    def __repr__(self):
        return "Neighbor(%r, %d, %r)" % (self.Word, self.Rank, self.Similarity)


def neighbors_from_result(words, rows, sims, count, k):
    """One query's device result (rows, sims, true count) as the reference's Neighbors list.  When fewer than k items
    qualify, search.go:126-133 sets k to the index of the LAST empty slot, i.e. k-1, and returns neighbors[:k-1]:
    the qualifying items followed by zero Neighbor{} values, k-1 entries in all.  This mirror keeps that shape."""
    out = [Neighbor(words[int(rows[i])], i + 1, float(sims[i])) for i in range(int(count))]
    if count < k:
        out += [Neighbor("", 0, 0.0) for _ in range(k - 1 - int(count))]
    return out


class Searcher:
    """search.Searcher (search.go:53-134) over an ITEM_EMB table in HBM.  Similarities are bit-identical to search.go
    run on the table's float32 values widened to float64; vectors loaded from text are rounded to float32 when
    uploaded, so on those inputs parity holds up to that rounding.  Equal similarities rank by row ascending.
    On an engine whose ITEM_EMB is row-sharded over several GPUs every search is collective: every rank's process
    makes the same call and receives the same complete result (Engine.knn_search)."""

    def __init__(self, engine, words, vectors=None):
        self.engine, self.words = engine, list(words)
        self.rows = {}
        for i, w in enumerate(self.words):
            if w in self.rows:                 # item2vec dictionaries never repeat a word; Search would ignore both
                raise ValueError("duplicate word %r in searcher" % w)
            self.rows[w] = i
        self.vectors = vectors                 # float64 [N, dim] of New(); None for a live table (from_engine)

    @classmethod
    def New(cls, *embs):
        """search.New(embs...): validates (equal dims, emb.Embeddings.Validate), then uploads the vectors as float32
        ITEM_EMB into an engine with D = dim and no feature tables."""
        if embs and any(e.Dim != embs[0].Dim for e in embs):
            raise ValueError("dimension for all vectors must be the same: %d" % embs[0].Dim)
        if not embs:
            raise ValueError("searcher needs at least one embedding")
        dim = embs[0].Dim
        vec = np.stack([e.Vector for e in embs]).astype(np.float64)
        eng = _e.Engine(_e.default_config(_e.MODEL_DIN_COS, uP=0, cF=0, S=1, D=dim, batch=1, pred_batch=1))
        eng.table_upload(_e.TABLE_ITEM_EMB, vec.astype(np.float32))
        return cls(eng, [e.Word for e in embs], vec)

    @classmethod
    def from_engine(cls, eng, words):
        """Searches eng's live ITEM_EMB (row i is words[i]) without copying it; SearchInternal then queries by row."""
        return cls(eng, words)

    def SearchInternal(self, word, k):
        row = self.rows.get(word)
        if row is None:
            raise ValueError("%s is not found in searcher" % word)         # search.go:75-77
        if self.vectors is not None:           # the word's own float64 vector, its row excluded (search.go:79)
            r, s, c = self.engine.knn_search(k, queries=self.vectors[row:row + 1], rows=[row])
        else:
            r, s, c = self.engine.knn_search(k, rows=[row])
        return neighbors_from_result(self.words, r[0], s[0], c[0], k)

    def SearchVector(self, query, k):
        r, s, c = self.engine.knn_search(k, queries=np.asarray(query, np.float64).reshape(1, -1))
        return neighbors_from_result(self.words, r[0], s[0], c[0], k)
