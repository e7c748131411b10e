/*
 * ctr_b200.h — C ABI of libctr_b200.so: the H100 (sm_90a) engine behind go-ctr's CTR hot path.
 *
 * This is the drop-in boundary.  Every entry point replaces one Go-side interface of the reference
 * (auxten/go-ctr @ c181363c; file:line relative to the repository root) and is exactly what a cgo
 * shim binds (see INTEGRATION.md and go/ctrb200/ctrb200.go).  Plain pointers and sizes only — no
 * torch / C++ types.  The caller owns every host buffer; the library copies and never retains a
 * caller pointer after return (cgo pointer-passing rule).  Every function returns 0 on success or a
 * CTR_E* code; the message is available from ctr_last_error().  Nothing aborts or exits.
 * There is no CPU fallback: without a CUDA device ctr_create fails with CTR_ENODEV.
 *
 * Layouts: all matrices row-major float32; indices int32 dense row ids (the id→row map stays on
 * the Go side where the reference keeps it, rcmd.go:472-505); -1 = missing row → zeros
 * (rcmd.go:502-505,519).
 */
#ifndef CTR_B200_H
#define CTR_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CTR_B200_ABI_VERSION 1

enum { CTR_OK = 0, CTR_EINVAL = 1, CTR_ENODEV = 2, CTR_ECUDA = 3, CTR_ENOMEM = 4, CTR_ESTATE = 5, CTR_ECOMM = 6, CTR_ENOTFOUND = 7, CTR_EIO = 8 };

/* which graph: model/youtube/dnn.go:162-184 | model/din/din.go:219-323 (cosine, live) |
 * din.go:230 + model/activation.go:23-50 (euclidean ActivationUnit variant) */
enum { CTR_MODEL_YOUTUBE = 0, CTR_MODEL_DIN_COS = 1, CTR_MODEL_DIN_EUC = 2 };

enum { CTR_TABLE_USER_FEAT = 0, CTR_TABLE_ITEM_FEAT = 1, CTR_TABLE_ITEM_EMB = 2 };

/* embedding-table optimiser.  FROZEN is the reference's behaviour (embeddings are inputs, not
 * learnables: din.go:161-169).  SGD fuses gradient scatter-add + update into the backward kernel
 * with red.global.add.v4.f32 (order-nondeterministic, Hogwild within a batch like the reference's
 * own item2vec trainer).  SGD_DETERMINISTIC sorts (row, sample, slot) keys and reduces each row's
 * segment in a fixed order — the parity-test mode.  ADAM applies the dense solver's update (model.go:88: Adam, step
 * table_lr, cfg betas / eps, gradient divided by the batch size first, no L2) once per DISTINCT row of the batch with
 * that row's summed gradient (sorted keys → segment reduction, deterministic); rows the batch did not touch keep their
 * moments ("lazy" Adam).  The moments are part of the checkpoint.  Every placement: one GPU, a replicated table, or a
 * row-sharded ITEM_EMB under world > 1.  On a row-sharded table a step of `world` ranks x batch B applies the update one
 * GPU with batch world*B applies to the whole table, with the replicated placement's scaling (row gradients scaled by
 * 1/world, Adam batch world*B, the dense step counter t): every distinct row that occurs in a valid slot (a history or
 * target id inside the table, in a sample below nvalid) of any rank's batch gets exactly one update with its gradient
 * summed over all ranks, also when that sum is exactly 0 (the row counts as touched by occurrence: its moments decay
 * and its weights move); untouched rows keep their weights and both moments bit for bit.  Each owner keeps, beside its
 * shard, an fp32 gradient shard plus a touched flag and a list slot per local row that the peers add into over NVLink:
 * 4*D + 8 bytes per local row, in addition to the 8*D bytes of the two moment shards.  The hot rows replicated on every
 * rank (reserved[0]) carry their two moments on every rank too.  The sums use red.add in arbitrary order: results are
 * not bitwise reproducible run to run (the sharded SGD step is not either). */
enum { CTR_TABLE_FROZEN = 0, CTR_TABLE_SGD = 1, CTR_TABLE_SGD_DETERMINISTIC = 2, CTR_TABLE_ADAM = 3 };

/* dense-layer GEMM engine: exact fp32 FFMA, or wgmma 3xTF32 (error-compensated, fp32 accumulate
 * in registers).  AUTO = wgmma when the shape qualifies. */
enum { CTR_GEMM_AUTO = 0, CTR_GEMM_FP32 = 1, CTR_GEMM_TCGEN05_3XTF32 = 2 };

typedef struct ctr_handle ctr_handle;

/* Hyper-parameters the reference hard-codes, as runtime fields (SURVEY.md §5 "Config / flags").
 * ctr_config_default() fills the reference's values. */
typedef struct {
    int32_t model;            /* CTR_MODEL_* */
    int32_t uP;               /* uProfileDim            model.go:27 */
    int32_t S;                /* uBehaviorSize          rcmd.go:24  (10) */
    int32_t D;                /* uBehaviorDim == iFeatureDim (din.go:176-178)  rcmd.go:22 (16) */
    int32_t cF;               /* cFeatureDim */
    int32_t H0, H1;           /* din.go:17-18 (200, 80) */
    int32_t batch;            /* model.Train batchSize */
    int32_t pred_batch;       /* model.InitForwardOnlyVm batchSize (model.go:215) */
    float   lr, l2, beta1, beta2, eps;   /* model.go:88: 0.01, 1e-4; gorgonia Adam defaults .9 .999 1e-8 */
    float   dropout0, dropout1;          /* din.go:204-205 (.005) / dnn.go:136-137 (.003) */
    uint32_t seed;            /* dropout-mask / weight-init counter RNG seed */
    int32_t table_opt;        /* CTR_TABLE_* */
    float   table_lr;         /* SGD step for embedding rows (engine extension) */
    int32_t gemm;             /* CTR_GEMM_* */
    int32_t device;           /* CUDA device ordinal */
    int32_t rank, world;      /* one handle (process) per GPU; large ITEM_* tables are row-sharded (owner(row) = row % world, world in
                                 {2,4,8}: peers read / update the owner's HBM over NVLink), small ones replicated */
    int32_t reserved[8];      /* tuning knobs, 0 = automatic: [0] hot rows (ids [0, n): keep rows ordered by popularity) with replica
                                 accumulators — and, on row-sharded tables, a replica on every rank (< 0: none; default 32768);
                                 [1] ITEM_EMB / ITEM_FEAT placement under world > 1: 1 = always shard, 2 = always replicate
                                 (default: replicate tables <= 32 MB, shard larger ones) */
} ctr_config;

typedef struct {
    float   cost;             /* BCE mean of this batch (model/cost.go:9-17) */
    float   ms_device;        /* device time of the step (CUDA events on the engine stream); 0 if not measured */
    int32_t launches;         /* kernels launched by the step */
    int32_t reserved;
} ctr_step_stats;

int  ctr_abi_version(void);
void ctr_config_default(ctr_config* cfg, int model);

/* din.NewDinNet / youtube.NewYoutubeDnn (din.go:171, dnn.go:119) — allocates device state. */
int  ctr_create(const ctr_config* cfg, ctr_handle** out);
void ctr_destroy(ctr_handle* h);
/* last error message of this handle (or of the last failed ctr_create when h == NULL) */
const char* ctr_last_error(const ctr_handle* h);

/* G.WithInit(G.Gaussian(0,1)) for mlp0/1/2 and ValuesOf(1) for att0 (din.go:181-191) with the
 * engine's counter RNG (streams 0,1,2) — the reference's draws are time-seeded, never reproducible. */
int ctr_init_weights(ctr_handle* h, uint32_t seed);
/* DinNet.Marshal / NewDinNetFromJson field layout (din.go:41-52, dnn.go:38-47): mlp0 [in,H0],
 * mlp1 [H0,H1], mlp2 [H1,1], att0 [1,S] row-major; att0 may be NULL for YouTube.  set also resets
 * the Adam moments and step counter (a fresh solver is built per model.Train call, model.go:88). */
int ctr_set_weights(ctr_handle* h, const float* mlp0, const float* mlp1, const float* mlp2, const float* att0);
int ctr_get_weights(ctr_handle* h, float* mlp0, float* mlp1, float* mlp2, float* att0);

/* Feature / embedding tables resident in HBM: replaces UserFeatureCache / ItemFeatureCache /
 * itemEmbeddingMap (rcmd.go:30-36, 473-505).  rows is [nrows, width] row-major.  With world > 1,
 * ITEM_EMB upload takes the FULL table on every rank and keeps rows r % world == rank — or all of them when the
 * table is small enough to be replicated (<= 32 MB, see ctr_config.reserved[1]); download mirrors that (a sharded
 * table's download fills this rank's rows only).  ITEM_FEAT follows the same rule; USER_FEAT is always replicated.
 * Row ids the entry points receive are range-checked on the device: an id outside [0, rows) reads as a missing row. */
int ctr_table_upload(ctr_handle* h, int which, const float* rows, int64_t nrows, int32_t width);
int ctr_table_download(ctr_handle* h, int which, float* rows, int64_t nrows, int32_t width);
/* Synthetic table generated on the device with the counter RNG (benchmarks with 10M-100M rows,
 * BASELINE.json configs[2..3]): element (r, c) of the FULL table = scale * draw(seed, stream=which,
 * ctr=r*width+c), dist 0 = U[0,1), 1 = N(0,1) (Box-Muller) — identical on every rank / shard. */
int ctr_table_fill(ctr_handle* h, int which, int64_t nrows, int32_t width, uint32_t seed, int32_t dist, float scale);

/* recommend.GetSampleVector for a batch (rcmd.go:462-536): X[b] = [user_feat | emb[hist[b,0..S)] |
 * emb[item] | item_feat], bit-exact copies.  X is [B, uP + S*D + D + cF]. */
int ctr_gather_rows(ctr_handle* h, const int32_t* user_row, const int32_t* item_row,
                    const int32_t* hist_rows, int64_t B, float* X);

/* model.Train (model.go:27-213) on the dense X / Y that recommend.GetSample built
 * (rcmd.go:339-460).  ranges = SampleInfo {UserProfile, UserBehavior, ItemFeature, CtxFeature} as
 * 4 [start,end) pairs (rcmd.go:132-137).  Zero-pads the ragged last batch and trains on it with
 * label 0 (model.go:132-184,357-371); *last_cost = cost of the last batch (model.go:198);
 * early_stop = no-improvement epochs (0 = off, model.go:199-209).  Single-GPU route (the reference's own shape of
 * use); with world > 1 it returns CTR_ESTATE — multi-GPU training goes through the index entry points. */
int ctr_train_dense(ctr_handle* h, const float* X, const float* Y, int64_t n, int32_t xcols,
                    const int32_t ranges[8], int32_t epochs, int32_t early_stop,
                    float* last_cost, int32_t* epochs_run);
/* model.Predict (model.go:242-353): batches of pred_batch, zero-padded tail, dropout off
 * (din.go:133-145).  out is [n]. */
int ctr_predict_dense(ctr_handle* h, const float* X, int64_t n, int32_t xcols,
                      const int32_t ranges[8], float* out);

/* The H100-native fast path: one model.Train inner-loop iteration (model.go:107-196) fed by row
 * indices instead of a materialised X; gathers from the HBM tables inside the kernels.
 * hist_rows is [B,S], most-recent-first, -1 padded (prepare.go:49-51, rcmd.go:517-522).
 * B must equal cfg.batch.  Host buffers: copied H2D inside the call. */
int ctr_train_step_idx(ctr_handle* h, const int32_t* user_row, const int32_t* item_row,
                       const int32_t* hist_rows, const float* label, int32_t B, ctr_step_stats* stats);
/* model.Train's batch loop for one pass over n samples (model.go:107-196) fed by row ids: batches of
 * cfg.batch are consumed in order, the ragged tail is zero-padded with label 0 (model.go:357-371), and
 * the host→device copy of batch i+1 overlaps the compute of batch i: the caller's (pageable) buffers are copied into
 * an internal pinned ring by a few host threads and DMA'd from there on a second stream.  One coarse call
 * per epoch is the shape a cgo caller wants.  costs (may be NULL) receives ceil(n/batch) batch costs.
 * With world > 1 every step is collective (both placements): all ranks must call with the same n. */
int ctr_train_idx(ctr_handle* h, const int32_t* user_row, const int32_t* item_row,
                  const int32_t* hist_rows, const float* label, int64_t n, float* costs);
/* recommend.Train (rcmd.go:197-246) fed by sample keys {UserId, ItemId, Timestamp, Label} (rcmd.go:189-194) — the
 * whole of GetSample (rcmd.go:339-460) runs on the device: the id maps (ctr_idmap_build) resolve the keys, samples
 * whose user or item has no features are dropped as the reference's assembler skips them (rcmd.go:378-382), the
 * survivors stay in HBM in input order, and each batch's history rows are windowed from the device ubcache at the
 * sample's timestamp (GetUserBehavior(uid, S, -1, ts): rcmd.go:509, prepare.go:13-38; no ubcache uploaded → empty
 * history) right before its step.  Then model.Train's loop: batches of cfg.batch, zero-padded tail with label 0,
 * *last_cost = cost of the epoch's last batch, early_stop = no-improvement epochs (0 = off) (model.go:96-209).
 * Host traffic: 28 bytes per sample, staged through an internal pinned ring (the caller's buffers may be pageable).
 * *rows_used = samples that survived.  world > 1: collective — every rank passes its own keys; all ranks run the
 * batch count of the rank with the most surviving samples. */
int ctr_train_keys(ctr_handle* h, const int64_t* user_ids, const int64_t* item_ids, const int64_t* ts, const float* label,
                   int64_t n, int32_t epochs, int32_t early_stop, float* last_cost, int32_t* epochs_run, int64_t* rows_used);
/* recommend.BatchPredict → model.Predict (rcmd.go:277-337) fed by indices. out is [n]. */
int ctr_predict_idx(ctr_handle* h, const int32_t* user_row, const int32_t* item_row,
                    const int32_t* hist_rows, int64_t n, float* out);

/* Same step with DEVICE-resident index / label buffers; asynchronous on the engine stream, no host
 * sync (stats->cost is not filled; read it with ctr_last_cost after ctr_sync).  Used when the caller
 * keeps the sample stream in HBM (bench.py's `value` leg; the device-side ubcache row f2).
 * The *_dev entry points, ctr_sync and ctr_last_cost do not take the handle's mutex: drive a handle's device-side
 * entry points from one thread (the host-buffer entry points serialise themselves). */
int ctr_train_step_idx_dev(ctr_handle* h, const int32_t* d_user_row, const int32_t* d_item_row,
                           const int32_t* d_hist_rows, const float* d_label, int32_t B);
int ctr_predict_idx_dev(ctr_handle* h, const int32_t* d_user_row, const int32_t* d_item_row,
                        const int32_t* d_hist_rows, int32_t B, float* d_out);
int ctr_last_cost(ctr_handle* h, float* cost);
int ctr_sync(ctr_handle* h);
/* the cudaStream_t the engine launches on (so a harness can record its own events on it), and a
 * way to adopt the caller's stream instead */
void* ctr_get_stream(ctr_handle* h);
int   ctr_set_stream(ctr_handle* h, void* cuda_stream);
/* number of kernels the engine has launched since creation */
int64_t ctr_launch_count(const ctr_handle* h);
/* per-kernel device-time profile: enable → every launch is bracketed by events (slow; for bench's
 * roofline leg).  ctr_profile_get returns accumulated ms and launch count for a kernel name. */
int ctr_profile_enable(ctr_handle* h, int on);
int ctr_profile_get(ctr_handle* h, const char* kernel, double* ms_total, int64_t* launches);
int ctr_profile_reset(ctr_handle* h);
int ctr_profile_dump(ctr_handle* h, char* buf, int64_t buflen);   /* "name ms launches\n" lines */

/* Test hook: forward+backward of one index batch WITHOUT any update; returns what G.Grad would
 * (model.go:56) plus the engine's row gradients.  Any output pointer may be NULL.
 * dUb [B,S,D], dIt [B,D], p [B], logit [B]. */
int ctr_debug_grads_idx(ctr_handle* h, const int32_t* user_row, const int32_t* item_row,
                        const int32_t* hist_rows, const float* label, int32_t B, int32_t training,
                        float* dmlp0, float* dmlp1, float* dmlp2, float* datt0,
                        float* dUb, float* dIt, float* p, float* logit, float* cost);

/* feature/ubcache on the device (SURVEY.md §8f row f2).  upload: every user's behaviour sequence in
 * time-DESCENDING order (ubcache.TimeSeq, cache.go:9-12) as one CSR: offsets [n_users+1], ts [n],
 * item_rows [n] (dense ITEM_EMB rows).  window: TimeSeq.Filter(maxTs, S) for a batch (cache.go:71-94;
 * maxTs == 0 means "from the newest"), i.e. what GetUserBehavior(uid, S, -1, sample.Timestamp) returns
 * (prepare.go:13-38), written as hist_rows [B,S], -1 padded.  The _dev variant leaves the result in
 * device memory for ctr_train_step_idx_dev / ctr_predict_idx_dev. */
int ctr_ubcache_upload(ctr_handle* h, const int64_t* offsets, const int64_t* ts, const int32_t* item_rows, int64_t n_users, int64_t n);
int ctr_ubcache_window(ctr_handle* h, const int32_t* user_row, const int64_t* max_ts, int32_t B, int32_t* hist_rows);
int ctr_ubcache_window_dev(ctr_handle* h, const int32_t* d_user_row, const int64_t* d_max_ts, int32_t B, int32_t* d_hist_rows);

/* The live cache: UserBehaviorCache.Set / BatchSet / Delete (cache.go:27-48) and online appends, applied in HBM so the
 * next window / ctr_batch_predict_keys / ctr_recommend_topk / ctr_train_keys sees them without a re-upload.
 * append: n events (user_rows[i], ts[i], item_rows[i]) go into their users' sequences; the cache is created if none was
 *   uploaded.  Every sequence stays time-descending, and equal timestamps are ordered most recent ARRIVAL first: an
 *   appended event comes before the stored events with the same ts, and among one call's events of one user with the
 *   same ts, the later in the call comes first.  This decides which items a window whose maxTs falls on a tied run
 *   returns.
 * set: replaces the whole sequences of n_set distinct users; user k's events are [offsets[k], offsets[k+1]) of ts /
 *   item_rows [n] (offsets [n_set+1] from 0 to n), non-increasing in ts.  An empty sequence is Delete: that user then
 *   windows to an empty history, as an unknown user does.  Clear (cache.go:51-55) is ctr_ubcache_upload of an empty
 *   cache (offsets {0, 0}).
 * Item rows are stored as given (-1 or out of range reads as a zero row, as with upload).  A user row must lie in
 * [0, max(cache users, USER_FEAT rows, user id map size)); the cache's user count grows to the largest row + 1.
 * Everything is validated on the host before any device work (CTR_EINVAL), and a failed call leaves the cache as it
 * was.  One call rewrites the CSR into a spare buffer and swaps the two (O(stored events + users) of HBM traffic), on
 * the engine stream.  With world > 1 each rank's cache is its own; these calls are not collective.  CTR_EXCLUDE_SEEN
 * on a row-sharded ITEM_EMB reads each row's events from the cache of the rank that owns the row, so apply every
 * upload, append and set on every rank.
 * download: the live cache back to the host.  *n_users and *n are always written; offsets [n_users+1] is written when
 *   non-NULL and cap_users >= n_users, ts / item_rows [n] when non-NULL and cap_events >= n; a non-NULL array that is
 *   too small is CTR_EINVAL, no cache is CTR_ESTATE. */
int ctr_ubcache_append(ctr_handle* h, const int32_t* user_rows, const int64_t* ts, const int32_t* item_rows, int64_t n);
int ctr_ubcache_set(ctr_handle* h, const int32_t* user_rows, const int64_t* offsets, const int64_t* ts,
                    const int32_t* item_rows, int64_t n_set, int64_t n);
int ctr_ubcache_download(ctr_handle* h, int64_t* offsets, int64_t* ts, int32_t* item_rows,
                         int64_t cap_users, int64_t cap_events, int64_t* n_users, int64_t* n);

/* ---- sparse ids, serving keys, checkpoint (SURVEY.md §8f rows f3, f4) ------------------------------------
 * The reference keys its caches by the decimal string of a Go int (rcmd.go:472,483,502,519); the engine's
 * tables are dense.  ctr_idmap_build puts `ids[i] → row i` into a device hash table (which: CTR_IDMAP_*);
 * duplicate ids or INT64_MIN are rejected (CTR_EINVAL).  lookup writes the row, or -1 for an unknown id —
 * which the gather reads as a zero row, the reference's "not found → zeros" (rcmd.go:501-505,519-521). */
enum { CTR_IDMAP_USER = 0, CTR_IDMAP_ITEM = 1 };
int ctr_idmap_build(ctr_handle* h, int which, const int64_t* ids, int64_t n);
int ctr_idmap_lookup(ctr_handle* h, int which, const int64_t* ids, int64_t n, int32_t* rows);
int ctr_idmap_lookup_dev(ctr_handle* h, int which, const int64_t* d_ids, int64_t n, int32_t* d_rows);

/* Live id maps and tables: a user or item that did not exist when the handle was set up gets a row and its features
 * while the handle serves and trains, as the reference's feature caches fetch a new key's features on first use
 * (rcmd.go:344-353, 472-492).  All three take the handle's mutex and run on the engine stream: work queued before sees
 * the old state, work queued after the new one.  Arguments are validated before any device write, and a refused call
 * changes nothing.
 * insert: an id the map holds keeps its row; the ids it lacks get rows idmap_n, idmap_n + 1, ... in the order of their
 *   first occurrence in ids (a repeated id gets one row).  rows (may be NULL) receives the row of every ids[i].  No map:
 *   the call creates one, which on distinct ids equals ctr_idmap_build.  CTR_EINVAL: NULL ids, n outside [1, 2^31), a bad
 *   which, INT64_MIN anywhere in ids, or more than INT32_MAX ids in all.  The load factor stays <= 0.5: a map that
 *   outgrows its table is rehashed into one of the capacity ctr_idmap_build picks for the new count.
 * download: *n = the id count; ids (may be NULL) [cap] receives the id of every row, ids[r] = the id of row r.  A
 *   non-NULL ids with cap < *n is CTR_EINVAL, no map is CTR_ESTATE.  Checkpoints do not hold id maps: download +
 *   ctr_idmap_build is how a map grown live is persisted and restored.
 * write_rows: row rows[i] of table `which` becomes data[i] (data [n, width], width = the table's model dimension), bit
 *   for bit.  CTR_EINVAL: a row outside [0, INT32_MAX) or the same row twice.  A row at or past the end grows the table
 *   to max(rows) + 1 rows; the rows in between are zero (a missing row reads as zero anyway).  No table: the call creates
 *   one.  Tables grow in place (reserved address space, memory mapped in chunks), without a second copy of the table.
 *   ITEM_EMB: written and new rows get zero row-Adam moments, every other row keeps its moments; the step counter,
 *   the dense weights and every other row are unchanged (ctr_table_upload, by contrast, resets the solver state).
 *   Host data is staged in chunks; the caller's buffers may be pageable.
 * World > 1: insert and write_rows are collective (every rank calls them, each with its OWN arguments; n = 0 is allowed
 *   there, with ids / rows / data then possibly NULL) and download is local.  The rule: afterwards every rank holds what
 *   one GPU would hold after the same call on the ranks' arguments concatenated in rank order.  Every rank checks its
 *   arguments, then the ranks exchange verdicts: if any rank fails, every rank returns the lowest failing rank's code and
 *   nothing changes anywhere; a state that differs across ranks (the map's size or the order-independent digest of its
 *   (id, row) pairs; a table's rows, width or placement) is CTR_EINVAL everywhere.  "Changes nothing" covers every
 *   refusal decided from the arguments and the state.  It does not cover a CUDA or NCCL failure after the agreement,
 *   such as running out of device memory while one rank grows its shard: as with the other collective calls, that rank
 *   returns the error, the others may then wait in the exchange, and the ranks' tables may differ; such a handle is to
 *   be rebuilt (ctr_table_upload, ctr_idmap_build) on every rank.
 *   insert: each rank numbers its own missing ids, the ranks all-gather the counts and then the lists padded to the
 *     longest (8 + 4 bytes an entry), and each runs the same deterministic merge (profile key idmap_merge_ranks): new ids
 *     get rows by first (rank, position), so an id new on several ranks takes its first.  rows receives the rows of this
 *     rank's own ids.  INT64_MIN on any rank, more than INT32_MAX rows in all, or more than INT32_MAX ids
 *     passed in all (as one GPU refuses them) is refused on every rank.  When every rank passes n = 0 the call does
 *     nothing.  Scratch: 4 x 8 bytes per gathered entry beside the single-GPU scratch.
 *   write_rows: the row ids are concatenated on every rank (4 bytes a row, broadcast per rank) and a row named twice,
 *     within or across ranks, is CTR_EINVAL everywhere.  A replicated table (USER_FEAT; ITEM_* at or under the placement
 *     threshold) concatenates the data the same way and every rank writes every row: each rank receives the whole
 *     union.  A row-sharded table sends each (row, data) to its owner row % world only (grouped send / recv, no
 *     full-table traffic), which writes its local row row / world; a row below the replicated hot-row count goes to
 *     every rank's hot-row replica too, and under CTR_TABLE_ADAM the written rows' moments are zeroed on the owner and in
 *     the hot-moment replica.  A write past the end grows every table to max(rows) + 1 with zero rows in between and
 *     keeps its placement (a replicated table never becomes sharded); no table yet is allocated by ctr_table_upload's
 *     placement rule for that size.  A shard that outgrows its allocation (an exportable one the peers map, which
 *     cannot grow in place) is reallocated at max(new local rows, 2 x old local rows) — the old and the new shard side
 *     by side at the peak, plus ITEM_EMB's moments grown in place — and the next collective call republishes the peer
 *     mappings.  Host staging: this rank's rows grouped by destination, one copy of its data. */
int ctr_idmap_insert(ctr_handle* h, int which, const int64_t* ids, int64_t n, int32_t* rows);
int ctr_idmap_download(ctr_handle* h, int which, int64_t* ids, int64_t cap, int64_t* n);
int ctr_table_write_rows(ctr_handle* h, int which, const int32_t* rows, const float* data, int64_t n, int32_t width);

/* recommend.BatchPredict (rcmd.go:277-337) over sample keys {UserId, ItemId, Timestamp} (rcmd.go:189-194),
 * entirely on the device: id maps → rows, ubcache window at the sample's timestamp → history rows,
 * forward → scores [n].  Needs both id maps; without an uploaded ubcache the history is empty (the
 * reference's "UserBehavior not implemented → zeros", rcmd.go:498,509).  A key whose user or item is
 * unknown scores as an all-zero X row (rcmd.go:299-307) — unless it is key 0, which fails the call with
 * CTR_ENOTFOUND as the reference returns the error (rcmd.go:300-303).  recommend.Rank (rcmd.go:248-275) =
 * this with one user id, the candidate item ids and ts = now. */
int ctr_batch_predict_keys(ctr_handle* h, const int64_t* user_ids, const int64_t* item_ids, const int64_t* ts,
                           int64_t n, float* scores);

/* Binary snapshot of everything a resumed run needs: dims, optimiser step, dense weights with their Adam
 * moments, and the three tables (this rank's shard of ITEM_EMB when world > 1 — use one path per rank).
 * The reference has no checkpoint at all (SURVEY.md §5: JSON weights only, din.go:62); that JSON stays
 * available through ctr_get_weights / ctr_set_weights.  load requires a handle created with the same
 * dims, rank and world; tables are (re)allocated from the file. */
int ctr_checkpoint_save(ctr_handle* h, const char* path);
int ctr_checkpoint_load(ctr_handle* h, const char* path);

/* utils.RocAuc32 (util.go:131-148 → nn/metrics/ranking.go:144): labels binarised at 0.5, tied
 * scores grouped, trapezoid. Sorted on the device.  Each rank evaluates the samples it passes (ctr_roc_auc_dist evaluates
 * every rank's). */
int ctr_roc_auc(ctr_handle* h, const float* pred, const float* y, int64_t n, double* auc);

/* Grouped AUC (GAUC: the metric of the DIN paper and of go-ctr's README.md:17/25/33): samples are grouped by
 * group[i] (normally the sample's UserId), groups ordered by ascending signed int64.  For group g with n_g samples, P_g
 * positives and N_g = n_g - P_g negatives, AUC_g is ctr_roc_auc over the group's samples by the same rules (labels
 * binarised at 0.5, -0 read as +0, scores ordered by the same transform of their float32 bits, equal scores one threshold
 * group) from integer counts: area2_g = sum (fp_i - fp_{i-1}) (tp_i + tp_{i-1}) over the threshold-group ends in int64,
 * AUC_g = (double)area2_g / (2.0 * P_g * N_g), NaN when P_g = 0 or N_g = 0.  Whenever 2 P_g N_g < 2^53, AUC_g equals
 * ctr_roc_auc on that group's samples bit for bit.  A group is used when P_g > 0 and N_g > 0;
 * *gauc = sum_used n_g AUC_g / sum_used n_g (weighted by impressions), NaN when no group is used.  The sum is
 * deterministic (identical inputs give identical bits) and compensated.
 * n in [1, 2^31); pred, y, group and gauc non-NULL, else CTR_EINVAL before any input is read.  n_groups (number of
 * groups), n_used (used groups) and the out_* arrays may each be NULL.  A non-NULL out_* array has room for n entries;
 * its first *n_groups entries are written in ascending group order: the group id, n_g, P_g and AUC_g (NaN when unused).
 * Host buffers; needs no tables (a handle created with batch = pred_batch = 1 is enough).  Runs on the engine stream
 * under the handle's mutex.  Not collective under world > 1: each rank evaluates the samples it passes (ctr_group_auc_dist
 * evaluates every rank's). */
int ctr_group_auc(ctr_handle* h, const float* pred, const float* y, const int64_t* group, int64_t n,
                  double* gauc, int64_t* n_groups, int64_t* n_used,
                  int64_t* out_group, int32_t* out_n, int32_t* out_pos, double* out_auc);

/* ctr_roc_auc and ctr_group_auc over every rank's samples of a multi-GPU handle (a held-out set each rank scored for
 * its own keys).  Neither needs tables; both run on the engine stream under the handle's mutex and use its
 * communicator.  h NULL is CTR_EINVAL before any collective work.
 * World == 1: the calls are ctr_roc_auc and ctr_group_auc, with their results, refusals and messages; the per-group
 *   arrays are written as ctr_group_auc writes them, and cap bounds them (see below).
 * World > 1: collective; every rank calls with its own samples.  n in [0, 2^31) per rank (n = 0 allows NULL arrays)
 *   and the total in [1, 2^32).  Every rank receives what the single-GPU call returns on all ranks' samples concatenated
 *   in rank order, bit for bit, by its rules (labels binarised at 0.5, -0 read as +0, the NaN key order, ascending
 *   signed group order).  Every rank checks its arguments, then the ranks exchange verdicts as the live-table calls do:
 *   if any rank fails, every rank returns the lowest failing rank's code, and nothing is written on any rank.  A CUDA
 *   or NCCL failure after the agreement follows the rule of ctr_idmap_insert: that rank returns the error and the
 *   others may wait in the exchange.
 *
 * ctr_roc_auc_dist: equal to ctr_roc_auc on the concatenation whenever that call is exact there (2 P N < 2^53; its
 *   trapezoid terms are half-integers summed in double).  Each rank sorts its score keys and sums the counts of equal
 *   keys into runs (key, positives, negatives); splitters from regular samples of the ranks' runs cut the key range
 *   into one range per rank, so equal scores always meet on one rank; each owner merges the runs it receives, learns
 *   the positives of the lower ranks, and sums its part of area2 = sum (fp_j - fp_{j-1}) (tp_j + tp_{j-1}) in uint64;
 *   one all-reduce completes it, and *auc = ((double)area2 * 0.5) / ((double)P * (double)N), NaN when P or N is 0.
 *   NVLink traffic: 12 bytes per run a rank sends (a tie group of scores on a rank is one run), plus four all-gathers
 *   of at most 256 bytes per rank (the agreement's included) and one 8-byte all-reduce.  Device scratch per rank: about 40 bytes per sample while the
 *   runs are built, then 40 bytes per received run.
 *
 * ctr_group_auc_dist: *gauc, *n_groups, *n_used and the per-group outputs equal ctr_group_auc on the concatenation bit
 *   for bit, the compensated sum included.  Each rank sorts records (group, score key and label; 16 bytes) by group,
 *   the records of each group range go to one rank, so every group lives whole on one rank, and each rank runs
 *   ctr_group_auc's grouped driver on its groups.  The groups' terms (group id, n_g, P_g, area2_g; 24 bytes a group) are
 *   all-gathered in rank order, which is ascending group order, and every rank folds them as ctr_group_auc does.
 *   NVLink traffic: 16 bytes per sample that changes rank, 24 bytes per group to every rank, and four all-gathers of
 *   at most 256 bytes per rank.  Device scratch: about
 *   56 bytes per own sample while sorting, then ctr_group_auc's 100 bytes per received sample, then 24 bytes per group
 *   of all ranks.  A group is never split, so one group holding most samples puts them all on one rank; more than
 *   2^31 - 1 samples on one rank, or more than 2^31 - 1 groups in all, is CTR_EINVAL on every rank.
 *   out_group, out_n, out_pos and out_auc may each be NULL and receive the first *n_groups groups in ascending group
 *   order; a non-NULL array with cap < *n_groups is CTR_EINVAL, decided once the group count is known and before
 *   anything is written. */
int ctr_roc_auc_dist(ctr_handle* h, const float* pred, const float* y, int64_t n, double* auc);
int ctr_group_auc_dist(ctr_handle* h, const float* pred, const float* y, const int64_t* group, int64_t n,
                       double* gauc, int64_t* n_groups, int64_t* n_used,
                       int64_t cap, int64_t* out_group, int32_t* out_n, int32_t* out_pos, double* out_auc);

/* The curves and average precision of nn/metrics/ranking.go, on the device.  All four follow binaryClfCurve
 * (ranking.go:13-57): scores ordered as ctr_roc_auc orders them (descending; -0 and +0 one threshold group; every NaN
 * bit pattern its own group, positive NaNs above +inf, negative NaNs below -inf), one point per threshold group from the
 * highest score down with the cumulative integer counts tp_j / fp_j, its threshold the group's score widened to double
 * (+0.0 for the ±0 group, a NaN with its bits).  A sample is positive when (double)y[i] == pos_label.  Every NaN the
 * calls compute (as opposed to a NaN threshold) is 0x7ff8000000000000.
 * n in [1, 2^31); h, pred, y and the scalar outputs non-NULL, else CTR_EINVAL.  Host buffers; needs no tables (a
 * handle created with batch = pred_batch = 1 is enough).  Runs on the engine stream under the handle's mutex.  Not
 * collective under world > 1: each rank evaluates the samples it passes.  A refusal writes no output except as stated.
 *
 * ROCCurve (ranking.go:71-103): when fp_0 != 0 the point (0, 0) comes first with threshold thresholds[0] + 1 (a NaN
 * threshold stays itself); fpr = fp * (1.0 / fp_max) and tpr = tp * (1.0 / tp_max), each a product, all NaN when
 * fp_max (resp. tp_max) is 0.  *npoints = the number of points; fpr, tpr and thresholds each receive that many values
 * and may each be NULL.  A curve of more than cap points is CTR_EINVAL with only *npoints written; cap = n + 1 always
 * suffices. */
int ctr_roc_curve(ctr_handle* h, const float* pred, const float* y, int64_t n, double pos_label,
                  double* fpr, double* tpr, double* thresholds, int64_t cap, int64_t* npoints);

/* PrecisionRecallCurve (ranking.go:183-209): precision_j = tp_j / (tp_j + fp_j), recall_j = tp_j / tp_last (a
 * division; NaN when tp_last = 0), cut at last_ind = the first j with tp_j >= tp_last, reversed, then precision 1 and
 * recall 0 appended.  *npoints = last_ind + 2 precision and recall values; thresholds receives last_ind + 1.  With no
 * positives: precision {0, 1}, recall {NaN, 0}, one threshold.  NULL arrays and cap as in ctr_roc_curve. */
int ctr_pr_curve(ctr_handle* h, const float* pred, const float* y, int64_t n, double pos_label,
                 double* precision, double* recall, double* thresholds, int64_t cap, int64_t* npoints);

/* AveragePrecisionScore (ranking.go:212-222) of a binary target, pos_label = 1: the terms
 * (recall_j - recall_{j-1}) * precision_j for j = 0 … last_ind (recall_{-1} = 0), each computed as in ctr_pr_curve,
 * summed as a double-double in a fixed order (within 1 ulp of the exactly rounded sum; identical inputs give identical
 * bits; the reference sums them one by one from the high-recall end).  NaN with no positives.  Labels that are not
 * binary (some label equal to neither the lowest nor the highest label, or any NaN label; base.go:89-119) are
 * CTR_EINVAL with *ap untouched, where the reference prints "unsupported" and returns 0. */
int ctr_average_precision(ctr_handle* h, const float* pred, const float* y, int64_t n, double* ap);

/* Mean average precision over groups (normally the sample's UserId), shaped like ctr_group_auc: groups ordered by
 * ascending signed int64; AP_g = ctr_average_precision over the group's samples (recall divided by the group's own
 * positives P_g); a group is used when P_g > 0; *map = the unweighted mean of AP_g over the used groups, a compensated
 * sum in a fixed order, NaN when no group is used.  The binary-label rule applies to the whole call.  n_groups, n_used
 * and the out_* arrays may each be NULL; a non-NULL out_* array has room for n entries, and its first *n_groups
 * entries receive, in ascending group order, the group id, n_g, P_g and AP_g (NaN when P_g = 0). */
int ctr_group_average_precision(ctr_handle* h, const float* pred, const float* y, const int64_t* group, int64_t n,
                                double* map, int64_t* n_groups, int64_t* n_used,
                                int64_t* out_group, int32_t* out_n, int32_t* out_pos, double* out_ap);

/* The classification and regression metrics of nn/metrics (classification.go, regression.go) on the device.  Shared
 * rules: host buffers of double (the reference's mat.Dense; float32 labels and predictions widen exactly); n in
 * [1, 2^31); a handle created with batch = pred_batch = 1 is enough.  The calls run on the engine stream under the
 * handle's mutex and are not collective under world > 1: each rank evaluates the samples it passes.  Every refusal comes
 * before any output is written (except as stated) and its message is in ctr_last_error; the arguments are checked
 * before the handle, so with h NULL the message is in ctr_last_error(NULL).  Identical inputs give identical bits.
 * Unweighted counts are exact integers; every weighted or floating-point sum is taken over fixed partitions in a fixed
 * order (a double-double wherever the reference has sample weights). */
enum { CTR_AVERAGE_MACRO = 0, CTR_AVERAGE_MICRO = 1, CTR_AVERAGE_WEIGHTED = 2 };
enum { CTR_MULTIOUTPUT_RAW = 0, CTR_MULTIOUTPUT_UNIFORM = 1, CTR_MULTIOUTPUT_VARIANCE_WEIGHTED = 2 };
enum { CTR_ERROR_SQUARED = 0, CTR_ERROR_ABSOLUTE = 1 };

/* AccuracyScore (classification.go:12-34): y_true and y_pred are [n, n_out] row-major, n_out in [1, 1024].  A row is
 * correct when each of its n_out columns compares equal with == (-0 == +0; a NaN never equals).  weight [n] (NULL: every
 * weight 1) must be finite, else CTR_EINVAL; zero and negative weights are used as given.  N = the weights of the correct
 * rows, D = all weights; *score = N / D with normalize != 0 (NaN when every weight is 0, as the reference's 0/0; a
 * nonzero N over D = 0 is ±inf), else N. */
int ctr_accuracy_score(ctr_handle* h, const double* y_true, const double* y_pred, int64_t n, int32_t n_out, const double* weight,
                       int32_t normalize, double* score);

/* ConfusionMatrix (classification.go:150-178) of 1-D labels.  The classes are LabelEncoder.Fit's on y_true
 * (label.go:288-321): the C distinct values ascending, -0 and +0 one class whose value keeps the sign of its first
 * occurrence in sample order.  Each label maps as sort.SearchFloat64s maps it (label.go:324-339), to the first class
 * >= it: a prediction between two classes counts as the higher one.  cm[r*C + c] = the summed weights (weight NULL:
 * counts) of the samples of true class r predicted as c.  CTR_EINVAL, naming the first offending sample, for a NaN in
 * y_true or y_pred, a weight that is not finite, or a prediction above the largest class (there the reference writes
 * into the cell before (r, 0), or panics when r = 0).  *n_classes = C is written whenever y_true holds no NaN, even by
 * a refusal.  classes (C values; C <= n) and cm (cap cells) may each be NULL; C*C > cap is CTR_EINVAL. */
int ctr_confusion_matrix(ctr_handle* h, const double* y_true, const double* y_pred, int64_t n, const double* weight, double* classes,
                         double* cm, int64_t cap, int32_t* n_classes);

/* PrecisionRecallFScoreSupport (classification.go:74-148) over the classes and cells of ctr_confusion_matrix (same
 * pipeline, same refusals).  Per class: tp = the diagonal cell, truesum = the row's weights, predsum = the column's (each
 * a compensated sum over the samples; the reference sums the matrix's cells); p = tp / predsum (0 when predsum <= 0),
 * r = tp / truesum (0 when truesum <= 0), f = (1+beta^2)*p*r / (beta^2*p + r) (0 when that denominator is not > 0), each
 * operation rounded on its own; support = the unweighted count of y_true in the class (le.Support).  pos_label >= 0:
 * *p, *r, *f, *support are that class's (pos_label >= C is CTR_EINVAL; the reference panics).  pos_label < 0: the average
 * -- CTR_AVERAGE_MACRO the plain mean over the classes; CTR_AVERAGE_WEIGHTED the same mean, bit for bit, because the
 * reference builds the support weights and then calls stat.Mean(p, nil) (:116-131; sklearn would weight by support);
 * CTR_AVERAGE_MICRO the per-class formulas on tp, truesum and predsum summed over the classes -- and *support = 0.
 * Another average is CTR_EINVAL (the reference returns zeros), as is a beta that is not finite.  p, r, f and support
 * may each be NULL.  per_class (NULL or cap rows) receives [C, 4] rows (p, r, f, support); with per_class non-NULL,
 * C > cap is CTR_EINVAL (C <= n, so cap = n always suffices).  *n_classes as in ctr_confusion_matrix.
 * PrecisionScore, RecallScore and F1Score are this call with beta = 1, FBetaScore with the beta given. */
int ctr_precision_recall_fscore(ctr_handle* h, const double* y_true, const double* y_pred, int64_t n, const double* weight, double beta,
                                int32_t average, int32_t pos_label, double* p, double* r, double* f, double* support,
                                double* per_class, int64_t cap, int32_t* n_classes);

/* R2Score (regression.go:83-128) of [n, n_out] targets, n_out in [1, 1024].  With weight [n] (NULL: every weight 1),
 * per column j: num_j = sum w*(pred - true)^2, avg_j = sum w*true / sum w, den_j = sum w*(true - avg_j)^2,
 * r2_j = 1 - num_j / max(den_j, 1e-20).  CTR_MULTIOUTPUT_RAW writes out[n_out] = r2_j; CTR_MULTIOUTPUT_VARIANCE_WEIGHTED
 * writes out[0] = sum den_j*r2_j * (1 / sum den_j), NaN when every den_j is 0; CTR_MULTIOUTPUT_UNIFORM writes out[0] =
 * the mean of the r2_j.  A constant column is not refused (unlike ctr_mlp_score); NaN and +-inf inputs propagate as IEEE
 * arithmetic makes them.  The sums are the fixed-partition column reductions of ctr_mlp_score. */
int ctr_r2_score(ctr_handle* h, const double* y_true, const double* y_pred, int64_t n, int32_t n_out, const double* weight,
                 int32_t multioutput, double* out);

/* MeanSquaredError (kind CTR_ERROR_SQUARED, regression.go:153-176) and MeanAbsoluteError (CTR_ERROR_ABSOLUTE, :220-244):
 * per column the mean of (pred - true)^2 or |pred - true| over the n rows; CTR_MULTIOUTPUT_RAW writes out[n_out],
 * CTR_MULTIOUTPUT_UNIFORM out[0] = their mean.  CTR_MULTIOUTPUT_VARIANCE_WEIGHTED is CTR_EINVAL: these functions have no
 * such mode.  No sample weights: the reference reads sampleWeight.At(0, j) (:163, :230), one weight for every sample of
 * column j, which either cancels out of N / D or gives 0 / 0. */
int ctr_mean_error(ctr_handle* h, const double* y_true, const double* y_pred, int64_t n, int32_t n_out, int32_t kind,
                   int32_t multioutput, double* out);

/* search.Searcher (feature/embedding/search/search.go:66-134): the k items of ITEM_EMB most cosine-similar to each
 * query, on the device.  queries == NULL: search by row — query i is ITEM_EMB row query_rows[i] widened to float64 and
 * excluded from its own result (SearchInternal, with the word→row map on the caller's side); a row outside [0, rows)
 * is CTR_ENOTFOUND ("<row> is not found in searcher").  queries != NULL: search by the float64 vectors queries [nq, D]
 * (SearchVector); query_rows may then be NULL or name a row to exclude per query (-1 = none).
 * Similarities are bit-identical to search.go on the widened float32 table: Norm and Cosine in float64, sequential
 * sums, dot / |q| / |v|; only similarities > 0 qualify.  Results come in rank order: similarity descending, equal
 * similarities by row ascending.  out_rows / out_sim are [nq, k]; out_count[i] is the true number of results of query i,
 * positions at or past it hold row -1 and similarity 0.  k in [1, 1024].  Needs only ITEM_EMB (a handle with
 * uP = cF = 0 is enough).  Runs on the engine stream under the handle's mutex, so it sees every update queued before it.
 * Row-sharded ITEM_EMB (world > 1, large table): the call is collective — every rank calls it with the same arguments
 * and receives the same complete result, bit-identical to one GPU holding the whole table.  Row ids stay global; more
 * than INT32_MAX rows is CTR_ESTATE.  Each rank scans its own shard and the ranks' lists are merged.  The ranks first
 * exchange their arguments and validation verdicts: arguments that differ are CTR_EINVAL on every rank ("ranks
 * disagree ..."), otherwise every rank returns the verdict of the lowest failing rank.  A failure after that exchange
 * (out of device memory, a failed peer mapping) leaves the other ranks waiting, as in the sharded train step.  The call starts with a device
 * barrier over the ranks and finishes its reads before any rank's next step can change a row, so no ctr_sync or host
 * barrier is needed between training and this call (unlike ctr_predict_idx on a sharded table).  A replicated ITEM_EMB
 * is searched locally, by each rank alone. */
int ctr_knn_search(ctr_handle* h, const double* queries, const int32_t* query_rows, int64_t nq, int32_t k,
                   int32_t* out_rows, double* out_sim, int32_t* out_count);

/* Recommendation without a candidate list (recommend/api.go:115-118 "todo: some default recall algorithm"): for each
 * of nu users, score EVERY row of ITEM_EMB as the sample (user_rows[j], item, hist_rows[j]) with the model's forward
 * pass (dropout off, exactly what ctr_predict_idx computes for that triple) and return the k best.
 *   Candidates: the ITEM_EMB rows [0, I).  An item's features are ITEM_FEAT row `item`, zeros when that row is missing.
 *     A user row or history row outside its table reads as a missing row, as in the other _idx entry points.
 *     hist_rows is [nu, S], -1 padded.
 *   Order: pre-sigmoid logit descending, then row ascending.  The sigmoid is monotone, so this is also a top-k by score,
 *     but it does not collapse where the score saturates at 1 (logit > 15).  out_scores[j, i] is sigmoid(logit)
 *     exactly as ctr_predict_idx returns it; out_logits (may be NULL) the logit.
 *   Exclusions: an item whose logit is NaN is never returned; with exclude_history != 0 neither is an item that appears
 *     among the user's valid hist_rows.
 *   out_rows / out_scores / out_logits are [nu, k]; out_count[j] is the true number of results of user j, positions at
 *     or past it hold row -1, score 0 and logit 0.
 *   k in [1, 1024]; nu >= 1.  Missing tables, or no ITEM_EMB, is CTR_ESTATE.
 *   Row-sharded ITEM_EMB (world > 1, large table): collective, under the same rule as ctr_knn_search — every rank calls
 *     with the same arguments and receives the same complete result, bit-identical to one GPU holding the whole table;
 *     each rank scores its own shard's items and the ranks' lists are merged; disagreeing arguments are CTR_EINVAL
 *     everywhere; no ctr_sync or host barrier is needed after training.  It needs D in {16, 32, 64, 128} and the user's
 *     history rows in shared memory (else CTR_ESTATE).  A replicated ITEM_EMB is served locally, by each rank alone.
 *   Items are scored in chunks of max(batch, pred_batch) rows, in the activation buffers the handle already has: a large
 *     catalogue wants a large pred_batch.  Only nu·k results cross PCIe.
 *   Runs on the engine stream under the handle's mutex, so it sees every update queued before it. */
int ctr_recommend_topk(ctr_handle* h, const int32_t* user_rows, const int32_t* hist_rows, int64_t nu, int32_t k,
                       int32_t exclude_history, int32_t* out_rows, float* out_scores, float* out_logits, int32_t* out_count);

/* Exclusion modes of the _ex recommendation and rank calls:
 *   CTR_EXCLUDE_NONE    nothing but NaN logits (exclude_history = 0 of the plain calls)
 *   CTR_EXCLUDE_WINDOW  the valid rows of the key's history window (exclude_history != 0)
 *   CTR_EXCLUDE_SEEN    everything the user has seen up to the cut: the window's valid rows and the item row of every
 *                       event of the user's device-ubcache sequence with ts <= max_ts (max_ts == 0: every event, as
 *                       TimeSeq.Filter, cache.go:71-94).  No ubcache, or a user row outside the cache, adds no event;
 *                       item rows of -1, rows past the table and repeated rows are harmless.  A superset of WINDOW, and
 *                       an evaluation cut at a held-out event's time never excludes the events after it.
 *                       Row-sharded ITEM_EMB (world > 1): the owner of a row decides.  Row g is excluded when it is a
 *                       valid row of the window, or when the ubcache of rank g % world holds an event of the user with
 *                       ts <= max_ts whose item is g.  With the same cache on every rank (apply ctr_ubcache_upload,
 *                       _append and _set on every rank) the result is bit-identical to one GPU holding the whole table
 *                       and that cache.  Caches that differ still give every rank the same complete result, each row
 *                       following its owner's cache; no union of the ranks' caches is formed. */
enum { CTR_EXCLUDE_NONE = 0, CTR_EXCLUDE_WINDOW = 1, CTR_EXCLUDE_SEEN = 2 };

/* ctr_recommend_topk with an exclusion mode: ctr_recommend_topk(..., exclude_history, ...) ==
 * ctr_recommend_topk_ex(..., NULL, ..., exclude_history ? CTR_EXCLUDE_WINDOW : CTR_EXCLUDE_NONE, ...).  max_ts [nu] is
 * user j's cut under CTR_EXCLUDE_SEEN and may be NULL otherwise.  Refusals write nothing: CTR_EINVAL for an exclude
 * outside the enum or SEEN with a NULL max_ts, besides ctr_recommend_topk's.  The seen set is built on the device per
 * user (a bitmap over the rank's ITEM_EMB rows, ⌈I / 32⌉ words of the handle's scratch, ⌈I_local / 32⌉ on a shard): no
 * length cap.  On a row-sharded ITEM_EMB SEEN is collective like the other modes, under the owner rule of
 * CTR_EXCLUDE_SEEN: each rank marks the rows it owns from its own ubcache, with no exchange beyond the lists' merge.
 * The ranks must also agree on max_ts (else CTR_EINVAL everywhere, "ranks disagree ...").  A replicated ITEM_EMB is
 * served locally, from each rank's own cache. */
int ctr_recommend_topk_ex(ctr_handle* h, const int32_t* user_rows, const int32_t* hist_rows, const int64_t* max_ts, int64_t nu, int32_t k,
                          int32_t exclude, int32_t* out_rows, float* out_scores, float* out_logits, int32_t* out_count);

/* Full-catalogue rank of held-out items (the offline protocol of item recommendation): for each of n keys (user_rows[i],
 * hist_rows[i] [n, S], item_rows[i]) every ITEM_EMB row is scored exactly as ctr_recommend_topk scores it for
 * (user_rows[i], hist_rows[i]) — the same kernels, chunks and logits — and the target item is ranked in that list's order
 * (logit descending, then row ascending):
 *   out_rank[i] = 1 + the number of items that come before the target, never counting an item whose logit is NaN nor,
 *     with exclude_history != 0, a row of the key's valid history.  For every k in [1, 1024], 0 < rank <= k exactly when
 *     ctr_recommend_topk(user, hist, k, exclude_history) lists the target, at position rank - 1.
 *   out_rank[i] = -1 ("cannot be recommended") for a target outside [0, I), one with a NaN logit, or, with
 *     exclude_history, one in its own history.
 *   out_logit (may be NULL): the target's logit from the same scoring pass, bit for bit the logit the list reports for
 *     that row; NaN for a target outside [0, I).
 *   Keys with the same user row and history share one scoring pass (1024 targets at most; more take several), so the
 *     cost is about one ctr_recommend_topk per distinct (user, history) without its selection, plus one chunk re-scored
 *     per distinct chunk that holds a target.  Ranks do not depend on how keys are grouped into calls.
 *   Refusals write nothing: CTR_EINVAL for n < 1 and null inputs or out_rank; CTR_ESTATE for missing tables or ITEM_EMB,
 *     or more than INT32_MAX rows.
 *   Row-sharded ITEM_EMB (world > 1, large table): collective, under the same rule as ctr_knn_search — every rank calls
 *     with the same arguments and receives the same out_rank and out_logit, bit-identical to one GPU holding the whole
 *     table with the same weights and pred_batch; row ids stay global.  Each rank scores and counts its own shard's
 *     items, a target's logit comes from the rank that owns its row, and the ranks' counts are summed.  Disagreeing
 *     arguments (user, history or item rows) are CTR_EINVAL everywhere ("ranks disagree ..."), otherwise every rank
 *     returns the verdict of the lowest failing rank; no ctr_sync or host barrier is needed between training and this
 *     call, nor between this call and the next step.  It needs the user's history rows in shared memory (else
 *     CTR_ESTATE, as ctr_recommend_topk).  A replicated ITEM_EMB is ranked locally, by each rank alone.
 *   Runs on the engine stream under the handle's mutex, so it sees every update queued before it. */
int ctr_rank_items(ctr_handle* h, const int32_t* user_rows, const int32_t* hist_rows, const int32_t* item_rows, int64_t n,
                   int32_t exclude_history, int64_t* out_rank, float* out_logit);

/* ctr_rank_items with an exclusion mode (CTR_EXCLUDE_*), as ctr_recommend_topk_ex extends ctr_recommend_topk: max_ts [n]
 * is key i's cut under CTR_EXCLUDE_SEEN (may be NULL otherwise), a target in the key's seen set ranks -1, and for every
 * k in [1, 1024], 0 < rank <= k exactly when ctr_recommend_topk_ex(user, hist, max_ts, k, exclude) lists the target at
 * position rank - 1.  Under SEEN keys share a pass only with the same user row, history and max_ts.  Refusals as
 * ctr_recommend_topk_ex's, besides ctr_rank_items'.  On a row-sharded ITEM_EMB SEEN follows the owner rule of
 * CTR_EXCLUDE_SEEN: a target's verdict comes from the rank that owns its row, in the same exchange as its logit, and a
 * seen target still reports its logit.  The ranks must agree on max_ts as on the rows (CTR_EINVAL otherwise). */
int ctr_rank_items_ex(ctr_handle* h, const int32_t* user_rows, const int32_t* hist_rows, const int64_t* max_ts, const int32_t* item_rows, int64_t n,
                      int32_t exclude, int64_t* out_rank, float* out_logit);

/* Ranking metrics of ranks from ctr_rank_items / ctr_mlp_rank_items (host only, no device).  group[i] names key i's
 * group (normally the user, or the user and the window cut); m_g keys in group g; hit(k) = 0 < rank <= k.
 *   hit[a]    HR@ks[a]: the mean over keys of hit(ks[a])
 *   recall[a] Recall@ks[a]: the mean over groups of (hits in the group) / m_g
 *   ndcg[a]   NDCG@ks[a]: the mean over groups of DCG / IDCG, DCG = sum over hits of 1/log2(rank + 1),
 *             IDCG = sum_{j=1..min(m_g, k)} 1/log2(j + 1)
 *   mrr       the mean over keys of 1/rank (0 for -1)
 * A key of rank -1 is a miss and stays in every denominator.  Groups are taken in order of first appearance and every
 * sum is compensated in a fixed order, so a repeated call gives the same bits.  Each output may be NULL; hit, recall and
 * ndcg have nks entries.  CTR_EINVAL (nothing written) for n < 1, nks < 1, null rank / group / ks, a k < 1, or a rank
 * of 0 or below -1; the message is readable through ctr_last_error(NULL). */
int ctr_rank_metrics(const int64_t* rank, const int64_t* group, int64_t n, const int32_t* ks, int32_t nks,
                     double* hit, double* recall, double* ndcg, double* mrr);

/* ---- item2vec (BASELINE config 5; SURVEY.md §8f row f1) ------------------------------------------------
 * embedding.TrainEmbedding(ch, window, dim, iter) (feature/embedding/wordemb.go:9-32): SkipGram +
 * HierarchicalSoftmax word2vec over the users' item sequences; its output is the ITEM_EMB table the hot
 * path gathers from (recommend.Train, rcmd.go:207-213).  tokens are word ids in [0, vocab) in corpus
 * order — ids are assigned by first appearance, as dictionary.Add does (dictionary.go:70-81); the Go side
 * keeps the string↔id map.  emb_out [vocab, dim] float32 == GenEmbeddingMap32 (word2vec.go:298-324);
 * words rarer than min_count keep their initial vector (they are filtered from the training document only,
 * memory.go:53-62).  Stand-alone call: no handle; errors via ctr_last_error(NULL). */
typedef struct {
    int32_t dim, window, iter;            /* rcmd.go:22-26: 16, 5 ; iter 1 (rcmd.go:543) */
    int32_t min_count, max_depth;         /* options.go: 5, 100 */
    float   init_lr, min_lr, subsample;   /* 0.025, 0.025e-4, 1e-3 */
    int32_t update_lr_batch;              /* 100000 */
    uint32_t seed;
    int32_t device;
    int32_t reserved[8];
} ctr_i2v_config;
typedef struct {
    int64_t doc_len;                      /* tokens left after the MinCount filter */
    int64_t trained_positions;            /* positions that passed the subsampling trial, all iterations */
    int64_t pairs, node_visits;           /* (centre, context) pairs trained; Huffman nodes updated */
    double  algorithmic_bytes;            /* 2*dim*4 * (node_visits + pairs): row read-modify-writes */
    float   ms_device;                    /* device time of the training kernels */
    int32_t launches;
} ctr_i2v_stats;
void ctr_i2v_config_default(ctr_i2v_config* cfg);
/* host-only: the Huffman paths the trainer walks — dictionary.HuffnamTree (huffman.go:23-57) +
 * Node.GetPath(max_depth) (node.go:26-43) for word counts `count[vocab]`; path_off [vocab+1], then
 * (inner node id in creation order, child code) per step.  Runs without a GPU (used by the CPU tests). */
int  ctr_i2v_paths(const int64_t* count, int32_t vocab, int32_t max_depth, int64_t* path_off, int32_t* path_node, uint8_t* path_code, int64_t cap);
int  ctr_i2v_train(const ctr_i2v_config* cfg, const int32_t* tokens, int64_t n, int32_t vocab,
                   float* emb_out, ctr_i2v_stats* stats);
/* BASELINE configs[4] shape: the item stream sharded over `world` processes (one per GPU), every rank passes ITS shard.
 * Dictionary counts are all-reduced (NCCL) so every rank builds the identical Huffman tree; every rank trains a full
 * replica of both vector tables on its shard and the replicas are averaged (all-reduce) every sync_every centre
 * positions (0 = 4 Mi) — the reference's trainer is Hogwild over goroutines in one address space (word2vec.go:165-169);
 * across GPUs the shared memory becomes periodic model averaging.  The learning rate follows the GLOBAL position count.
 * emb_out receives the averaged table (identical on every rank; ranks that do not need it may pass NULL and save the
 * 4·vocab·dim-byte copy to the host); id = ncclUniqueId bytes from ctr_comm_unique_id on rank 0.
 * ctr_i2v_config.reserved[0] = 1 (single GPU only): sequential float64 parity mode — one warp walks the document in
 * order, reproducing the CPU restatement of the reference bit for bit (tests/test_gpu_i2v.py). */
int  ctr_i2v_train_dist(const ctr_i2v_config* cfg, const int32_t* tokens_shard, int64_t n_shard, int32_t vocab,
                        float* emb_out, ctr_i2v_stats* stats, int32_t rank, int32_t world,
                        const void* nccl_id, int32_t id_bytes, int64_t sync_every);
/* recommend.Train's embedding stage (rcmd.go:207-213, 538-545: GetItemEmbeddingModelFromUb → TrainEmbedding →
 * GenEmbeddingMap32 → the itemEmbeddingMap lookups) straight into the handle's ITEM_EMB, with no table crossing PCIe.
 * item_ids [n] is the item stream in corpus order, as ItemSeqGenerator yields it (one item per message, users
 * concatenated), as int64; every int64 value is a word, INT64_MIN included.  Word ids are assigned on the device by first
 * appearance (dictionary.Add, dictionary.go:70-81), and the trainer then runs exactly as ctr_i2v_train on that word-id
 * stream: MinCount filter, Huffman tree over all words, subsampling, lr schedule, and reserved[0] = 1 (sequential
 * float64 mode) alike.  n in [1, 2^31); the stream needs at least two distinct words.
 * ITEM_EMB becomes [idmap_n(CTR_IDMAP_ITEM), D]: row r holds the trained vector of the word whose item id the item map
 * sends to r; rows whose item never occurs are zero (rcmd.go:501-505, 519-521: missing item embedding → zeros); words
 * below min_count keep their initial vector, as GenEmbeddingMap32 has them; words without an item-map entry shape the
 * dictionary and the tree but land in no row.  Afterwards the handle is exactly as ctr_table_upload(ITEM_EMB, M) of that
 * matrix M would leave it: same allocation rules, row-Adam moments and hot-row accumulators reset.  When ITEM_EMB already
 * has that shape the rows are rewritten in place, otherwise the table is allocated as ctr_table_upload allocates it.
 * The rows are written only after training has succeeded: a refusal, or any error before that write, leaves ITEM_EMB
 * and its solver state as they were.
 * *vocab = V is written when vocab is non-NULL (also when V < 2 is refused); vocab_ids (may be NULL) receives the first
 * min(cap, V) words' item ids in word-id order (SaveVectors, the word ↔ row bookkeeping of a Searcher).  When vocab_ids
 * is non-NULL and cap < V, the handle keeps all V ids on the host until its next ctr_item_emb_train, and
 * ctr_item_emb_vocab reads them.  stats as ctr_i2v_train fills it.
 * CTR_EINVAL: null or short arguments, cfg->dim != D, a configuration ctr_i2v_train refuses, n out of range, fewer than
 * two distinct words.  CTR_ESTATE: no item id map.
 * world > 1: the call is collective.  Every rank passes its own shard of the item stream (n = 0 allowed, item_ids may
 * then be NULL; each rank's n below 2^31, the concatenation may be longer) and afterwards holds what one GPU holds after
 * the same call on the ranks' shards concatenated in rank order, except for two things: the trained vectors come from
 * ctr_i2v_train_dist's local SGD with model averaging (the replicas averaged every cfg->reserved[1] centre positions;
 * 0 selects 4 Mi), and stats is this rank's.  In detail:
 *   - vocabulary: word ids by first appearance in the concatenation; *vocab and vocab_ids are identical on every rank and
 *     equal, bit for bit, what one GPU returns for the concatenated stream (mapped items, unmapped ids, INT64_MIN, an id
 *     first seen on a later rank, a run of one id across a shard boundary alike);
 *   - training: MinCount, subsampling, the Huffman tree and the lr schedule use the global counts and token count; it
 *     runs on the handle's communicator and engine stream.  Words below min_count are never trained, but their rows
 *     pass through every replica average (an all-reduced sum, then a scale by 1/world): at world = 2 that gives the
 *     one-GPU initial vector bit for bit, at world > 2 the sum of the equal copies can round, by about one ulp per
 *     average;
 *   - table: ITEM_EMB ends as [idmap_n(CTR_IDMAP_ITEM), D] under the one-GPU rules (in place when it has that shape,
 *     otherwise allocated as ctr_table_upload allocates it, with the configuration's placement; moments and hot-row
 *     accumulators reset, and the next collective call republishes the shards and rebuilds the hot-row replica from
 *     the new rows).  A replicated table: every rank writes every row.  A row-sharded table: each rank writes only the
 *     rows it owns from its own replica (global row l·world + rank into local row l); the replicas are equal after the
 *     last average, so no rows travel;
 *   - agreement: the call starts with every rank's verdict, a hash of the configuration (cfg->device aside), ITEM_EMB's
 *     presence, shape and placement, the item map's size and digest and the ranks' token counts in one all-gather.
 *     Every rank returns the same code, and no refusal changes a map or a table: CTR_ESTATE when a rank has no item map;
 *     CTR_EINVAL when configurations, item maps or ITEM_EMB's shape or placement differ between ranks, for
 *     reserved[0] == 1 (the sequential mode is single-GPU), fewer than two distinct words in the concatenation, or
 *     every rank empty.  A CUDA or NCCL failure after the agreement (out of memory on one rank, say) can leave the
 *     ranks apart, as with the other collective calls;
 *   - vocab_ids: a rank cannot know how many unmapped ids the other ranks' streams bring, so cap may fall short of V;
 *     the whole vocabulary is then read back with ctr_item_emb_vocab (local, the same on every rank).
 *   Memory beside the one-GPU figures: the 8·R-byte first-occurrence tags (all-reduced); the ranks' side lists gathered
 *   (12 bytes per entry, world × the longest list); the merge's four 8-byte buffers per gathered entry (mt = the ranks'
 *   distinct unmapped ids summed, in place of u in the one-GPU figure's 32·u); and the trainer's two full replicas
 *   (8·V·D bytes) on every rank.
 * With world = 1 the call is single-GPU, n >= 1.
 * cfg->device is ignored: the handle's device is used.  Runs on the engine stream under the handle's mutex: ordered after
 * everything queued before it, and everything queued after it sees the new table.  The int64 stream is staged from
 * pageable memory through pinned bounce buffers.  Peak device memory beside the handle's own buffers, with R item-map
 * rows, m tokens without an item-map entry and u distinct such ids: at most 12·n + 24·m + 72·(R + u) bytes (+ sort
 * scratch) while numbering — the whole stream is never sorted, only its m unmapped tokens — then 9·n + 4·R bytes plus
 * ctr_i2v_train's vocabulary tables while training, and 4·V·D + 4·R bytes next to ITEM_EMB for the final write. */
int  ctr_item_emb_train(ctr_handle* h, const ctr_i2v_config* cfg, const int64_t* item_ids, int64_t n,
                        int64_t* vocab_ids, int64_t cap, int32_t* vocab, ctr_i2v_stats* stats);
/* The vocabulary the last ctr_item_emb_train kept because its vocab_ids could not take all of it (cap < V): *vocab = V,
 * and vocab_ids receives the first min(cap, V) item ids in word-id order.  Host memory only, not collective.
 * CTR_ESTATE when nothing is kept (that call returned every id, or failed before numbering, or none was made). */
int  ctr_item_emb_vocab(ctr_handle* h, int64_t* vocab_ids, int64_t cap, int32_t* vocab);

/* ---- model/mlp: the float64 MLP classifier of the reference's default path (BASELINE configs[0]; SURVEY.md §8a row
 * a11) — main.go:42-52 → model/mlp/mlp.go:45-65 (SimpleMlpFitWrap.Fit / SimpleMlpPredWrap.Predict: float32 samples →
 * float64 → nn.MLPClassifier) → nn/neural_network/basemlp64.go.  Float64 arithmetic on the device; packed parameter
 * vector in the reference's layout (basemlp64.go:459-463: per layer [intercepts | coefs row-major]).
 * Labels, classes and outputs (BaseMultilayerPerceptron64.Fit, basemlp64.go:578-598), decided at every cold initialise
 * from the labels the classifier sees (for ctr_mlp_fit_keys, the survivors'):
 *   - every label == 0 or == 1 (−0 counts as 0): no classes; one logistic output on binary_log_loss, and predict
 *     returns probabilities;
 *   - otherwise the classes are the distinct labels, ascending, widened to float64 (LabelBinarizer64, :1294-1313); ±0
 *     are one class, whose value keeps the sign of its first occurrence in sample order.  C >= 2 classes: C softmax
 *     outputs (exp, sum in column order, divide; no max subtraction, so an overflow gives NaN) on log_loss (:162-178),
 *     each sample's target the one-hot row of its class; C = 1 (every label one v not in {0, 1}): one logistic output
 *     on an all-ones target.  Predict returns float32(classes[MaxIdx64(outputs)]): the first strict maximum, so a
 *     NaN in output 0 wins and a NaN elsewhere never does (:917-931, mathCompat.go:93-101).  With C = 1, v.
 *   - a warm start of a fitted model keeps the output layer and needs the same classes (0 of them for binary labels).
 * The packed vector's last layer has max(1, C) outputs: np = Σ (1 + fi)·fo.  cfg.units[n_layers-1] is 1, the binary
 * width, as NOutputs comes from the labels in the reference.  Refused with CTR_EINVAL, changing nothing (DESIGN.md §2):
 * a NaN label, more than 1024 classes, and a warm start whose classes differ from the fitted ones.
 * The regressor (nn.MLPRegressor, multilayer_perceptron.go:9-71; ctr_mlp_regressor_create) shares the network, the
 * solvers and every fit rule, but has no labels: its targets are [n, units[n_layers-1]] float32, and the output kind is
 * decided at every cold initialise from all of them (basemlp64.go:502-511): some target not 0 or 1 → identity output
 * on square_loss (Σ (h − y)² / 2 / rows, :152-161); all 0 or 1 with one column → logistic on binary_log_loss, the
 * binary classifier bit for bit; all 0 or 1 with more columns → softmax on log_loss over the dense 0/1 rows (not
 * necessarily one-hot).  A warm start of a fitted regressor keeps its output kind.  A NaN or ±inf target is refused
 * with CTR_EINVAL, changing nothing (DESIGN.md §2). -------------- */
enum { CTR_MLP_RELU = 0, CTR_MLP_LOGISTIC = 1, CTR_MLP_IDENTITY = 2, CTR_MLP_TANH = 3 };
enum { CTR_MLP_SOLVER_ADAM = 0, CTR_MLP_SOLVER_SGD = 1 };                              /* Solver "adam" | "sgd" */
enum { CTR_MLP_LR_CONSTANT = 0, CTR_MLP_LR_INVSCALING = 1, CTR_MLP_LR_ADAPTIVE = 2 };  /* LearningRate */
enum { CTR_MLP_OUT_IDENTITY = 0, CTR_MLP_OUT_LOGISTIC = 1, CTR_MLP_OUT_SOFTMAX = 2 };   /* OutActivation */
typedef struct ctr_mlp ctr_mlp;
typedef struct {
    int32_t n_layers;                 /* len(layerUnits): hidden layers + 2 (basemlp64.go:495-497) */
    int32_t units[8];                 /* [nFeatures, HiddenLayerSizes..., 1]; the output width follows the labels (above) */
    int32_t hidden_act;               /* Activation "relu" (:229) | "logistic" | "identity" | "tanh"; one output is logistic (:423-425), more are softmax */
    int32_t batch, max_iter, n_iter_no_change;   /* BatchSize 200, MaxIter 200, NIterNoChange 10 (:233,238,254) */
    int32_t shuffle, adaptive;        /* Shuffle true (:241); LearningRate == "adaptive" */
    int32_t warm_start;               /* WarmStart (:245): keep the current parameters instead of re-initialising */
    uint32_t seed;                    /* init + shuffle counter RNG (the reference's source is time-seeded, :448,500) */
    int32_t device;
    double alpha, lr_init, beta1, beta2, eps, tol;   /* 1e-4, 1e-3, .9, .999, 1e-8, 1e-4 (:232-252) */
} ctr_mlp_config;
void ctr_mlp_config_default(ctr_mlp_config* cfg, int32_t n_features);      /* NewBaseMultilayerPerceptron64, :227-256 */
int  ctr_mlp_create(const ctr_mlp_config* cfg, ctr_mlp** out);             /* nn.NewMLPClassifier */
/* The solver surface of BaseMultilayerPerceptron64 beyond ctr_mlp_config (basemlp64.go:25-50).  "lbfgs",
 * EarlyStopping and BatchNormalize are not built; callers must reject them rather than drop them. */
typedef struct {
    int32_t solver;                   /* CTR_MLP_SOLVER_*: "adam" (:1075-1091) or "sgd" (SGDOptimizer64, :987-1039) */
    int32_t lr_schedule;              /* CTR_MLP_LR_*: "constant"; "invscaling": lr = lr_init / (t+1)^power_t at every epoch
                                       * end, t = samples seen since the last cold initialise (:999-1003, :814) — sgd only,
                                       * Adam treats it as "constant" (:1053); "adaptive" (:1005-1023, :1054-1073) */
    int32_t nesterov;                 /* NesterovsMomentum (sgd) */
    int32_t reserved0;                /* 0 */
    double power_t;                   /* PowerT .5 */
    double momentum;                  /* Momentum .9, in [0, 1] (sgd) */
    double weight_decay;              /* WeightDecay 0, in [0, 1): packed parameters *= (1 − wd) before every minibatch (:342-346) */
    double reserved[5];               /* 0 */
} ctr_mlp_options;
void ctr_mlp_options_default(ctr_mlp_options* opts);                       /* adam, constant, .5, .9, Nesterov, 0 */
/* ctr_mlp_create(cfg, out) == ctr_mlp_create_ex(cfg, NULL, out): default options, lr_schedule adaptive iff cfg->adaptive.
 * cfg->adaptive together with a non-adaptive opts->lr_schedule is CTR_EINVAL. */
int  ctr_mlp_create_ex(const ctr_mlp_config* cfg, const ctr_mlp_options* opts, ctr_mlp** out);
/* nn.NewMLPRegressor: cfg->units[n_layers-1] is the target count, in [1, 1024]; opts (may be NULL) and every other
 * argument are checked as by ctr_mlp_create_ex, before any device is looked for. */
int  ctr_mlp_regressor_create(const ctr_mlp_config* cfg, const ctr_mlp_options* opts, ctr_mlp** out);
void ctr_mlp_destroy(ctr_mlp* m);
const char* ctr_mlp_last_error(const ctr_mlp* m);
/* SimpleMlpFitWrap.Fit (mlp.go:45-65): X [n, xcols] float32, Y [n] float32 labels (classes as above) → fit (basemlp64.go:484-567 →
 * fitStochastic :729-857, solver adam or sgd).  The sample count t of "invscaling" carries over warm-start fits
 * (and ctr_mlp_set_params) and restarts at 0 whenever the parameters are initialised.  *n_iter = epochs run (NIter); loss_curve (may be NULL) receives max_iter
 * per-epoch losses at most. */
int  ctr_mlp_fit(ctr_mlp* m, const float* X, const float* Y, int64_t n, int32_t xcols, int32_t* n_iter, double* loss_curve);
/* SimpleMlpPredWrap.Predict (mlp.go:15-39): float32 [n] probabilities (the 64-bit class returns them raw,
 * basemlp64.go:897-931), or with classes installed the predicted class labels.  For a regressor, Y and out are
 * [n, units[n_layers-1]] row-major, and out is float32 of ctr_mlp_predict_f64's values, bit for bit. */
int  ctr_mlp_predict(ctr_mlp* m, const float* X, int64_t n, int32_t xcols, float* out);
/* The float64 output layer [n, units[n_layers-1]] of any fitted model: MLPRegressor.Predict (:53-62) for a regressor,
 * predictProbas (basemlp64.go:897-915) for a classifier. */
int  ctr_mlp_predict_f64(ctr_mlp* m, const float* X, int64_t n, int32_t xcols, double* out);
/* MLPRegressor.Score (:64-70 → r2Score64, basemlp64.go:1116-1141) on the device: per target column, mean = Σ y / n,
 * r2 = 1 − Σ (pred − y)² / Σ (y − mean)²; *r2 = the mean over the columns.  The sums are fixed-order reductions: the
 * same bits on every run.  CTR_EINVAL for a column whose Σ (y − mean)² is 0 (the reference panics), CTR_ESTATE for a
 * classifier (its accuracy score is ctr_mlp_accuracy) or an unfitted regressor. */
int  ctr_mlp_score(ctr_mlp* m, const float* X, const float* Y, int64_t n, int32_t xcols, double* r2);
/* MLPClassifier.Score (multilayer_perceptron.go:127-133 → AccuracyScore64, basemlp64.go:1143-1155) on the device: the
 * forward pass in chunks as ctr_mlp_predict runs it, the comparison and the count on the device, *acc = correct / n.
 * Y [n] holds the labels.  With classes a row is correct when classes[argmax] (ctr_mlp_predict's label) == (double)Y[i];
 * with one class that is "Y[i] == the class".  A binary model (labels all 0 or 1) compares, as the reference does, the
 * float64 PROBABILITY of ctr_mlp_predict_f64 with the label: a row counts only where that probability is exactly 0.0 or
 * 1.0 and equals its label (not the float32 probability of ctr_mlp_predict, nor a 0.5 threshold).  Equal, bit for bit,
 * to ctr_accuracy_score of Y against those predictions.  CTR_ESTATE on a regressor (its score is ctr_mlp_score) or
 * before a fit; CTR_EINVAL for null arguments, n < 1 or xcols != the network's inputs. */
int  ctr_mlp_accuracy(ctr_mlp* m, const float* X, const float* Y, int64_t n, int32_t xcols, double* acc);
/* The output kind (CTR_MLP_OUT_*).  A classifier's follows its classes.  To restore a regressor (the reference's JSON
 * carries OutActivation): ctr_mlp_set_output, then ctr_mlp_set_params; set_output leaves the model unfitted until
 * set_params.  set_output is CTR_ESTATE on a classifier, and CTR_EINVAL for a logistic output with more than one
 * target or a softmax with one (0/1 targets never make them). */
int  ctr_mlp_get_output(ctr_mlp* m, int32_t* kind);
int  ctr_mlp_set_output(ctr_mlp* m, int32_t kind);
/* The classifier fed by sample keys {UserId, ItemId, Timestamp, Label} from a feature store: no X on the host.  The
 * handle h is used only as the feature store — its id maps, USER_FEAT / ITEM_EMB / ITEM_FEAT tables, optional device
 * ubcache and uP, S, D, cF; its model kind and dense weights are not used.  m->units[0] must equal uP + S·D + D + cF.
 * fit: recommend.Train (rcmd.go:197-246) with mlp.SimpleMlpFitWrap — GetSample (rcmd.go:339-460) on the device, then
 *   ctr_mlp_fit.  Samples resolve as in ctr_train_keys: a key whose user or item is unknown is dropped, order kept; each
 *   survivor's history is GetUserBehavior(uid, S, -1, ts) from the ubcache (empty without one).  The classifier then
 *   trains on the survivors exactly as ctr_mlp_fit would on the X ctr_gather_rows builds for them, bit for bit: init
 *   or warm start, minibatches clipped to the survivor count, the shuffle over the survivors, solvers, weight decay,
 *   stopping rules and the t carry.  Each minibatch's float64 rows are gathered on the device into a [batch, nin]
 *   buffer the classifier owns; resident cost is about (S + 7)·4 bytes per survivor instead of nin·8.  *rows_used
 *   (may be NULL) = survivors; none is CTR_ENOTFOUND with the parameters untouched.  n in [1, 2^31).
 * predict: recommend.BatchPredict / Rank (rcmd.go:248-337) with model/mlp: keys → scores [n] (probabilities, or class
 *   labels as ctr_mlp_predict returns them, or a regressor's predicted values), in
 *   chunks of h's pred_batch, history windowed at each key's ts.  An unknown key scores as an all-zero X row, unless
 *   it is key 0, which fails the call with CTR_ENOTFOUND (rcmd.go:300-303).
 * A regressor takes each key's label as its target (one target: units[n_layers-1] must be 1, else CTR_EINVAL).
 * Refusals change nothing: CTR_EINVAL for null or short arguments, a width mismatch, or m and h on different devices;
 * CTR_ESTATE for a missing id map, missing tables, and predict before any fit or ctr_mlp_set_params.  The message is
 * readable through both ctr_mlp_last_error(m) and ctr_last_error(h).
 * Multi-GPU feature stores (world > 1): fit_keys is CTR_ESTATE — data-parallel float64 training would not keep fit's
 *   bit-for-bit result; fit on one GPU and serve the parameters on every rank through ctr_mlp_set_params, or train on
 *   every rank at once with ctr_mlp_fit_keys_dist (below), which replicates the fit instead.  predict with
 *   ITEM_EMB and ITEM_FEAT both replicated serves from this GPU's tables alone; with a row-sharded ITEM_EMB (ITEM_FEAT
 *   sharded or replicated) each rank scores its own keys and reads the rows from their owners, the hot rows from its
 *   replica, under ctr_batch_predict_keys' rule: the first call after a table change publishes the shard mappings and
 *   must run on every rank, and after training every rank calls ctr_sync and the processes meet at a barrier before
 *   predicting.  A replicated ITEM_EMB beside a sharded ITEM_FEAT is CTR_ESTATE.
 * Locking: both calls take h's mutex, then m's.  A caller that holds either object's lock across calls must take
 * them in the same order. */
int  ctr_mlp_fit_keys(ctr_mlp* m, ctr_handle* h, const int64_t* user_ids, const int64_t* item_ids, const int64_t* ts,
                      const float* label, int64_t n, int32_t* n_iter, double* loss_curve, int64_t* rows_used);
int  ctr_mlp_predict_keys(ctr_mlp* m, ctr_handle* h, const int64_t* user_ids, const int64_t* item_ids, const int64_t* ts,
                          int64_t n, float* scores);
/* ctr_mlp_fit_keys on a multi-GPU feature store, including a row-sharded ITEM_EMB that no GPU holds whole.  On world == 1
 * the call is ctr_mlp_fit_keys.  With world > 1 it is collective: every rank calls it with its OWN keys (n = 0 is allowed
 * there, with the arrays then possibly NULL).  The rule: afterwards every rank's m holds what ctr_mlp_fit_keys on one GPU
 * would hold after fitting on all ranks' keys concatenated in rank order, against a store holding the whole table:
 * parameters, classes / output kind, t, *n_iter, loss_curve and *rows_used (the survivors of all ranks), bit for bit.
 *   Training is replicated, not data-parallel: a step of this model is launch-bound, and what a row-sharded store
 *   prevents is reading the rows, not computing the step.  Each rank resolves and windows its own keys on the device
 *   with its own id maps and ubcache, exactly as fit_keys does: each key is windowed by the ubcache of the rank that
 *   passed it, so parity with one GPU assumes the ranks' ubcaches agree, as they do when they are kept live through the
 *   collective calls.  The survivor records (user row, item row, S history rows, label) are then all-gathered in rank
 *   order, counts first, and every rank runs the single-GPU fit over the same records in the same shuffled order with
 *   the same kernels.  Only layer 0's row gather differs: on a row-sharded ITEM_EMB it reads the hot rows from the rank's
 *   replica and the rest from their owners (ITEM_FEAT sharded or replicated), the same float32 rows, so the same float64
 *   ones (profile key mlp_fit_gather_peer; the record all-gather is mlp_fit_gather_ranks).  Nothing is all-reduced.  With
 *   ITEM_EMB and ITEM_FEAT both replicated each rank gathers from its own tables; a replicated ITEM_EMB beside a sharded
 *   ITEM_FEAT is CTR_ESTATE.
 *   Every rank checks its arguments and state, then the ranks exchange verdicts: if any rank fails, every rank returns
 *   the lowest failing rank's code and no model changes.  CTR_EINVAL everywhere: a ctr_mlp_config (the device aside) or
 *   ctr_mlp_options that differs across ranks, a model kind that differs, a warm start whose fitted state (fitted or
 *   not, output kind, classes, t, packed parameters) differs, a table placement that differs, or more than INT32_MAX
 *   keys in all.  No survivor on any rank is CTR_ENOTFOUND everywhere.  A CUDA or NCCL failure after the agreement
 *   follows the rule of the live-table calls above (ctr_idmap_insert): that rank returns the error and the models may
 *   differ.  Null m or h, n < 0, n > INT32_MAX, or a NULL array with n > 0 is CTR_EINVAL (null m or h before any
 *   collective work; a rank with other bad arguments still takes part in the agreement with its refusal).
 *   Ordering: on a row-sharded ITEM_EMB the call enters as the whole-table serving calls do (the shard mappings
 *   published, a device barrier behind every rank's queued row updates, the hot rows written back to their owners), so
 *   no ctr_sync or barrier is needed after training or a live-table write; the next collective call orders itself
 *   after this one likewise.
 *   Memory: the one-GPU cost of about (S + 7)·4 bytes per survivor, now for ALL ranks' survivors on every rank: the
 *   gathered records and the shuffle index take (S + 5)·4 bytes per survivor of the whole concatenation, beside this
 *   rank's own resolution arrays (the all-gather staging: 20 bytes per own key and S·4 per own survivor).  The
 *   all-gather moves (S + 3)·4 bytes per survivor to every rank.
 *   Locking: h's mutex, then m's, as ctr_mlp_fit_keys. */
int  ctr_mlp_fit_keys_dist(ctr_mlp* m, ctr_handle* h, const int64_t* user_ids, const int64_t* item_ids, const int64_t* ts,
                           const float* label, int64_t n, int32_t* n_iter, double* loss_curve, int64_t* rows_used);
/* Top-k recommendation over the whole item table with the classifier: the default recall recommend/api.go leaves as a
 * todo (api.go:115-118), for main.go's model.  h is the feature store, as for ctr_mlp_predict_keys.
 *   Users are external ids (h's user map); user j's history is GetUserBehavior(uid, S, -1, ts[j]) from the device
 *     ubcache, empty without one.  Every ITEM_EMB row is scored, as ctr_recommend_topk scores them; a missing ITEM_FEAT
 *     row reads as zeros.  Each item's score is bit for bit what ctr_mlp_predict_keys returns for (user, the item's id,
 *     ts[j]): the user's part of layer 0 is computed once and each item continues the same float64 chain.
 *   Order: output-layer logit (before the logistic) descending, then row ascending; a NaN logit never qualifies.
 *     exclude_history skips the rows of the user's window.  out_rows / out_scores (float32 probabilities) / out_logits
 *     (float64, may be NULL) are [nu, k]; out_count[j] may be less than k, and positions at or past it hold row -1,
 *     score 0 and logit 0.  A regressor with an identity output ranks by its predicted value, which is both the
 *     logit and, as float32, the score; one with a logistic output (0/1 targets) is the binary classifier.
 *   Refusals write nothing: CTR_EINVAL for k outside [1, 1024], nu < 1, null inputs or outputs and ctr_mlp_predict_keys'
 *     argument refusals; CTR_ESTATE for a classifier not fitted or with classes (it predicts labels, not a click
 *     probability), a model with more than one output, a missing id map or table; CTR_ENOTFOUND for any unknown user
 *     id, naming the first.
 *   Items are scored in chunks of h's pred_batch (whole tiles of 128) in the classifier's activation buffers,
 *     pred_batch · (units[1] + … + units[L-1]) · 8 bytes: a large catalogue wants a large pred_batch.  Only nu·k
 *     results cross PCIe.  Locking: h's mutex, then m's.
 *   Multi-GPU feature stores: with ITEM_EMB and ITEM_FEAT both replicated each rank serves alone from its own tables.
 *     On a row-sharded ITEM_EMB the call is collective, under ctr_recommend_topk's rule: every rank calls it with the
 *     same arguments and gets the same complete result, bit-identical to one GPU holding the whole table.  Each rank
 *     resolves the ids with its own id map; arguments or resolved rows that differ across ranks are CTR_EINVAL on
 *     every rank, else every rank returns the lowest failing rank's verdict (CTR_ENOTFOUND for an unknown user
 *     included).  Each user's window is the one rank 0's ubcache cuts (with equal caches, the single-GPU window);
 *     CTR_EXCLUDE_SEEN follows ctr_recommend_topk_ex's owner rule.  Each rank scores its own rows: per group of 256
 *     users one broadcast of rank 0's windows and one all-gather of the lists.  No ctr_sync is needed after training.
 *     Scratch: [world][min(nu, 256)][k] gathered lists, 12 bytes an entry, beside the single-GPU scratch. */
int  ctr_mlp_recommend_topk(ctr_mlp* m, ctr_handle* h, const int64_t* user_ids, const int64_t* ts, int64_t nu, int32_t k,
                            int32_t exclude_history, int32_t* out_rows, float* out_scores, double* out_logits, int32_t* out_count);
/* Full-catalogue rank of held-out items with the classifier, ctr_rank_items' definition over ctr_mlp_recommend_topk's
 * scoring: key i is (user_ids[i], item_ids[i], ts[i]); the user's window is GetUserBehavior(uid, S, -1, ts[i]), empty
 * without a ubcache.  out_rank[i] = 1 + the items before the target in the (float64 logit descending, row ascending)
 * order, NaN logits and (exclude_history) the window's rows never counting; -1 for a target that is excluded, has a
 * NaN logit, or whose item id h's item map does not hold.  For every k in [1, 1024], 0 < rank <= k exactly when
 * ctr_mlp_recommend_topk(user, ts, k, exclude_history) lists the target, at position rank - 1.  out_logit (may be NULL)
 * is the target's float64 logit, bit for bit the list's (NaN for an unknown item).  Keys with the same user and ts
 * share one scoring pass (1024 targets at most).
 *   Refusals write nothing: CTR_EINVAL for n outside [1, 2^31), null inputs or out_rank and ctr_mlp_predict_keys'
 *     argument refusals; CTR_ESTATE as ctr_mlp_recommend_topk (not fitted, classes, more than one output, a missing id
 *     map or table); CTR_ENOTFOUND for any unknown user id, naming the first.
 *   Locking: h's mutex, then m's; everything runs on h's stream.
 *   Multi-GPU feature stores as ctr_mlp_recommend_topk: collective on a row-sharded ITEM_EMB, the item ids hashed with
 *     the user ids and ts and the resolved rows compared; one broadcast of rank 0's windows per call, then per pass an
 *     all-gather of the targets' logits (8 bytes each, [world][m], and the owners' seen flags) and a sum of the
 *     counts. */
int  ctr_mlp_rank_items(ctr_mlp* m, ctr_handle* h, const int64_t* user_ids, const int64_t* item_ids, const int64_t* ts, int64_t n,
                        int32_t exclude_history, int64_t* out_rank, double* out_logit);
/* The classifier's recommendation and rank with an exclusion mode (CTR_EXCLUDE_*): the plain calls are these with
 * exclude_history ? CTR_EXCLUDE_WINDOW : CTR_EXCLUDE_NONE.  Under CTR_EXCLUDE_SEEN each key's ts is also its cut: every
 * item of the user's ubcache events with ts <= the key's ts (0: every event) is excluded, the window included.
 * CTR_EINVAL (nothing written) for an exclude outside the enum, besides the plain calls' refusals. */
int  ctr_mlp_recommend_topk_ex(ctr_mlp* m, ctr_handle* h, const int64_t* user_ids, const int64_t* ts, int64_t nu, int32_t k,
                               int32_t exclude, int32_t* out_rows, float* out_scores, double* out_logits, int32_t* out_count);
int  ctr_mlp_rank_items_ex(ctr_mlp* m, ctr_handle* h, const int64_t* user_ids, const int64_t* item_ids, const int64_t* ts, int64_t n,
                           int32_t exclude, int64_t* out_rank, double* out_logit);
/* packed parameter vector; ctr_mlp_get_params(m, NULL, 0, &np) returns the current length (it follows the classes) */
int  ctr_mlp_get_params(ctr_mlp* m, double* params, int64_t cap, int64_t* np);
int  ctr_mlp_set_params(ctr_mlp* m, const double* params, int64_t np);
/* the installed classes, ascending; *n = 0 for binary labels and for a regressor, on which set_classes is CTR_ESTATE.  get with classes == NULL returns only *n.  To restore a
 * model: ctr_mlp_set_classes, then ctr_mlp_set_params.  set_classes refuses (CTR_EINVAL, changing nothing) more than
 * 1024 classes, NaN and classes that are not strictly ascending; it sizes the output layer for them (n = 0: binary),
 * zeroing the parameters when the width changes, and the model counts as not fitted until ctr_mlp_set_params. */
int  ctr_mlp_get_classes(ctr_mlp* m, double* classes, int32_t cap, int32_t* n);
int  ctr_mlp_set_classes(ctr_mlp* m, const double* classes, int32_t n);

/* Multi-GPU (world > 1): one handle per rank/process.  The id is ncclUniqueId bytes produced on
 * rank 0 by ctr_comm_unique_id and distributed by the host (torch.distributed / Go). */
int ctr_comm_unique_id(void* id_out, int32_t* id_bytes /* in: capacity, out: used */);
int ctr_comm_init(ctr_handle* h, const void* id, int32_t id_bytes);

#ifdef __cplusplus
}
#endif
#endif
