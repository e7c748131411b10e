// idmap.cuh — sparse external id → dense table row, on the device (SURVEY.md §8f row f3).
// The reference keys every cache by the decimal string of a Go int (`strconv.Itoa(sampleKey.UserId)`,
// rcmd.go:472,483,502; `itemEmbeddingMap.Get`, :502,519) — MovieLens ids are sparse, the tables here are
// dense.  An open-addressing table (linear probing, load factor <= 0.5) in HBM maps int64 ids to int32
// rows; a missing id yields -1, which the gather turns into a zero row exactly like the reference's
// "embedding not found → zeros" (rcmd.go:501-505,519-521).
#pragma once
#include "common.cuh"
#include "ubcache.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_reduce.cuh>
#include <algorithm>

namespace ctr {

constexpr unsigned long long kIdEmpty = 0x8000000000000000ull;   // INT64_MIN is not a usable id

__device__ __forceinline__ unsigned long long idmap_hash(unsigned long long k) {
    k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
    return k;
}

__global__ void __launch_bounds__(256)
k_idmap_clear(unsigned long long* __restrict__ keys, int* __restrict__ vals, unsigned long long cap) {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < cap; i += (unsigned long long)gridDim.x * blockDim.x) {
        keys[i] = kIdEmpty; vals[i] = -1;
    }
}

// row of ids[i] is base + i.  flags[0] |= 1 on a duplicate id, |= 2 on the reserved id.
__global__ void __launch_bounds__(256)
k_idmap_insert(unsigned long long* __restrict__ keys, int* __restrict__ vals, unsigned long long mask,
               const long long* __restrict__ ids, long n, int* __restrict__ flags, int base) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const unsigned long long id = (unsigned long long)ids[i];
        if (id == kIdEmpty) { atomicOr(flags, 2); continue; }
        unsigned long long slot = idmap_hash(id) & mask;
        for (;;) {
            const unsigned long long prev = atomicCAS(&keys[slot], kIdEmpty, id);
            if (prev == kIdEmpty) { vals[slot] = base + (int)i; break; }
            if (prev == id) { atomicOr(flags, 1); atomicMin(&vals[slot], base + (int)i); break; }
            slot = (slot + 1) & mask;
        }
    }
}

// ctr_idmap_insert outgrowing its table: every entry of the old table (old_cap slots) into the cleared new one
__global__ void __launch_bounds__(256)
k_idmap_rehash(const unsigned long long* __restrict__ old_keys, const int* __restrict__ old_vals, unsigned long long old_cap,
               unsigned long long* __restrict__ keys, int* __restrict__ vals, unsigned long long mask) {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < old_cap; i += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long id = old_keys[i];
        if (id == kIdEmpty) continue;
        unsigned long long slot = idmap_hash(id) & mask;
        while (atomicCAS(&keys[slot], kIdEmpty, id) != kIdEmpty) slot = (slot + 1) & mask;   // ids are distinct
        vals[slot] = old_vals[i];
    }
}

// ctr_idmap_download: ids[row] = the id of every row (rows are dense, so every ids[r] is written)
__global__ void __launch_bounds__(256)
k_idmap_dump(const unsigned long long* __restrict__ keys, const int* __restrict__ vals, unsigned long long cap, long long* __restrict__ ids) {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < cap; i += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long id = keys[i];
        if (id != kIdEmpty) ids[vals[i]] = (long long)id;
    }
}

__global__ void __launch_bounds__(256)
k_idmap_lookup(const unsigned long long* __restrict__ keys, const int* __restrict__ vals, unsigned long long mask,
               const long long* __restrict__ ids, long n, int* __restrict__ rows) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const unsigned long long id = (unsigned long long)ids[i];
        int row = -1;
        if (id != kIdEmpty) {
            unsigned long long slot = idmap_hash(id) & mask;
            for (;;) {
                const unsigned long long k = __ldg(&keys[slot]);
                if (k == id) { row = __ldg(&vals[slot]); break; }
                if (k == kIdEmpty) break;
                slot = (slot + 1) & mask;
            }
        }
        rows[i] = row;
    }
}

// ---- ctr_idmap_insert with world > 1 (the ranks' ids concatenated in rank order) -----------------------------------
// *digest += a mix of every (id, row) pair of the map: the sum is order-independent, so maps holding the same pairs agree
// on it whatever their slot layout (the ranks compare it before any write).
__global__ void __launch_bounds__(256)
k_idmap_digest(const unsigned long long* __restrict__ keys, const int* __restrict__ vals, unsigned long long cap, unsigned long long* __restrict__ digest) {
    unsigned long long s = 0;
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < cap; i += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long id = keys[i];
        if (id != kIdEmpty) s += idmap_hash(id ^ idmap_hash(0x9e3779b97f4a7c15ull + (unsigned long long)(unsigned)vals[i]));
    }
    for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0 && s) atomicAdd(digest, s);
}

// The ranks' lists, all-gathered: rank j's distinct missing ids (ascending) and their first positions in its own ids sit at
// [j·stride, j·stride + cnt[j]).  Compacted to off[j] + e, each id is tagged (j << 32) | position: the tag orders
// entries as their positions in the concatenation of the ranks' ids do.
struct RankLists { long long off[kMaxPeers + 1]; int cnt[kMaxPeers]; };
__global__ void __launch_bounds__(256)
k_idmap_merge_ranks(const unsigned long long* __restrict__ ids, const int* __restrict__ pos, long stride, RankLists L, int world,
                    unsigned long long* __restrict__ key, unsigned long long* __restrict__ tag) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < (long)world * stride; i += (long)gridDim.x * blockDim.x) {
        const int j = (int)(i / stride);
        const long e = i - (long)j * stride;
        if (e >= L.cnt[j]) continue;
        key[L.off[j] + e] = ids[i];
        tag[L.off[j] + e] = ((unsigned long long)j << 32) | (unsigned)pos[i];
    }
}
struct MinPos { __device__ int operator()(int a, int b) const { return a < b ? a : b; } };       // first positions (ReduceByKey)
struct MinTag { __device__ unsigned long long operator()(unsigned long long a, unsigned long long b) const { return a < b ? a : b; } };

// Scratch of idmap_merge_ranks for m = L.off[world] gathered entries: key0, key1, tag0, tag1 [m] and tmp (this many bytes).
inline size_t idmap_merge_tmp_bytes(int m, cudaStream_t st) {
    size_t b1 = 0, b2 = 0, b3 = 0;
    unsigned long long* k = nullptr; int* u = nullptr;
    cub::DeviceRadixSort::SortPairs(nullptr, b1, k, k, k, k, m, 0, 64, st);
    cub::DeviceReduce::ReduceByKey(nullptr, b2, k, k, k, k, u, MinTag{}, m, st);
    cub::DeviceRadixSort::SortPairs(nullptr, b3, k, k, k, k, m, 0, 64, st);
    return std::max(b1, std::max(b2, b3));
}
// The first half of the merge: the gathered entries compacted and tagged, sorted by id, the smallest tag of each id kept
// (ReduceByKey(MinTag)).  key0 / tag0 [0, *u) receive the distinct ids ascending as uint64 and the tag of each one's
// first occurrence in the concatenation (ctr_item_emb_train's side words stop here).  Radix sorts and a keyed reduction
// over the same input: the result is the same on every rank.  Synchronises st (reads *u back).
inline cudaError_t idmap_merge_min(const unsigned long long* g_ids, const int* g_pos, long stride, const RankLists& L, int world,
                                   unsigned long long* key0, unsigned long long* key1, unsigned long long* tag0, unsigned long long* tag1,
                                   int* d_u, void* tmp, size_t tmp_bytes, int grid, cudaStream_t st, int* u) {
    const int m = (int)L.off[world];
    *u = 0;
    if (m == 0) return cudaSuccess;
    k_idmap_merge_ranks<<<grid, 256, 0, st>>>(g_ids, g_pos, stride, L, world, key0, tag0);
    size_t b = tmp_bytes;
    cudaError_t e = cub::DeviceRadixSort::SortPairs(tmp, b, key0, key1, tag0, tag1, m, 0, 64, st);
    if (e == cudaSuccess) { b = tmp_bytes; e = cub::DeviceReduce::ReduceByKey(tmp, b, key1, key0, tag1, tag0, d_u, MinTag{}, m, st); }
    if (e == cudaSuccess) e = cudaMemcpyAsync(u, d_u, sizeof(int), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    return e != cudaSuccess ? e : cudaGetLastError();
}
// The merge every rank runs on the same gathered lists: idmap_merge_min, then the distinct ids sorted by their tags.
// key1[0, *u) receives the distinct ids in order of first occurrence in the concatenation, the order a single-GPU
// insert of it gives new rows in.  Synchronises st.
inline cudaError_t idmap_merge_ranks(const unsigned long long* g_ids, const int* g_pos, long stride, const RankLists& L, int world,
                                     unsigned long long* key0, unsigned long long* key1, unsigned long long* tag0, unsigned long long* tag1,
                                     int* d_u, void* tmp, size_t tmp_bytes, int grid, cudaStream_t st, int* u) {
    int wbits = 0; while ((1 << wbits) < world) wbits++;
    cudaError_t e = idmap_merge_min(g_ids, g_pos, stride, L, world, key0, key1, tag0, tag1, d_u, tmp, tmp_bytes, grid, st, u);
    if (e != cudaSuccess || *u == 0) return e;
    size_t b = tmp_bytes;
    e = cub::DeviceRadixSort::SortPairs(tmp, b, tag0, tag1, key0, key1, *u, 0, 32 + wbits, st);
    return e != cudaSuccess ? e : cudaGetLastError();
}

__device__ __forceinline__ int idmap_find(const unsigned long long* __restrict__ keys, const int* __restrict__ vals,
                                          unsigned long long mask, unsigned long long id) {
    if (id == kIdEmpty) return -1;
    unsigned long long slot = idmap_hash(id) & mask;
    for (;;) {
        const unsigned long long k = __ldg(&keys[slot]);
        if (k == id) return __ldg(&vals[slot]);
        if (k == kIdEmpty) return -1;
        slot = (slot + 1) & mask;
    }
}

// First step of the item2vec dictionary over an item-id stream (ctr_item_emb_train): rows[i] = the row of ids[i], -1
// when the map has no entry; first_pos[row] = the smallest position of the row's id (first_pos starts at 0xFFFFFFFF);
// *n_side counts the tokens without an entry.  Positions ascend with the lane, so among the lanes of a warp holding
// one row the lowest lane carries the minimum, and a plain read skips the atomic once an earlier position is stored.
// ctr_idmap_insert's probe passes first_pos == nullptr: rows and the count only.
__global__ void __launch_bounds__(256)
k_idmap_first_pos(const unsigned long long* __restrict__ keys, const int* __restrict__ vals, unsigned long long mask,
                  const long long* __restrict__ ids, long n, int* __restrict__ rows, unsigned* __restrict__ first_pos,
                  unsigned long long* __restrict__ n_side) {
    const int lane = threadIdx.x & 31;
    for (long i0 = blockIdx.x * (long)blockDim.x + threadIdx.x; i0 < ((n + 31) & ~31L); i0 += (long)gridDim.x * blockDim.x) {
        const bool in = i0 < n;
        const int row = in ? idmap_find(keys, vals, mask, (unsigned long long)ids[i0]) : -1;
        if (in) rows[i0] = row;
        const unsigned side = __ballot_sync(0xffffffffu, in && row < 0);
        if (lane == 0 && side) atomicAdd(n_side, (unsigned long long)__popc(side));
        if (!first_pos) continue;
        const unsigned peers = __match_any_sync(0xffffffffu, row);
        if (row >= 0 && lane == __ffs(peers) - 1 && (unsigned)i0 < *(volatile unsigned*)(first_pos + row)) atomicMin(first_pos + row, (unsigned)i0);
    }
}

// The whole key → index step of recommend.BatchPredict (rcmd.go:277-337) in one launch, one warp per key:
// lanes 0/1 resolve the user / item id, the warp then evaluates TimeSeq.Filter (cache.go:71-94) for the
// user's behaviour CSR (ub_off == nullptr: no UserBehavior provider → empty history) and writes hist [B,S].
// BatchPredict's per-sample failure rule (rcmd.go:299-307): a key whose user or item feature cannot be
// fetched becomes an all-zero X row — user, item and every history slot are dropped together.
// keys3 = [user ids | item ids | timestamps], each B long.
__global__ void __launch_bounds__(256)
k_keys_resolve(const unsigned long long* __restrict__ ukeys, const int* __restrict__ uvals, unsigned long long umask,
               const unsigned long long* __restrict__ ikeys, const int* __restrict__ ivals, unsigned long long imask,
               const long long* __restrict__ ub_off, const long long* __restrict__ ub_ts, const int* __restrict__ ub_items, long n_users,
               const long long* __restrict__ keys3, int B, int S,
               int* __restrict__ user_row, int* __restrict__ item_row, int* __restrict__ hist) {
    const int lane = threadIdx.x & 31;
    const int nwarps = gridDim.x * (blockDim.x >> 5);
    for (int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); b < B; b += nwarps) {
        int row = -1;
        if (lane == 0) row = idmap_find(ukeys, uvals, umask, (unsigned long long)keys3[b]);
        else if (lane == 1) row = idmap_find(ikeys, ivals, imask, (unsigned long long)keys3[B + b]);
        int u = __shfl_sync(0xffffffffu, row, 0), it = __shfl_sync(0xffffffffu, row, 1);
        if (u < 0 || it < 0) { u = -1; it = -1; }
        long long first = 0, end = 0;
        if (ub_off && u >= 0 && u < n_users) {
            const long long beg = ub_off[u]; end = ub_off[u + 1]; first = end;
            if (end > beg) {
                long long mt = keys3[2 * (long)B + b];
                if (mt == 0) mt = ub_ts[beg];
                first = ub_first_leq(ub_ts, beg, end, mt, lane);
            }
        }
        const long long avail = end - first;
        for (int s = lane; s < S; s += 32) hist[(long)b * S + s] = s < avail ? ub_items[first + s] : -1;
        if (lane == 0) { user_row[b] = u; item_row[b] = it; }
    }
}

// ---- recommend.GetSample's assembly for training (rcmd.go:339-460), on the device -----------------------------
// A sample whose user or item has no features is skipped by the reference's assembler goroutines
// (rcmd.go:378-382: `continue` on GetSampleVector's error); here: flag → exclusive scan → ordered compaction.
__global__ void __launch_bounds__(256)
k_keys_rows(const unsigned long long* __restrict__ ukeys, const int* __restrict__ uvals, unsigned long long umask,
            const unsigned long long* __restrict__ ikeys, const int* __restrict__ ivals, unsigned long long imask,
            const long long* __restrict__ uid, const long long* __restrict__ iid, long n, int* __restrict__ flag) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
        flag[i] = (idmap_find(ukeys, uvals, umask, (unsigned long long)uid[i]) >= 0 &&
                   idmap_find(ikeys, ivals, imask, (unsigned long long)iid[i]) >= 0) ? 1 : 0;
}
// survivors are appended after the *count samples of the earlier chunks, input order kept
__global__ void __launch_bounds__(256)
k_keys_compact(const unsigned long long* __restrict__ ukeys, const int* __restrict__ uvals, unsigned long long umask,
               const unsigned long long* __restrict__ ikeys, const int* __restrict__ ivals, unsigned long long imask,
               const long long* __restrict__ uid, const long long* __restrict__ iid, const long long* __restrict__ ts,
               const float* __restrict__ label, long n, const int* __restrict__ flag, const int* __restrict__ pos,
               const unsigned long long* __restrict__ count, int* __restrict__ out_user, int* __restrict__ out_item,
               long long* __restrict__ out_ts, float* __restrict__ out_label) {
    const unsigned long long base = *count;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        if (!flag[i]) continue;
        const unsigned long long o = base + (unsigned long long)pos[i];
        out_user[o] = idmap_find(ukeys, uvals, umask, (unsigned long long)uid[i]);
        out_item[o] = idmap_find(ikeys, ivals, imask, (unsigned long long)iid[i]);
        out_ts[o] = ts[i]; out_label[o] = label[i];
    }
}
__global__ void k_keys_advance(const int* __restrict__ chunk_total, unsigned long long* __restrict__ count) { *count += (unsigned long long)*chunk_total; }

}  // namespace ctr
