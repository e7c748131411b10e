// ubcache.cuh — feature/ubcache on the device (SURVEY.md §8f row f2): per-user behaviour sequences in
// time-descending order (TimeSeq, cache.go:9-12) stored as one CSR in HBM, and TimeSeq.Filter
// (cache.go:71-94) evaluated for a whole batch: the first `count` items with ts <= maxTs.  Emits the
// [B,S] history-row matrix the train / predict entry points consume (most recent first, -1 padded:
// prepare.go:49-51, rcmd.go:517-522), removing the host from the per-sample path.
#pragma once
#include "common.cuh"

namespace ctr {

// First index in [beg, end) whose timestamp is <= mt (timestamps descend), or end.  Warp-cooperative: a few
// binary steps (uniform across the warp) narrow the range to 32 entries, then ONE coalesced load + ballot finishes —
// 3 dependent memory round trips for a 100-event history instead of 7.
__device__ __forceinline__ long long ub_first_leq(const long long* __restrict__ ts, long long beg, long long end, long long mt, int lane) {
    long long lo = beg, hi = end;                        // invariant: answer in [lo, hi]
    while (hi - lo > 32) { const long long mid = (lo + hi) >> 1; if (ts[mid] <= mt) hi = mid; else lo = mid + 1; }
    const long long i = lo + lane;
    const bool hit = i < hi && ts[i] <= mt;
    const unsigned m = __ballot_sync(0xffffffffu, hit);
    return m ? lo + (__ffs(m) - 1) : hi;
}

// one warp per sample: lower bound over the (descending) timestamps, then a coalesced
// write of up to S item rows
__global__ void __launch_bounds__(256)
k_ub_window(const long long* __restrict__ off, const long long* __restrict__ ts, const int* __restrict__ items,
            const int* __restrict__ user_row, const long long* __restrict__ max_ts, int B, int S, long n_users,
            int* __restrict__ hist) {
    const int lane = threadIdx.x & 31;
    const int nwarps = gridDim.x * (blockDim.x >> 5);
    for (int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); b < B; b += nwarps) {
        const int u = user_row[b];
        long long beg = 0, end = 0;
        if (u >= 0 && u < n_users) { beg = off[u]; end = off[u + 1]; }      // unknown user → empty (cache.go:61-64)
        long long first = end;
        if (end > beg) {
            long long mt = max_ts[b];
            if (mt == 0) mt = ts[beg];                                      // cache.go:72-74
            first = ub_first_leq(ts, beg, end, mt, lane);      // every lane of the warp takes this branch (u, beg, end are warp-uniform)
        }
        const long long avail = end - first;
        for (int s = lane; s < S; s += 32) hist[(long)b * S + s] = s < avail ? items[first + s] : -1;
    }
}

// The seen set of CTR_EXCLUDE_SEEN as a bitmap over this rank's local rows (rec.cuh, rec_seen): the item rows of user
// u's events with ts <= max_ts (max_ts == 0: every event; cache.go:71-94) and the window rows hist[0, S).  The events
// are one run [first, end) of the time-descending sequence; every block finds `first` with its first warp, then the grid
// strides over the run and the window.  Rows outside [0, n_items) are skipped; an unknown user, or no cache (off ==
// nullptr), adds no event.  On a row-sharded ITEM_EMB only the rows this rank owns are marked (global row r is local
// row r / world of rank r % world), so each row's verdict comes from its owner's cache; world = 1, rank = 0: the bitmap
// over the global rows.  seen (⌈local rows / 32⌉ words) is zeroed by the caller.
__global__ void __launch_bounds__(256)
k_ub_seen(const long long* __restrict__ off, const long long* __restrict__ ts, const int* __restrict__ items, long n_users, int u,
          long long max_ts, const int* __restrict__ hist, int S, long n_items, int world, int rank, unsigned* __restrict__ seen) {
    __shared__ long long first_s;
    long long beg = 0, end = 0;
    if (off && u >= 0 && u < n_users) { beg = off[u]; end = off[u + 1]; }
    if (threadIdx.x < 32) {
        long long first = beg;
        if (end > beg && max_ts != 0) first = ub_first_leq(ts, beg, end, max_ts, threadIdx.x);   // uniform across the warp
        if (threadIdx.x == 0) first_s = first;
    }
    __syncthreads();
    const long long first = first_s, ne = end - first;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < ne + S; i += (long long)gridDim.x * blockDim.x) {
        const int r = i < ne ? items[first + i] : hist[i - ne];
        if (r >= 0 && r < n_items && r % world == rank) {
            const int l = r / world;
            atomicOr(seen + (l >> 5), 1u << (l & 31));
        }
    }
}

// ---- updates: ctr_ubcache_append / ctr_ubcache_set rewrite the CSR into a spare buffer --------------------------
// A call touches T users (ascending rows tuser[k]).  Touched user k's stored segment is [ob[k], oe[k]) and its new
// events are [bb[k], bb[k] + bcnt[k]) of the batch arrays (bts, bit; time-descending within the segment).  dcum[k] is
// the exclusive prefix sum of the touched users' length changes, so every stored event of an untouched user between
// touched users k-1 and k moves by dcum[k], and user u's new offset is its old one plus dcum[#touched rows < u].

// old offset of user u; users at or past the stored count n_users start at n (and a missing cache has n_users = 0)
__device__ __forceinline__ long long ub_old_off(const long long* __restrict__ off, long long n_users, long long n, long long u) {
    return u < n_users ? off[u] : n;
}

// append's sort key, most significant first: user row, then ts descending (tmax - ts), so one radix sort orders the
// batch by (user, ts desc).  The batch is fed in reverse arrival order, so the stable sort breaks ties by later arrival
// first.  two_pass: the fields do not fit one 64-bit word; the ts key is sorted first and the user row second.
__global__ void __launch_bounds__(256)
k_ub_sort_keys(const int* __restrict__ user, const long long* __restrict__ ts, long long m, int tbits, long long tmax,
               bool two_pass, unsigned long long* __restrict__ key, int* __restrict__ idx) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < m; i += (long long)gridDim.x * blockDim.x) {
        const long long j = m - 1 - i;
        const unsigned long long tk = (unsigned long long)tmax - (unsigned long long)ts[j];
        key[i] = two_pass || tbits == 64 ? tk : ((unsigned long long)(unsigned)user[j] << tbits) | tk;
        idx[i] = (int)j;
    }
}

// two-pass sort: the user row of every element in its ts-sorted position
__global__ void __launch_bounds__(256)
k_ub_user_keys(const int* __restrict__ user, const int* __restrict__ idx, long long m, unsigned* __restrict__ ukey) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < m; i += (long long)gridDim.x * blockDim.x) ukey[i] = (unsigned)user[idx[i]];
}

// the batch in sorted order
__global__ void __launch_bounds__(256)
k_ub_gather_batch(const int* __restrict__ idx, const int* __restrict__ user, const long long* __restrict__ ts, const int* __restrict__ item,
                  long long m, int* __restrict__ bu, long long* __restrict__ bts, int* __restrict__ bit) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < m; i += (long long)gridDim.x * blockDim.x) {
        const int j = idx[i];
        bu[i] = user[j]; bts[i] = ts[j]; bit[i] = item[j];
    }
}

// per touched user: its stored segment and its length change (delta[T] = 0 closes the scan).  set (perm != nullptr):
// touched user k is set entry perm[k], whose events are [soff[e], soff[e+1]) and replace the stored ones.
__global__ void __launch_bounds__(256)
k_ub_touched(const int* __restrict__ tuser, const int* __restrict__ perm, const long long* __restrict__ soff, int T,
             const long long* __restrict__ off, long long n_users, long long n,
             int* __restrict__ bb, int* __restrict__ bcnt, long long* __restrict__ ob, long long* __restrict__ oe, long long* __restrict__ delta) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k > T) return;
    if (k == T) { delta[T] = 0; return; }
    const long long u = tuser[k];
    const long long b = ub_old_off(off, n_users, n, u), e = ub_old_off(off, n_users, n, u + 1);
    ob[k] = b; oe[k] = e;
    if (perm) {
        const int s = perm[k];
        bb[k] = (int)soff[s]; bcnt[k] = (int)(soff[s + 1] - soff[s]);
        delta[k] = (soff[s + 1] - soff[s]) - (e - b);
    } else delta[k] = bcnt[k];                                  // append: bb / bcnt come from the run-length encoding
}

// first k in [lo, hi) with a[k] > v (a non-decreasing), or hi
template <typename T>
__device__ __forceinline__ int ub_upper(const T* __restrict__ a, int lo, int hi, long long v) {
    while (lo < hi) { const int mid = (lo + hi) >> 1; if ((long long)a[mid] <= v) lo = mid + 1; else hi = mid; }
    return lo;
}

constexpr int kUbTile = 2048;                                  // elements per block of the offset / move kernels (256 threads)

// new offsets [0, new_users]: off(u) + dcum[#touched rows < u].  The block finds the touched users of its tile once,
// so a tile with none (the common case) does no per-element search.
__global__ void __launch_bounds__(256)
k_ub_offsets(const long long* __restrict__ off, long long n_users, long long n, const int* __restrict__ tuser, int T,
             const long long* __restrict__ dcum, long long new_users, long long* __restrict__ new_off) {
    __shared__ int klo, khi;
    const long long u0 = (long long)blockIdx.x * kUbTile;
    const long long u1 = min(u0 + kUbTile, new_users + 1) - 1;
    if (threadIdx.x == 0) { klo = ub_upper(tuser, 0, T, u0 - 1); khi = ub_upper(tuser, klo, T, u1 - 1); }
    __syncthreads();
    const int lo = klo, hi = khi;
    for (long long u = u0 + threadIdx.x; u <= u1; u += blockDim.x)
        new_off[u] = ub_old_off(off, n_users, n, u) + dcum[ub_upper(tuser, lo, hi, u - 1)];
}

// every stored event to its new place.  Untouched users: shifted by dcum.  A touched user's stored event moves past the
// user's new events with ts >= its own (append), or is dropped (set replaces the sequence).
template <bool REPLACE>
__global__ void __launch_bounds__(256)
k_ub_move_stored(const long long* __restrict__ ts, const int* __restrict__ items, long long n,
                 const long long* __restrict__ ob, const long long* __restrict__ oe, const long long* __restrict__ dcum, int T,
                 const int* __restrict__ bb, const int* __restrict__ bcnt, const long long* __restrict__ bts,
                 long long* __restrict__ ts_out, int* __restrict__ items_out) {
    __shared__ int klo, khi;
    __shared__ bool plain;
    const long long i0 = (long long)blockIdx.x * kUbTile;
    const long long i1 = min(i0 + kUbTile, n) - 1;
    if (threadIdx.x == 0) {
        klo = ub_upper(oe, 0, T, i0); khi = ub_upper(oe, klo, T, i1);
        plain = klo == khi && (klo == T || ob[klo] > i1);     // no touched segment meets the tile
    }
    // each thread moves 8 events, lane-contiguous: every load and store instruction of a warp covers 32 consecutive
    // events, so the stores stay coalesced whatever the shift.  The loads do not depend on the search, so they are
    // issued before the barrier and overlap it.
    long long t[8]; int it[8];
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const long long e = i0 + threadIdx.x + 256 * j;
        if (e <= i1) { t[j] = ts[e]; it[j] = items[e]; }
    }
    __syncthreads();
    const int lo = klo, hi = khi;
    const long long shift0 = dcum[lo];
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const long long e = i0 + threadIdx.x + 256 * j;
        if (e > i1) break;
        long long dst = e + shift0;
        if (!plain) {
            const int k = ub_upper(oe, lo, hi, e);
            dst = e + dcum[k];
            if (k < T && ob[k] <= e) {                             // a touched user's stored event
                if (REPLACE) continue;
                // its new events with ts >= its own come first (the batch segment is time-descending)
                int a = bb[k], z = bb[k] + bcnt[k];
                while (a < z) { const int mid = (a + z) >> 1; if (bts[mid] >= t[j]) a = mid + 1; else z = mid; }
                dst += a - bb[k];
            }
        }
        ts_out[dst] = t[j]; items_out[dst] = it[j];
    }
}

// every new event to its place, one warp per touched user: after the user's stored events with a strictly greater ts
// (append; set drops the stored ones), in batch order among the new ones
template <bool REPLACE>
__global__ void __launch_bounds__(256)
k_ub_place_new(const long long* __restrict__ ts, const long long* __restrict__ ob, const long long* __restrict__ oe,
               const long long* __restrict__ dcum, int T, const int* __restrict__ bb, const int* __restrict__ bcnt,
               const long long* __restrict__ bts, const int* __restrict__ bit, long long* __restrict__ ts_out, int* __restrict__ items_out) {
    const int lane = threadIdx.x & 31;
    const int nwarps = gridDim.x * (blockDim.x >> 5);
    for (int k = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); k < T; k += nwarps) {
        const long long b = ob[k], e = oe[k], base = b + dcum[k];
        const int s = bb[k], c = bcnt[k];
        for (int r = lane; r < c; r += 32) {
            const long long t = bts[s + r];
            long long g = 0;
            if (!REPLACE) {                                     // stored events with ts > t: first index with ts <= t
                long long a = b, z = e;
                while (a < z) { const long long mid = (a + z) >> 1; if (ts[mid] > t) a = mid + 1; else z = mid; }
                g = a - b;
            }
            ts_out[base + r + g] = t; items_out[base + r + g] = bit[s + r];
        }
    }
}

}  // namespace ctr
