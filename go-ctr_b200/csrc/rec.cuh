// rec.cuh — top-k recommendation over the whole item table (ctr_recommend_topk): the default recall the reference leaves
// as a todo (recommend/api.go:115-118).  DESIGN.md §1a row f6.
//
// One user's items are scored chunk by chunk by the ordinary forward (k_attn_fwd_user, the MLP GEMMs, k_head), which
// leaves the chunk's logits in h->Z.  The selection keeps the first k items under (logit descending, row ascending) in
// knn.cuh's list/buffer machinery with LogitKey: a NaN logit never qualifies, and the rows of the user's exclusion list
// are skipped.  The order is total, so the result depends neither on the chunk size nor on the slicing.
//   k_rec_scan:   grid = slices of the chunk; each CTA writes the top-k of its slice as it stands (empty entries included)
//   k_knn_merge<LogitKey>: merges the user's running list with the slices' lists
//   k_rec_finish: the users' lists → rows (-1 past the count), logits and scores (0 past the count), counts
// ctr_mlp_recommend_topk runs the same three kernels on the float64 MLP's logits, with Logit64Key.  Under
// CTR_EXCLUDE_SEEN the _seen siblings of k_rec_scan, k_rec_rank_sort and k_rec_rank test each row against the user's
// seen bitmap (k_ub_seen, ubcache.cuh) in place of the window's rows; on a row-sharded ITEM_EMB each rank's bitmap
// covers its own local rows, built from its own behaviour cache.
#pragma once
#include "knn.cuh"
#include "mlp64.cuh"

namespace ctr {
namespace rec {

using knn::LogitKey;
using knn::Logit64Key;
using knn::kEmptyRow;
using knn::kMaxK;
using knn::kStep;
using knn::kThreads;

// dynamic shared memory of k_rec_scan: the list/buffer state plus the exclusion rows that fall into the slice
template <class K>
__host__ inline size_t scan_smem_bytes(int k, int nex) { return knn::smem_bytes<K>(1, 0, k) + (size_t)nex * 4 + 16; }

// The seen set of CTR_EXCLUDE_SEEN (k_ub_seen, ubcache.cuh): a bitmap over the rank's local rows [0, N_local), bit
// l & 31 of word l >> 5 set when local row l (global row l·world + rank) is excluded; on a single table the global rows
// [0, I).  Any history length costs one word load per item and ⌈N_local / 32⌉ words, a 32·D-th of the rank's shard.
// The owner of a row decides: a target's verdict is read on its owner (k_rec_target_logits) and travels with its logit.
__device__ __forceinline__ bool rec_seen(const unsigned* __restrict__ seen, int row) { return (__ldg(seen + (row >> 5)) >> (row & 31)) & 1u; }

// z[b] is the logit of local row row0 + b, b < n; local row l is global row l·world + rank (a row-sharded ITEM_EMB; 1
// and 0 otherwise).  excl[0, nex): global rows that must not be returned (duplicates and rows outside the table are
// harmless).  run_s / run_r: the user's running list over the earlier chunks (nullptr for the first): only rows that
// beat its k-th entry can enter the result, so the slice lists start out filled with that entry — its row lies in an
// earlier chunk, so the fillers are told apart by row and written back as empty entries.
// Out: per slice the top-k list of global rows, [slices][k].  SEEN (k_rec_scan_seen): the local rows of the bitmap seen
// are excluded in place of excl.
template <class K, bool SEEN>
__device__ __forceinline__ void rec_scan(const typename K::T* __restrict__ z, int n, int row0, int world, int rank, int rows_per_slice,
                                         const int* __restrict__ excl, int nex, const unsigned* __restrict__ seen, int k,
                                         const typename K::T* run_s, const int* run_r,
                                         typename K::T* __restrict__ out_s, int* __restrict__ out_row) {
    using T = typename K::T;
    extern __shared__ __align__(16) char smem_raw[];
    const knn::Smem<K> sm = knn::carve<K>(smem_raw, 1, 0, k);
    int* ex = reinterpret_cast<int*>(smem_raw + knn::smem_bytes<K>(1, 0, k));
    __shared__ int nx;
    const int r0 = blockIdx.x * rows_per_slice, r1 = min(n, r0 + rows_per_slice);
    const T t_s = run_r ? run_s[k - 1] : K::empty();
    const int t_r = run_r ? run_r[k - 1] : kEmptyRow;
    for (int i = threadIdx.x; i < k; i += kThreads) { sm.ls[i] = t_s; sm.lr[i] = t_r; }
    if (threadIdx.x == 0) { sm.bn[0] = 0; nx = 0; }
    __syncthreads();
    if constexpr (!SEEN) {
        for (int i = threadIdx.x; i < nex; i += kThreads) {       // usually none of the user's rows fall into this slice
            const int e = __ldg(excl + i);
            const long b = (long)(e / world) - row0;
            if (e >= 0 && e % world == rank && b >= r0 && b < r1) ex[atomicAdd(&nx, 1)] = e;
        }
        __syncthreads();
    }
    const int m = nx;
    for (int base = r0; base < r1; base += kStep) {
#pragma unroll
        for (int r = 0; r < knn::kRows; r++) {
            const int b = base + threadIdx.x + r * kThreads;
            if (b >= r1) continue;
            const int row = (row0 + b) * world + rank;
            bool skip = false;
            if constexpr (SEEN) skip = rec_seen(seen, row0 + b);
            else for (int e = 0; e < m; e++) skip |= ex[e] == row;
            if (!skip) knn::offer(sm, 0, k, __ldg(z + b), row);
        }
        __syncthreads();
        knn::flush<1>(sm, k);
        __syncthreads();
    }
    for (int i = threadIdx.x; i < k; i += kThreads) {
        const bool filler = sm.lr[i] == t_r;
        out_s[(size_t)blockIdx.x * k + i] = filler ? K::empty() : sm.ls[i];
        out_row[(size_t)blockIdx.x * k + i] = filler ? kEmptyRow : sm.lr[i];
    }
}

template <class K>
__global__ void __launch_bounds__(kThreads) k_rec_scan(const typename K::T* __restrict__ z, int n, int row0, int world, int rank, int rows_per_slice,
                                                        const int* __restrict__ excl, int nex, int k,
                                                        const typename K::T* run_s, const int* run_r,
                                                        typename K::T* __restrict__ out_s, int* __restrict__ out_row) {
    rec_scan<K, false>(z, n, row0, world, rank, rows_per_slice, excl, nex, nullptr, k, run_s, run_r, out_s, out_row);
}

// k_rec_scan with the local rows of the bitmap seen excluded; dynamic shared memory scan_smem_bytes<K>(k, 0)
template <class K>
__global__ void __launch_bounds__(kThreads) k_rec_scan_seen(const typename K::T* __restrict__ z, int n, int row0, int world, int rank, int rows_per_slice,
                                                             const unsigned* __restrict__ seen, int k,
                                                             const typename K::T* run_s, const int* run_r,
                                                             typename K::T* __restrict__ out_s, int* __restrict__ out_row) {
    rec_scan<K, true>(z, n, row0, world, rank, rows_per_slice, nullptr, 0, seen, k, run_s, run_r, out_s, out_row);
}

// the single-table form (world = 1, rank = 0)
template <class K>
__global__ void __launch_bounds__(kThreads) k_rec_scan_seen(const typename K::T* __restrict__ z, int n, int row0, int rows_per_slice,
                                                             const unsigned* __restrict__ seen, int k,
                                                             const typename K::T* run_s, const int* run_r,
                                                             typename K::T* __restrict__ out_s, int* __restrict__ out_row) {
    rec_scan<K, true>(z, n, row0, 1, 0, rows_per_slice, nullptr, 0, seen, k, run_s, run_r, out_s, out_row);
}

// the score of a logit, bit-identical to what the predict route returns for the same sample: sigmoid32, the function
// k_head applies (ctr_predict_idx); the float64 MLP's logistic output narrowed to float32 (ctr_mlp_predict_keys)
__device__ __forceinline__ float rec_score(float z) { return sigmoid32(z); }
__device__ __forceinline__ float rec_score(double z) { return (float)mlp64_logistic(z); }

// n = users * k list entries
template <class K>
__global__ void k_rec_finish(const typename K::T* __restrict__ ls, const int* __restrict__ lr, int k, long n,
                             int32_t* __restrict__ out_row, typename K::T* __restrict__ out_logit, float* __restrict__ out_score,
                             int32_t* __restrict__ out_count) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const long j = i / k;
    const int p = (int)(i - j * k);
    const bool v = lr[i] != kEmptyRow;
    out_row[i] = v ? lr[i] : -1;
    out_logit[i] = v ? ls[i] : typename K::T(0);
    out_score[i] = v ? rec_score(ls[i]) : 0.0f;
    // valid entries are a prefix of the sorted list
    if (v && (p == k - 1 || lr[i + 1] == kEmptyRow)) out_count[j] = p + 1;
    if (!v && p == 0) out_count[j] = 0;
}

// ---- the rank of held-out items (ctr_rank_items / ctr_mlp_rank_items): the same scoring pass, counted instead of
// selected.  One pass holds m <= kMaxK targets of one (user, window).  rank = 1 + the items that come before the
// target in the list order (knn::better), NaN logits and the window's rows (nex > 0) never counting; -1 for a target
// outside [0, n_items), in the window, or with a NaN logit.  The target's logit is copied out of the pass's own scoring
// (k_rec_target_logits), so it is the list's logit bit for bit, and the counts are integer sums: deterministic.
//   k_rec_target_logits: per chunk holding a target, the logits of the chunk's targets
//   k_rec_rank_sort:     one CTA; the valid targets sorted in list order, each target's place, the bins zeroed
//   k_rec_rank<K>:       per chunk; each item's bin = the first sorted target it comes before (binary search), counted
//                        per CTA in shared memory, then one integer atomicAdd per bin
//   k_rec_rank_finish:   one CTA; rank of the target in place p = 1 + bins[0] + ... + bins[p]
// On a row-sharded ITEM_EMB (world > 1) each rank scores its own shard (local row l = global row l·world + rank): a
// target's logit comes from the rank that owns its row, the ranks' target logits are all-gathered into tl [world][tls]
// (target j read from slot rows[j] % world), every rank sorts the same targets, and the bins the ranks count over their
// shards are summed before k_rec_rank_finish.  With world = 1 and tls = m these are the single-table kernels.
// Under CTR_EXCLUDE_SEEN a target's verdict is its owner's: k_rec_target_logits also writes the owner's seen flag of
// each target it copies, the flags travel in the same all-gather as the logits ([world][tls], the same slots), and
// k_rec_rank_sort_seen reads them next to the logits.
constexpr int kRankThreads = 256;
constexpr int kRankRows = 2048;               // items per CTA of k_rec_rank

// z[b] is the logit of local row row0 + b, b < n (global row (row0 + b)·world + rank); tl[j] = the logit of target j
// when this rank owns rows[j] and it lies in this chunk.  seen (CTR_EXCLUDE_SEEN; nullptr otherwise): this rank's
// bitmap over its local rows, and flag[j] = whether that target is seen.
template <class T>
__global__ void k_rec_target_logits(const T* __restrict__ z, int n, int row0, int world, int rank, const int* __restrict__ rows, int m,
                                    T* __restrict__ tl, const unsigned* __restrict__ seen = nullptr, int* __restrict__ flag = nullptr) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    const int t = rows[j];
    if (t < 0 || t % world != rank) return;
    const long b = (long)(t / world) - row0;
    if (b >= 0 && b < n) {
        tl[j] = z[b];
        if (seen) flag[j] = rec_seen(seen, row0 + (int)b);
    }
}

// <<<1, kMaxK>>>.  tl [world][tls]: target j's logit at tl[(rows[j] % world)·tls + j].  place[j]: target j's place
// among the v valid targets (ties by index), -1 when invalid; ss / sr [v]: the valid targets' (logit, row) in list
// order; bins[0, m] zeroed.  n_items: the global row count.  SEEN: a target is excluded when its owner's flag
// (flag [world][tls], the slots of tl) is set, or on a single table (flag == nullptr) when the bitmap seen marks it.
template <class K, bool SEEN>
__device__ __forceinline__ void rec_rank_sort(const int* __restrict__ rows, const typename K::T* __restrict__ tl, int tls, int world, int m,
                                              long n_items, const int* __restrict__ excl, int nex, const unsigned* __restrict__ seen,
                                              const int* __restrict__ flag, int* __restrict__ place, int* __restrict__ nvalid,
                                              typename K::T* __restrict__ ss, int* __restrict__ sr, unsigned long long* __restrict__ bins) {
    using T = typename K::T;
    __shared__ T s[kMaxK];
    __shared__ int r[kMaxK];
    __shared__ int cnt;
    const int j = threadIdx.x;
    if (j == 0) cnt = 0;
    bool ok = false;
    if (j < m) {
        r[j] = rows[j];
        ok = r[j] >= 0 && r[j] < n_items;
        s[j] = ok ? tl[(size_t)(r[j] % world) * tls + j] : T(0);
        ok = ok && K::qualifies(s[j]);
        if constexpr (SEEN) ok = ok && !(flag ? flag[(size_t)(r[j] % world) * tls + j] : rec_seen(seen, r[j]));
        else for (int e = 0; e < nex && ok; e++) ok = __ldg(excl + e) != r[j];
        if (!ok) r[j] = -1;                                   // marks the target invalid for the others
    }
    for (int i = j; i <= m; i += blockDim.x) bins[i] = 0;
    __syncthreads();
    if (ok) atomicAdd(&cnt, 1);
    int p = -1;
    if (ok) {
        p = 0;
        for (int i = 0; i < m; i++)
            if (r[i] >= 0 && (knn::better(s[i], r[i], s[j], r[j]) || (i < j && s[i] == s[j] && r[i] == r[j]))) p++;
        ss[p] = s[j]; sr[p] = r[j];
    }
    if (j < m) place[j] = p;
    __syncthreads();
    if (j == 0) *nvalid = cnt;
}

template <class K>
__global__ void __launch_bounds__(kMaxK) k_rec_rank_sort(const int* __restrict__ rows, const typename K::T* __restrict__ tl, int tls, int world, int m,
                                                         long n_items, const int* __restrict__ excl, int nex, int* __restrict__ place,
                                                         int* __restrict__ nvalid, typename K::T* __restrict__ ss, int* __restrict__ sr,
                                                         unsigned long long* __restrict__ bins) {
    rec_rank_sort<K, false>(rows, tl, tls, world, m, n_items, excl, nex, nullptr, nullptr, place, nvalid, ss, sr, bins);
}

// k_rec_rank_sort with the targets their owners flag seen excluded: flag [world][tls] as tl (k_rec_target_logits)
template <class K>
__global__ void __launch_bounds__(kMaxK) k_rec_rank_sort_seen(const int* __restrict__ rows, const typename K::T* __restrict__ tl, int tls, int world, int m,
                                                              long n_items, const int* __restrict__ flag, int* __restrict__ place,
                                                              int* __restrict__ nvalid, typename K::T* __restrict__ ss, int* __restrict__ sr,
                                                              unsigned long long* __restrict__ bins) {
    rec_rank_sort<K, true>(rows, tl, tls, world, m, n_items, nullptr, 0, nullptr, flag, place, nvalid, ss, sr, bins);
}

// the single-table form (tl [m]): the rows of the bitmap seen (global rows) excluded
template <class K>
__global__ void __launch_bounds__(kMaxK) k_rec_rank_sort_seen(const int* __restrict__ rows, const typename K::T* __restrict__ tl, int m, long n_items,
                                                              const unsigned* __restrict__ seen, int* __restrict__ place, int* __restrict__ nvalid,
                                                              typename K::T* __restrict__ ss, int* __restrict__ sr, unsigned long long* __restrict__ bins) {
    rec_rank_sort<K, true>(rows, tl, m, 1, m, n_items, nullptr, 0, seen, nullptr, place, nvalid, ss, sr, bins);
}

// grid = slices of kRankRows items of the chunk z[0, n) (local rows row0 + b, global (row0 + b)·world + rank); the
// chunk's items counted into bins[0, v).  excl: global rows (duplicates, -1 and rows past the table are harmless).
template <class K>
__global__ void __launch_bounds__(kRankThreads) k_rec_rank(const typename K::T* __restrict__ z, int n, int row0, int world, int rank,
                                                           const int* __restrict__ excl, int nex, const typename K::T* __restrict__ ss,
                                                           const int* __restrict__ sr, const int* __restrict__ nvalid,
                                                           unsigned long long* __restrict__ bins) {
    using T = typename K::T;
    __shared__ T ks[kMaxK];
    __shared__ int kr[kMaxK];
    __shared__ int cb[kMaxK + 1];
    extern __shared__ int ex[];                              // the exclusion rows that fall into this slice
    __shared__ int nx;
    const int v = *nvalid;
    if (v == 0) return;
    const int r0 = blockIdx.x * kRankRows, r1 = min(n, r0 + kRankRows);
    for (int i = threadIdx.x; i < v; i += kRankThreads) { ks[i] = ss[i]; kr[i] = sr[i]; }
    for (int i = threadIdx.x; i <= v; i += kRankThreads) cb[i] = 0;
    if (threadIdx.x == 0) nx = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < nex; i += kRankThreads) {
        const int e = __ldg(excl + i);
        const long b = (long)(e / world) - row0;
        if (e >= 0 && e % world == rank && b >= r0 && b < r1) ex[atomicAdd(&nx, 1)] = e;
    }
    __syncthreads();
    const int mx = nx, lane = threadIdx.x & 31;
    for (int base = r0; base < r1; base += kRankThreads) {    // uniform per warp: every lane reaches the match
        const int b = base + threadIdx.x;
        int q = v;                                            // bin v: comes before no target
        if (b < r1) {
            const T s = __ldg(z + b);
            const int row = (row0 + b) * world + rank;
            bool skip = !K::qualifies(s);
            for (int e = 0; e < mx; e++) skip |= ex[e] == row;
            if (!skip) {
                int lo = 0, hi = v;                           // the first target this item comes before
                while (lo < hi) {
                    const int mid = (lo + hi) >> 1;
                    if (knn::better(s, row, ks[mid], kr[mid])) hi = mid; else lo = mid + 1;
                }
                q = lo;
            }
        }
        const unsigned peers = __match_any_sync(0xffffffffu, q);
        if (q < v && lane == __ffs(peers) - 1) atomicAdd(&cb[q], __popc(peers));
    }
    __syncthreads();
    for (int i = threadIdx.x; i < v; i += kRankThreads)
        if (cb[i]) atomicAdd(bins + i, (unsigned long long)cb[i]);
}

// k_rec_rank with the local rows of the bitmap seen excluded; no dynamic shared memory.  A copy of k_rec_rank's
// counting loop rather than a body shared with it: sharing changes k_rec_rank's register allocation.
template <class K>
__device__ __forceinline__ void rec_rank_seen(const typename K::T* __restrict__ z, int n, int row0, int world, int rank,
                                              const unsigned* __restrict__ seen, const typename K::T* __restrict__ ss, const int* __restrict__ sr,
                                              const int* __restrict__ nvalid, unsigned long long* __restrict__ bins) {
    using T = typename K::T;
    __shared__ T ks[kMaxK];
    __shared__ int kr[kMaxK];
    __shared__ int cb[kMaxK + 1];
    const int v = *nvalid;
    if (v == 0) return;
    const int r0 = blockIdx.x * kRankRows, r1 = min(n, r0 + kRankRows);
    for (int i = threadIdx.x; i < v; i += kRankThreads) { ks[i] = ss[i]; kr[i] = sr[i]; }
    for (int i = threadIdx.x; i <= v; i += kRankThreads) cb[i] = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    for (int base = r0; base < r1; base += kRankThreads) {    // uniform per warp: every lane reaches the match
        const int b = base + threadIdx.x;
        int q = v;                                            // bin v: comes before no target
        if (b < r1) {
            const T s = __ldg(z + b);
            const int row = (row0 + b) * world + rank;
            if (K::qualifies(s) && !rec_seen(seen, row0 + b)) {
                int lo = 0, hi = v;                           // the first target this item comes before
                while (lo < hi) {
                    const int mid = (lo + hi) >> 1;
                    if (knn::better(s, row, ks[mid], kr[mid])) hi = mid; else lo = mid + 1;
                }
                q = lo;
            }
        }
        const unsigned peers = __match_any_sync(0xffffffffu, q);
        if (q < v && lane == __ffs(peers) - 1) atomicAdd(&cb[q], __popc(peers));
    }
    __syncthreads();
    for (int i = threadIdx.x; i < v; i += kRankThreads)
        if (cb[i]) atomicAdd(bins + i, (unsigned long long)cb[i]);
}

template <class K>
__global__ void __launch_bounds__(kRankThreads) k_rec_rank_seen(const typename K::T* __restrict__ z, int n, int row0, int world, int rank,
                                                                const unsigned* __restrict__ seen, const typename K::T* __restrict__ ss,
                                                                const int* __restrict__ sr, const int* __restrict__ nvalid,
                                                                unsigned long long* __restrict__ bins) {
    rec_rank_seen<K>(z, n, row0, world, rank, seen, ss, sr, nvalid, bins);
}

// the single-table form (world = 1, rank = 0)
template <class K>
__global__ void __launch_bounds__(kRankThreads) k_rec_rank_seen(const typename K::T* __restrict__ z, int n, int row0, const unsigned* __restrict__ seen,
                                                                const typename K::T* __restrict__ ss, const int* __restrict__ sr,
                                                                const int* __restrict__ nvalid, unsigned long long* __restrict__ bins) {
    rec_rank_seen<K>(z, n, row0, 1, 0, seen, ss, sr, nvalid, bins);
}

// <<<1, kMaxK>>>: out_rank[j] and out_logit[j] (NaN for a row outside [0, n_items)); tl [world][tls] as for k_rec_rank_sort
template <class T>
__global__ void __launch_bounds__(kMaxK) k_rec_rank_finish(const int* __restrict__ rows, const T* __restrict__ tl, int tls, int world,
                                                           const int* __restrict__ place, int m, long n_items, const unsigned long long* __restrict__ bins,
                                                           long long* __restrict__ out_rank, T* __restrict__ out_logit) {
    __shared__ unsigned long long cum[kMaxK];
    const int j = threadIdx.x;
    if (j < m) cum[j] = bins[j];
    __syncthreads();
    for (int o = 1; o < m; o <<= 1) {                        // inclusive scan
        unsigned long long a = 0;
        if (j < m && j >= o) a = cum[j - o];
        __syncthreads();
        if (j < m) cum[j] += a;
        __syncthreads();
    }
    if (j >= m) return;
    const int p = place[j];
    out_rank[j] = p < 0 ? -1 : (long long)cum[p] + 1;
    const int t = rows[j];
    out_logit[j] = t >= 0 && t < n_items ? tl[(size_t)(t % world) * tls + j] : T(__longlong_as_double(0x7ff8000000000000ll));
}

// the fallback route: index buffers of B samples (user, item row0 + b, hist) for the ordinary attention kernels
__global__ void k_rec_fill_idx(int user, const int* __restrict__ hist, int S, int row0, int B, int* __restrict__ d_user,
                               int* __restrict__ d_item, int* __restrict__ d_hist) {
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < (long)B * S; i += (long)gridDim.x * blockDim.x) {
        const int b = (int)(i / S), s = (int)(i - (long)b * S);
        d_hist[i] = __ldg(hist + s);
        if (s == 0) { d_user[b] = user; d_item[b] = row0 + b; }
    }
}

}  // namespace rec
}  // namespace ctr
