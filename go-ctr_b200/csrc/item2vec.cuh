// item2vec.cuh — embedding.TrainEmbedding (feature/embedding/wordemb.go:9-32) on the device: wego word2vec
// SkipGram + HierarchicalSoftmax (model/word2vec/model.go:48-78, optimizer.go:107-129).  BASELINE config 5,
// SURVEY.md §8f row f1.  The dictionary counts, MinCount filter, Huffman tree (the reference's insertion
// procedure, huffman.go:23-57, in O(V log V)) and the per-word root→leaf paths are built on the host;
// both vector tables live in HBM: syn0 [V,D] (the item embeddings) and syn1 [V-1,D] (inner nodes).
//
// Kernel: one warp per centre position, Hogwild like the reference's goroutines (word2vec.go:165-169) but
// ~10^4 positions in flight.  A vector of D = 4*LPR floats is held by LPR lanes, so a warp walks the
// centre's Huffman path for 32/LPR contexts at once: per node one 128-bit load, a group dot product,
// the 1000-entry sigmoid table, a register axpy into tmp and a red.global.add.v4.f32 into the node
// vector; the context row takes tmp with one more red.add.  HBM/L2-bound: 2*D*4 bytes per visited node.
//
// Staleness compensation.  Sequential SGD (and the reference's <=NumCPU Hogwild goroutines) lets every
// update of the root see the previous one; with C (centre, context) pairs in flight the root would take
// C stale steps at once and |f| overshoots the +-6 cut-off for good.  So a vector that a fraction p of
// all pairs touches is stepped with lr / max(1, C*p): the C*p concurrent gradients are averaged rather
// than summed — top Huffman nodes (p = subtree frequency) and very frequent context items are damped,
// rare nodes and items (C*p < 1) get the exact update.  C itself is kept proportional to the vocabulary
// (small corpora run almost sequentially).  Deliberate adaptation to 10^3..10^5-way concurrency; quality is
// checked against the sequential float64 oracle (tests/test_gpu_i2v.py), the arithmetic of this kernel against a
// float64 model of one launch at every vector width (tests/test_gpu_i2v_kernel.py).
//
// What one warp sees of its own updates (measured on H100, tests/test_gpu_i2v_kernel.py tier A at D = 128): the
// contexts of one pass read the same node vectors; a later pass of the same centre reads the red.add of the earlier
// pass (same thread, same address), except for hot nodes, whose updates wait in shared memory until the next flush.
#pragma once
#include "common.cuh"
#include "idmap.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_reduce.cuh>
#include <algorithm>

namespace ctr {

__constant__ float c_i2v_lut[1000];       // sigmoid_table.go:28-45

struct I2vArgs {
    const int* doc; long nd;              // MinCount-filtered token ids
    const double* z;                      // [V] subsample keep threshold (subsample.go:34-38)
    const long long* poff; const int* pnode; const unsigned char* pcode;   // path CSR per word
    float* syn0; float* syn1; int D, W;
    const float* lr_tab; int upd;         // lr of positions [k*upd, (k+1)*upd)
    const float* node_scale;              // [V-1] 1/max(1, C*p_node)
    const float* word_scale;              // [V]   1/max(1, C*p_word)
    uint32_t seed; int iter;
    unsigned long long* counters;         // [0] trained positions, [1] (centre, context) pairs, [2] node visits
    int hot_base, hot_n;                  // inner nodes [hot_base, hot_base + hot_n) = the top of the Huffman tree
    long pos_begin, pos_end;              // this launch trains the centre positions [pos_begin, pos_end) of the document
};

// The top of the tree is on every path: the root alone would take one red.add per (pair, 16 bytes) on the same
// 16 L2 addresses.  Huffman nodes are numbered in creation order = non-decreasing subtree count, so the last
// kI2vHot nodes ARE the hottest ones: their updates are summed per block in shared memory (native f32 shared
// atomics) and flushed to HBM every kI2vFlush positions per warp — one global add per block instead of one per pair.
constexpr int kI2vHot = 64;
constexpr int kI2vFlush = 8;

template <int LPR>
__global__ void __launch_bounds__(256)
k_i2v_skipgram_hs(I2vArgs a) {
    constexpr int RPW = 32 / LPR, D = 4 * LPR;
    extern __shared__ float s_acc[];           // [hot_n, D] this block's pending updates of the hot nodes
    const int lane = threadIdx.x & 31, lir = lane % LPR, sub = lane / LPR;
    const long nwarps = (long)gridDim.x * (blockDim.x >> 5);
    const long gwarp = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const long niter = (a.pos_end - a.pos_begin + nwarps - 1) / nwarps;
    unsigned long long n_tr = 0, n_pair = 0, n_node = 0;
    for (int i = threadIdx.x; i < a.hot_n * D; i += blockDim.x) s_acc[i] = 0.0f;
    __syncthreads();
    for (long it = 0; it < niter; it++) {
        const long pos = a.pos_begin + it * nwarps + gwarp;
        bool train = pos < a.pos_end;
        int id = 0;
        if (train) {
            id = a.doc[pos];
            // Subsampler.Trial (subsample.go:45-52): train when z[id] > U[0,1)
            const double u = (double)(mix64(a.seed, 200u + (uint32_t)a.iter, (uint64_t)pos) >> 11) * (1.0 / 9007199254740992.0);
            train = a.z[id] > u;
        }
        if (train) {
            const int del = (int)(mix64(a.seed, 300u + (uint32_t)a.iter, (uint64_t)pos) % (uint64_t)a.W);   // modelutil.NextRandom(window)
            const float lr = a.lr_tab[pos / a.upd];
            const long long p0 = a.poff[id]; const int np = (int)(a.poff[id + 1] - p0);
            const int nctx = 2 * (a.W - del);                                   // a in [del, 2W+1-del), a != W
            n_tr++;
            for (int k0 = 0; k0 < nctx; k0 += RPW) {
                const int k = k0 + sub;
                int aa = del + k; if (aa >= a.W) aa++;
                const long cpos = pos - a.W + aa;
                const bool active = k < nctx && cpos >= 0 && cpos < a.nd;       // model.go:63-66
                const int cid = active ? a.doc[cpos] : 0;
                float* cptr = a.syn0 + (long)cid * D + lir * 4;
                const float4 c = active ? *reinterpret_cast<const float4*>(cptr) : zero4();
                float4 tmp = zero4();
                bool alive = active;
                if (active && lir == 0) n_pair++;
                for (int i = 0; i < np; i++) {                                  // optimizer.go:113-128
                    if (__ballot_sync(0xffffffffu, alive) == 0u) break;
                    const int node = a.pnode[p0 + i];
                    float* nptr = a.syn1 + (long)node * D + lir * 4;
                    const float4 nv = *reinterpret_cast<const float4*>(nptr);
                    const float f = group_sum<LPR>(dot4(c, nv));
                    if (alive && (f <= -6.0f || f >= 6.0f)) alive = false;      // `return`: the rest of the path is abandoned
                    if (alive) {
                        // clamped: in float32 f = nextafterf(6, 0) rounds f + 6 up to 12 and the product to 1000, one past the table
                        const int bin = min((int)((f + 6.0f) * (1000.0f / 6.0f / 2.0f)), 999);
                        const float g = (1.0f - (float)a.pcode[p0 + i] - c_i2v_lut[bin]) * lr;
                        tmp = fma4(g, nv, tmp);
                        const float gs = g * __ldg(a.node_scale + node);
                        const int hs = node - a.hot_base;
                        if (hs >= 0) {
                            float* sp = s_acc + hs * D + lir * 4;
                            atomicAdd(sp + 0, gs * c.x); atomicAdd(sp + 1, gs * c.y); atomicAdd(sp + 2, gs * c.z); atomicAdd(sp + 3, gs * c.w);
                        } else {
                            red_add4(nptr, make_float4(gs * c.x, gs * c.y, gs * c.z, gs * c.w));
                        }
                        if (lir == 0) n_node++;
                    }
                }
                if (active) {                                                   // model.go:74-76
                    const float ws = __ldg(a.word_scale + cid);
                    red_add4(cptr, make_float4(ws * tmp.x, ws * tmp.y, ws * tmp.z, ws * tmp.w));
                }
            }
        }
        if (a.hot_n > 0 && ((it % kI2vFlush) == kI2vFlush - 1 || it == niter - 1)) {       // uniform across the block
            __syncthreads();
            for (int i = threadIdx.x; i < a.hot_n * D; i += blockDim.x) {
                const float v = s_acc[i];
                if (v != 0.0f) { atomicAdd(a.syn1 + (long)a.hot_base * D + i, v); s_acc[i] = 0.0f; }
            }
            __syncthreads();
        }
    }
    n_tr = (lane == 0) ? n_tr : 0;
    for (int o = 16; o > 0; o >>= 1) {
        n_pair += __shfl_xor_sync(0xffffffffu, n_pair, o); n_node += __shfl_xor_sync(0xffffffffu, n_node, o);
    }
    if (lane == 0) {
        if (n_tr) atomicAdd(a.counters + 0, n_tr);
        if (n_pair) atomicAdd(a.counters + 1, n_pair);
        if (n_node) atomicAdd(a.counters + 2, n_node);
    }
}

// -------------------------------------------------------------------------------------------------------------------
// Sequential float64 mode (ctr_i2v_config.reserved[0] = 1): ONE warp walks the document in order, float64 tables and
// arithmetic, no staleness compensation, no hot-node aggregation — the reference's algorithm as a single goroutine
// would run it (word2vec.go:198-221, model.go:48-78, optimizer.go:107-129), operation for operation: the dot product
// is accumulated in element order, multiplications and additions are rounded separately (the CPU restatement is
// built without FMA contraction), the sigmoid comes from the same 1000-entry table.  It exists for PARITY: on the same
// tokens it reproduces oracle/i2v_oracle.c bit for bit (tests/test_gpu_i2v.py), which pins the host plan both kernels
// are given: the device-side dictionary filter, subsample thresholds, Huffman paths and learning-rate schedule.  The
// parallel kernel above shares no code with this one below that plan; its own draws, window enumeration and update
// arithmetic are pinned by tests/test_gpu_i2v_kernel.py.  Throughput is irrelevant here (~10^5 tokens/s).
// -------------------------------------------------------------------------------------------------------------------
struct I2vSeqArgs {
    const int* doc; long nd; long n_stream;
    const double* z;
    const long long* poff; const int* pnode; const unsigned char* pcode;
    double* syn0; double* syn1; const double* lut;      // lut: 1000-entry sigmoid table in float64
    int D, W, upd, iters;
    double init_lr, min_lr;
    uint32_t seed;
    unsigned long long* counters;
};
__global__ void __launch_bounds__(32)
k_i2v_seq_f64(I2vSeqArgs a) {
    constexpr int MAXJ = 4;                              // D <= 128
    const int lane = threadIdx.x;
    const int D = a.D, nj = (D + 31) / 32;
    unsigned long long n_tr = 0, n_pair = 0, n_node = 0;
    double lr = a.init_lr;                               // w.currentlr persists across iterations
    for (int iter = 0; iter < a.iters; iter++) {
        long seen = 0;
        for (long pos = 0; pos < a.nd; pos++) {
            const int id = a.doc[pos];
            const double u = (double)(mix64(a.seed, 200u + (uint32_t)iter, (uint64_t)pos) >> 11) * (1.0 / 9007199254740992.0);
            if (a.z[id] > u) {                           // Subsampler.Trial, subsample.go:45-52
                const int del = (int)(mix64(a.seed, 300u + (uint32_t)iter, (uint64_t)pos) % (uint64_t)a.W);
                const long long p0 = a.poff[id]; const int np = (int)(a.poff[id + 1] - p0);
                for (int aa = del; aa < a.W * 2 + 1 - del; aa++) {          // model.go:59-77
                    if (aa == a.W) continue;
                    const long cpos = pos - a.W + aa;
                    if (cpos < 0 || cpos >= a.nd) continue;
                    double* ctx = a.syn0 + (long)a.doc[cpos] * D;
                    double c[MAXJ], tmp[MAXJ];
#pragma unroll
                    for (int j = 0; j < MAXJ; j++) { const int k = lane + 32 * j; c[j] = (j < nj && k < D) ? ctx[k] : 0.0; tmp[j] = 0.0; }
                    n_pair++;
                    for (int i = 0; i < np; i++) {                           // optimizer.go:113-128
                        double* nvp = a.syn1 + (long)a.pnode[p0 + i] * D;
                        double nv[MAXJ], prod[MAXJ];
#pragma unroll
                        for (int j = 0; j < MAXJ; j++) { const int k = lane + 32 * j; nv[j] = (j < nj && k < D) ? nvp[k] : 0.0; prod[j] = __dmul_rn(c[j], nv[j]); }
                        double inner = 0.0;                                  // element order k = 0 .. D-1, like the scalar loop
                        for (int k = 0; k < D; k++) {
                            const int j = k >> 5;
                            const double pj = j == 0 ? prod[0] : j == 1 ? prod[1] : j == 2 ? prod[2] : prod[3];
                            inner = __dadd_rn(inner, __shfl_sync(0xffffffffu, pj, k & 31));
                        }
                        if (inner <= -6.0 || inner >= 6.0) break;            // `return`: abandons the rest of the path
                        const double g = __dmul_rn(__dadd_rn(__dadd_rn(1.0, -(double)a.pcode[p0 + i]), -a.lut[(int)((inner + 6.0) * (1000.0 / 6.0 / 2.0))]), lr);
#pragma unroll
                        for (int j = 0; j < MAXJ; j++) {
                            const int k = lane + 32 * j;
                            if (j < nj && k < D) { tmp[j] = __dadd_rn(tmp[j], __dmul_rn(g, nv[j])); nvp[k] = __dadd_rn(nv[j], __dmul_rn(g, c[j])); }
                        }
                        n_node++;
                        __syncwarp();
                    }
#pragma unroll
                    for (int j = 0; j < MAXJ; j++) { const int k = lane + 32 * j; if (j < nj && k < D) ctx[k] = __dadd_rn(c[j], tmp[j]); }
                    __syncwarp();
                }
                n_tr++;
            }
            seen++;                                      // observe(), word2vec.go:223-233
            if (seen % a.upd == 0) lr = lr < a.min_lr ? a.min_lr : a.init_lr * (1.0 - (double)seen / (double)a.n_stream);
        }
    }
    if (lane == 0) { a.counters[0] = n_tr; a.counters[1] = n_pair; a.counters[2] = n_node; }
}
__global__ void k_i2v_init64(double* __restrict__ syn0, long n, int D, uint32_t seed) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const double u = (double)(mix64(seed, 100u, (uint64_t)i) >> 11) * (1.0 / 9007199254740992.0);
        syn0[i] = (u - 0.5) / (double)D;
    }
}
__global__ void k_f64_to_f32_i2v(const double* __restrict__ a, float* __restrict__ b, long n) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) b[i] = (float)a[i];
}

// -------------------------------------------------------------------------------------------------------------------
// Dictionary / Huffman plan on the device (the host used to spend 85 % of the end-to-end time here).  What stays on the
// host is the O(V) two-queue merge over the count-sorted leaves — everything proportional to the stream length
// (counting, the MinCount filter) or to V * depth (the per-word root->leaf paths) runs here.
// -------------------------------------------------------------------------------------------------------------------
// dictionary.Add (dictionary.go:70-81): occurrences per word id.  Warp-aggregated: lanes holding the same id add once.
__global__ void __launch_bounds__(256)
k_i2v_count(const int* __restrict__ tok, long n, int V, unsigned long long* __restrict__ cnt, int* __restrict__ bad) {
    for (long i0 = (blockIdx.x * (long)blockDim.x + threadIdx.x); i0 < ((n + 31) & ~31L); i0 += (long)gridDim.x * blockDim.x) {
        const bool in = i0 < n;
        const int id = in ? tok[i0] : -1;
        if (in && (id < 0 || id >= V)) { *bad = 1; }
        const bool ok = in && id >= 0 && id < V;
        const unsigned peers = __match_any_sync(0xffffffffu, ok ? id : -1);
        if (ok && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(cnt + id, (unsigned long long)__popc(peers));
    }
}
// keep[i] = 1 when the word survives the MinCount filter (memory.go:53-62, cpsutil.go:74-78)
__global__ void __launch_bounds__(256)
k_i2v_keep(const int* __restrict__ tok, long n, const unsigned long long* __restrict__ cnt, int min_count, unsigned char* __restrict__ keep) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
        keep[i] = !(0 <= min_count && cnt[tok[i]] < (unsigned long long)min_count);
}
// subsample threshold z = max(0, 1 - sqrt(t / count)) (subsample.go:34-38), staleness scale of a word, sort keys
__global__ void __launch_bounds__(256)
k_i2v_word_tables(const unsigned long long* __restrict__ cnt, int V, double subsample, double ceff, double total,
                  double* __restrict__ z, float* __restrict__ word_scale, unsigned long long* __restrict__ sort_key, int* __restrict__ sort_val) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < V; i += gridDim.x * blockDim.x) {
        const double c = (double)cnt[i];
        const double v = c > 0.0 ? 1.0 - sqrt(subsample / c) : 0.0;
        z[i] = v < 0.0 ? 0.0 : v;
        if (word_scale) word_scale[i] = (float)(1.0 / fmax(1.0, ceff * c / total));
        if (sort_key) { sort_key[i] = cnt[i]; sort_val[i] = i; }
    }
}
__global__ void __launch_bounds__(256)
k_i2v_node_scale(const long long* __restrict__ node_val, int nn, double ceff, double total, float* __restrict__ node_scale) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nn; i += gridDim.x * blockDim.x)
        node_scale[i] = (float)(1.0 / fmax(1.0, ceff * (double)node_val[i] / total));
}
// Node.GetPath(maxDepth) (node.go:26-43) from the parent / code arrays of the tree: pass 0 writes the number of
// (inner node, child code) steps of every word, pass 1 (after an exclusive scan) the steps in root -> leaf order.
__global__ void __launch_bounds__(256)
k_i2v_paths(const int* __restrict__ parent, const unsigned char* __restrict__ code, const unsigned long long* __restrict__ cnt, int V, int max_depth, int pass,
            long long* __restrict__ poff, int* __restrict__ pnode, unsigned char* __restrict__ pcode) {
    for (int w = blockIdx.x * blockDim.x + threadIdx.x; w < V; w += gridDim.x * blockDim.x) {
        if (cnt[w] == 0) { if (pass == 0) poff[w] = 0; continue; }             // an id that never occurs has no path (never trained)
        int len = 0;
        for (int p = w; p != -1; p = parent[p]) len++;                         // leaf .. root, both included
        const int depth = max_depth < len ? max_depth : len;
        const int steps = depth > 0 ? depth - 1 : 0;
        if (pass == 0) { poff[w] = steps; continue; }
        // chain[len-1-i] for i < steps = the i-th node from the root: reached after len-1-i parent hops from the leaf
        long long o = poff[w];
        // walk once from the leaf, emitting when the position from the root is < steps
        int p = w, child = -1;
        for (int h = 0; h <= len - 1; h++) {                                   // h hops done: p = chain[h]
            const int i_from_root = len - 1 - h;                               // p is chain[len-1-i] with i = i_from_root
            if (h > 0 && i_from_root < steps) { pnode[o + i_from_root] = p - V; pcode[o + i_from_root] = code[child]; }
            child = p; p = parent[p];
        }
    }
}
// element-wise mean of `world` replicas after an all-reduce(sum): x *= 1/world
__global__ void __launch_bounds__(256)
k_i2v_scale(float* __restrict__ x, long n, float s) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) x[i] *= s;
}

// -------------------------------------------------------------------------------------------------------------------
// dictionary.Add's first-appearance numbering over an int64 item-id stream, on the device (ctr_item_emb_train).  The
// item map resolves most tokens to a row and k_idmap_first_pos (idmap.cuh) keeps each row's first position; the tokens
// without an entry form the side list, whose distinct ids and first positions come from a sort.  Both sets, ordered by
// first position, are the vocabulary: a word's rank in that order is its id.
// -------------------------------------------------------------------------------------------------------------------
// side list: (id, position) of every token without an item-map entry, in any order (the sort that follows is keyed by id
// and the reduction takes the minimum position, so the slot order does not reach the result)
__global__ void __launch_bounds__(256)
k_i2v_dict_side(const int* __restrict__ rows, const long long* __restrict__ ids, long n, unsigned long long* __restrict__ key,
                int* __restrict__ pos, unsigned long long* __restrict__ count) {
    const int lane = threadIdx.x & 31;
    for (long i0 = blockIdx.x * (long)blockDim.x + threadIdx.x; i0 < ((n + 31) & ~31L); i0 += (long)gridDim.x * blockDim.x) {
        const bool side = i0 < n && rows[i0] < 0;
        const unsigned b = __ballot_sync(0xffffffffu, side);
        if (!b) continue;
        unsigned long long base = 0;
        if (lane == 0) base = atomicAdd(count, (unsigned long long)__popc(b));
        base = __shfl_sync(0xffffffffu, base, 0);
        if (side) { const unsigned long long o = base + __popc(b & ((1u << lane) - 1u)); key[o] = (unsigned long long)ids[i0]; pos[o] = (int)i0; }
    }
}
// A row's first occurrence across ranks: (rank << 32) | its first position in this rank's stream (first_pos from
// k_idmap_first_pos), kI2vNever when this rank's stream never holds its id.  Positions stay below 2^31, so the minimum
// over the ranks is the row's first occurrence in the ranks' streams concatenated in rank order; on one GPU the tag is
// the position.
constexpr unsigned long long kI2vNever = ~0ull;
__global__ void __launch_bounds__(256)
k_i2v_first_tag(const unsigned* __restrict__ first_pos, long R, int rank, unsigned long long* __restrict__ tag) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < R; i += (long)gridDim.x * blockDim.x) {
        const unsigned p = first_pos[i];
        tag[i] = p == 0xFFFFFFFFu ? kI2vNever : ((unsigned long long)rank << 32) | p;
    }
}
// sort input of the vocabulary: rows [0, R) keyed by their first-occurrence tag (kI2vNever: the row's id never occurs),
// then the u side words keyed by theirs; val = row, or -(j+1) for side word j.  Tags are distinct, so the order is total.
__global__ void __launch_bounds__(256)
k_i2v_dict_rank_keys(const unsigned long long* __restrict__ row_tag, long R, const unsigned long long* __restrict__ side_tag, long u,
                     unsigned long long* __restrict__ key, int* __restrict__ val) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < R + u; i += (long)gridDim.x * blockDim.x) {
        if (i < R) { key[i] = row_tag[i]; val[i] = (int)i; }
        else { key[i] = side_tag[i - R]; val[i] = -(int)(i - R) - 1; }
    }
}
// after the sort: entry w < V is word w.  Its item id is the map's id of its row (row_id: the map's row -> id list) or
// the side list's id (side_id); *V = the entries before the first kI2vNever key.  Rows whose id never occurs keep
// word_of_row = -1.
__global__ void __launch_bounds__(256)
k_i2v_dict_rank(const unsigned long long* __restrict__ key, const int* __restrict__ val, long N, const long long* __restrict__ row_id,
                const unsigned long long* __restrict__ side_id, int* __restrict__ word_of_row, int* __restrict__ word_of_side,
                long long* __restrict__ vocab_ids, int* __restrict__ V) {
    for (long w = blockIdx.x * (long)blockDim.x + threadIdx.x; w < N; w += (long)gridDim.x * blockDim.x) {
        const unsigned long long k = key[w];
        if (k == kI2vNever) continue;
        const int v = val[w];
        if (v >= 0) { word_of_row[v] = (int)w; vocab_ids[w] = row_id[v]; }
        else { word_of_side[-v - 1] = (int)w; vocab_ids[w] = (long long)side_id[-v - 1]; }
        if (w + 1 == N || key[w + 1] == kI2vNever) *V = (int)(w + 1);
    }
}
// the int32 word-id document, in place over rows[]: a mapped token takes its row's word, a side token the word of its id
// in side_ids (ascending as uint64, distinct)
__global__ void __launch_bounds__(256)
k_i2v_dict_doc(int* __restrict__ doc, const long long* __restrict__ ids, long n, const int* __restrict__ word_of_row,
               const unsigned long long* __restrict__ side_ids, long u, const int* __restrict__ word_of_side) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const int row = doc[i];
        if (row >= 0) { doc[i] = word_of_row[row]; continue; }
        const unsigned long long id = (unsigned long long)ids[i];
        long lo = 0, hi = u;                                   // first side id >= id; the id is in the list
        while (lo < hi) { const long mid = (lo + hi) >> 1; if (side_ids[mid] < id) lo = mid + 1; else hi = mid; }
        doc[i] = word_of_side[lo];
    }
}
// ---- the numbering over the ranks' streams (ctr_item_emb_train; one GPU runs the same code at world = 1) -----------
// Each rank resolves its own stream (k_idmap_first_pos) and tags its rows' first positions (k_i2v_first_tag); the ranks'
// tags meet in a min all-reduce.  Each rank builds its own side list (i2v_dict_side_list); the ranks all-gather the lists
// and every rank reduces them to the distinct side ids with their smallest tags (idmap_merge_min, idmap.cuh).  Every rank
// then orders the same rows and side words the same way (i2v_dict_order) and converts its own stream (k_i2v_dict_doc).

// Scratch of i2v_dict_side_list for m side tokens: k0, k1 [m] (uint64), p0, p1 [m] (int) and tmp (this many bytes)
inline size_t i2v_dict_side_tmp_bytes(int m, cudaStream_t st) {
    size_t b1 = 0, b2 = 0;
    unsigned long long* k = nullptr; int* p = nullptr;
    cub::DeviceRadixSort::SortPairs(nullptr, b1, k, k, p, p, m, 0, 64, st);
    cub::DeviceReduce::ReduceByKey(nullptr, b2, k, k, p, p, p, MinPos{}, m, st);
    return std::max(b1, b2);
}
// One rank's side list: rows [n] from k_idmap_first_pos, m of them -1.  k0 / p0 [0, *u) receive the distinct unmapped ids
// ascending as uint64 and the first position of each in this rank's stream; slot counts a zeroed slot claim.
// Synchronises st (reads *u back).
inline cudaError_t i2v_dict_side_list(const int* rows, const long long* ids, long n, int m, unsigned long long* k0, unsigned long long* k1, int* p0, int* p1,
                                      unsigned long long* slot, int* d_u, void* tmp, size_t tmp_bytes, int grid, cudaStream_t st, int* u) {
    *u = 0;
    if (m == 0) return cudaSuccess;
    k_i2v_dict_side<<<grid, 256, 0, st>>>(rows, ids, n, k0, p0, slot);
    size_t b = tmp_bytes;
    cudaError_t e = cub::DeviceRadixSort::SortPairs(tmp, b, k0, k1, p0, p1, m, 0, 64, st);
    if (e == cudaSuccess) { b = tmp_bytes; e = cub::DeviceReduce::ReduceByKey(tmp, b, k1, k0, p1, p0, d_u, MinPos{}, m, st); }
    if (e == cudaSuccess) e = cudaMemcpyAsync(u, d_u, sizeof(int), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    return e != cudaSuccess ? e : cudaGetLastError();
}
inline void i2v_first_tags(const unsigned* first_pos, long R, int rank, unsigned long long* tag, int grid, cudaStream_t st) {
    k_i2v_first_tag<<<grid, 256, 0, st>>>(first_pos, R, rank, tag);
}
// Scratch of i2v_dict_order for N = R + u entries: key0, key1 [N] (uint64), val0, val1 [N] (int), row_id [R] and tmp
inline size_t i2v_dict_order_tmp_bytes(long N, cudaStream_t st) {
    size_t b = 0;
    unsigned long long* k = nullptr; int* v = nullptr;
    cub::DeviceRadixSort::SortPairs(nullptr, b, k, k, v, v, (int)N, 0, 64, st);
    return b;
}
// The vocabulary, the same on every rank: the R map rows (row_tag, the ranks' minimum) and the u side words (side_id /
// side_tag, the merge's output) sorted by tag; a word's rank in that order is its id.  The sort reads the low 32 +
// ceil(log2 world) bits, which hold every tag (positions < 2^31) and order kI2vNever last; on one GPU that is a 32-bit
// sort of positions.  The item id of a row's word comes from the map (row_id [R]: k_idmap_dump of keys / vals [cap]).
// word_of_row [R] (-1 before the call), word_of_side [u], vocab_ids [R + u], *V.  Synchronises st (reads *V back).
inline cudaError_t i2v_dict_order(const unsigned long long* keys, const int* vals, unsigned long long cap, const unsigned long long* row_tag, long R,
                                  const unsigned long long* side_id, const unsigned long long* side_tag, long u, int world, long long* row_id,
                                  unsigned long long* key0, unsigned long long* key1, int* val0, int* val1, void* tmp, size_t tmp_bytes,
                                  int* word_of_row, int* word_of_side, long long* vocab_ids, int* d_V, int grid, cudaStream_t st, int* V) {
    int wbits = 0; while ((1 << wbits) < world) wbits++;
    const long N = R + u;
    *V = 0;
    cudaError_t e = cudaMemsetAsync(d_V, 0, sizeof(int), st);
    if (e != cudaSuccess || N == 0) return e;
    k_idmap_dump<<<grid, 256, 0, st>>>(keys, vals, cap, row_id);
    k_i2v_dict_rank_keys<<<grid, 256, 0, st>>>(row_tag, R, side_tag, u, key0, val0);
    size_t b = tmp_bytes;
    e = cub::DeviceRadixSort::SortPairs(tmp, b, key0, key1, val0, val1, (int)N, 0, 32 + wbits, st);
    if (e != cudaSuccess) return e;
    k_i2v_dict_rank<<<grid, 256, 0, st>>>(key1, val1, N, row_id, side_id, word_of_row, word_of_side, vocab_ids, d_V);
    e = cudaMemcpyAsync(V, d_V, sizeof(int), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    return e != cudaSuccess ? e : cudaGetLastError();
}

// ITEM_EMB [R, D] (row stride D: D is a power of two >= 4) from the trained syn0 [V, D]: row r takes its word's vector,
// or zeros when its id never occurs.  One float4 per thread.  world > 1 with a row-sharded table: rank `rank` writes only
// the rows it owns, global row l·world + rank into its local row l (world = 1: every row).
__global__ void __launch_bounds__(256)
k_i2v_emb_scatter(const float* __restrict__ syn0, const int* __restrict__ word_of_row, long R, int D, int world, int rank, float* __restrict__ tab) {
    const int q = D / 4;
    const long local = (R - rank + world - 1) / world;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < local * q; i += (long)gridDim.x * blockDim.x) {
        const long l = i / q; const int c = (int)(i - l * q);
        const int w = word_of_row[l * world + rank];
        const float4 v = w >= 0 ? reinterpret_cast<const float4*>(syn0)[(long)w * q + c] : make_float4(0.f, 0.f, 0.f, 0.f);
        reinterpret_cast<float4*>(tab)[i] = v;
    }
}

// syn0 = (U[0,1) - 0.5) / dim (word2vec.go:103-111) with the counter RNG
__global__ void k_i2v_init(float* __restrict__ syn0, long n, int D, uint32_t seed) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const double u = (double)(mix64(seed, 100u, (uint64_t)i) >> 11) * (1.0 / 9007199254740992.0);
        syn0[i] = (float)((u - 0.5) / (double)D);
    }
}

}  // namespace ctr
