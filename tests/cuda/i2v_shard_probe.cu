// i2v_shard_probe.cu — test-only entry points for ctr_item_emb_train's numbering across ranks and its owner-written
// rows (world > 1), launched on device buffers the caller owns (tests/test_gpu_i2v_shard_probe.py through ctypes,
// tests/i2v_shard_probe.py).  The kernels and the inline host steps come from go-ctr_b200/csrc/item2vec.cuh and idmap.cuh
// themselves, not copies, called as ctr_item_emb_train calls them.
//
// A rank's first tags and side list need only its own stream and the (shared) item map; the merge and the ordering need
// only the gathered lists and the reduced tags; a rank's document and rows need only the global word tables.  So W
// streams on one device act as W ranks: the test plays the min all-reduce with an elementwise minimum and the all-gather
// with a padded concatenation.  Every entry point synchronises the device and returns 0, or -1 with
// i2v_shard_probe_error() set.  Not linked into libctr_b200.so and not part of include/ctr_b200.h.
// Build: nvcc <flags of go-ctr_b200/build.py> -I go-ctr_b200/csrc -o tests/cuda/_build/libi2v_shard_probe.so tests/cuda/i2v_shard_probe.cu
#include "idmap.cuh"
#include "item2vec.cuh"
#include <cstdio>

using namespace ctr;

namespace {
char g_err[256] = "";
int fail(const char* what, cudaError_t e = cudaSuccess) {
    if (e != cudaSuccess) snprintf(g_err, sizeof g_err, "%s: %s", what, cudaGetErrorString(e));
    else snprintf(g_err, sizeof g_err, "%s", what);
    return -1;
}
#define PC(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return fail(#call, e_); } while (0)
int done() { PC(cudaGetLastError()); PC(cudaDeviceSynchronize()); return 0; }
constexpr int G = 1024;

template <typename T> struct Tmp {
    T* p = nullptr;
    ~Tmp() { if (p) cudaFree(p); }
    cudaError_t alloc(size_t n) { return cudaMalloc(&p, std::max<size_t>(n, 1) * sizeof(T)); }
};
}  // namespace

extern "C" const char* i2v_shard_probe_error() { return g_err; }

// ctr_idmap_build's map: keys / vals [cap] cleared, ids [n] inserted at rows 0 .. n-1
extern "C" int i2v_shard_probe_map(const long long* ids, long long n, unsigned long long* keys, int* vals, unsigned long long cap, int* flags) {
    if (cap == 0 || (cap & (cap - 1)) || n < 0) return fail("bad map arguments");
    k_idmap_clear<<<G, 256>>>(keys, vals, cap);
    if (n > 0) k_idmap_insert<<<G, 256>>>(keys, vals, cap - 1, ids, (long)n, flags, 0);
    return done();
}

// One rank's stream ids [n] against the map: rows [n] (the map's row or -1), row_tag [R] (rank-tagged first positions,
// kI2vNever for a row this stream never holds), side_ids / side_pos [*u] (distinct unmapped ids ascending and their first
// positions in this stream)
extern "C" int i2v_shard_probe_local(const unsigned long long* keys, const int* vals, unsigned long long cap, const long long* ids, long long n, long long R,
                                     int rank, int* rows, unsigned long long* row_tag, unsigned long long* side_ids, int* side_pos, int* u_out) {
    if (n < 0 || R < 0 || rank < 0) return fail("bad local arguments");
    Tmp<unsigned> first; Tmp<unsigned long long> cnt, k1; Tmp<int> p1, d_u; Tmp<unsigned char> tmp;
    PC(first.alloc(R)); PC(cnt.alloc(2));
    PC(cudaMemset(first.p, 0xff, sizeof(unsigned) * (size_t)R)); PC(cudaMemset(cnt.p, 0, 2 * sizeof(unsigned long long)));
    k_idmap_first_pos<<<G, 256>>>(keys, vals, cap - 1, ids, (long)n, rows, first.p, cnt.p);
    i2v_first_tags(first.p, (long)R, rank, row_tag, G, 0);
    PC(cudaGetLastError());
    unsigned long long m = 0;
    PC(cudaMemcpy(&m, cnt.p, sizeof m, cudaMemcpyDeviceToHost));
    int u = 0;
    if (m > 0) {
        PC(k1.alloc(m)); PC(p1.alloc(m)); PC(d_u.alloc(1));
        const size_t tb = i2v_dict_side_tmp_bytes((int)m, 0);
        PC(tmp.alloc(tb));
        PC(i2v_dict_side_list(rows, ids, (long)n, (int)m, side_ids, k1.p, side_pos, p1.p, cnt.p + 1, d_u.p, tmp.p, tb, G, 0, &u));
    }
    *u_out = u;
    return done();
}

// idmap_merge_min over the gathered lists g_ids / g_pos [world][stride] (rank j's cnt[j] entries first): side_id / side_tag
// [*u], the distinct ids ascending and the tag of each one's first occurrence
extern "C" int i2v_shard_probe_merge(const unsigned long long* g_ids, const int* g_pos, long long stride, const int* cnt, int world,
                                     unsigned long long* side_id, unsigned long long* side_tag, int* u_out) {
    if (world < 1 || world > kMaxPeers || stride < 0) return fail("bad merge arguments");
    RankLists L{};
    for (int j = 0; j < world; j++) { L.cnt[j] = cnt[j]; L.off[j + 1] = L.off[j] + cnt[j]; }
    const int m = (int)L.off[world];
    Tmp<unsigned long long> k1, t1; Tmp<int> d_u; Tmp<unsigned char> tmp;
    PC(k1.alloc(m)); PC(t1.alloc(m)); PC(d_u.alloc(1));
    const size_t tb = idmap_merge_tmp_bytes(m, 0);
    PC(tmp.alloc(tb));
    int u = 0;
    PC(idmap_merge_min(g_ids, g_pos, (long)stride, L, world, side_id, k1.p, side_tag, t1.p, d_u.p, tmp.p, tb, G, 0, &u));
    *u_out = u;
    return done();
}

// i2v_dict_order: word_of_row [R] (set to -1 here first), word_of_side [u], vocab_ids [R + u], *V
extern "C" int i2v_shard_probe_order(const unsigned long long* keys, const int* vals, unsigned long long cap, const unsigned long long* row_tag, long long R,
                                     const unsigned long long* side_id, const unsigned long long* side_tag, long long u, int world,
                                     int* word_of_row, int* word_of_side, long long* vocab_ids, int* V_out) {
    if (R < 0 || u < 0 || world < 1 || world > kMaxPeers) return fail("bad order arguments");
    const long N = (long)(R + u);
    Tmp<unsigned long long> k0, k1; Tmp<int> v0, v1, d_V; Tmp<long long> row_id; Tmp<unsigned char> tmp;
    PC(k0.alloc(N)); PC(k1.alloc(N)); PC(v0.alloc(N)); PC(v1.alloc(N)); PC(d_V.alloc(1)); PC(row_id.alloc(R));
    const size_t tb = i2v_dict_order_tmp_bytes(N, 0);
    PC(tmp.alloc(tb));
    PC(cudaMemset(word_of_row, 0xff, sizeof(int) * (size_t)R));
    int V = 0;
    PC(i2v_dict_order(keys, vals, cap, row_tag, (long)R, side_id, side_tag, (long)u, world, row_id.p, k0.p, k1.p, v0.p, v1.p, tmp.p, tb,
                      word_of_row, word_of_side, vocab_ids, d_V.p, G, 0, &V));
    *V_out = V;
    return done();
}

// k_i2v_dict_doc: one rank's document in place over its rows [n]
extern "C" int i2v_shard_probe_doc(int* doc, const long long* ids, long long n, const int* word_of_row, const unsigned long long* side_id, long long u,
                                   const int* word_of_side) {
    k_i2v_dict_doc<<<G, 256>>>(doc, ids, (long)n, word_of_row, side_id, (long)u, word_of_side);
    return done();
}

// k_i2v_emb_scatter: rank `rank`'s rows of the [R, D] table (world = 1: the whole table)
extern "C" int i2v_shard_probe_scatter(const float* syn0, const int* word_of_row, long long R, int D, int world, int rank, float* tab) {
    if (D < 4 || (D & (D - 1)) || world < 1 || rank < 0 || rank >= world) return fail("bad scatter arguments");
    k_i2v_emb_scatter<<<G, 256>>>(syn0, word_of_row, (long)R, D, world, rank, tab);
    return done();
}
