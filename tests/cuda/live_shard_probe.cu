// live_shard_probe.cu — test-only entry points for the collective live id maps and table writes (ctr_idmap_insert,
// ctr_table_write_rows with world > 1), launched on device buffers the caller owns (tests/test_gpu_live_shard_probe.py
// through ctypes, tests/live_shard_probe.py).  The kernels and the merge driver come from go-ctr_b200/csrc/idmap.cuh,
// item2vec.cuh, attn.cuh and vmm.cuh themselves, not copies, launched as ctr_idmap_insert and ctr_table_write_rows launch
// them.
//
// A rank's numbering needs only its own ids and the (shared) map, the merge only the gathered lists, and an owner's row
// write only the rows routed to it, so W shards of one device act as W ranks: the test plays the all-gathers and the
// routing with plain copies.  Every entry point synchronises the device and returns 0, or -1 with live_probe_error() set.
// Not linked into libctr_b200.so and not part of include/ctr_b200.h.
// Build: nvcc <flags of go-ctr_b200/build.py> -I go-ctr_b200/csrc -o tests/cuda/_build/liblive_shard_probe.so tests/cuda/live_shard_probe.cu
#include "attn.cuh"
#include "idmap.cuh"
#include "item2vec.cuh"
#include "vmm.cuh"
#include <cstdio>
#include <string>

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

// device scratch owned by one call
template <typename T> struct Tmp {
    T* p = nullptr;
    ~Tmp() { if (p) cudaFree(p); }
    cudaError_t alloc(size_t n) { return cudaMalloc(&p, std::max<size_t>(n, 1) * sizeof(T)); }
};
}  // namespace

extern "C" const char* live_probe_error() { return g_err; }

// One rank's numbering, as ctr_idmap_insert numbers (keys == nullptr: no map yet): rows [n] = the map's row or -1,
// out_ids / out_pos [*u] = the distinct missing ids ascending as uint64 and their first positions, *m = ids without a row.
extern "C" int live_probe_number(const unsigned long long* keys, const int* vals, unsigned long long cap, const long long* ids, long long n,
                                 int* rows, unsigned long long* out_ids, int* out_pos, long long* m_out, int* u_out) {
    if (n < 0) return fail("bad number arguments");
    Tmp<unsigned long long> cnt, k0, k1; Tmp<int> p0, p1, d_u; Tmp<unsigned char> tmp;
    PC(cnt.alloc(2)); PC(cudaMemset(cnt.p, 0, 2 * sizeof(unsigned long long)));
    unsigned long long m = (unsigned long long)n;
    if (keys) {
        k_idmap_first_pos<<<G, 256>>>(keys, vals, cap - 1, ids, (long)n, rows, nullptr, cnt.p);
        PC(cudaGetLastError());
        PC(cudaMemcpy(&m, cnt.p, sizeof m, cudaMemcpyDeviceToHost));
    } else PC(cudaMemset(rows, 0xff, sizeof(int) * (size_t)n));
    *m_out = (long long)m; *u_out = 0;
    if (m == 0) return done();
    PC(k0.alloc(m)); PC(k1.alloc(m)); PC(p0.alloc(m)); PC(p1.alloc(m)); PC(d_u.alloc(1));
    size_t b1 = 0, b2 = 0;
    PC(cub::DeviceRadixSort::SortPairs(nullptr, b1, k0.p, k1.p, p0.p, p1.p, (int)m, 0, 64));
    PC(cub::DeviceReduce::ReduceByKey(nullptr, b2, k1.p, k0.p, p1.p, p0.p, d_u.p, MinPos{}, (int)m));
    PC(tmp.alloc(std::max(b1, b2)));
    k_i2v_dict_side<<<G, 256>>>(rows, ids, (long)n, k0.p, p0.p, cnt.p + 1);
    size_t tb = std::max(b1, b2);
    PC(cub::DeviceRadixSort::SortPairs(tmp.p, tb, k0.p, k1.p, p0.p, p1.p, (int)m, 0, 64));
    tb = std::max(b1, b2);
    PC(cub::DeviceReduce::ReduceByKey(tmp.p, tb, k1.p, k0.p, p1.p, p0.p, d_u.p, MinPos{}, (int)m));
    int u = 0;
    PC(cudaMemcpy(&u, d_u.p, sizeof u, cudaMemcpyDeviceToHost));
    PC(cudaMemcpy(out_ids, k0.p, sizeof(unsigned long long) * (size_t)u, cudaMemcpyDeviceToDevice));
    PC(cudaMemcpy(out_pos, p0.p, sizeof(int) * (size_t)u, cudaMemcpyDeviceToDevice));
    *u_out = u;
    return done();
}

// The single-GPU order: the numbered ids [u] sorted by first position (the sort ctr_idmap_insert runs on one GPU)
extern "C" int live_probe_order(const unsigned long long* ids, const int* pos, int u, unsigned long long* out_ids) {
    if (u < 1) return fail("bad order arguments");
    Tmp<int> p1; Tmp<unsigned char> tmp;
    PC(p1.alloc(u));
    size_t tb = 0;
    PC(cub::DeviceRadixSort::SortPairs(nullptr, tb, pos, p1.p, ids, out_ids, u, 0, 32));
    PC(tmp.alloc(tb));
    PC(cub::DeviceRadixSort::SortPairs(tmp.p, tb, pos, p1.p, ids, out_ids, u, 0, 32));
    return done();
}

// idmap_merge_ranks over the gathered lists g_ids / g_pos [world][stride] (rank j's cnt[j] entries first): out_ids [*u]
extern "C" int live_probe_merge(const unsigned long long* g_ids, const int* g_pos, long long stride, const int* cnt, int world,
                                unsigned long long* out_ids, int* u_out) {
    if (world < 1 || world > kMaxPeers || stride < 0) return fail("bad merge arguments");
    RankLists L{};
    for (int j = 0; j < world; j++) { L.cnt[j] = cnt[j]; L.off[j + 1] = L.off[j] + cnt[j]; }
    const int m = (int)L.off[world];
    Tmp<unsigned long long> k0, k1, t0, t1; Tmp<int> d_u; Tmp<unsigned char> tmp;
    PC(k0.alloc(m)); PC(k1.alloc(m)); PC(t0.alloc(m)); PC(t1.alloc(m)); PC(d_u.alloc(1));
    const size_t tb = idmap_merge_tmp_bytes(m, 0);
    PC(tmp.alloc(tb));
    int u = 0;
    PC(idmap_merge_ranks(g_ids, g_pos, (long)stride, L, world, k0.p, k1.p, t0.p, t1.p, d_u.p, tmp.p, tb, G, 0, &u));
    if (u > 0) PC(cudaMemcpy(out_ids, k1.p, sizeof(unsigned long long) * (size_t)u, cudaMemcpyDeviceToDevice));
    *u_out = u;
    return done();
}

// ctr_idmap_insert's write: fresh [u] inserted at rows R, R + 1, ... into keys / vals [cap]; a new table (keys != old_keys)
// is cleared first and the old map (old_keys == nullptr: none) rehashed into it
extern "C" int live_probe_add(const unsigned long long* old_keys, const int* old_vals, unsigned long long old_cap, unsigned long long* keys,
                              int* vals, unsigned long long cap, const unsigned long long* fresh, int u, int R, int* flags) {
    if (cap == 0 || (cap & (cap - 1))) return fail("bad add arguments");
    if (keys != old_keys) {
        k_idmap_clear<<<G, 256>>>(keys, vals, cap);
        if (old_keys) k_idmap_rehash<<<G, 256>>>(old_keys, old_vals, old_cap, keys, vals, cap - 1);
    }
    if (u > 0) k_idmap_insert<<<G, 256>>>(keys, vals, cap - 1, (const long long*)fresh, (long)u, flags, R);
    return done();
}

extern "C" int live_probe_dump(const unsigned long long* keys, const int* vals, unsigned long long cap, long long* ids) {
    k_idmap_dump<<<G, 256>>>(keys, vals, cap, ids);
    return done();
}

extern "C" int live_probe_lookup(const unsigned long long* keys, const int* vals, unsigned long long cap, const long long* ids, long long n, int* rows) {
    k_idmap_lookup<<<G, 256>>>(keys, vals, cap - 1, ids, (long)n, rows);
    return done();
}

extern "C" int live_probe_digest(const unsigned long long* keys, const int* vals, unsigned long long cap, unsigned long long* out) {
    PC(cudaMemset(out, 0, sizeof(unsigned long long)));
    k_idmap_digest<<<G, 256>>>(keys, vals, cap, out);
    return done();
}

// k_table_write_rows (the single table) or, world > 1, k_shard_write_rows on rank `rank`'s shard
extern "C" int live_probe_write(float* t, long long ld, const int* rows, const float* data, long long n, int width, int world, int rank,
                                float* mo, float* vo, float* hot, int hot_k, float* hm, float* hv) {
    if (n < 1 || width < 1 || world < 1 || rank < 0 || rank >= world) return fail("bad write arguments");
    const int grid = (int)std::min<long long>((n + 7) / 8, G);
    if (world == 1) k_table_write_rows<<<grid, 256>>>(t, (long)ld, rows, data, (long)n, width, mo, vo);
    else k_shard_write_rows<<<grid, 256>>>(t, (long)ld, rows, data, (long)n, width, world, rank, mo, vo, hot, hot_k, hm, hv);
    return done();
}

// vmm_grow_rows on a shard of `rows` rows (row_b bytes each) filled from host (its spare bytes set to 0xff first), grown
// to `want`: out [want rows] = the grown shard; *old_bytes / *new_bytes = the allocation before and after; *gran = the
// allocation granularity vmm_alloc rounds to
extern "C" int live_probe_grow(const void* host, long long rows, long long want, long long row_b, int dev, void* out,
                               long long* old_bytes, long long* new_bytes, long long* gran) {
    std::string err;
    VmmBuf b;
    if (!vmm_alloc((size_t)std::max<long long>(rows, 1) * row_b, dev, &b, &err)) return fail(err.c_str());
    CUmemAllocationProp prop = vmm_prop(dev);
    size_t g = 0;
    drv().MemGetAllocationGranularity(&g, &prop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED);
    *gran = (long long)g;
    *old_bytes = (long long)b.bytes;
    int rc = 0;
    if (cudaMemset(b.ptr, 0xff, b.bytes) != cudaSuccess || cudaMemcpy(b.ptr, host, (size_t)rows * row_b, cudaMemcpyHostToDevice) != cudaSuccess) rc = fail("shard fill");
    if (rc == 0 && !vmm_grow_rows(&b, (size_t)rows, (size_t)want, (size_t)row_b, dev, 0, &err)) rc = fail(err.c_str());
    if (rc == 0 && (cudaDeviceSynchronize() != cudaSuccess || cudaMemcpy(out, b.ptr, (size_t)want * row_b, cudaMemcpyDeviceToHost) != cudaSuccess)) rc = fail("shard read");
    *new_bytes = (long long)b.bytes;
    vmm_free(&b);
    return rc;
}
