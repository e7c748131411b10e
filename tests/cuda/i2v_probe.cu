// i2v_probe.cu — test-only entry points that launch the item2vec kernels of go-ctr_b200/csrc/item2vec.cuh on arrays the
// caller owns (tests/test_gpu_i2v_kernel.py through ctypes).  The header is included, not copied: what runs here is
// k_i2v_skipgram_hs<LPR>, k_i2v_word_tables, k_i2v_node_scale and k_i2v_paths as the trainer launches them.  Not linked
// into libctr_b200.so and not part of include/ctr_b200.h.
// Build: nvcc <flags of go-ctr_b200/build.py> -I go-ctr_b200/csrc -o tests/cuda/_build/libi2v_probe.so tests/cuda/i2v_probe.cu
#include "item2vec.cuh"
#include <cub/cub.cuh>
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

using namespace ctr;

namespace {
char g_err[256] = "";
int fail(const char* what, cudaError_t e = cudaSuccess) {
    if (e != cudaSuccess) snprintf(g_err, sizeof g_err, "%s: %s", what, cudaGetErrorString(e));
    else snprintf(g_err, sizeof g_err, "%s", what);
    return -1;
}
// device copy of a host array; freed with the object
template <typename T>
struct Dev {
    T* p = nullptr; size_t n = 0;
    ~Dev() { if (p) cudaFree(p); }
    cudaError_t up(const T* h, size_t count) {
        n = count;
        cudaError_t e = cudaMalloc(&p, sizeof(T) * std::max<size_t>(count, 1));
        if (e == cudaSuccess && count && h) e = cudaMemcpy(p, h, sizeof(T) * count, cudaMemcpyHostToDevice);
        else if (e == cudaSuccess) e = cudaMemset(p, 0, sizeof(T) * std::max<size_t>(count, 1));
        return e;
    }
    cudaError_t down(T* h) const { return n ? cudaMemcpy(h, p, sizeof(T) * n, cudaMemcpyDeviceToHost) : cudaSuccess; }
};
#define PC(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return fail(#call, e_); } while (0)
}  // namespace

extern "C" const char* i2v_probe_error() { return g_err; }
extern "C" int i2v_probe_hot_max() { return kI2vHot; }
extern "C" int i2v_probe_flush_every() { return kI2vFlush; }

// One launch of k_i2v_skipgram_hs<D/4><<<grid, block, max(hot_n,1)*D*4>>> over every field of I2vArgs.  syn0 [V,D] and
// syn1 [nn,D] are read and written in place, counters [3] are written.  The indices the kernel dereferences are checked
// here, so a malformed test input is an error message and not a stray access.
extern "C" int i2v_probe_skipgram(const int* doc, long nd, const double* z, int V, const long long* poff, const int* pnode, const unsigned char* pcode,
                                  float* syn0, float* syn1, int nn, int D, int W, const float* lr_tab, int n_lr, int upd,
                                  const float* node_scale, const float* word_scale, unsigned seed, int iter, int hot_base, int hot_n,
                                  long pos_begin, long pos_end, int grid, int block, unsigned long long* counters) {
    if (D < 4 || D > 128 || (D & (D - 1)) || W < 1 || V < 1 || nn < 1 || nd < 1 || upd < 1) return fail("bad shape");
    if (grid < 1 || block < 32 || block > 256 || block % 32) return fail("block must be a multiple of 32 in [32, 256]");
    if (pos_begin < 0 || pos_end > nd || pos_begin >= pos_end) return fail("bad position range");
    if ((pos_end - 1) / upd >= n_lr) return fail("lr_tab too short");
    if (hot_n < 0 || hot_n > kI2vHot || hot_base < 0 || hot_base + hot_n < nn) return fail("every node >= hot_base needs a shared-memory slot");
    for (long i = 0; i < nd; i++) if (doc[i] < 0 || doc[i] >= V) return fail("token outside the vocabulary");
    for (int w = 0; w < V; w++) if (poff[w + 1] < poff[w] || poff[w] < 0) return fail("path offsets must not decrease");
    for (long long i = 0; i < poff[V]; i++) if (pnode[i] < 0 || pnode[i] >= nn) return fail("path node outside syn1");
    Dev<int> d_doc, d_pnode; Dev<double> d_z; Dev<long long> d_poff; Dev<unsigned char> d_pcode;
    Dev<float> d_syn0, d_syn1, d_lr, d_nsc, d_wsc; Dev<unsigned long long> d_ctr;
    PC(d_doc.up(doc, (size_t)nd)); PC(d_z.up(z, (size_t)V)); PC(d_poff.up(poff, (size_t)V + 1));
    PC(d_pnode.up(pnode, (size_t)poff[V])); PC(d_pcode.up(pcode, (size_t)poff[V]));
    PC(d_syn0.up(syn0, (size_t)V * D)); PC(d_syn1.up(syn1, (size_t)nn * D));
    PC(d_lr.up(lr_tab, (size_t)n_lr)); PC(d_nsc.up(node_scale, (size_t)nn)); PC(d_wsc.up(word_scale, (size_t)V));
    PC(d_ctr.up(nullptr, 3));
    std::vector<float> lut(1000);                                                    // as i2v_train_impl uploads it (sigmoid_table.go:28-45)
    for (int i = 0; i < 1000; i++) { double e = std::exp(((double)i / 1000.0 * 2.0 - 1.0) * 6.0); lut[(size_t)i] = (float)(e / (e + 1.0)); }
    PC(cudaMemcpyToSymbol(c_i2v_lut, lut.data(), sizeof(float) * 1000));
    I2vArgs a{}; a.doc = d_doc.p; a.nd = nd; a.z = d_z.p; a.poff = d_poff.p; a.pnode = d_pnode.p; a.pcode = d_pcode.p; a.syn0 = d_syn0.p; a.syn1 = d_syn1.p;
    a.D = D; a.W = W; a.lr_tab = d_lr.p; a.upd = upd; a.node_scale = d_nsc.p; a.word_scale = d_wsc.p; a.seed = seed; a.iter = iter;
    a.counters = d_ctr.p; a.hot_base = hot_base; a.hot_n = hot_n; a.pos_begin = pos_begin; a.pos_end = pos_end;
    const size_t sm = (size_t)std::max(hot_n, 1) * D * sizeof(float);
    switch (D / 4) {
        case 1: k_i2v_skipgram_hs<1><<<grid, block, sm>>>(a); break;   case 2: k_i2v_skipgram_hs<2><<<grid, block, sm>>>(a); break;
        case 4: k_i2v_skipgram_hs<4><<<grid, block, sm>>>(a); break;   case 8: k_i2v_skipgram_hs<8><<<grid, block, sm>>>(a); break;
        case 16: k_i2v_skipgram_hs<16><<<grid, block, sm>>>(a); break; default: k_i2v_skipgram_hs<32><<<grid, block, sm>>>(a); break;
    }
    PC(cudaGetLastError()); PC(cudaDeviceSynchronize());
    PC(d_syn0.down(syn0)); PC(d_syn1.down(syn1)); PC(d_ctr.down(counters));
    return 0;
}

// k_i2v_word_tables (without the sort keys) and k_i2v_node_scale
extern "C" int i2v_probe_tables(const unsigned long long* cnt, int V, double subsample, double ceff, double total, const long long* node_val, int nn,
                                double* z, float* word_scale, float* node_scale) {
    if (V < 1 || nn < 1) return fail("bad shape");
    Dev<unsigned long long> d_cnt; Dev<long long> d_nval; Dev<double> d_z; Dev<float> d_wsc, d_nsc;
    PC(d_cnt.up(cnt, (size_t)V)); PC(d_nval.up(node_val, (size_t)nn)); PC(d_z.up(nullptr, (size_t)V)); PC(d_wsc.up(nullptr, (size_t)V)); PC(d_nsc.up(nullptr, (size_t)nn));
    k_i2v_word_tables<<<4, 256>>>(d_cnt.p, V, subsample, ceff, total, d_z.p, d_wsc.p, nullptr, nullptr);
    k_i2v_node_scale<<<4, 256>>>(d_nval.p, nn, ceff, total, d_nsc.p);
    PC(cudaGetLastError()); PC(cudaDeviceSynchronize());
    PC(d_z.down(z)); PC(d_wsc.down(word_scale)); PC(d_nsc.down(node_scale));
    return 0;
}

// both passes of k_i2v_paths with the exclusive scan between them, as i2v_train_impl runs them.  parent / code: [2V-1]
// (leaves [0,V), inner nodes V + creation index).  Returns the number of steps written, or -1; cap: room in pnode / pcode.
extern "C" long long i2v_probe_paths(const int* parent, const unsigned char* code, const unsigned long long* cnt, int V, int max_depth,
                                     long long* poff, int* pnode, unsigned char* pcode, long long cap) {
    if (V < 2 || max_depth < 1) return fail("bad shape");
    for (int i = 0; i < 2 * V - 1; i++) if (parent[i] < -1 || parent[i] >= 2 * V - 1 || (parent[i] != -1 && parent[i] <= i)) return fail("parent must point upward");
    Dev<int> d_parent, d_pnode; Dev<unsigned char> d_code, d_pcode, d_tmp; Dev<unsigned long long> d_cnt; Dev<long long> d_poff;
    PC(d_parent.up(parent, (size_t)2 * V - 1)); PC(d_code.up(code, (size_t)2 * V - 1)); PC(d_cnt.up(cnt, (size_t)V)); PC(d_poff.up(nullptr, (size_t)V + 1));
    k_i2v_paths<<<4, 256>>>(d_parent.p, d_code.p, d_cnt.p, V, max_depth, 0, d_poff.p, nullptr, nullptr);
    size_t tb = 0;
    PC(cub::DeviceScan::ExclusiveSum(nullptr, tb, d_poff.p, d_poff.p, V + 1));
    PC(d_tmp.up(nullptr, tb));
    PC(cub::DeviceScan::ExclusiveSum(d_tmp.p, tb, d_poff.p, d_poff.p, V + 1));
    PC(d_poff.down(poff));
    const long long nsteps = poff[V];
    if (nsteps > cap) return fail("path buffers too small");
    PC(d_pnode.up(nullptr, (size_t)nsteps)); PC(d_pcode.up(nullptr, (size_t)nsteps));
    k_i2v_paths<<<4, 256>>>(d_parent.p, d_code.p, d_cnt.p, V, max_depth, 1, d_poff.p, d_pnode.p, d_pcode.p);
    PC(cudaGetLastError()); PC(cudaDeviceSynchronize());
    PC(d_pnode.down(pnode)); PC(d_pcode.down(pcode));
    return nsteps;
}
