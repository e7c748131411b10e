// common.cuh — device helpers shared by the engine's kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace ctr {

constexpr int kWarp = 32;

// gorgonia v0.9.17 float32 sigmoid semantics (saturates outside [-88, 15]); the product of the
// reference's model.go / din.go graph nodes `G.Sigmoid` (din.go:273,307,311,315).
__device__ __forceinline__ float sigmoid32(float x) {
    if (x < -88.0f) return 0.0f;
    if (x > 15.0f) return 1.0f;
    return __fdividef(1.0f, 1.0f + __expf(-x));       // MUFU.EX2 + MUFU.RCP, rel. error ~1e-7
}

// Counter RNG (spec shared with the test oracle; implemented independently here): dropout masks
// (G.Dropout, din.go:308,312) and N(0,1) init (din.go:187-191).
__host__ __device__ __forceinline__ uint64_t mix64(uint32_t seed, uint32_t stream, uint64_t ctr) {
    uint64_t z = (((uint64_t)seed << 32) | stream) * 0x9E3779B97F4A7C15ull + ctr * 0xD1B54A32D192ED03ull
                 + 0x632BE59BD9B4E019ull;
    z ^= z >> 30; z *= 0xBF58476D1CE4E5B9ull;
    z ^= z >> 27; z *= 0x94D049BB133111EBull;
    z ^= z >> 31;
    return z;
}
// dropout draws: a 32-bit multiply-xorshift hash of (seed, stream, counter) — ~8 integer ops per
// element, cheap enough for a GEMM epilogue
__host__ __device__ __forceinline__ uint32_t hash32(uint32_t seed, uint32_t stream, uint32_t ctr) {
    uint32_t x = ctr ^ (seed * 0x9E3779B1u) ^ (stream * 0x85EBCA77u + 0xC2B2AE3Du);
    x ^= x >> 16; x *= 0x7FEB352Du; x ^= x >> 15; x *= 0x846CA68Bu; x ^= x >> 16;
    return x;
}
__host__ __device__ __forceinline__ float uniform24(uint32_t seed, uint32_t stream, uint64_t ctr) {
    return (float)(hash32(seed, stream, (uint32_t)ctr) >> 8) * (1.0f / 16777216.0f);
}
// dropout keep-factor: 0 or 1/(1-p)
__device__ __forceinline__ float drop_keep(float p, uint32_t seed, uint32_t stream, uint64_t ctr) {
    if (p <= 0.0f) return 1.0f;
    return uniform24(seed, stream, ctr) < (1.0f - p) ? 1.0f / (1.0f - p) : 0.0f;
}
// derivative factor through dropout+sigmoid given the stored post-dropout activation hd = h*keep:
// keep * h * (1-h); a dropped (or saturated-to-0) unit has hd == 0 and contributes 0.
__device__ __forceinline__ float dsigmoid_drop(float hd, float p) {
    if (hd == 0.0f) return 0.0f;
    if (p <= 0.0f) return hd * (1.0f - hd);
    float h = hd * (1.0f - p);
    return (1.0f / (1.0f - p)) * h * (1.0f - h);
}

template <int W>
__device__ __forceinline__ float group_sum(float v) {     // sum over aligned groups of W lanes
#pragma unroll
    for (int o = W / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_sum(float v) { return group_sum<32>(v); }
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
// streaming 128-bit load that does not allocate in L1 (rows are used once per kernel)
__device__ __forceinline__ float4 ldg4_stream(const float* p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}
// 128-bit vector reduction into global memory (sm_90+): one L2 atomic transaction per 16 bytes
__device__ __forceinline__ void red_add4(float* p, float4 v) {
    asm volatile("red.global.add.v4.f32 [%0], {%1,%2,%3,%4};"
                 :: "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ float dot4(float4 a, float4 b) { return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w; }
__device__ __forceinline__ float4 fma4(float s, float4 a, float4 c) {
    return make_float4(fmaf(s, a.x, c.x), fmaf(s, a.y, c.y), fmaf(s, a.z, c.z), fmaf(s, a.w, c.w));
}
__device__ __forceinline__ float4 zero4() { return make_float4(0.f, 0.f, 0.f, 0.f); }

// 16-byte global→shared copy that does not occupy a register or stall the issuing warp (LDGSTS); valid == false
// writes zeros without touching src
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc, bool valid) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(gsrc), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async4(void* smem_dst, const void* gsrc) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(d), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// Where one sample's rows come from.  index mode: the HBM tables + per-sample row ids
// (GetSampleVector rcmd.go:462-536 done inside the kernel).  dense mode: a materialised X row and
// SampleInfo column offsets (model.Train's tensor.Slice calls, model.go:129-171).
// Row ids outside [0, n_*) read as "missing" (zeros), exactly like -1: a stale id from the host can never
// address memory outside the table (the reference's "not found -> zeros", rcmd.go:501-505,519-521).
constexpr int kMaxPeers = 8;         // one NVSwitch box
struct RowSrc {
    const float* emb;   long lde;     // ITEM_EMB  [I, D]   (this rank's shard when world > 1)
    const float* ufeat; long ldu;     // USER_FEAT [U, uP]
    const float* ifeat; long ldi;     // ITEM_FEAT [I, cF]
    const int* user_row; const int* item_row; const int* hist;   // [B] [B] [B,S]
    const int* item_feat_row;    // row of ITEM_FEAT when it differs from item_row
    const float* X; long ldx; int up0, ub0, it0, cx0;            // dense mode
    int dense;
    int nvalid;          // rows >= nvalid are the zero-padded tail (model.go:357-371)
    int n_emb, n_user, n_ifeat;      // logical (global) row counts: ids outside [0, n) are missing rows
    // row-sharded tables over NVLink peer memory (comm.cuh): owner(row) = row & wmask, local row = row >> wshift.
    // peer_emb[j] / peer_ifeat[j] are rank j's shards mapped into this process (CUDA IPC); world == 1: unused.
    int world, wmask, wshift, ifeat_sharded;
    float* peer_emb[kMaxPeers];
    const float* peer_ifeat[kMaxPeers];
    float* rows_cache;   // [B, S+1, D]: the forward keeps every fetched row for the backward (one NVLink pull per row)
    // the hot_k most popular rows (ids [0, hot_k): keep rows ordered by popularity) are replicated on every rank:
    // reads are local, their gradients are summed locally and all-reduced (comm.cuh)
    int hot_k; const float* hot_tab;
};

// CTR_TABLE_ADAM on a row-sharded ITEM_EMB: every owner's shareable gradient buffer, the same layout on every rank
// (rows = the largest shard's local rows): bytes [0, 4) the touched-row count, [4, 8) the update kernel's block ticket,
// then a touched flag per local row (u32), the list of touched local rows (i32) and the fp32 gradient shard [rows, lde];
// all of it zero between steps
struct ShardGrad { long flag_off, list_off, grad_off, bytes; };
inline ShardGrad shard_grad_layout(long rows, long lde) {
    auto up = [](long b) { return (b + 255) & ~255L; };
    ShardGrad s;
    s.flag_off = 256; s.list_off = s.flag_off + up(rows * 4); s.grad_off = s.list_off + up(rows * 4);
    s.bytes = s.grad_off + rows * lde * (long)sizeof(float);
    return s;
}

struct Dims { int uP, S, D, cF, in; };

__device__ __forceinline__ bool row_ok(int idx, int n) { return (unsigned)idx < (unsigned)n; }
// address of row idx of a row-sharded table whose shards are mapped at peer[0, world)
template <typename T>
__device__ __forceinline__ T* shard_row(const RowSrc& r, T* const* peer, int idx, long ld) {
    return peer[idx & r.wmask] + (long)(idx >> r.wshift) * ld;
}
// address of ITEM_EMB row idx (must be valid)
__device__ __forceinline__ const float* emb_row(const RowSrc& r, int idx) {
    return r.world > 1 ? shard_row(r, r.peer_emb, idx, r.lde) : r.emb + (long)idx * r.lde;
}
__device__ __forceinline__ const float* ifeat_row(const RowSrc& r, int idx) {
    return r.ifeat_sharded ? shard_row(r, r.peer_ifeat, idx, r.ldi) : r.ifeat + (long)idx * r.ldi;
}

__device__ __forceinline__ const float* src_ub(const RowSrc& r, const Dims& d, int b, int s) {
    if (b >= r.nvalid) return nullptr;
    if (r.dense) return r.X + (long)b * r.ldx + r.ub0 + (long)s * d.D;
    int idx = __ldg(r.hist + (long)b * d.S + s);
    return row_ok(idx, r.n_emb) ? emb_row(r, idx) : nullptr;
}
__device__ __forceinline__ const float* src_it(const RowSrc& r, const Dims& d, int b) {
    if (b >= r.nvalid) return nullptr;
    if (r.dense) return r.X + (long)b * r.ldx + r.it0;
    int idx = r.item_row[b];
    return row_ok(idx, r.n_emb) ? emb_row(r, idx) : nullptr;
}
__device__ __forceinline__ const float* src_up(const RowSrc& r, int b) {
    if (b >= r.nvalid) return nullptr;
    if (r.dense) return r.X + (long)b * r.ldx + r.up0;
    int idx = r.user_row[b];
    return row_ok(idx, r.n_user) ? r.ufeat + (long)idx * r.ldu : nullptr;
}
__device__ __forceinline__ const float* src_cx(const RowSrc& r, int b) {
    if (b >= r.nvalid) return nullptr;
    if (r.dense) return r.X + (long)b * r.ldx + r.cx0;
    int idx = r.item_feat_row ? r.item_feat_row[b] : r.item_row[b];
    return row_ok(idx, r.n_ifeat) ? ifeat_row(r, idx) : nullptr;
}

}  // namespace ctr
