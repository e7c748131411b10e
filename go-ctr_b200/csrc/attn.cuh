// attn.cuh — embedding-row gather fused with DIN's attention ActivationUnit / YouTube mean-pool
// (forward), and its backward fused with the gradient scatter-add + SGD row update.
//
// Replaces, per batch: recommend.GetSampleVector's lookups + concat (rcmd.go:462-536),
// model.CosineSimilarity (activation.go:57-83) / EucDistance (:23-50), the attention weight and
// sigmoid gate (din.go:231-276), G.Mean pooling (din.go:298, dnn.go:164-167) and G.Concat
// (din.go:301, dnn.go:170).  HBM-bound: (S+1) rows of D floats per sample, one pass forward, one
// pass backward (+ the L2-side red.add that writes each touched row back once).
//
// Mapping: one warp per sample; a row of D = 4*LPR*VPL floats is covered by LPR lanes x VPL 128-bit loads,
// so a warp carries 32/LPR rows per step and the dot products reduce inside the LPR-lane group with
// __shfl_xor.  Three kernel families:
//   k_attn_{fwd,bwd}_idx  index mode (rows come from the HBM tables), D in {16,32,64,128}, S <= 64: the
//                         fast path — next-sample ids and the dense features travel through lane-private
//                         shared-memory slots (cp.async), see the comments at the kernels;
//   k_attn_{fwd,bwd}_vec  the same lane mapping for the dense-X compatibility route and S > 64;
//   k_attn_{fwd,bwd}_gen  any D <= 256, unaligned sources (the reference test's D = 7), scalar loads;
//   k_attn_fwd_user       one user against a run of consecutive items (ctr_recommend_topk), history in shared memory.
// _vec and _idx share their per-row math (attn_gate, bwd_coef, sum_subgroups); _gen keeps exact sqrtf / division.
#pragma once
#include "common.cuh"

namespace ctr {

enum { MODEL_YOUTUBE = 0, MODEL_DIN_COS = 1, MODEL_DIN_EUC = 2 };

// prefetched history indices of one sample, two per lane (S <= 64), broadcast by shuffle
struct HistIdx {
    int i0, i1;
    __device__ __forceinline__ void load(const RowSrc& r, const Dims& d, int b, int lane) {
        i0 = i1 = -1;
        if (!r.dense && b < r.nvalid) {
            const int* h = r.hist + (long)b * d.S;
            if (lane < d.S) i0 = __ldg(h + lane);
            if (lane + 32 < d.S) i1 = __ldg(h + lane + 32);
        }
    }
    // all 32 lanes must call; s may differ per lane
    __device__ __forceinline__ int get(int s) const {
        int a0 = __shfl_sync(0xffffffffu, i0, s & 31);
        int a1 = __shfl_sync(0xffffffffu, i1, s & 31);
        return s < 32 ? a0 : a1;
    }
};

// one history slot: pointer to the row (nullptr = zeros) and its table row id (-1 in dense mode)
struct RowRef { const float* p; int idx; };

// history ids come from hi when it holds them (index mode, S <= 64), else from r.hist
__device__ __forceinline__ RowRef ub_ref(const RowSrc& r, const Dims& d, const HistIdx& hi, int b, int s) {
    const bool use_hi = (!r.dense) && d.S <= 64;
    // every lane of the warp reaches the shuffle inside hi.get()
    int sidx = use_hi ? hi.get(s < d.S ? s : 0) : -1;
    RowRef o; o.p = nullptr; o.idx = -1;
    if (s >= d.S || b >= r.nvalid) return o;
    if (r.dense) { o.p = r.X + (long)b * r.ldx + r.ub0 + (long)s * d.D; return o; }
    int idx = use_hi ? sidx : __ldg(r.hist + (long)b * d.S + s);
    if (row_ok(idx, r.n_emb)) { o.p = emb_row(r, idx); o.idx = idx; }
    return o;
}

// MUFU-based reciprocal / sigmoid / sqrt for the attention gate, flush-to-zero forms (no denormal fix-up code
// around the MUFU): relative error ~1e-6, two orders below the 1e-4 parity bar
__device__ __forceinline__ float rcp_ftz(float x) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float rsqrt_ftz(float x) { float r; asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float ex2_ftz(float x) { float r; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float frcp(float x) { return rcp_ftz(x); }
// gorgonia's float32 sigmoid saturates outside [-88, 15]; below -88 the formula itself yields 1/(1+inf) = 0
__device__ __forceinline__ float sigmoid_fast(float x) {
    const float r = rcp_ftz(1.0f + ex2_ftz(-1.4426950408889634f * x));
    return x > 15.0f ? 1.0f : r;
}
// sqrt(x) for x >= 0 through MUFU.RSQ; squared norms below 1e-30 count as zero (they sit under the 1e-8 the
// cosine denominator adds anyway, activation.go:80)
__device__ __forceinline__ float fsqrt_pos(float x) { return x > 1e-30f ? x * rsqrt_ftz(x) : 0.0f; }

// attention gate of one row given the group-reduced dot products (generic kernels)
__device__ __forceinline__ float gate_cos(float dot, float nx2, float ny, float att_s) {
    return sigmoid32((dot / (sqrtf(nx2) * ny + 1e-8f) + 1.0f) * 0.5f * att_s);
}

// -------------------------------------------------------------------------------------------------
// Per-row math of the _vec and _idx kernels.  A row of D = 4*LPR*VPL floats is covered by LPR lanes
// holding VPL float4 each (column block q of lane l = (q*LPR + l)*4, so every load instruction of the
// group is one contiguous LPR*16-byte segment); a warp therefore carries 32/LPR rows per instruction
// group and the scalar gate math is amortised over them.
// -------------------------------------------------------------------------------------------------
// 128 threads per block with at least 8 blocks per SM: the micro-benchmark (tests/cuda/gather_probe.cu)
// shows occupancy, not software pipelining, is what hides the gate's MUFU/shuffle latency — 32 warps/SM
// at <= 64 registers reach ~5.9 TB/s.
constexpr int kAttnThreads = 128, kAttnMinBlocks = 8;

// attention gate a of history row s, u, against the item row v (ny = |v|); att[s] reads as 0 beyond S.  MODEL is a
// template parameter (no per-row branches); mean pooling has a = 1.
template <int LPR, int VPL, int MODEL>
__device__ __forceinline__ float attn_gate(const float4 (&u)[VPL], const float4 (&v)[VPL], float ny, const float* __restrict__ att,
                                           int s, int S) {
    float a = 1.0f;
    if (MODEL == MODEL_DIN_COS) {
        float dot = 0.0f, nx2 = 0.0f;
#pragma unroll
        for (int q = 0; q < VPL; q++) { dot += dot4(u[q], v[q]); nx2 += dot4(u[q], u[q]); }
        dot = group_sum<LPR>(dot); nx2 = group_sum<LPR>(nx2);
        const float cs = dot * frcp(fsqrt_pos(nx2) * ny + 1e-8f);
        a = sigmoid_fast((cs + 1.0f) * 0.5f * (s < S ? __ldg(att + s) : 0.0f));
    } else if (MODEL == MODEL_DIN_EUC) {
        float d2 = 0.0f;
#pragma unroll
        for (int q = 0; q < VPL; q++) {
            const float4 e = make_float4(u[q].x - v[q].x, u[q].y - v[q].y, u[q].z - v[q].z, u[q].w - v[q].w);
            d2 += dot4(e, e);
        }
        a = sigmoid_fast((1.0f - fsqrt_pos(group_sum<LPR>(d2))) * (s < S ? __ldg(att + s) : 0.0f));
    }
    return a;
}

// x[q] += the same lane's x[q] in the other 32/LPR - 1 sub-groups of the warp
template <int LPR, int VPL>
__device__ __forceinline__ void sum_subgroups(float4 (&x)[VPL]) {
#pragma unroll
    for (int q = 0; q < VPL; q++) {
#pragma unroll
        for (int o = LPR; o < 32; o <<= 1) {
            x[q].x += __shfl_xor_sync(0xffffffffu, x[q].x, o);
            x[q].y += __shfl_xor_sync(0xffffffffu, x[q].y, o);
            x[q].z += __shfl_xor_sync(0xffffffffu, x[q].z, o);
            x[q].w += __shfl_xor_sync(0xffffffffu, x[q].w, o);
        }
    }
}

// -------------------------------------------------------------------------------------------------
// forward, vector path.  Writes the MLP input row X0[b] = [uProfile | pooled | item | ctx | 0-pad].
// -------------------------------------------------------------------------------------------------
template <int LPR, int VPL, int MODEL>
__global__ void __launch_bounds__(kAttnThreads, kAttnMinBlocks)
k_attn_fwd_vec(RowSrc r, Dims d, const float* __restrict__ att,
               float* __restrict__ X0, long ldx0, int Kp, int B) {
    extern __shared__ __align__(16) float smem[];
    constexpr int RPW = 32 / LPR, NT = kAttnThreads;
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int lir = lane % LPR, sub = lane / LPR;
    const int nwarps = gridDim.x * (NT / 32);
    float* row = smem + (long)wib * Kp;
    const float invS = 1.0f / (float)d.S;
    // 128-bit copies of the dense per-sample features when every offset is 16-byte aligned
    const bool feat4 = (!r.dense) && (d.uP % 4 == 0) && (d.D % 2 == 0) && (r.ldu % 4 == 0) && (r.ldi % 4 == 0);
    const int nu4 = (d.uP + 3) / 4, nc4 = (d.cF + 3) / 4;

    for (int b = blockIdx.x * (NT / 32) + wib; b < B; b += nwarps) {
        HistIdx hi; hi.load(r, d, b, lane);
        const float* ip = src_it(r, d, b);
        float4 v[VPL];
        float ny2 = 0.0f;
#pragma unroll
        for (int q = 0; q < VPL; q++) { v[q] = ip ? ldg4(ip + (q * LPR + lir) * 4) : zero4(); ny2 += dot4(v[q], v[q]); }
        // dense per-sample features: issued before the row loop so they overlap it
        const float* pu = src_up(r, b);
        const float* pc = src_cx(r, b);
        if (feat4) {            // table rows are zero-padded to a multiple of 4 floats (ctr_table_upload)
            for (int j = lane; j < nu4; j += 32) *reinterpret_cast<float4*>(row + 4 * j) = pu ? ldg4(pu + 4 * j) : zero4();
            for (int j = lane; j < nc4; j += 32) *reinterpret_cast<float4*>(row + d.uP + 2 * d.D + 4 * j) = pc ? ldg4(pc + 4 * j) : zero4();
            for (int j = d.uP + 2 * d.D + 4 * nc4 + lane; j < Kp; j += 32) row[j] = 0.0f;
        } else {
            for (int j = lane; j < d.uP; j += 32) row[j] = pu ? __ldg(pu + j) : 0.0f;
            for (int j = lane; j < d.cF; j += 32) row[d.uP + 2 * d.D + j] = pc ? __ldg(pc + j) : 0.0f;
            for (int j = d.in + lane; j < Kp; j += 32) row[j] = 0.0f;
        }
        const float ny = fsqrt_pos(group_sum<LPR>(ny2));
        float4 acc[VPL];
#pragma unroll
        for (int q = 0; q < VPL; q++) acc[q] = zero4();
        for (int s0 = 0; s0 < d.S; s0 += RPW) {
            const int s = s0 + sub;
            const float* p = ub_ref(r, d, hi, b, s).p;
            float4 u[VPL];
#pragma unroll
            for (int q = 0; q < VPL; q++) u[q] = p ? ldg4_stream(p + (q * LPR + lir) * 4) : zero4();
            const float a = attn_gate<LPR, VPL, MODEL>(u, v, ny, att, s, d.S);
#pragma unroll
            for (int q = 0; q < VPL; q++) acc[q] = fma4(a, u[q], acc[q]);   // slots beyond S / missing rows carry u == 0
        }
        sum_subgroups<LPR, VPL>(acc);
        // assemble the concat row in shared memory, then one coalesced 128-bit store pass
        if (sub == 0) {
#pragma unroll
            for (int q = 0; q < VPL; q++) {
                float* p1 = row + d.uP + (q * LPR + lir) * 4;
                p1[0] = acc[q].x * invS; p1[1] = acc[q].y * invS; p1[2] = acc[q].z * invS; p1[3] = acc[q].w * invS;
                float* p2 = p1 + d.D;
                p2[0] = v[q].x; p2[1] = v[q].y; p2[2] = v[q].z; p2[3] = v[q].w;
            }
        }
        __syncwarp();
        float4* dst = reinterpret_cast<float4*>(X0 + (long)b * ldx0);
        const float4* src4 = reinterpret_cast<const float4*>(row);
        for (int j = lane; j < Kp / 4; j += 32) dst[j] = src4[j];
        __syncwarp();
    }
}

// -------------------------------------------------------------------------------------------------
// forward, index path (the fast path: rows come from the HBM tables).  Same lane mapping and math as
// k_attn_fwd_vec, with everything the dense-X route needs compiled out:
//   * the sample's ids for the NEXT sample and this lane's 16-byte chunk of the dense features travel
//     through lane-private shared-memory slots with cp.async — no registers held, no load the warp must
//     wait for in front of the row loop, and the id → address dependency is off the critical path;
//   * the MLP input row is written straight from registers: lanes [0, uP/4) own the user-profile chunks,
//     the following lanes the ctx chunks and the zero pad, the sub-group-0 lanes pooled + item.
// Requires S <= 64, uP % 4 == 0, 16-byte aligned table rows and (Kp - 2D)/4 <= 32 (one chunk per lane).
// -------------------------------------------------------------------------------------------------
// streaming 128-bit load of a row that may live in a peer GPU's HBM (NVLink): plain ld.global, no L1 allocation
__device__ __forceinline__ float4 ld4_peer(const float* p) {
    float4 r;
    asm volatile("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}
template <bool PEER>
__device__ __forceinline__ float* emb_ptr(const RowSrc& r, int idx) {
    return PEER ? shard_row(r, r.peer_emb, idx, r.lde) : const_cast<float*>(r.emb) + (long)idx * r.lde;
}
// read side of a sharded table: the replicated hot rows are local
template <bool PEER>
__device__ __forceinline__ const float* emb_src(const RowSrc& r, int idx) {
    if (PEER && idx < r.hot_k) return r.hot_tab + (long)idx * r.lde;
    return emb_ptr<PEER>(r, idx);
}

// PEER: ITEM_EMB (and ITEM_FEAT when large) are row-sharded over the GPUs of the box and every shard is mapped into
// this process (CUDA IPC): the gather reads the owner's HBM directly over NVLink — the transfer is the load itself, so
// it overlaps the gate math of the other warps tile by tile — and keeps each fetched row in rows_cache for the
// backward, so a row crosses NVLink once per step.
template <int LPR, int VPL, int MODEL, bool PEER>
__global__ void __launch_bounds__(kAttnThreads, kAttnMinBlocks)
k_attn_fwd_idx(RowSrc r, Dims d, const float* __restrict__ att, float* __restrict__ X0, long ldx0, int Kp, int B) {
    constexpr int RPW = 32 / LPR, DD = 4 * LPR * VPL, NT = kAttnThreads;
    __shared__ __align__(16) float4 s_feat[NT];      // lane-private: this lane's feature chunk of the current sample
    __shared__ __align__(16) int4 s_ids[NT];         // lane-private: {hist id lane, hist id lane+32, item row, feature row} of the next sample
    const int lane = threadIdx.x & 31, lir = lane % LPR, sub = lane / LPR;
    const int nwarps = gridDim.x * (NT / 32);
    int b = blockIdx.x * (NT / 32) + (threadIdx.x >> 5);
    if (b >= B) return;
    const float invS = 1.0f / (float)d.S;
    const int nu4 = d.uP >> 2, nc4 = (d.cF + 3) >> 2;
    const bool f_user = lane < nu4;
    const int fc = f_user ? lane : lane - nu4;
    const bool f_load = f_user || fc < nc4;
    const int f_off = f_user ? 4 * lane : d.uP + 2 * DD + 4 * fc;
    const int f_n = f_user ? r.n_user : r.n_ifeat;
    const int* f_ids = f_user ? r.user_row : (r.item_feat_row ? r.item_feat_row : r.item_row);
    int* my_ids = reinterpret_cast<int*>(&s_ids[threadIdx.x]);
    float4* my_feat = &s_feat[threadIdx.x];

    auto fetch_ids = [&](int bb) {           // asynchronous: lands in my_ids; the zero-padded tail (model.go:357-371) has no ids
        if (bb < r.nvalid) {
            const int* h = r.hist + (long)bb * d.S;
            if (lane < d.S) cp_async4(my_ids, h + lane);
            if (lane + 32 < d.S) cp_async4(my_ids + 1, h + lane + 32);
            cp_async4(my_ids + 2, r.item_row + bb);
            cp_async4(my_ids + 3, f_ids + bb);
        } else *reinterpret_cast<int4*>(my_ids) = make_int4(-1, -1, -1, -1);
        cp_async_commit();
    };
    *reinterpret_cast<int4*>(my_ids) = make_int4(-1, -1, -1, -1);
    fetch_ids(b);
    for (;;) {
        cp_async_wait_all();
        int4 id = *reinterpret_cast<const int4*>(my_ids);        // x: hist[lane], y: hist[lane+32], z: item, w: feature row
        id.x = row_ok(id.x, r.n_emb) ? id.x : -1; id.y = row_ok(id.y, r.n_emb) ? id.y : -1;
        id.z = row_ok(id.z, r.n_emb) ? id.z : -1; id.w = row_ok(id.w, f_n) ? id.w : -1;
        const int bn = b + nwarps;
        if (bn < B) fetch_ids(bn);
        if (f_load) {
            const int fw = id.w >= 0 ? id.w : 0;
            const float* fp = f_user ? r.ufeat + (long)fw * r.ldu : (PEER ? ifeat_row(r, fw) : r.ifeat + (long)fw * r.ldi);
            cp_async16(my_feat, fp + 4 * fc, id.w >= 0);
        }
        cp_async_commit();
        float4 v[VPL], acc[VPL];
        float ny2 = 0.0f;
        const float* ip = emb_src<PEER>(r, id.z >= 0 ? id.z : 0);
        float* cache_b = (PEER && r.rows_cache) ? r.rows_cache + (long)b * (d.S + 1) * DD : nullptr;    // predict keeps no rows
#pragma unroll
        for (int q = 0; q < VPL; q++) {
            v[q] = id.z >= 0 ? (PEER ? ld4_peer(ip + (q * LPR + lir) * 4) : ldg4(ip + (q * LPR + lir) * 4)) : zero4();
            acc[q] = zero4();
        }
        // history rows: the loads of a group are issued, then (first group only) the item row's norm is formed
        // while they are in flight, then the group is consumed
        int row;
        auto load_rows = [&](float4 (&u)[VPL], int s0) {
            const int s = s0 + sub;
            const int a0 = __shfl_sync(0xffffffffu, id.x, s & 31), a1 = __shfl_sync(0xffffffffu, id.y, s & 31);
            row = s < d.S ? (s < 32 ? a0 : a1) : -1;
            const float* p = emb_src<PEER>(r, row >= 0 ? row : 0) + lir * 4;
#pragma unroll
            for (int q = 0; q < VPL; q++) u[q] = row >= 0 ? (PEER ? ld4_peer(p + q * LPR * 4) : ldg4_stream(p + q * LPR * 4)) : zero4();
        };
        float4 u[VPL];
        load_rows(u, 0);
#pragma unroll
        for (int q = 0; q < VPL; q++) ny2 += dot4(v[q], v[q]);
        const float ny = fsqrt_pos(group_sum<LPR>(ny2));
        if (PEER && cache_b && sub == 0 && id.z >= 0) {
#pragma unroll
            for (int q = 0; q < VPL; q++) *reinterpret_cast<float4*>(cache_b + (long)d.S * DD + (q * LPR + lir) * 4) = v[q];
        }
        for (int s0 = 0;;) {
            const int s = s0 + sub;
            const float a = attn_gate<LPR, VPL, MODEL>(u, v, ny, att, s, d.S);
#pragma unroll
            for (int q = 0; q < VPL; q++) acc[q] = fma4(a, u[q], acc[q]);      // slots beyond S / missing rows carry u == 0
            if (PEER && cache_b && row >= 0) {
                float* c = cache_b + (long)s * DD + lir * 4;
#pragma unroll
                for (int q = 0; q < VPL; q++) *reinterpret_cast<float4*>(c + q * LPR * 4) = u[q];
            }
            s0 += RPW;
            if (s0 >= d.S) break;
            load_rows(u, s0);
        }
        sum_subgroups<LPR, VPL>(acc);
        float* xr = X0 + (long)b * ldx0;
        if (sub == 0) {
#pragma unroll
            for (int q = 0; q < VPL; q++) {
                *reinterpret_cast<float4*>(xr + d.uP + (q * LPR + lir) * 4) = make_float4(acc[q].x * invS, acc[q].y * invS, acc[q].z * invS, acc[q].w * invS);
                *reinterpret_cast<float4*>(xr + d.uP + DD + (q * LPR + lir) * 4) = v[q];
            }
        }
        if (f_off < Kp) {
            // my feature chunk landed long ago unless the next sample's ids (committed before it) are still in
            // flight: wait for all but that newest-but-one group is not expressible per lane → wait for both
            cp_async_wait_all();
            *reinterpret_cast<float4*>(xr + f_off) = f_load ? *my_feat : zero4();
        }
        if (bn >= B) break;
        b = bn;
    }
}

// -------------------------------------------------------------------------------------------------
// forward, one user against a run of consecutive items (ctr_recommend_topk): X0[b] is the MLP input row of the sample
// (user, item i0 + b, hist[0, S)) for b < B; every item i0 + b must be a row of ITEM_EMB.  Each CTA stages the user's
// S history rows (zeros for missing slots) in shared memory once; a warp then reads only its item's ITEM_EMB and
// ITEM_FEAT rows.  Same lane map and per-row math as k_attn_fwd_idx / _vec (attn_gate, fma4 in s0 order,
// sum_subgroups), so every row is bit-identical to the row they write for the same sample.  The profile row and the
// zero pad are the same for every item: each warp writes them once into its staging row.
// Dynamic shared memory: user_smem_floats(S, D, Kp) floats.  Two blocks fewer per SM than the gather kernels (80
// registers): the history comes from shared memory, so fewer loads need to be in flight, and the cosine gate at D >= 64
// fits without spills.
// PEER (row-sharded ITEM_EMB): the items are this rank's local rows i0 + b (r.emb is the shard, the hot rows written
// back), global row (i0 + b)·world + rank; the history rows come through emb_src<PEER> (the hot-row replica, else the
// owner's HBM over NVLink); the item's ITEM_FEAT row is its local row of a sharded ITEM_FEAT or its global row of a
// replicated one, missing when the global row is not below n_ifeat.
// -------------------------------------------------------------------------------------------------
__host__ __device__ inline size_t user_smem_floats(int S, int D, int Kp) { return (size_t)S * D + (size_t)(kAttnThreads / 32) * Kp; }

template <int LPR, int VPL, int MODEL, bool PEER>
__global__ void __launch_bounds__(kAttnThreads, kAttnMinBlocks - 2)
k_attn_fwd_user(RowSrc r, Dims d, const float* __restrict__ att, int user, const int* __restrict__ hist, int i0, int rank,
                float* __restrict__ X0, long ldx0, int Kp, int B) {
    extern __shared__ __align__(16) float smem[];
    constexpr int RPW = 32 / LPR, DD = 4 * LPR * VPL, NT = kAttnThreads;
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int lir = lane % LPR, sub = lane / LPR;
    const int nwarps = gridDim.x * (NT / 32);
    float4* s_hist = reinterpret_cast<float4*>(smem);                 // [S][DD/4]
    float* row = smem + (long)d.S * DD + (long)wib * Kp;              // this warp's MLP input row
    for (int i = threadIdx.x; i < d.S * (DD / 4); i += NT) {
        const int s = i / (DD / 4), c = i - s * (DD / 4);
        const int idx = __ldg(hist + s);
        s_hist[i] = !row_ok(idx, r.n_emb) ? zero4() : PEER ? ld4_peer(emb_src<PEER>(r, idx) + 4 * c) : ldg4(r.emb + (long)idx * r.lde + 4 * c);
    }
    const float* pu = row_ok(user, r.n_user) ? r.ufeat + (long)user * r.ldu : nullptr;
    for (int j = lane; j < d.uP; j += 32) row[j] = pu ? __ldg(pu + j) : 0.0f;
    for (int j = d.in + lane; j < Kp; j += 32) row[j] = 0.0f;
    __syncthreads();
    const float invS = 1.0f / (float)d.S;

    for (int b = blockIdx.x * (NT / 32) + wib; b < B; b += nwarps) {
        const int item = i0 + b;
        const float* ip = r.emb + (long)item * r.lde;
        float4 v[VPL];
        float ny2 = 0.0f;
#pragma unroll
        for (int q = 0; q < VPL; q++) { v[q] = ldg4(ip + (q * LPR + lir) * 4); ny2 += dot4(v[q], v[q]); }
        const float ny = fsqrt_pos(group_sum<LPR>(ny2));
        float4 acc[VPL];
#pragma unroll
        for (int q = 0; q < VPL; q++) acc[q] = zero4();
        for (int s0 = 0; s0 < d.S; s0 += RPW) {
            const int s = s0 + sub;
            float4 u[VPL];
#pragma unroll
            for (int q = 0; q < VPL; q++) u[q] = s < d.S ? s_hist[s * (DD / 4) + q * LPR + lir] : zero4();
            const float a = attn_gate<LPR, VPL, MODEL>(u, v, ny, att, s, d.S);
#pragma unroll
            for (int q = 0; q < VPL; q++) acc[q] = fma4(a, u[q], acc[q]);   // slots beyond S / missing rows carry u == 0
        }
        sum_subgroups<LPR, VPL>(acc);
        if (sub == 0) {
#pragma unroll
            for (int q = 0; q < VPL; q++) {
                float* p1 = row + d.uP + (q * LPR + lir) * 4;
                p1[0] = acc[q].x * invS; p1[1] = acc[q].y * invS; p1[2] = acc[q].z * invS; p1[3] = acc[q].w * invS;
                float* p2 = p1 + d.D;
                p2[0] = v[q].x; p2[1] = v[q].y; p2[2] = v[q].z; p2[3] = v[q].w;
            }
        }
        const float* pc;
        if (PEER) {
            const int gi = item * r.world + rank;
            pc = row_ok(gi, r.n_ifeat) ? r.ifeat + (long)(r.ifeat_sharded ? item : gi) * r.ldi : nullptr;
        } else pc = row_ok(item, r.n_ifeat) ? r.ifeat + (long)item * r.ldi : nullptr;
        for (int j = lane; j < d.cF; j += 32) row[d.uP + 2 * d.D + j] = pc ? __ldg(pc + j) : 0.0f;
        __syncwarp();
        float4* dst = reinterpret_cast<float4*>(X0 + (long)b * ldx0);
        const float4* src4 = reinterpret_cast<const float4*>(row);
        for (int j = lane; j < Kp / 4; j += 32) dst[j] = src4[j];
        __syncwarp();
    }
}

// -------------------------------------------------------------------------------------------------
// forward, generic path (any D <= 256, unaligned sources — the dense-X compatibility route and odd
// dims such as the reference test's D=7, model_test.go:24-28).
// -------------------------------------------------------------------------------------------------
constexpr int kGenAcc = 8;   // D <= 32*kGenAcc

__global__ void __launch_bounds__(256)
k_attn_fwd_gen(RowSrc r, Dims d, int model, const float* __restrict__ att,
               float* __restrict__ X0, long ldx0, int Kp, int B) {
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int nwarps = gridDim.x * (blockDim.x >> 5);
    const float invS = 1.0f / (float)d.S;
    for (int b = blockIdx.x * (blockDim.x >> 5) + wib; b < B; b += nwarps) {
        const float* ip = src_it(r, d, b);
        float vv[kGenAcc], acc[kGenAcc];
        float ny2 = 0.0f;
#pragma unroll
        for (int j = 0; j < kGenAcc; j++) {
            int k = lane + 32 * j;
            vv[j] = (ip && k < d.D) ? __ldg(ip + k) : 0.0f;
            ny2 += vv[j] * vv[j]; acc[j] = 0.0f;
        }
        const float ny = sqrtf(warp_sum(ny2));
        for (int s = 0; s < d.S; s++) {
            const float* up = src_ub(r, d, b, s);
            float uu[kGenAcc]; float dot = 0.0f, nx2 = 0.0f, d2 = 0.0f;
#pragma unroll
            for (int j = 0; j < kGenAcc; j++) {
                int k = lane + 32 * j;
                uu[j] = (up && k < d.D) ? __ldg(up + k) : 0.0f;
                dot += uu[j] * vv[j]; nx2 += uu[j] * uu[j];
                float e = uu[j] - vv[j]; d2 += e * e;
            }
            float a = 1.0f;
            if (model == MODEL_DIN_COS) {
                dot = warp_sum(dot); nx2 = warp_sum(nx2);
                a = gate_cos(dot, nx2, ny, __ldg(att + s));
            } else if (model == MODEL_DIN_EUC) {
                d2 = warp_sum(d2);
                a = sigmoid32((1.0f - sqrtf(d2)) * __ldg(att + s));
            }
#pragma unroll
            for (int j = 0; j < kGenAcc; j++) acc[j] = fmaf(a, uu[j], acc[j]);
        }
        float* dst = X0 + (long)b * ldx0;
        const float* pu = src_up(r, b);
        for (int j = lane; j < d.uP; j += 32) dst[j] = pu ? __ldg(pu + j) : 0.0f;
#pragma unroll
        for (int j = 0; j < kGenAcc; j++) {
            int k = lane + 32 * j;
            if (k < d.D) { dst[d.uP + k] = acc[j] * invS; dst[d.uP + d.D + k] = vv[j]; }
        }
        const float* pc = src_cx(r, b);
        for (int j = lane; j < d.cF; j += 32) dst[d.uP + 2 * d.D + j] = pc ? __ldg(pc + j) : 0.0f;
        for (int j = d.in + lane; j < Kp; j += 32) dst[j] = 0.0f;
    }
}

// -------------------------------------------------------------------------------------------------
// backward.  dX[b] = [g (d cost/d pooled) | gi (d cost/d item through the MLP input)].
// Emits d cost/d att0 (sum over batch), and for every gathered row either
//   * sgd != 0: fused scatter-add + SGD with red.global.add.v4.f32:
//       rows >= hot_rows : table_row += -lr * grad directly;
//       rows <  hot_rows : grad accumulates in one of hot_reps replica accumulators (contention on
//                          popular rows is spread over the replicas; k_hot_apply folds them into
//                          the table after the kernel), or
//   * dUb/dIt buffers (deterministic update path, debug hook, multi-GPU return leg).
// Analytic reverse of din.go:231-298 (see DESIGN.md §kernels for the derivation):
//   da_s = g·u_s / S ; dz_s = da_s a_s (1-a_s) ; datt_s += dz_s w_s ; dw_s = dz_s att_s
//   cosine:  c = dw_s/2 ; du_s = a_s g/S + c (v/den - cos·|v| u_s/(|u_s| den))
//                         dv  += c (u_s/den - cos·|u_s| v/(|v| den))
//   euclid:  du_s = a_s g/S - dw_s (u_s-v)/dist ; dv += dw_s (u_s-v)/dist
//   mean  :  du_s = g/S
// -------------------------------------------------------------------------------------------------
struct BwdOut {
    float* datt;        // [S] accumulated with atomics (zeroed by the optimiser step)
    float* dUb;         // [B,S,D] or null
    float* dIt;         // [B,D]   or null
    int    sgd;         // fused scatter-add + SGD into r.emb
    float  neg_lr;      // -table_lr
    float* hot_acc;     // [hot_reps, hot_rows, D] replica accumulators (sums of -lr * gradient)
    int    hot_rows, hot_reps;
    float* scatter_base;    // where row gradients are added (row idx * lde): the table itself, or the per-lookup
                            // gradient buffer of the sharded path
    // CTR_TABLE_ADAM on a row-sharded table (PEER): row gradients go to the owner's gradient buffer (peer_adam[j],
    // layout adam) instead of its rows, and every occurrence marks the row touched; hot_touch[row] = 1 marks a hot row
    unsigned char* peer_adam[kMaxPeers];
    ShardGrad adam;
    float* hot_touch;
};

// destination of one row's (already -lr scaled) gradient: a hot-row replica accumulator or the table row
__device__ __forceinline__ float* scatter_dst(const RowSrc& r, const Dims& d, const BwdOut& o, int idx, int rep) {
    if (idx < o.hot_rows) return o.hot_acc + ((long)rep * o.hot_rows + idx) * d.D;
    return o.scatter_base + (long)idx * r.lde;
}
// the same on a row-sharded table: the hot-row replica accumulators, else the owner's row over NVLink (SGD) or the
// owner's gradient row (row Adam).  lead: the one lane of the row's group that marks the row touched — the first
// marker of a row appends its local row to the owner's list
__device__ __forceinline__ float* peer_scatter_dst(const RowSrc& r, const Dims& d, const BwdOut& o, int idx, int rep, bool lead) {
    if (idx < o.hot_rows) {
        if (o.hot_touch && lead) o.hot_touch[idx] = 1.0f;
        return scatter_dst(r, d, o, idx, rep);
    }
    if (!o.peer_adam[0]) return shard_row(r, r.peer_emb, idx, r.lde);
    unsigned char* base = o.peer_adam[idx & r.wmask];
    const long lr = idx >> r.wshift;
    if (lead && atomicExch_system(reinterpret_cast<unsigned*>(base + o.adam.flag_off) + lr, 1u) == 0u) {
        const unsigned slot = atomicAdd_system(reinterpret_cast<unsigned*>(base), 1u);
        reinterpret_cast<int*>(base + o.adam.list_off)[slot] = (int)lr;
    }
    return reinterpret_cast<float*>(base + o.adam.grad_off) + lr * r.lde;
}

// Backward coefficients of history row s (u) for the lanes of its group: du = c1*g + c2*v + c3*u and
// dv += c4*u - kv*v, where kv is added to kvsum.  The group's lane 0 (lead) adds d att_s to sdatt[s] while
// s < S.  u is in registers; g and v are accessors q → float4 of this lane's chunk q, so that a kernel may
// keep them in shared memory.  ny = |v|, rny = 1/|v| (0 for v = 0).
struct DuCoef { float c1, c2, c3, c4; };
template <int LPR, int VPL, int MODEL, typename GF, typename VF>
__device__ __forceinline__ DuCoef bwd_coef(const float4 (&u)[VPL], GF g, VF v, float ny, float rny, float invS,
                                           const float* __restrict__ att, int s, int S, bool lead, float* sdatt, float& kvsum) {
    DuCoef c{invS, 0.0f, 0.0f, 0.0f};
    if (MODEL != MODEL_YOUTUBE) {
        const float att_s = s < S ? __ldg(att + s) : 0.0f;
        float gu = 0.0f, dot = 0.0f, nx2 = 0.0f;
#pragma unroll
        for (int q = 0; q < VPL; q++) {
            const float4 gq = g(q), vq = v(q);
            gu += dot4(gq, u[q]);
            if (MODEL == MODEL_DIN_COS) { dot += dot4(u[q], vq); nx2 += dot4(u[q], u[q]); }
            else {
                const float4 e = make_float4(u[q].x - vq.x, u[q].y - vq.y, u[q].z - vq.z, u[q].w - vq.w);
                nx2 += dot4(e, e);
            }
        }
        gu = group_sum<LPR>(gu); nx2 = group_sum<LPR>(nx2);
        if (MODEL == MODEL_DIN_COS) {
            dot = group_sum<LPR>(dot);
            const float nx = fsqrt_pos(nx2);
            const float iden = frcp(nx * ny + 1e-8f);
            const float cs = dot * iden;
            const float w = (cs + 1.0f) * 0.5f;
            const float a = sigmoid_fast(w * att_s);
            const float dz = gu * invS * a * (1.0f - a);
            if (lead && s < S) atomicAdd(&sdatt[s], dz * w);
            const float cc = 0.5f * dz * att_s;
            c.c1 = a * invS; c.c2 = cc * iden; c.c4 = c.c2;
            c.c3 = nx2 > 1e-30f ? -cc * cs * ny * iden * rsqrt_ftz(nx2) : 0.0f;   // -cc*cos*|v|/(|u| den)
            kvsum += cc * cs * nx * iden * rny;                                 //  cc*cos*|u|/(|v| den)
        } else {
            const float dist = fsqrt_pos(nx2);
            const float w = 1.0f - dist;
            const float a = sigmoid_fast(w * att_s);
            const float dz = gu * invS * a * (1.0f - a);
            if (lead && s < S) atomicAdd(&sdatt[s], dz * w);
            const float k = nx2 > 1e-30f ? dz * att_s * rsqrt_ftz(nx2) : 0.0f;  // dw/dist
            c.c1 = a * invS; c.c3 = -k; c.c2 = k;      // du = c1 g - k (u - v)
            c.c4 = s < S ? k : 0.0f;                   // dv += k (u - v)
            kvsum += c.c4;
        }
    }
    return c;
}

template <int LPR, int VPL, int MODEL>
__global__ void __launch_bounds__(kAttnThreads, kAttnMinBlocks)
k_attn_bwd_vec(RowSrc r, Dims d, const float* __restrict__ att,
               const float* __restrict__ dX, long lddx, BwdOut o, int B) {
    extern __shared__ __align__(16) float smem[];     // datt partials [S]
    constexpr int RPW = 32 / LPR, NT = kAttnThreads;
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int lir = lane % LPR, sub = lane / LPR;
    const int gwarp = blockIdx.x * (NT / 32) + wib;
    const int nwarps = gridDim.x * (NT / 32);
    const int rep = o.hot_reps > 0 ? gwarp % o.hot_reps : 0;
    const float invS = 1.0f / (float)d.S;
    const float sc = o.sgd ? o.neg_lr : 1.0f;         // fused SGD: gradients leave pre-scaled by -lr
    for (int j = threadIdx.x; j < d.S; j += NT) smem[j] = 0.0f;
    __syncthreads();

    for (int b = gwarp; b < B; b += nwarps) {
        HistIdx hi; hi.load(r, d, b, lane);
        const float* ip = src_it(r, d, b);
        float4 g[VPL], v[VPL], dvu[VPL];
        float ny2 = 0.0f;
#pragma unroll
        for (int q = 0; q < VPL; q++) {
            g[q] = ldg4(dX + (long)b * lddx + (q * LPR + lir) * 4);
            // the table is written by this kernel (sgd mode): coherent loads, no .nc
            v[q] = ip ? *reinterpret_cast<const float4*>(ip + (q * LPR + lir) * 4) : zero4();
            ny2 += dot4(v[q], v[q]); dvu[q] = zero4();
        }
        ny2 = group_sum<LPR>(ny2);
        const float ny = fsqrt_pos(ny2);
        const float rny = ny2 > 1e-30f ? rsqrt_ftz(ny2) : 0.0f;
        float kvsum = 0.0f;                               // coefficient of -v in dv
        for (int s0 = 0; s0 < d.S; s0 += RPW) {
            const int s = s0 + sub;
            const RowRef rr = ub_ref(r, d, hi, b, s);
            float4 u[VPL];
#pragma unroll
            for (int q = 0; q < VPL; q++) u[q] = rr.p ? *reinterpret_cast<const float4*>(rr.p + (q * LPR + lir) * 4) : zero4();
            const DuCoef c = bwd_coef<LPR, VPL, MODEL>(u, [&](int q) { return g[q]; }, [&](int q) { return v[q]; }, ny, rny, invS,
                                                       att, s, d.S, lir == 0, smem, kvsum);
            if (s < d.S) {
                const float e1 = c.c1 * sc, e2 = c.c2 * sc, e3 = c.c3 * sc;
                float* dst = (o.sgd && rr.p) ? scatter_dst(r, d, o, rr.idx, rep) : nullptr;
#pragma unroll
                for (int q = 0; q < VPL; q++) {
                    float4 du;
                    du.x = fmaf(e3, u[q].x, fmaf(e2, v[q].x, e1 * g[q].x)); du.y = fmaf(e3, u[q].y, fmaf(e2, v[q].y, e1 * g[q].y));
                    du.z = fmaf(e3, u[q].z, fmaf(e2, v[q].z, e1 * g[q].z)); du.w = fmaf(e3, u[q].w, fmaf(e2, v[q].w, e1 * g[q].w));
                    dvu[q] = fma4(c.c4, u[q], dvu[q]);
                    if (o.dUb) *reinterpret_cast<float4*>(o.dUb + ((long)b * d.S + s) * d.D + (q * LPR + lir) * 4) = du;
                    if (dst) red_add4(dst + (q * LPR + lir) * 4, du);
                }
            }
        }
        // dv = gi + sum_subgroups(dvu) - (sum kv) * v
#pragma unroll
        for (int of = LPR; of < 32; of <<= 1) kvsum += __shfl_xor_sync(0xffffffffu, kvsum, of);
        sum_subgroups<LPR, VPL>(dvu);
        if (sub == 0) {
            float* dst = (o.sgd && ip) ? scatter_dst(r, d, o, r.item_row[b], rep) : nullptr;
#pragma unroll
            for (int q = 0; q < VPL; q++) {
                const float4 gi = ldg4(dX + (long)b * lddx + d.D + (q * LPR + lir) * 4);
                float4 dv;
                dv.x = (gi.x + dvu[q].x - kvsum * v[q].x) * sc; dv.y = (gi.y + dvu[q].y - kvsum * v[q].y) * sc;
                dv.z = (gi.z + dvu[q].z - kvsum * v[q].z) * sc; dv.w = (gi.w + dvu[q].w - kvsum * v[q].w) * sc;
                if (o.dIt) *reinterpret_cast<float4*>(o.dIt + (long)b * d.D + (q * LPR + lir) * 4) = dv;
                if (dst) red_add4(dst + (q * LPR + lir) * 4, dv);
            }
        }
    }
    __syncthreads();
    if (MODEL != MODEL_YOUTUBE && o.datt)
        for (int j = threadIdx.x; j < d.S; j += NT)
            if (smem[j] != 0.0f) atomicAdd(o.datt + j, smem[j]);
}

// backward, index path: k_attn_bwd_vec's math with the dense-X route compiled out, the next sample's ids
// prefetched through lane-private shared-memory slots (see k_attn_fwd_idx), and the two per-sample vectors
// every row needs — g = d cost/d pooled and the item row v — parked in shared memory instead of registers.
// That frees the registers for the forward kernel's wide lane mapping (LPR lanes x VPL float4 per row, 32/LPR
// rows per step), which halves the per-row share of the gate's scalar/shuffle/MUFU work against the
// 8-lanes-per-row mapping the register-resident version was limited to.  FUSED: scatter-add + SGD straight into
// the table / hot-row replicas (red.global.add.v4.f32); otherwise gradients go to the dUb / dIt buffers.
// Requires S <= 64.
// PEER (row-sharded tables over NVLink, see k_attn_fwd_idx): rows are re-read from rows_cache (what the forward
// fetched — the gradient is taken at the step-start table values, and nothing crosses NVLink twice), and each row
// gradient leaves as red.global.add.v4.f32 straight into the OWNER's table over NVLink, pre-scaled by -lr/world (row
// Adam: into the owner's gradient shard, scaled by 1/world, marking the row touched — peer_scatter_dst).
template <int LPR, int VPL, int MODEL, bool FUSED, bool PEER>
__global__ void __launch_bounds__(kAttnThreads, kAttnMinBlocks)
k_attn_bwd_idx(RowSrc r, Dims d, const float* __restrict__ att,
               const float* __restrict__ dX, long lddx, BwdOut o, int B) {
    constexpr int RPW = 32 / LPR, CH = LPR * VPL, NT = kAttnThreads;
    __shared__ float s_datt[64];
    __shared__ __align__(16) int4 s_ids[NT];
    __shared__ __align__(16) float4 s_g[NT / 32][CH], s_v[NT / 32][CH];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, lir = lane % LPR, sub = lane / LPR;
    const int gwarp = blockIdx.x * (NT / 32) + wib;
    const int nwarps = gridDim.x * (NT / 32);
    const int rep = o.hot_reps > 0 ? gwarp % o.hot_reps : 0;
    const float invS = 1.0f / (float)d.S;
    const float sc = FUSED ? o.neg_lr : 1.0f;         // fused SGD: gradients leave pre-scaled by -lr
    if (MODEL != MODEL_YOUTUBE && threadIdx.x < 64) s_datt[threadIdx.x] = 0.0f;     // mean pooling has no att
    int* my_ids = reinterpret_cast<int*>(&s_ids[threadIdx.x]);
    *reinterpret_cast<int4*>(my_ids) = make_int4(-1, -1, -1, -1);
    __syncthreads();
    auto fetch_ids = [&](int bb) {           // the zero-padded tail (model.go:357-371) has no ids
        if (bb < r.nvalid) {
            const int* h = r.hist + (long)bb * d.S;
            if (lane < d.S) cp_async4(my_ids, h + lane);
            if (lane + 32 < d.S) cp_async4(my_ids + 1, h + lane + 32);
            cp_async4(my_ids + 2, r.item_row + bb);
        } else *reinterpret_cast<int4*>(my_ids) = make_int4(-1, -1, -1, -1);
        cp_async_commit();
    };
    const float4* gs = s_g[wib];
    const float4* vs = s_v[wib];
    auto g_of = [&](int q) { return gs[q * LPR + lir]; };       // this lane's chunk q of g / v
    auto v_of = [&](int q) { return vs[q * LPR + lir]; };
    int b = gwarp;
    if (b < B) fetch_ids(b);
    while (b < B) {
        cp_async_wait_all();
        int4 id = *reinterpret_cast<const int4*>(my_ids);
        id.x = row_ok(id.x, r.n_emb) ? id.x : -1; id.y = row_ok(id.y, r.n_emb) ? id.y : -1; id.z = row_ok(id.z, r.n_emb) ? id.z : -1;
        const int bn = b + nwarps;
        if (bn < B) fetch_ids(bn);
        const float* cache_b = PEER ? r.rows_cache + (long)b * (d.S + 1) * (4 * CH) : nullptr;
        // stage g and v (one float4 per lane; the table is written by this kernel in FUSED mode: coherent load)
        if (lane < CH) {
            s_g[wib][lane] = ldg4(dX + (long)b * lddx + 4 * lane);
            const float* vp = PEER ? cache_b + (long)d.S * (4 * CH) : r.emb + (long)(id.z >= 0 ? id.z : 0) * r.lde;
            s_v[wib][lane] = id.z >= 0 ? *reinterpret_cast<const float4*>(vp + 4 * lane) : zero4();
        }
        auto load_rows = [&](float4 (&u)[VPL], int& row, int s0) {
            const int s = s0 + sub;
            const int a0 = __shfl_sync(0xffffffffu, id.x, s & 31), a1 = __shfl_sync(0xffffffffu, id.y, s & 31);
            row = s < d.S ? (s < 32 ? a0 : a1) : -1;
            const float* p = (PEER ? cache_b + (long)(s < d.S ? s : 0) * (4 * CH) : r.emb + (long)(row >= 0 ? row : 0) * r.lde) + lir * 4;
#pragma unroll
            for (int q = 0; q < VPL; q++) u[q] = row >= 0 ? *reinterpret_cast<const float4*>(p + q * LPR * 4) : zero4();
        };
        float4 u[VPL], dvu[VPL];
        int row;
        load_rows(u, row, 0);
        __syncwarp();
        float ny2 = 0.0f;
#pragma unroll
        for (int q = 0; q < VPL; q++) { const float4 t = v_of(q); ny2 += dot4(t, t); dvu[q] = zero4(); }
        ny2 = group_sum<LPR>(ny2);
        const float ny = fsqrt_pos(ny2), rny = ny2 > 1e-30f ? rsqrt_ftz(ny2) : 0.0f;
        float kvsum = 0.0f;                               // coefficient of -v in dv
        for (int s0 = 0;;) {
            const int s = s0 + sub;
            const DuCoef c = bwd_coef<LPR, VPL, MODEL>(u, g_of, v_of, ny, rny, invS, att, s, d.S, lir == 0, s_datt, kvsum);
            if (s < d.S) {
                const float e1 = c.c1 * sc, e2 = c.c2 * sc, e3 = c.c3 * sc;
                float* dst = nullptr;
                if (FUSED) { if (row >= 0) dst = (PEER ? peer_scatter_dst(r, d, o, row, rep, lir == 0) : scatter_dst(r, d, o, row, rep)) + lir * 4; }
                else if (o.dUb) dst = o.dUb + ((long)b * d.S + s) * d.D + lir * 4;
#pragma unroll
                for (int q = 0; q < VPL; q++) {
                    const float4 gq = g_of(q), vq = v_of(q);
                    float4 du;
                    du.x = fmaf(e3, u[q].x, fmaf(e2, vq.x, e1 * gq.x)); du.y = fmaf(e3, u[q].y, fmaf(e2, vq.y, e1 * gq.y));
                    du.z = fmaf(e3, u[q].z, fmaf(e2, vq.z, e1 * gq.z)); du.w = fmaf(e3, u[q].w, fmaf(e2, vq.w, e1 * gq.w));
                    dvu[q] = fma4(c.c4, u[q], dvu[q]);
                    if (dst) { if (FUSED) red_add4(dst + q * LPR * 4, du); else *reinterpret_cast<float4*>(dst + q * LPR * 4) = du; }
                }
            }
            s0 += RPW;
            if (s0 >= d.S) break;
            load_rows(u, row, s0);
        }
        // dv = gi + sum_subgroups(dvu) - (sum kv) * v
#pragma unroll
        for (int of = LPR; of < 32; of <<= 1) kvsum += __shfl_xor_sync(0xffffffffu, kvsum, of);
        sum_subgroups<LPR, VPL>(dvu);
        if (sub == 0) {
            float* dst = nullptr;
            if (FUSED) { if (id.z >= 0) dst = (PEER ? peer_scatter_dst(r, d, o, id.z, rep, lir == 0) : scatter_dst(r, d, o, id.z, rep)) + lir * 4; }
            else if (o.dIt) dst = o.dIt + (long)b * d.D + lir * 4;
#pragma unroll
            for (int q = 0; q < VPL; q++) {
                const float4 gi = ldg4(dX + (long)b * lddx + d.D + (q * LPR + lir) * 4);
                const float4 vq = v_of(q);
                float4 dv;
                dv.x = (gi.x + dvu[q].x - kvsum * vq.x) * sc; dv.y = (gi.y + dvu[q].y - kvsum * vq.y) * sc;
                dv.z = (gi.z + dvu[q].z - kvsum * vq.z) * sc; dv.w = (gi.w + dvu[q].w - kvsum * vq.w) * sc;
                if (dst) { if (FUSED) red_add4(dst + q * LPR * 4, dv); else *reinterpret_cast<float4*>(dst + q * LPR * 4) = dv; }
            }
        }
        __syncwarp();          // s_g / s_v are rewritten for the next sample
        b = bn;
    }
    __syncthreads();
    if (MODEL != MODEL_YOUTUBE && o.datt && threadIdx.x < d.S && s_datt[threadIdx.x] != 0.0f) atomicAdd(o.datt + threadIdx.x, s_datt[threadIdx.x]);
}

// folds the hot-row replica accumulators into the table: row += scale * sum_rep acc ; acc = 0
// (the accumulators already hold -lr * gradient, so scale = 1)
__global__ void __launch_bounds__(256)
k_hot_apply(float* __restrict__ emb, long lde, float* __restrict__ hot_acc, int hot_rows, int hot_reps,
            int D, float neg_lr) {
    const long n4 = (long)hot_rows * (D / 4);
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n4; i += (long)gridDim.x * blockDim.x) {
        const long row = i / (D / 4); const int c = (int)(i % (D / 4)) * 4;
        float4 s = zero4();
        for (int rep = 0; rep < hot_reps; rep++) {
            float4* p = reinterpret_cast<float4*>(hot_acc + ((long)rep * hot_rows + row) * D + c);
            const float4 t = *p;
            if (t.x != 0.0f || t.y != 0.0f || t.z != 0.0f || t.w != 0.0f) {
                s.x += t.x; s.y += t.y; s.z += t.z; s.w += t.w;
                *p = zero4();
            }
        }
        if (s.x != 0.0f || s.y != 0.0f || s.z != 0.0f || s.w != 0.0f) {
            float4* e = reinterpret_cast<float4*>(emb + row * lde + c);
            float4 t = *e;
            t.x = fmaf(neg_lr, s.x, t.x); t.y = fmaf(neg_lr, s.y, t.y); t.z = fmaf(neg_lr, s.z, t.z); t.w = fmaf(neg_lr, s.w, t.w);
            *e = t;
        }
    }
}

// sharded tables, replicated hot rows: every rank copies rows [0, hot_k) from their owners' shards (once per table
// generation), and writes its own rows back before the shard is read by the host (download / checkpoint)
__global__ void __launch_bounds__(256)
k_hot_pull(RowSrc r, float* __restrict__ hot_tab, int hot_k, int D) {
    const int q4 = D / 4;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < (long)hot_k * q4; i += (long)gridDim.x * blockDim.x) {
        const int row = (int)(i / q4), c = (int)(i % q4) * 4;
        *reinterpret_cast<float4*>(hot_tab + (long)row * r.lde + c) = *reinterpret_cast<const float4*>(emb_ptr<true>(r, row) + c);
    }
}
__global__ void __launch_bounds__(256)
k_hot_writeback(float* __restrict__ shard, long lde, const float* __restrict__ hot_tab, int hot_k, int D, int world, int rank) {
    const int q4 = D / 4;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < (long)hot_k * q4; i += (long)gridDim.x * blockDim.x) {
        const int row = (int)(i / q4), c = (int)(i % q4) * 4;
        if (row % world == rank) *reinterpret_cast<float4*>(shard + (long)(row / world) * lde + c) = *reinterpret_cast<const float4*>(hot_tab + (long)row * lde + c);
    }
}
// the reverse for data that only the owner holds (the row-Adam moments): hot[row] = this rank's shard row for the rows
// it owns, zero for the others — summed over the ranks (all-reduce), every rank then holds every hot row's values
__global__ void __launch_bounds__(256)
k_hot_own(float* __restrict__ hot, const float* __restrict__ shard, long lde, int hot_k, int D, int world, int rank) {
    const int q4 = D / 4;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < (long)hot_k * q4; i += (long)gridDim.x * blockDim.x) {
        const int row = (int)(i / q4), c = (int)(i % q4) * 4;
        *reinterpret_cast<float4*>(hot + (long)row * D + c) =
            (shard && row % world == rank) ? *reinterpret_cast<const float4*>(shard + (long)(row / world) * lde + c) : zero4();
    }
}
// sharded search by row: out[i] = ITEM_EMB row rows[i] (valid), widened to float64, for the vector instantiation of
// k_knn_scan (knn.cuh)
__global__ void __launch_bounds__(256)
k_gather_rows_f64(RowSrc r, const int* __restrict__ rows, int n, int D, double* __restrict__ out) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < (long)n * D; i += (long)gridDim.x * blockDim.x) {
        const int q = (int)(i / D), c = (int)(i - (long)q * D);
        out[i] = (double)emb_src<true>(r, __ldg(rows + q))[c];
    }
}

// replicated-table step: table += grad (already -lr/world scaled and summed over ranks); grad = 0
__global__ void __launch_bounds__(256)
k_apply_table_grad(float* __restrict__ tab, float* __restrict__ grad, long n4) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n4; i += (long)gridDim.x * blockDim.x) {
        float4 g = reinterpret_cast<float4*>(grad)[i];
        if (g.x != 0.0f || g.y != 0.0f || g.z != 0.0f || g.w != 0.0f) {
            float4 t = reinterpret_cast<float4*>(tab)[i];
            t.x += g.x; t.y += g.y; t.z += g.z; t.w += g.w;
            reinterpret_cast<float4*>(tab)[i] = t;
            reinterpret_cast<float4*>(grad)[i] = zero4();
        }
    }
}

__global__ void __launch_bounds__(256)
k_attn_bwd_gen(RowSrc r, Dims d, int model, const float* __restrict__ att,
               const float* __restrict__ dX, long lddx, BwdOut o, int B) {
    extern __shared__ __align__(16) float smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int nwarps = gridDim.x * (blockDim.x >> 5);
    const float invS = 1.0f / (float)d.S;
    for (int j = threadIdx.x; j < d.S; j += blockDim.x) smem[j] = 0.0f;
    __syncthreads();
    for (int b = blockIdx.x * (blockDim.x >> 5) + wib; b < B; b += nwarps) {
        const float* ip = src_it(r, d, b);
        float vv[kGenAcc], gg[kGenAcc], dv[kGenAcc];
        float ny2 = 0.0f;
#pragma unroll
        for (int j = 0; j < kGenAcc; j++) {
            int k = lane + 32 * j;
            vv[j] = (ip && k < d.D) ? ip[k] : 0.0f;
            gg[j] = k < d.D ? __ldg(dX + (long)b * lddx + k) : 0.0f;
            dv[j] = k < d.D ? __ldg(dX + (long)b * lddx + d.D + k) : 0.0f;
            ny2 += vv[j] * vv[j];
        }
        const float ny = sqrtf(warp_sum(ny2));
        for (int s = 0; s < d.S; s++) {
            const float* up = src_ub(r, d, b, s);
            float uu[kGenAcc], du[kGenAcc];
            float dot = 0.0f, nx2 = 0.0f, d2 = 0.0f, gu = 0.0f;
#pragma unroll
            for (int j = 0; j < kGenAcc; j++) {
                int k = lane + 32 * j;
                uu[j] = (up && k < d.D) ? up[k] : 0.0f;
                dot += uu[j] * vv[j]; nx2 += uu[j] * uu[j]; gu += gg[j] * uu[j];
                float e = uu[j] - vv[j]; d2 += e * e;
            }
            if (model == MODEL_YOUTUBE) {
#pragma unroll
                for (int j = 0; j < kGenAcc; j++) du[j] = gg[j] * invS;
            } else {
                const float att_s = __ldg(att + s);
                gu = warp_sum(gu);
                if (model == MODEL_DIN_COS) {
                    dot = warp_sum(dot);
                    const float nx = sqrtf(warp_sum(nx2));
                    const float den = nx * ny + 1e-8f, cs = dot / den, w = (cs + 1.0f) * 0.5f;
                    const float a = sigmoid32(w * att_s);
                    const float dz = gu * invS * a * (1.0f - a);
                    if (lane == 0) atomicAdd(&smem[s], dz * w);
                    const float cc = 0.5f * dz * att_s, iden = 1.0f / den;
                    const float ku = nx > 0.0f ? cs * ny / (nx * den) : 0.0f;
                    const float kv = ny > 0.0f ? cs * nx / (ny * den) : 0.0f;
#pragma unroll
                    for (int j = 0; j < kGenAcc; j++) {
                        du[j] = a * invS * gg[j] + cc * (vv[j] * iden - ku * uu[j]);
                        dv[j] += cc * (uu[j] * iden - kv * vv[j]);
                    }
                } else {
                    const float dist = sqrtf(warp_sum(d2));
                    const float w = 1.0f - dist, a = sigmoid32(w * att_s);
                    const float dz = gu * invS * a * (1.0f - a);
                    if (lane == 0) atomicAdd(&smem[s], dz * w);
                    const float dw = dz * att_s, k2 = dist > 0.0f ? dw / dist : 0.0f;
#pragma unroll
                    for (int j = 0; j < kGenAcc; j++) {
                        float e = uu[j] - vv[j];
                        du[j] = a * invS * gg[j] - k2 * e;
                        dv[j] += k2 * e;
                    }
                }
            }
#pragma unroll
            for (int j = 0; j < kGenAcc; j++) {
                int k = lane + 32 * j;
                if (k < d.D) {
                    if (o.dUb) o.dUb[((long)b * d.S + s) * d.D + k] = du[j];
                    if (o.sgd && up) atomicAdd(o.scatter_base + (up - r.emb) + k, o.neg_lr * du[j]);
                }
            }
        }
#pragma unroll
        for (int j = 0; j < kGenAcc; j++) {
            int k = lane + 32 * j;
            if (k < d.D) {
                if (o.dIt) o.dIt[(long)b * d.D + k] = dv[j];
                if (o.sgd && ip) atomicAdd(o.scatter_base + (ip - r.emb) + k, o.neg_lr * dv[j]);
            }
        }
    }
    __syncthreads();
    if (model != MODEL_YOUTUBE && o.datt)
        for (int j = threadIdx.x; j < d.S; j += blockDim.x)
            if (smem[j] != 0.0f) atomicAdd(o.datt + j, smem[j]);
}

// -------------------------------------------------------------------------------------------------
// recommend.GetSampleVector materialised (rcmd.go:462-536): X[b] = [user | S history rows | item
// emb | item feat].  Bit-exact copies (widened exactly when T is double); one warp per sample.
// Output row b holds sample rows(b): RowsAsIs (sample b) for ctr_gather_rows and the MLP's key-fed predict,
// RowsByIdx (sample idx[b]) for the shuffled minibatches of ctr_mlp_fit_keys.
// -------------------------------------------------------------------------------------------------
struct RowsAsIs { __device__ __forceinline__ int operator()(int b) const { return b; } };
struct RowsByIdx {
    const long* idx;
    __device__ __forceinline__ int operator()(int b) const { return (int)__ldg(idx + b); }
};

template <typename T, typename Rows>
__global__ void __launch_bounds__(256)
k_gather_rows(RowSrc r, Dims d, T* __restrict__ X, long ldx, int B, Rows rows) {
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int nwarps = gridDim.x * (blockDim.x >> 5);
    for (int b = blockIdx.x * (blockDim.x >> 5) + wib; b < B; b += nwarps) {
        T* x = X + (long)b * ldx;
        const int sb = rows(b);
        const float* pu = src_up(r, sb);
        for (int j = lane; j < d.uP; j += 32) x[j] = pu ? (T)__ldg(pu + j) : (T)0;
        for (int s = 0; s < d.S; s++) {
            const float* up = src_ub(r, d, sb, s);
            for (int j = lane; j < d.D; j += 32) x[d.uP + (long)s * d.D + j] = up ? (T)__ldg(up + j) : (T)0;
        }
        const float* ip = src_it(r, d, sb);
        T* xi = x + d.uP + (long)d.S * d.D;
        for (int j = lane; j < d.D; j += 32) xi[j] = ip ? (T)__ldg(ip + j) : (T)0;
        const float* pc = src_cx(r, sb);
        for (int j = lane; j < d.cF; j += 32) xi[d.D + j] = pc ? (T)__ldg(pc + j) : (T)0;
    }
}

// -------------------------------------------------------------------------------------------------
// Deterministic row update (CTR_TABLE_SGD_DETERMINISTIC): keys[p] = table row of gradient slot
// p = b*(S+1)+slot (slot S = target item), sorted stably; one warp walks each equal-key segment in
// ascending p (== (b, slot) order) accumulating in double, then applies row -= lr * sum once.
// -------------------------------------------------------------------------------------------------
__global__ void k_scatter_keys(const int* __restrict__ hist, const int* __restrict__ item_row,
                               int S, int B, int nvalid, int n_emb, unsigned* __restrict__ keys, unsigned* __restrict__ pos) {
    long n = (long)B * (S + 1);
    for (long p = blockIdx.x * (long)blockDim.x + threadIdx.x; p < n; p += (long)gridDim.x * blockDim.x) {
        int b = (int)(p / (S + 1)), sl = (int)(p % (S + 1));
        // rows of the zero-padded tail (b >= nvalid, model.go:357-371) have no ids: the staging slot holds stale ones
        int row = b < nvalid ? (sl < S ? hist[(long)b * S + sl] : item_row[b]) : -1;
        keys[p] = row_ok(row, n_emb) ? (unsigned)row : 0xFFFFFFFFu;
        pos[p] = (unsigned)p;
    }
}

// element k of the gradient sum of the segment of equal keys that starts at i, in double, in ascending p
__device__ __forceinline__ double segment_sum(const unsigned* __restrict__ keys, const unsigned* __restrict__ pos, long n, long i,
                                              unsigned key, const float* __restrict__ dUb, const float* __restrict__ dIt, int S, int D, int k) {
    double acc = 0.0;
    for (long j = i; j < n && keys[j] == key; j++) {
        unsigned p = pos[j];
        int b = (int)(p / (unsigned)(S + 1)), sl = (int)(p % (unsigned)(S + 1));
        if (k < D) acc += (double)(sl < S ? dUb[((long)b * S + sl) * D + k] : dIt[(long)b * D + k]);
    }
    return acc;
}

__global__ void __launch_bounds__(256)
k_segment_sgd(const unsigned* __restrict__ keys, const unsigned* __restrict__ pos, long n,
              const float* __restrict__ dUb, const float* __restrict__ dIt, int S, int D,
              float* __restrict__ emb, long lde, float lr) {
    const int lane = threadIdx.x & 31;
    long w = (blockIdx.x * (long)blockDim.x + threadIdx.x) >> 5;
    long nw = ((long)gridDim.x * blockDim.x) >> 5;
    for (long i = w; i < n; i += nw) {
        unsigned key = keys[i];
        if (key == 0xFFFFFFFFu) continue;
        if (i > 0 && keys[i - 1] == key) continue;        // not a segment head
        for (int k0 = 0; k0 < D; k0 += 32) {
            int k = k0 + lane;
            const double acc = segment_sum(keys, pos, n, i, key, dUb, dIt, S, D, k);
            if (k < D) {
                float* e = emb + (long)key * lde + k;
                *e = (float)((double)*e - (double)lr * acc);
            }
        }
    }
}

// CTR_TABLE_ADAM: the dense solver's update (gorgonia AdamSolver.Step as model.go:88 configures it: g *= 1/batch;
// m = b1 m + (1-b1) g; v = b2 v + (1-b2) g²; w -= lr · (m/c1) / (sqrt(v/c2) + eps)) applied to the embedding rows
// the batch touched — once per distinct row with the row's summed gradient ("lazy" Adam: untouched rows keep their
// moments; no L2 on embeddings).  c1 = 1-b1^t, c2 = 1-b2^t with the dense step counter t.
struct RowAdam { float lr, b1, b2, eps, c1, c2, inv_batch; };
__device__ __forceinline__ void row_adam_elem(float& w, float& m, float& v, float g, const RowAdam& a) {
    g *= a.inv_batch;
    m = a.b1 * m + (1.0f - a.b1) * g;
    v = a.b2 * v + (1.0f - a.b2) * g * g;
    w -= a.lr * (m / a.c1) / (sqrtf(v / a.c2) + a.eps);
}
__global__ void __launch_bounds__(256)
k_segment_adam(const unsigned* __restrict__ keys, const unsigned* __restrict__ pos, long n,
               const float* __restrict__ dUb, const float* __restrict__ dIt, int S, int D,
               float* __restrict__ emb, float* __restrict__ mo, float* __restrict__ vo, long lde, RowAdam a) {
    const int lane = threadIdx.x & 31;
    long w = (blockIdx.x * (long)blockDim.x + threadIdx.x) >> 5;
    long nw = ((long)gridDim.x * blockDim.x) >> 5;
    for (long i = w; i < n; i += nw) {
        unsigned key = keys[i];
        if (key == 0xFFFFFFFFu) continue;
        if (i > 0 && keys[i - 1] == key) continue;        // not a segment head
        for (int k0 = 0; k0 < D; k0 += 32) {
            int k = k0 + lane;
            const double acc = segment_sum(keys, pos, n, i, key, dUb, dIt, S, D, k);
            if (k < D) {
                const long o = (long)key * lde + k;
                float ww = emb[o], mm = mo[o], vv = vo[o];
                row_adam_elem(ww, mm, vv, (float)acc, a);
                emb[o] = ww; mo[o] = mm; vo[o] = vv;
            }
        }
    }
}
// replicated-table step: grad holds the all-reduced 1/world * gradient sums; rows with any non-zero element were touched
__global__ void __launch_bounds__(256)
k_apply_table_adam(float* __restrict__ tab, float* __restrict__ grad, float* __restrict__ mo, float* __restrict__ vo, long rows, int ld, RowAdam a) {
    const int lane = threadIdx.x & 31;
    long w = (blockIdx.x * (long)blockDim.x + threadIdx.x) >> 5;
    const long nw = ((long)gridDim.x * blockDim.x) >> 5;
    for (long r = w; r < rows; r += nw) {
        bool any = false;
        for (int k = lane; k < ld; k += 32) any |= grad[r * ld + k] != 0.0f;
        if (!__any_sync(0xffffffffu, any)) continue;
        for (int k = lane; k < ld; k += 32) {
            const long o = r * ld + k;
            float ww = tab[o], mm = mo[o], vv = vo[o];
            row_adam_elem(ww, mm, vv, grad[o], a);
            tab[o] = ww; mo[o] = mm; vo[o] = vv; grad[o] = 0.0f;
        }
    }
}
// row-sharded table, owner side (after the barrier that follows every rank's backward): one row Adam update per row of
// this rank's touched list with the gradient the ranks added into gbuf, then the gradient row, the flag and (last block
// out) the count go back to zero.  One warp per row.
__global__ void __launch_bounds__(256)
k_shard_adam(unsigned char* __restrict__ gbuf, ShardGrad L, float* __restrict__ tab, float* __restrict__ mo, float* __restrict__ vo,
             long lde, int D, RowAdam a) {
    unsigned* cnt = reinterpret_cast<unsigned*>(gbuf);
    const long n = *reinterpret_cast<volatile unsigned*>(cnt);
    const int* list = reinterpret_cast<const int*>(gbuf + L.list_off);
    unsigned* flag = reinterpret_cast<unsigned*>(gbuf + L.flag_off);
    float* grad = reinterpret_cast<float*>(gbuf + L.grad_off);
    const int lane = threadIdx.x & 31;
    const long nw = ((long)gridDim.x * blockDim.x) >> 5;
    for (long i = (blockIdx.x * (long)blockDim.x + threadIdx.x) >> 5; i < n; i += nw) {
        const long lr = list[i];
        for (int c = lane * 4; c < D; c += 128) {
            const long o = lr * lde + c;
            float4 w = *reinterpret_cast<float4*>(tab + o), m = *reinterpret_cast<float4*>(mo + o), v = *reinterpret_cast<float4*>(vo + o);
            const float4 g = *reinterpret_cast<const float4*>(grad + o);
            row_adam_elem(w.x, m.x, v.x, g.x, a); row_adam_elem(w.y, m.y, v.y, g.y, a);
            row_adam_elem(w.z, m.z, v.z, g.z, a); row_adam_elem(w.w, m.w, v.w, g.w, a);
            *reinterpret_cast<float4*>(tab + o) = w; *reinterpret_cast<float4*>(mo + o) = m; *reinterpret_cast<float4*>(vo + o) = v;
            *reinterpret_cast<float4*>(grad + o) = zero4();
        }
        if (lane == 0) flag[lr] = 0u;
    }
    __syncthreads();                 // every block has read the count before the last one resets it
    if (threadIdx.x == 0) {
        __threadfence();
        if (atomicAdd(cnt + 1, 1u) == gridDim.x - 1) { cnt[0] = 0u; cnt[1] = 0u; }
    }
}
// the replicated hot rows under row Adam: every rank applies the same update to its replica from the all-reduced
// gradient sums (sum) and touch marks (touch, > 0 = some rank's batch holds the row), then zeroes both.  One warp per row.
__global__ void __launch_bounds__(256)
k_hot_adam(float* __restrict__ hot_tab, float* __restrict__ sum, float* __restrict__ touch, float* __restrict__ mo, float* __restrict__ vo,
           int hot_k, int D, RowAdam a) {
    const int lane = threadIdx.x & 31;
    const long nw = ((long)gridDim.x * blockDim.x) >> 5;
    for (long row = (blockIdx.x * (long)blockDim.x + threadIdx.x) >> 5; row < hot_k; row += nw) {
        if (touch[row] == 0.0f) continue;
        for (int c = lane; c < D; c += 32) {
            const long o = row * D + c;
            float ww = hot_tab[o], mm = mo[o], vv = vo[o];
            row_adam_elem(ww, mm, vv, sum[o], a);
            hot_tab[o] = ww; mo[o] = mm; vo[o] = vv; sum[o] = 0.0f;
        }
        __syncwarp();
        if (lane == 0) touch[row] = 0.0f;
    }
}

// synthetic table rows generated in place (ctr_table_fill): global row = local*world + rank
__global__ void k_table_fill(float* __restrict__ t, long ld, long local_rows, int width, int world, int rank,
                             uint32_t seed, uint32_t stream, int dist, float scale) {
    long n = local_rows * (long)width;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        long lr = i / width; int c = (int)(i % width);
        uint64_t ctr = (uint64_t)(lr * world + rank) * (uint64_t)width + c;
        uint64_t z = mix64(seed, stream, ctr);
        float v;
        if (dist == 0) v = (float)(z >> 40) * (1.0f / 16777216.0f);
        else {
            float u1 = ((float)(z >> 40) + 1.0f) * (1.0f / 16777217.0f);
            float u2 = (float)((z >> 8) & 0xFFFFFFull) * (1.0f / 16777216.0f);
            v = sqrtf(-2.0f * __logf(u1)) * __cosf(6.2831853f * u2);
        }
        t[lr * ld + c] = v * scale;
    }
}

// ctr_table_write_rows: row rows[i] of t = data[i] ([n, width] compact), bit for bit; mo / vo (ITEM_EMB row-Adam moments,
// layout of the table) are zeroed on those rows when non-null.  One warp per row.
__global__ void __launch_bounds__(256)
k_table_write_rows(float* __restrict__ t, long ld, const int* __restrict__ rows, const float* __restrict__ data, long n, int width,
                   float* __restrict__ mo, float* __restrict__ vo) {
    const int lane = threadIdx.x & 31;
    for (long r = (blockIdx.x * (long)blockDim.x + threadIdx.x) >> 5; r < n; r += ((long)gridDim.x * blockDim.x) >> 5) {
        const long dst = (long)rows[r] * ld;
        for (int c = lane; c < width; c += 32) t[dst + c] = data[r * width + c];
        if (mo) for (long c = lane; c < ld; c += 32) { mo[dst + c] = 0.0f; vo[dst + c] = 0.0f; }
    }
}
// *dup = 1 when the ascending rows hold a value twice
__global__ void __launch_bounds__(256)
k_rows_dup(const int* __restrict__ sorted, long n, int* __restrict__ dup) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i + 1 < n; i += (long)gridDim.x * blockDim.x)
        if (sorted[i] == sorted[i + 1]) *dup = 1;
}

}  // namespace ctr
