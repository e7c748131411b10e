// umma_gemm.cuh — the dense MLP GEMMs on Hopper's warpgroup tensor cores (wgmma + TMA + mbarrier),
// hand-written for sm_90a.  C[M,N] = epilogue(A[M,K] · B[N,K]ᵀ), fp32 in / fp32 out.
//
// Precision: the reference's MLP is float32 (gonum Sgemm under gorgonia, din.go:307-315) and the
// parity bar is 1e-4 relative on scores, which single-pass TF32 (10-bit mantissa) cannot hold.  So
// each product is error-compensated "3xTF32": x = hi + lo with hi = x & 0xFFFFE000 (exactly
// representable in TF32) and lo = x - hi (exact in fp32), and
//     A·B ≈ A_hi·B_hi + A_hi·B_lo + A_lo·B_hi            (fp32 accumulation in registers).
// B (weights, tiny) is pre-split once per step by k_split_weights (or by the optimiser); A (activations,
// streamed from HBM exactly once) is split in registers: wgmma takes its A operand from registers, so
// every consumer thread loads its fragment of the tile from shared memory and keeps a hi and a lo copy.
//
// One persistent CTA per SM, three warpgroups:
//   warpgroup 0     TMA producer (one thread): cp.async.bulk.tensor 2D, SWIZZLE_128B, {32 fp32 x 128 rows}
//                   A boxes and {32 x 32*NCH} B_hi / B_lo boxes into a STAGES-deep ring (mbarrier complete_tx)
//   warpgroups 1-2  consumers, 64 rows of the 128-row tile each: one wgmma.m64nNk8 tf32 (N = 32*NCH, the whole
//                   tile width) per k-step of 8 and product; the fragments of k-block kb+1 are loaded and split
//                   while the wgmma group of kb runs (two fragment sets, wait_group 1 retires kb-1 first, since
//                   wgmma reads its A registers asynchronously); fused sigmoid+dropout /
//                   dsigmoid / plain store straight from the accumulator registers
#pragma once
#include <cuda.h>
#include <type_traits>
#include "common.cuh"

namespace ctr {
namespace umma {

enum { UEPI_STORE = 0, UEPI_SIGMOID_DROP = 1, UEPI_DSIGMOID = 2 };

constexpr int kBlockM = 128;                 // rows of a tile: two consumer warpgroups of 64
constexpr int kKB = 32;                      // K (fp32) per shared-memory stage: one 128-byte swizzle row
constexpr int kThreads = 384;

struct Args {
    int M, N, Nz, K;            // columns [N, Nz) of C written as zeros; operand columns >= K read as zeros (TMA fill)
    float* C; long ldc;
    const float* H; long ldh;   // UEPI_DSIGMOID: stored post-dropout activation
    float drop_p; uint32_t seed, stream;
    int stages;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "LAB_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra LAB_DONE;\n"
        "bra LAB_WAIT;\n"
        "LAB_DONE:\n"
        "}\n" :: "r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 :: "r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
// named barrier over the two consumer warpgroups (id 0 is __syncthreads)
__device__ __forceinline__ void consumers_sync(int id) { asm volatile("bar.sync %0, 256;" :: "r"(id) : "memory"); }

// registers move from the producer warpgroup (which needs few) to the two consumer warpgroups (accumulators + fragments):
// 40 + 2 x 232 per thread-slot stays within the 64 K registers of the SM
__device__ __forceinline__ void producer_regs() { asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory"); }
__device__ __forceinline__ void consumer_regs() { asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory"); }

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" :: "n"(N) : "memory"); }

// wgmma shared-memory descriptor, K-major operand, SWIZZLE_128B: rows of 128 bytes, 8-row groups 1024 bytes
// apart (SBO), LBO unused (=1), layout type 1 in bits [62,64).  A k-step of 8 tf32 is +32 bytes of start address.
__device__ __forceinline__ uint64_t desc_sw128(uint32_t saddr) {
    return (uint64_t)((saddr >> 4) & 0x3FFF) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}

// D[64 x 32*NCH] += A[64 x 8] · B[32*NCH x 8]ᵀ, one instruction over the whole tile width: A from registers (tf32
// fragment: rows lane/4 and +8 of the warp's 16, k = lane%4 and +4), B from shared memory (rows 128 bytes apart in
// 1024-byte groups of 8, so one descriptor spans all NCH 32-row chunks).  Accumulator d[c][4j + 2h + e] = (row lane/4 + 8h,
// column 32c + 8j + 2*(lane%4) + e).  wgmma takes N in steps of 8 up to 256; the operand lists are spelled out per width.
template <int NCH>
__device__ __forceinline__ void wgmma_tf32(float (&d)[NCH][16], const uint32_t (&a)[4], uint64_t b);
#define UMMA_ACC16(c) "+f"(d[c][0]), "+f"(d[c][1]), "+f"(d[c][2]), "+f"(d[c][3]), "+f"(d[c][4]), "+f"(d[c][5]), "+f"(d[c][6]), "+f"(d[c][7]), \
                      "+f"(d[c][8]), "+f"(d[c][9]), "+f"(d[c][10]), "+f"(d[c][11]), "+f"(d[c][12]), "+f"(d[c][13]), "+f"(d[c][14]), "+f"(d[c][15])
#define UMMA_D0 "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15"
#define UMMA_D1 "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31"
#define UMMA_D2 "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47"
#define UMMA_D3 "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63"
#define UMMA_D4 "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79"
#define UMMA_D5 "%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95"
#define UMMA_D6 "%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111"
#define UMMA_D7 "%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127"
template <> __device__ __forceinline__ void wgmma_tf32<1>(float (&d)[1][16], const uint32_t (&a)[4], uint64_t b) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %21, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {" UMMA_D0 "}, {%16,%17,%18,%19}, %20, p, 1, 1;\n}\n"
                 : UMMA_ACC16(0)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(1));
}
template <> __device__ __forceinline__ void wgmma_tf32<2>(float (&d)[2][16], const uint32_t (&a)[4], uint64_t b) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {" UMMA_D0 "," UMMA_D1 "}, {%32,%33,%34,%35}, %36, p, 1, 1;\n}\n"
                 : UMMA_ACC16(0), UMMA_ACC16(1)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(1));
}
template <> __device__ __forceinline__ void wgmma_tf32<3>(float (&d)[3][16], const uint32_t (&a)[4], uint64_t b) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %53, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n96k8.f32.tf32.tf32 {" UMMA_D0 "," UMMA_D1 "," UMMA_D2 "}, {%48,%49,%50,%51}, %52, p, 1, 1;\n}\n"
                 : UMMA_ACC16(0), UMMA_ACC16(1), UMMA_ACC16(2)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(1));
}
template <> __device__ __forceinline__ void wgmma_tf32<4>(float (&d)[4][16], const uint32_t (&a)[4], uint64_t b) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %69, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {" UMMA_D0 "," UMMA_D1 "," UMMA_D2 "," UMMA_D3 "}, {%64,%65,%66,%67}, %68, p, 1, 1;\n}\n"
                 : UMMA_ACC16(0), UMMA_ACC16(1), UMMA_ACC16(2), UMMA_ACC16(3)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(1));
}
template <> __device__ __forceinline__ void wgmma_tf32<5>(float (&d)[5][16], const uint32_t (&a)[4], uint64_t b) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %85, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n160k8.f32.tf32.tf32 {" UMMA_D0 "," UMMA_D1 "," UMMA_D2 "," UMMA_D3 "," UMMA_D4 "}, {%80,%81,%82,%83}, %84, p, 1, 1;\n}\n"
                 : UMMA_ACC16(0), UMMA_ACC16(1), UMMA_ACC16(2), UMMA_ACC16(3), UMMA_ACC16(4)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(1));
}
template <> __device__ __forceinline__ void wgmma_tf32<6>(float (&d)[6][16], const uint32_t (&a)[4], uint64_t b) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %101, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n192k8.f32.tf32.tf32 {" UMMA_D0 "," UMMA_D1 "," UMMA_D2 "," UMMA_D3 "," UMMA_D4 "," UMMA_D5 "}, {%96,%97,%98,%99}, %100, p, 1, 1;\n}\n"
                 : UMMA_ACC16(0), UMMA_ACC16(1), UMMA_ACC16(2), UMMA_ACC16(3), UMMA_ACC16(4), UMMA_ACC16(5)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(1));
}
template <> __device__ __forceinline__ void wgmma_tf32<7>(float (&d)[7][16], const uint32_t (&a)[4], uint64_t b) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %117, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n224k8.f32.tf32.tf32 {" UMMA_D0 "," UMMA_D1 "," UMMA_D2 "," UMMA_D3 "," UMMA_D4 "," UMMA_D5 "," UMMA_D6 "}, {%112,%113,%114,%115}, %116, p, 1, 1;\n}\n"
                 : UMMA_ACC16(0), UMMA_ACC16(1), UMMA_ACC16(2), UMMA_ACC16(3), UMMA_ACC16(4), UMMA_ACC16(5), UMMA_ACC16(6)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(1));
}
template <> __device__ __forceinline__ void wgmma_tf32<8>(float (&d)[8][16], const uint32_t (&a)[4], uint64_t b) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %133, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 {" UMMA_D0 "," UMMA_D1 "," UMMA_D2 "," UMMA_D3 "," UMMA_D4 "," UMMA_D5 "," UMMA_D6 "," UMMA_D7 "}, {%128,%129,%130,%131}, %132, p, 1, 1;\n}\n"
                 : UMMA_ACC16(0), UMMA_ACC16(1), UMMA_ACC16(2), UMMA_ACC16(3), UMMA_ACC16(4), UMMA_ACC16(5), UMMA_ACC16(6), UMMA_ACC16(7)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(1));
}

#undef UMMA_ACC16
#undef UMMA_D0
#undef UMMA_D1
#undef UMMA_D2
#undef UMMA_D3
#undef UMMA_D4
#undef UMMA_D5
#undef UMMA_D6
#undef UMMA_D7

__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
    const float h = __uint_as_float(__float_as_uint(x) & 0xFFFFE000u);
    hi = __float_as_uint(h); lo = __float_as_uint(x - h);
}

// One k-block (4 k-steps) of the 3-term product for this warpgroup's 64 rows, issued as one wgmma group and
// committed (the caller waits).  The fragments hold the hi/lo split of A; B_hi / B_lo are [32*NCH rows x 128 bytes]
// in the swizzled K-major layout.
template <int NCH>
__device__ __forceinline__ void mma_kblock(float (&acc)[NCH][16], const uint32_t (&ahi)[4][4], const uint32_t (&alo)[4][4],
                                           uint32_t sBhi, uint32_t sBlo) {
    wg_fence();
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const uint64_t dh = desc_sw128(sBhi + (uint32_t)(k * 32));
        const uint64_t dl = desc_sw128(sBlo + (uint32_t)(k * 32));
        wgmma_tf32<NCH>(acc, ahi[k], dh);
        wgmma_tf32<NCH>(acc, ahi[k], dl);
        wgmma_tf32<NCH>(acc, alo[k], dh);
    }
    wg_commit();
}

template <int EPI, int NCH>
__global__ void __launch_bounds__(kThreads, 1)
k_umma_gemm(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmBhi,
            const __grid_constant__ CUtensorMap tmBlo, Args a) {
    extern __shared__ uint8_t smem_raw[];
    constexpr uint32_t kABytes = (uint32_t)kBlockM * kKB * 4u;
    constexpr uint32_t kBBytes = (uint32_t)NCH * 32u * kKB * 4u;
    constexpr uint32_t kStBytes = kABytes + 2u * kBBytes;           // stage s: [A | B_hi | B_lo]
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const int stages = a.stages;
    auto sA = [&](int s) { return base + (uint32_t)s * kStBytes; };
    const uint32_t bars = base + (uint32_t)stages * kStBytes;
    auto full = [&](int s) { return bars + 8u * s; };
    auto empty = [&](int s) { return bars + 8u * (stages + s); };
    const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        for (int s = 0; s < stages; s++) { mbar_init(full(s), 1); mbar_init(empty(s), 8); }
        fence_barrier_init();
    }
    __syncthreads();

    const int num_k = (a.K + kKB - 1) / kKB;
    const int num_tiles = (a.M + kBlockM - 1) / kBlockM;

    if (wg == 0) {                                                  // ---------------- TMA producer
        producer_regs();
        if (threadIdx.x == 0) {
            uint32_t it = 0;
            for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
                if (EPI == UEPI_DSIGMOID) {                         // the epilogue's H rows: one contiguous block, into L2
                    const long row = (long)tile * kBlockM;
                    const uint32_t bytes = (uint32_t)(min((long)kBlockM, a.M - row) * a.ldh * 4);
                    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" :: "l"(a.H + row * a.ldh), "r"(bytes) : "memory");
                }
                for (int kb = 0; kb < num_k; kb++, it++) {
                    const int s = it % stages; const uint32_t ph = (it / stages) & 1u;
                    mbar_wait(empty(s), ph ^ 1u);
                    mbar_expect_tx(full(s), kStBytes);
                    tma_load_2d(sA(s), &tmA, full(s), kb * kKB, tile * kBlockM);
                    tma_load_2d(sA(s) + kABytes, &tmBhi, full(s), kb * kKB, 0);
                    tma_load_2d(sA(s) + kABytes + kBBytes, &tmBlo, full(s), kb * kKB, 0);
                }
            }
        }
        return;
    }
    // ---------------- consumers: warpgroup wg-1 owns tile rows [64*(wg-1), 64*wg)
    consumer_regs();
    const int r0 = (wg - 1) * 64 + warp * 16 + (lane >> 2);         // and r0 + 8
    const int q = lane & 3;
    const float inv_keep = a.drop_p > 0.0f ? 1.0f / (1.0f - a.drop_p) : 1.0f;
    const float keep_thr = 1.0f - a.drop_p;
    const float kp = a.drop_p > 0.0f ? 1.0f - a.drop_p : 1.0f;
    // wait for ring slot i and load this thread's A fragment of it, split hi / lo
    auto load_frag = [&](uint32_t i, uint32_t (&hi)[4][4], uint32_t (&lo)[4][4]) {
        const int s = i % stages;
        mbar_wait(full(s), (i / stages) & 1u);
#pragma unroll
        for (int k = 0; k < 4; k++)
#pragma unroll
            for (int v = 0; v < 4; v++) {
                const int r = r0 + 8 * (v & 1), kk = k * 8 + q + 4 * (v >> 1);
                float x;
                asm volatile("ld.shared.f32 %0, [%1];" : "=f"(x)
                             : "r"(sA(s) + (uint32_t)(r * 128) + ((uint32_t)(((kk >> 2) ^ (r & 7)) << 4) | (uint32_t)((kk & 3) << 2))));
                split_tf32(x, hi[k][v], lo[k][v]);
            }
    };
    auto release = [&](uint32_t i) {                                // this warp's reads of slot i are complete
        __syncwarp();
        if (lane == 0) mbar_arrive(empty(i % stages));
    };
    uint32_t fhi[2][4][4], flo[2][4][4];                            // fragments of k-blocks kb (set kb&1) and kb+1
    uint32_t it = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        float acc[NCH][16];
#pragma unroll
        for (int c = 0; c < NCH; c++)
#pragma unroll
            for (int j = 0; j < 16; j++) acc[c][j] = 0.0f;
        load_frag(it, fhi[0], flo[0]);
        // issue k-block kb; retire kb-1, which frees its ring slot and its fragment set; then load and split kb+1
        // into that set while the group of kb runs
        auto step = [&](int kb, auto set) {
            constexpr int b = decltype(set)::value;
            const uint32_t i = it + (uint32_t)kb;
            mma_kblock<NCH>(acc, fhi[b], flo[b], sA(i % stages) + kABytes, sA(i % stages) + kABytes + kBBytes);
            wg_wait<1>();
            if (kb > 0) release(i - 1);
            if (kb + 1 < num_k) load_frag(i + 1, fhi[b ^ 1], flo[b ^ 1]);
        };
        for (int kb = 0; kb < num_k; kb += 2) {
            step(kb, std::integral_constant<int, 0>{});
            if (kb + 1 < num_k) step(kb + 1, std::integral_constant<int, 1>{});
        }
        wg_wait<0>();
        release(it + (uint32_t)num_k - 1u);
        it += (uint32_t)num_k;
        // epilogue straight from the accumulators: each thread holds two rows x (2 adjacent columns per 8).  dsigmoid
        // loads the H values of a group of kEpiG chunks for both rows before the group's first store (C and H are not
        // known not to alias, so a load is never moved above a store); the producer has prefetched the tile's H rows
        // into L2.  Groups of two chunks fit next to the accumulators up to NCH = 7, one at NCH = 8.
        constexpr int kEpiG = EPI == UEPI_DSIGMOID ? (NCH < 8 ? 2 : 1) : NCH;
#pragma unroll
        for (int c0 = 0; c0 < NCH; c0 += kEpiG) {
            float2 hv[kEpiG][2][4];
            if (EPI == UEPI_DSIGMOID) {
#pragma unroll
                for (int g = 0; g < kEpiG; g++)
#pragma unroll
                    for (int h = 0; h < 2; h++)
#pragma unroll
                        for (int j = 0; j < 4; j++) {
                            const long gm = min((long)tile * kBlockM + r0 + 8 * h, (long)a.M - 1);   // rows past M are not stored
                            const int col8 = (c0 + g) * 32 + j * 8;                            // Nz % 8 == 0: whole 8-column groups
                            hv[g][h][j] = c0 + g < NCH && col8 < a.Nz
                                ? *reinterpret_cast<const float2*>(a.H + gm * a.ldh + col8 + 2 * q) : make_float2(0.0f, 0.0f);
                        }
            }
#pragma unroll
            for (int g = 0; g < kEpiG; g++) {
                const int c = c0 + g;
                if (c >= NCH) continue;
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const long gm = (long)tile * kBlockM + r0 + 8 * h;
                    if (gm >= a.M) continue;
                    const uint32_t ctr0 = (uint32_t)((uint64_t)gm * (uint64_t)a.N);
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        const int col = c * 32 + j * 8 + 2 * q;
                        if (col >= a.Nz) continue;                  // Nz and ldc are multiples of 4: pairs are whole
                        float v[2] = {acc[c][4 * j + 2 * h], acc[c][4 * j + 2 * h + 1]};
                        if (EPI == UEPI_DSIGMOID) {
                            const float hs[2] = {hv[g][h][j].x, hv[g][h][j].y};
#pragma unroll
                            for (int e = 0; e < 2; e++) { const float hh = hs[e] * kp; v[e] *= inv_keep * hh * (1.0f - hh); }   // keep*h*(1-h), h = hd*(1-p)
                        } else if (EPI == UEPI_SIGMOID_DROP) {
#pragma unroll
                            for (int e = 0; e < 2; e++) {
                                const float x = v[e];
                                float sg = __fdividef(1.0f, 1.0f + __expf(-x));   // x < -88 → exp = inf → 0
                                sg = x > 15.0f ? 1.0f : sg;
                                sg = x < -88.0f ? 0.0f : sg;
                                v[e] = sg;
                                if (a.drop_p > 0.0f) v[e] *= uniform24(a.seed, a.stream, ctr0 + (uint32_t)(col + e)) < keep_thr ? inv_keep : 0.0f;
                            }
                        }
                        v[0] = col < a.N ? v[0] : 0.0f;
                        v[1] = col + 1 < a.N ? v[1] : 0.0f;
                        *reinterpret_cast<float2*>(a.C + gm * a.ldc + col) = make_float2(v[0], v[1]);
                    }
                }
            }
        }
    }
}

// W (logical [rows, cols], stride ld) → hi / lo TF32 split, optionally transposed, into padded
// K-major operand buffers [orows_pad, ocols_pad] (stride old); padding stays zero.  All operand copies of a
// step are produced by ONE launch (blockIdx.y = job): the work is tiny, launch gaps would dominate.
struct SplitJob { const float* W; long ld; int rows, cols, transpose; float* hi; float* lo; long old; };
struct SplitJobs { SplitJob j[4]; };
__global__ void __launch_bounds__(256)
k_split_weights(SplitJobs jobs) {
    const SplitJob& jb = jobs.j[blockIdx.y];
    const long n = (long)jb.rows * jb.cols;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const int r = (int)(i / jb.cols), c = (int)(i % jb.cols);
        const float x = jb.W[(long)r * jb.ld + c];
        const float h = __uint_as_float(__float_as_uint(x) & 0xFFFFE000u);
        const long o = jb.transpose ? (long)c * jb.old + r : (long)r * jb.old + c;
        jb.hi[o] = h; jb.lo[o] = x - h;
    }
}

// -------------------------------------------------------------------------------------------------
// Weight-gradient GEMM: C[M,N] += Aᵀ·B with A [K, M] and B [K, N] row-major — the reduction runs over
// the batch (K = samples), so both operands are MN-major (model.go:56: d cost / d mlp0 = concatᵀ·dZ0,
// d cost/d mlp1 = h0ᵀ·dZ1).  wgmma reads tf32 operands K-major only, so:
//   A (the 128 rows of C this CTA owns) goes to registers: every thread loads its fragment straight from
//   the raw TMA box of [32 samples x kDwAPitch columns] and splits it hi/lo;
//   B is transposed by the consumers into Bᵀ_hi / Bᵀ_lo [32*NCH rows x 32 samples] (K-major, SWIZZLE_128B).
// Bᵀ and the A fragments are double-buffered: k-block kb+1 is transposed and loaded while the wgmma group of kb
// runs, and one consumer barrier per k-block publishes it.
// Grid: blockIdx.x = 128-row block of C, blockIdx.y = slice of the batch (split-K); each CTA adds its
// partial product into C with red.global.add.v2.f32.
// -------------------------------------------------------------------------------------------------
// The A box is 8 columns wider than the 128 it uses: with a row pitch of 136 words the four samples a quad reads
// (pitch ≡ 8 banks) and the eight columns its lanes read fall in 32 distinct banks.  Columns past the matrix are
// zero-filled by TMA and never read from HBM.
constexpr int kDwAPitch = kBlockM + 8;

struct DwArgs {
    int K;                      // batch rows to reduce (rows >= K are zero-filled by TMA)
    int M, N;                   // valid rows / cols of C
    float* C; long ldc;
    int stages;
    int kb_per;                 // 32-sample k-blocks per CTA along the batch
};

template <int NCH>
__global__ void __launch_bounds__(kThreads, 1)
k_umma_dw(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, DwArgs a) {
    extern __shared__ uint8_t smem_raw[];
    constexpr int BN = NCH * 32;
    constexpr uint32_t kABytes = 32u * kDwAPitch * 4u;              // 32 samples x kDwAPitch columns of A
    constexpr uint32_t kBBytes = 32u * BN * 4u;                    // 32 samples x BN columns of B, pitch BN*4 B
    constexpr uint32_t kStBytes = kABytes + kBBytes;
    constexpr uint32_t kTBytes = (uint32_t)BN * 128u;              // Bᵀ_hi or Bᵀ_lo: BN rows of 32 samples
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    auto sThi = [&](int b) { return base + (uint32_t)(2 * b) * kTBytes; };
    auto sTlo = [&](int b) { return base + (uint32_t)(2 * b + 1) * kTBytes; };
    const int stages = a.stages;
    auto sA = [&](int s) { return base + 4u * kTBytes + (uint32_t)s * kStBytes; };
    const uint32_t bars = base + 4u * kTBytes + (uint32_t)stages * kStBytes;
    auto full = [&](int s) { return bars + 8u * s; };
    auto empty = [&](int s) { return bars + 8u * (stages + s); };
    const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        for (int s = 0; s < stages; s++) { mbar_init(full(s), 1); mbar_init(empty(s), 8); }
        fence_barrier_init();
    }
    __syncthreads();

    const int m0 = blockIdx.x * kBlockM;
    const int total_kb = (a.K + 31) / 32;
    const int kb0 = blockIdx.y * a.kb_per, kb1 = min(total_kb, kb0 + a.kb_per);
    const int nkb = max(0, kb1 - kb0);

    if (wg == 0) {                                                  // ---------------- TMA producer
        producer_regs();
        if (threadIdx.x == 0) {
            for (int it = 0; it < nkb; it++) {
                const int s = it % stages; const uint32_t ph = (it / stages) & 1u;
                mbar_wait(empty(s), ph ^ 1u);
                mbar_expect_tx(full(s), kStBytes);
                const int row = (kb0 + it) * 32;
                tma_load_2d(sA(s), &tmA, full(s), m0, row);
                tma_load_2d(sA(s) + kABytes, &tmB, full(s), 0, row);
            }
        }
        return;
    }
    consumer_regs();
    if (nkb == 0) return;
    const int ct = threadIdx.x - 128;                               // 0..255 over both consumer warpgroups
    const int r0 = (wg - 1) * 64 + warp * 16 + (lane >> 2);
    const int q = lane & 3;
    float acc[NCH][16];
#pragma unroll
    for (int c = 0; c < NCH; c++)
#pragma unroll
        for (int j = 0; j < 16; j++) acc[c][j] = 0.0f;
    uint32_t fhi[2][4][4], flo[2][4][4];
    // raw k-block it → Bᵀ buffer b and fragment set (fhi, flo); the ring slot goes back to the producer right after
    auto stage_in = [&](int it, int b, uint32_t (&hi)[4][4], uint32_t (&lo)[4][4]) {
        const int s = it % stages;
        mbar_wait(full(s), (it / stages) & 1u);
        const uint32_t pa = sA(s), pb = sA(s) + kABytes;
        // B [32 x BN] → Bᵀ_hi / Bᵀ_lo: a warp takes 32 consecutive columns (conflict-free reads) and writes each as
        // 16 bytes (4 samples) of its own row
#pragma unroll 2
        for (int u = ct; u < BN * 8; u += 256) {
            const int n = u % BN, kq = u / BN;
            float x[4];
#pragma unroll
            for (int i = 0; i < 4; i++)
                asm volatile("ld.shared.f32 %0, [%1];" : "=f"(x[i]) : "r"(pb + (uint32_t)((4 * kq + i) * BN + n) * 4u));
            uint32_t h[4], l[4];
#pragma unroll
            for (int i = 0; i < 4; i++) split_tf32(x[i], h[i], l[i]);
            const uint32_t off = (uint32_t)n * 128u + ((uint32_t)(kq ^ (n & 7)) << 4);
            asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" :: "r"(sThi(b) + off), "r"(h[0]), "r"(h[1]), "r"(h[2]), "r"(h[3]) : "memory");
            asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" :: "r"(sTlo(b) + off), "r"(l[0]), "r"(l[1]), "r"(l[2]), "r"(l[3]) : "memory");
        }
#pragma unroll
        for (int k = 0; k < 4; k++)
#pragma unroll
            for (int v = 0; v < 4; v++) {
                const int r = r0 + 8 * (v & 1), kk = k * 8 + q + 4 * (v >> 1);
                float x;
                asm volatile("ld.shared.f32 %0, [%1];" : "=f"(x) : "r"(pa + (uint32_t)(kk * kDwAPitch + r) * 4u));
                split_tf32(x, hi[k][v], lo[k][v]);
            }
        __syncwarp();
        if (lane == 0) mbar_arrive(empty(s));
        fence_proxy_async();                                        // generic-proxy writes of Bᵀ → visible to wgmma
    };
    stage_in(0, 0, fhi[0], flo[0]);
    consumers_sync(1);
    // Bᵀ buffer b^1 was last read by the group of it-1, which both warpgroups retired before the previous barrier
    auto step = [&](int it, auto set) {
        constexpr int b = decltype(set)::value;
        mma_kblock<NCH>(acc, fhi[b], flo[b], sThi(b), sTlo(b));
        if (it + 1 < nkb) stage_in(it + 1, b ^ 1, fhi[b ^ 1], flo[b ^ 1]);
        wg_wait<0>();
        if (it + 1 < nkb) consumers_sync(1);
    };
    for (int it = 0; it < nkb; it += 2) {
        step(it, std::integral_constant<int, 0>{});
        if (it + 1 < nkb) step(it + 1, std::integral_constant<int, 1>{});
    }
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const int m = m0 + r0 + 8 * h;
        if (m >= a.M) continue;
        float* crow = a.C + (long)m * a.ldc;
#pragma unroll
        for (int c = 0; c < NCH; c++)
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const int col = c * 32 + j * 8 + 2 * q;
                if (col < a.N)                                      // N is even on the padded grad storage
                    asm volatile("red.global.add.v2.f32 [%0], {%1,%2};" :: "l"(crow + col), "f"(acc[c][4 * j + 2 * h]), "f"(acc[c][4 * j + 2 * h + 1]) : "memory");
            }
    }
}

}  // namespace umma
}  // namespace ctr
