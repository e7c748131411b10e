// comm.cuh — multi-GPU state of one rank (SURVEY.md §8e).  One process per GPU; the dense weights and the
// small feature tables are replicated; ITEM_EMB (and ITEM_FEAT when it is large) takes one of two placements:
//
//  * row-sharded (the north-star placement; tables > 32 MB): owner(row) = row % world, local row = row / world,
//    world a power of two <= 8 (one NVSwitch box).  Every rank maps every peer's shard into its own address space
//    (VMM allocations shared as file descriptors, 2 MB pages — vmm.cuh) and the attention kernels touch the owner's HBM directly over NVLink: the forward gather is a
//    plain 128-bit load from the owner (the transfer overlaps the gate math of the other warps — there is no
//    separate exchange phase, no index all-to-all, no host sync), the backward scatter is a
//    red.global.add.v4.f32 into the owner's row pre-scaled by -lr/world.  Two device-side barriers per step
//    (flag exchange over peer memory) order the phases: nobody reads a row before every rank's update of the
//    previous step has landed, nobody updates a row before every rank has finished reading.  Semantics =
//    single-GPU training on the global batch with gradients taken at the step-start table.  The most popular rows
//    (ids [0, 32768) by default, cfg.reserved[0]) are additionally replicated on every rank: local reads, gradient
//    sums all-reduced — what a Zipf-distributed id stream needs.
//  * replicated (tables <= 32 MB): every rank keeps the whole table, row gradients are summed into a
//    table-shaped buffer and all-reduced with the dense gradients (NCCL), applied identically everywhere.
//
// NCCL (dlopen'ed, shared with torch's bundled copy) does the bootstrap — the size all-gather / rendezvous — and the
// small dense-gradient all-reduce (~250 KB) that keeps every rank's Adam step identical.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "owner.cuh"
#include "vmm.cuh"

struct ctr_handle;

namespace ctr {

constexpr size_t kReplicateBytes = (size_t)32 << 20;
constexpr size_t kArenaBytes = (size_t)2 << 20;          // small shared arena: barrier flags (+ room for exchange buffers)

struct Comm {
    int rank = 0, world = 1;
    void* nccl = nullptr;         // ncclComm_t
    bool ready = false;
    // placement of ITEM_EMB under world > 1 (ITEM_FEAT: ctr_handle::tab_sharded)
    bool replicate = false;
    DevBuf<float> table_grad;                         // replicated placement: summed row gradients [rows, ld]
    // ---- row-sharded placement: peer mappings
    int wshift = 0;                                   // log2(world)
    float* peer_emb[kMaxPeers] = {};                  // rank j's ITEM_EMB shard ([j == rank] = the local table)
    float* peer_ifeat[kMaxPeers] = {};                // rank j's ITEM_FEAT shard when sharded
    VmmBuf peer_map[kMaxPeers][4];                    // this process's mappings of rank j's {ITEM_EMB, ITEM_FEAT, arena, row-Adam gradients} (vmm.cuh)
    uint64_t published_gen = 0;                       // ctr_handle::tab_gen the mappings belong to (0 = none)
    VmmBuf arena_vmm; unsigned char* arena = nullptr; // shared arena of this rank
    int lsock = -1; unsigned long long job_hash = 0;  // descriptor socket of this rank (abstract UDS named after the NCCL id)
    unsigned char* peer_arena[kMaxPeers] = {};
    unsigned long long epoch = 0;                     // barrier generation (same sequence on every rank)
    PinnedBuf<int> h_err; int* d_err = nullptr;       // pinned + mapped: set by a barrier that timed out
    DevBuf<float> rows_cache;                         // [Bmax, S+1, D] rows fetched by the forward
    DevBuf<unsigned char> d_xchg;                     // device staging of the handle all-gather
    // replicated hot rows of a sharded ITEM_EMB: rows [0, hot_k) live on every rank (hot_tab), their -lr/world scaled
    // gradient sums (hot_sum) are all-reduced with the dense gradients — a Zipf-popular row is neither pulled over
    // NVLink by every sample nor hammered by every rank's red.add
    // (hot_sum holds hot_k more floats after the row sums: the touch marks of CTR_TABLE_ADAM, all-reduced with them)
    int hot_k = 0; DevBuf<float> hot_tab, hot_sum, hot_acc; int hot_reps = 0;
    // CTR_TABLE_ADAM on the sharded ITEM_EMB: this rank's shareable owner-side gradient buffer (layout ShardGrad,
    // attn.cuh), every rank's mapping of it, and the hot rows' two moments (replicated like hot_tab)
    VmmBuf adam_vmm; ShardGrad adam_lay{};
    unsigned char* peer_adam[kMaxPeers] = {};
    DevBuf<float> hot_m, hot_v;
};

// the fixed header a collective serving call all-gathers first (comm_agree): the call's shape, a hash of every input
// array, and this rank's validation verdict
struct CommHdr {
    int64_t n;                  // queries / users
    int32_t k, mode, flag;      // mode: which inputs are given; flag: exclude_history
    int32_t code;               // CTR_OK or this rank's error code ...
    uint64_t hash[2];
    int64_t plan;               // what fixes the number of list all-gathers (queries per chunk / users per group)
    char msg[208];              // ... and its message
};
static_assert(sizeof(CommHdr) == 256, "one all-gather slot of Comm::d_xchg");

}  // namespace ctr

static int comm_agree(ctr_handle* h, ctr::CommHdr hd, int verdict);
static int comm_gather_lists(ctr_handle* h, const void* send_s, void* recv_s, size_t score_bytes, const int* send_r, int* recv_r, size_t n);
static int comm_allreduce_grads(ctr_handle* h, float* extra, size_t extra_n);
static int comm_train_step(ctr_handle* h, const int32_t* d_user, const int32_t* d_item, const int32_t* d_hist, const float* d_label, int32_t B, int32_t nvalid);
static int comm_predict(ctr_handle* h, const int32_t* d_user, const int32_t* d_item, const int32_t* d_hist, int32_t B, float* d_out);
static int comm_barrier(ctr_handle* h);
static int comm_max_i64(ctr_handle* h, int64_t* v);
static int comm_unique_id(void* id_out, int32_t* id_bytes);
static int comm_init(ctr_handle* h, const void* id, int32_t id_bytes);
static void comm_destroy(ctr_handle* h);
