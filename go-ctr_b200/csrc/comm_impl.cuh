// comm_impl.cuh — included by engine.cu after ctr_handle and step_core are defined.
#pragma once
#include <dlfcn.h>
#include <sys/time.h>

namespace {

// ---- the NCCL entry points we use, resolved at run time -------------------------------------------
struct Uid { char internal[128]; };      // ncclUniqueId
struct NcclApi {
    void* lib = nullptr;
    int (*GetUniqueId)(void*) = nullptr;
    int (*CommInitRank)(void**, int, Uid /* by value */, int) = nullptr;
    int (*CommDestroy)(void*) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
};
enum { kNcclChar = 0, kNcclInt32 = 2, kNcclInt64 = 4, kNcclUint64 = 5, kNcclFloat32 = 7, kNcclFloat64 = 8, kNcclSum = 0, kNcclMax = 2 };

NcclApi g_nccl;

bool nccl_load(std::string* err) {
    if (g_nccl.lib) return true;
    const char* names[] = {"libnccl.so.2", "libnccl.so", "/usr/lib/x86_64-linux-gnu/libnccl.so.2"};
    void* lib = nullptr;
    for (const char* n : names) { lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL); if (lib) break; }
    if (!lib) { *err = std::string("cannot dlopen libnccl: ") + dlerror(); return false; }
#define SYM(field, name) *(void**)(&g_nccl.field) = dlsym(lib, name); if (!g_nccl.field) { *err = std::string("missing NCCL symbol ") + name; return false; }
    SYM(GetUniqueId, "ncclGetUniqueId") SYM(CommInitRank, "ncclCommInitRank") SYM(CommDestroy, "ncclCommDestroy")
    SYM(GroupStart, "ncclGroupStart") SYM(GroupEnd, "ncclGroupEnd")
    SYM(AllReduce, "ncclAllReduce") SYM(AllGather, "ncclAllGather") SYM(GetErrorString, "ncclGetErrorString")
#undef SYM
    g_nccl.lib = lib;
    return true;
}

#define NC(h, call) do { int r_ = (call); if (r_ != 0) return set_err(h, CTR_ECOMM, "%s: %s", #call, g_nccl.GetErrorString(r_)); } while (0)

// ---- device-side barrier over peer memory ---------------------------------------------------------------
// Every rank owns kMaxPeers 64-bit flags at the start of its arena; flag[j] is written by rank j only.  Barrier
// number e: thread j publishes e into peer j's flag[rank] (release, system scope — everything this GPU wrote
// before, including the red.adds of the previous kernel into peer tables, is ordered in front of it), then waits
// until its own flag[j] reaches e (acquire): one NVLink round trip; a peer that never arrives (crashed
// process) trips the 20 s timeout, which raises the host-visible error flag instead of hanging the GPU.
struct BarArgs {
    unsigned long long* mine;
    unsigned long long* peer[kMaxPeers];
    int world, rank;
    unsigned long long epoch;
    int* err;
};
__global__ void k_peer_barrier(BarArgs a) {
    const int j = threadIdx.x;
    if (j >= a.world) return;
    __threadfence_system();
    asm volatile("st.release.sys.global.u64 [%0], %1;" :: "l"(a.peer[j] + a.rank), "l"(a.epoch) : "memory");
    unsigned long long t0, t1, v = 0;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    for (;;) {
        asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(a.mine + j) : "memory");
        if (v >= a.epoch) break;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
        if (t1 - t0 > 20000000000ull) { *reinterpret_cast<volatile int*>(a.err) = 1 + j; break; }
    }
    __threadfence_system();
}

// what one rank publishes about its shareable buffers (ITEM_EMB shard, ITEM_FEAT shard, arena, and under CTR_TABLE_ADAM
// the owner-side gradient buffer): sizes via the NCCL all-gather (which doubles as the rendezvous barrier), the
// allocations themselves as file descriptors over Unix-domain sockets (vmm.cuh)
constexpr int kPub = 4;
struct PubRec { unsigned long long bytes[kPub]; int has[kPub]; };
struct FdHdr { int rank, nfds; int which[kPub]; };

void comm_sock_name(const Comm& cm, int rank, char* out, size_t n) { snprintf(out, n, "ctrb200.%016llx.%d", (unsigned long long)cm.job_hash, rank); }

int comm_hot_setup(ctr_handle* h);

int comm_close_peers(ctr_handle* h) {
    Comm& cm = h->comm;
    for (int j = 0; j < kMaxPeers; j++)
        for (int k = 0; k < kPub; k++) vmm_free(&cm.peer_map[j][k]);
    for (int j = 0; j < kMaxPeers; j++) { cm.peer_emb[j] = nullptr; cm.peer_ifeat[j] = nullptr; cm.peer_arena[j] = nullptr; cm.peer_adam[j] = nullptr; }
    cm.published_gen = 0;
    return CTR_OK;
}

// Collective: every rank exports its shards + arena and maps everybody else's.  Runs once per table generation
// (first sharded step after ctr_table_upload / ctr_table_fill / ctr_checkpoint_load).
int comm_publish(ctr_handle* h) {
    Comm& cm = h->comm;
    const int W = cm.world;
    std::string err;
    CU(h, cudaStreamSynchronize(h->stream));
    comm_close_peers(h);
    // row Adam: the owner-side gradient buffer of this table generation, sized by the largest shard (one layout on every
    // rank), zero; another table_opt leaves it unallocated
    const bool adam = h->cfg.table_opt == CTR_TABLE_ADAM;
    if (adam) {
        const int64_t rows = (h->tab_rows[CTR_TABLE_ITEM_EMB] + W - 1) / W;
        const ShardGrad lay = shard_grad_layout((long)std::max<int64_t>(rows, 1), h->tab_ld[CTR_TABLE_ITEM_EMB]);
        if (!cm.adam_vmm.live || cm.adam_lay.bytes != lay.bytes) {
            vmm_free(&cm.adam_vmm);
            if (!vmm_alloc((size_t)lay.bytes, h->dev, &cm.adam_vmm, &err)) return set_err(h, CTR_ENOMEM, "row-Adam gradient shard (%ld bytes): %s", lay.bytes, err.c_str());
        }
        cm.adam_lay = lay;
        CU(h, cudaMemsetAsync(cm.adam_vmm.ptr, 0, (size_t)lay.bytes, h->stream));
        CU(h, cudaStreamSynchronize(h->stream));
    } else vmm_free(&cm.adam_vmm);
    const VmmBuf* mine[kPub] = {&h->tab_vmm[CTR_TABLE_ITEM_EMB], h->tab_sharded[CTR_TABLE_ITEM_FEAT] ? &h->tab_vmm[CTR_TABLE_ITEM_FEAT] : nullptr, &cm.arena_vmm,
                                adam ? &cm.adam_vmm : nullptr};
    PubRec rec{};
    for (int k = 0; k < kPub; k++) if (mine[k] && mine[k]->live) { rec.bytes[k] = mine[k]->bytes; rec.has[k] = 1; }
    if (!rec.has[0] || !rec.has[2]) return set_err(h, CTR_ESTATE, "row-sharded ITEM_EMB is not in shareable memory (upload the table after ctr_create with world > 1)");
    if (!cm.d_xchg) RET(dalloc(h, cm.d_xchg, 256 * (size_t)(kMaxPeers + 1), false));
    PubRec* d_send = (PubRec*)cm.d_xchg.get(); PubRec* d_recv = d_send + 1;
    std::vector<PubRec> all((size_t)W);
    CU(h, cudaMemcpyAsync(d_send, &rec, sizeof rec, cudaMemcpyHostToDevice, h->stream));
    NC(h, g_nccl.AllGather(d_send, d_recv, sizeof(PubRec), kNcclChar, cm.nccl, h->stream));
    CU(h, cudaMemcpyAsync(all.data(), d_recv, sizeof(PubRec) * (size_t)W, cudaMemcpyDeviceToHost, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    for (int j = 0; j < W; j++)
        if (all[(size_t)j].has[1] != rec.has[1]) return set_err(h, CTR_ESTATE, "rank %d disagrees on the ITEM_FEAT placement", j);
        else if (all[(size_t)j].has[3] != rec.has[3] || all[(size_t)j].bytes[3] != rec.bytes[3]) return set_err(h, CTR_ESTATE, "rank %d disagrees on the table optimiser or the ITEM_EMB rows", j);
    // my descriptors to every peer (connect + one small message each: lands in the peer's backlog / socket buffer) ...
    for (int j = 0; j < W; j++) {
        if (j == cm.rank) continue;
        char name[64]; comm_sock_name(cm, j, name, sizeof name);
        const int s = uds_connect(name, 30000);
        if (s < 0) return set_err(h, CTR_ECOMM, "cannot reach rank %d's descriptor socket", j);
        FdHdr hd{}; hd.rank = cm.rank; int fds[kPub];
        bool ok = true;
        for (int k = 0; k < kPub && ok; k++) if (rec.has[k]) { ok = vmm_export_fd(*mine[k], &fds[hd.nfds], &err); hd.which[hd.nfds] = k; if (ok) hd.nfds++; }
        ok = ok && uds_send_fds(s, &hd, sizeof hd, fds, hd.nfds);
        for (int i = 0; i < hd.nfds; i++) close(fds[i]);
        close(s);
        if (!ok) return set_err(h, CTR_ECOMM, "sending descriptors to rank %d failed: %s", j, err.c_str());
    }
    // ... then collect theirs and map them
    for (int n = 0; n < W - 1; n++) {
        const int s = accept(cm.lsock, nullptr, nullptr);
        if (s < 0) return set_err(h, CTR_ECOMM, "accept on the descriptor socket failed");
        FdHdr hd{}; int fds[kPub]; int nf = 0;
        const bool ok = uds_recv_fds(s, &hd, sizeof hd, fds, kPub, &nf);
        close(s);
        if (!ok || hd.rank < 0 || hd.rank >= W || hd.rank == cm.rank || nf != hd.nfds) { for (int i = 0; i < nf; i++) close(fds[i]); return set_err(h, CTR_ECOMM, "bad descriptor message"); }
        for (int i = 0; i < nf; i++) {
            const int k = hd.which[i];
            if (k < 0 || k >= kPub || !vmm_import(fds[i], (size_t)all[(size_t)hd.rank].bytes[k], h->dev, &cm.peer_map[hd.rank][k], &err)) {
                for (int i2 = i + 1; i2 < nf; i2++) close(fds[i2]);
                return set_err(h, CTR_ECOMM, "mapping rank %d's buffer %d: %s — row-sharded tables need peer access between the GPUs of the box", hd.rank, k, err.c_str());
            }
        }
    }
    for (int j = 0; j < W; j++) {
        if (j == cm.rank) { cm.peer_emb[j] = (float*)mine[0]->ptr; cm.peer_ifeat[j] = rec.has[1] ? (float*)mine[1]->ptr : nullptr; cm.peer_arena[j] = (unsigned char*)mine[2]->ptr;
                            cm.peer_adam[j] = rec.has[3] ? (unsigned char*)mine[3]->ptr : nullptr; }
        else { cm.peer_emb[j] = (float*)cm.peer_map[j][0].ptr; cm.peer_ifeat[j] = (float*)cm.peer_map[j][1].ptr; cm.peer_arena[j] = (unsigned char*)cm.peer_map[j][2].ptr;
               cm.peer_adam[j] = (unsigned char*)cm.peer_map[j][3].ptr; }
        if (!cm.peer_emb[j] || !cm.peer_arena[j] || (rec.has[1] && !cm.peer_ifeat[j]) || (rec.has[3] && !cm.peer_adam[j])) return set_err(h, CTR_ESTATE, "rank %d published no shard", j);
    }
    cm.published_gen = h->tab_gen;
    return comm_hot_setup(h);
}

// (re)builds this rank's replica of the hot rows from the owners' shards; collective through its caller
int comm_hot_setup(ctr_handle* h) {
    Comm& cm = h->comm;
    const int D = h->cfg.D;
    int want = h->cfg.reserved[0];
    if (want == 0) want = 32768;
    if (want < 0) want = 0;
    want = (int)std::min<int64_t>(want, h->tab_rows[CTR_TABLE_ITEM_EMB]);
    cm.hot_tab.reset(); cm.hot_sum.reset(); cm.hot_acc.reset(); cm.hot_m.reset(); cm.hot_v.reset();
    cm.hot_k = want; cm.hot_reps = 0;
    if (want == 0) return CTR_OK;
    if (h->tab_ld[CTR_TABLE_ITEM_EMB] != D) return set_err(h, CTR_EINVAL, "replicated hot rows need D %% 4 == 0");
    RET(dalloc(h, cm.hot_tab, (size_t)want * D, false)); RET(dalloc(h, cm.hot_sum, (size_t)want * (D + 1)));     // + the row-Adam touch marks
    cm.hot_reps = (int)std::min<size_t>(16, std::max<size_t>(1, ((size_t)64 << 20) / ((size_t)want * D * sizeof(float))));
    RET(dalloc(h, cm.hot_acc, (size_t)cm.hot_reps * want * D));
    RowSrc r{}; r.lde = D; r.wmask = cm.world - 1; r.wshift = cm.wshift; r.world = cm.world;
    for (int j = 0; j < cm.world; j++) r.peer_emb[j] = cm.peer_emb[j];
    RET(launch(h, "hot_rows_pull", [&] { k_hot_pull<<<h->num_sms * 4, 256, 0, h->stream>>>(r, cm.hot_tab, want, D); }));
    if (h->cfg.table_opt == CTR_TABLE_ADAM) {
        // the hot rows' moments from their owners' moment shards (zero where an owner has none yet): each rank fills
        // the rows it owns, the all-reduce hands every rank all of them
        RET(dalloc(h, cm.hot_m, (size_t)want * D, false)); RET(dalloc(h, cm.hot_v, (size_t)want * D, false));
        const long lde = h->tab_ld[CTR_TABLE_ITEM_EMB];
        RET(launch(h, "hot_moments_pull", [&] {
            k_hot_own<<<h->num_sms * 4, 256, 0, h->stream>>>(cm.hot_m, h->emb_m.get(), lde, want, D, cm.world, cm.rank);
            k_hot_own<<<h->num_sms * 4, 256, 0, h->stream>>>(cm.hot_v, h->emb_v.get(), lde, want, D, cm.world, cm.rank);
        }));
        NC(h, g_nccl.GroupStart());
        NC(h, g_nccl.AllReduce(cm.hot_m, cm.hot_m, (size_t)want * D, kNcclFloat32, kNcclSum, cm.nccl, h->stream));
        NC(h, g_nccl.AllReduce(cm.hot_v, cm.hot_v, (size_t)want * D, kNcclFloat32, kNcclSum, cm.nccl, h->stream));
        NC(h, g_nccl.GroupEnd());
    }
    CU(h, cudaStreamSynchronize(h->stream));
    return CTR_OK;
}
// the owner's shard rows of the hot range are stale while training runs on the replicas: refresh this rank's own
int comm_hot_writeback(ctr_handle* h) {
    Comm& cm = h->comm;
    if (cm.hot_k <= 0 || !cm.hot_tab || cm.published_gen != h->tab_gen) return CTR_OK;
    if (cm.hot_m) RET(ensure_moments(h));      // row Adam: the owner's moment shards receive the hot rows' moments too
    const long lde = h->tab_ld[CTR_TABLE_ITEM_EMB];
    return launch(h, "hot_rows_writeback", [&] {
        k_hot_writeback<<<h->num_sms * 4, 256, 0, h->stream>>>(h->tab[CTR_TABLE_ITEM_EMB], lde, cm.hot_tab, cm.hot_k, h->cfg.D, cm.world, cm.rank);
        if (cm.hot_m) {
            k_hot_writeback<<<h->num_sms * 4, 256, 0, h->stream>>>(h->emb_m, lde, cm.hot_m, cm.hot_k, h->cfg.D, cm.world, cm.rank);
            k_hot_writeback<<<h->num_sms * 4, 256, 0, h->stream>>>(h->emb_v, lde, cm.hot_v, cm.hot_k, h->cfg.D, cm.world, cm.rank);
        }
    });
}

// what search needs of a sharded handle: the communicator, a supported world and the ITEM_EMB shard
int comm_check_emb(ctr_handle* h) {
    const Comm& cm = h->comm;
    if (!cm.ready) return set_err(h, CTR_ESTATE, "world=%d but ctr_comm_init was not called", cm.world);
    if (cm.world > kMaxPeers || (cm.world & (cm.world - 1))) return set_err(h, CTR_EINVAL, "row-sharded tables need world in {2, 4, 8} (one NVSwitch box), got %d", cm.world);
    if (!h->tab[CTR_TABLE_ITEM_EMB] || h->tab_width[CTR_TABLE_ITEM_EMB] != h->cfg.D) return set_err(h, CTR_ESTATE, "ITEM_EMB shard not uploaded");
    return CTR_OK;
}

int comm_check(ctr_handle* h) {
    const ctr_config& c = h->cfg;
    RET(comm_check_emb(h));
    if (c.uP > 0 && !h->tab[CTR_TABLE_USER_FEAT]) return set_err(h, CTR_ESTATE, "USER_FEAT not uploaded");
    if (c.cF > 0 && !h->tab[CTR_TABLE_ITEM_FEAT]) return set_err(h, CTR_ESTATE, "ITEM_FEAT not uploaded");
    if (!attn_idx_shape_ok(h, true))
        return set_err(h, CTR_EINVAL, "row-sharded tables need D in {16,32,64,128}, S <= 64, uP %% 4 == 0 and uP + cF <= 128");
    return CTR_OK;
}

int comm_ensure(ctr_handle* h, bool want_cache) {
    Comm& cm = h->comm;
    if (cm.published_gen != h->tab_gen) RET(comm_publish(h));
    if (want_cache) RET(reserve(h, cm.rows_cache, (size_t)h->Bmax * (h->cfg.S + 1) * h->cfg.D, false));
    return CTR_OK;
}

RowSrc comm_src(ctr_handle* h, const int* d_user, const int* d_item, const int* d_hist, int B, bool cache) {
    Comm& cm = h->comm;
    RowSrc r = idx_src(h, d_user, d_item, d_hist, B);
    r.world = cm.world; r.wmask = cm.world - 1; r.wshift = cm.wshift;
    r.ifeat_sharded = h->tab_sharded[CTR_TABLE_ITEM_FEAT] ? 1 : 0;
    for (int j = 0; j < cm.world; j++) { r.peer_emb[j] = cm.peer_emb[j]; r.peer_ifeat[j] = cm.peer_ifeat[j]; }
    r.rows_cache = cache ? cm.rows_cache.get() : nullptr;
    r.hot_k = cm.hot_k; r.hot_tab = cm.hot_tab;
    return r;
}

}  // namespace

// max over the ranks of a host-side count (sizes the collective batch loop of ctr_train_keys)
static int comm_max_i64(ctr_handle* h, int64_t* v) {
    Comm& cm = h->comm;
    if (!cm.ready) return set_err(h, CTR_ESTATE, "world=%d but ctr_comm_init was not called", cm.world);
    if (!cm.d_xchg) RET(dalloc(h, cm.d_xchg, 256 * (size_t)(kMaxPeers + 1), false));
    CU(h, cudaMemcpyAsync(cm.d_xchg, v, sizeof(int64_t), cudaMemcpyHostToDevice, h->stream));
    NC(h, g_nccl.AllReduce(cm.d_xchg, cm.d_xchg, 1, kNcclInt64, kNcclMax, cm.nccl, h->stream));
    CU(h, cudaMemcpyAsync(v, cm.d_xchg, sizeof(int64_t), cudaMemcpyDeviceToHost, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    return CTR_OK;
}

// 64-bit hash of a caller array (FNV-1a over 8-byte words), for comparing the ranks' arguments of a collective call
static uint64_t comm_hash(const void* p, size_t bytes) {
    const unsigned char* b = (const unsigned char*)p;
    uint64_t hs = 1469598103934665603ull;
    for (size_t i = 0; i < bytes; i += 8) {
        uint64_t w = 0;
        memcpy(&w, b + i, std::min<size_t>(8, bytes - i));
        hs = (hs ^ w) * 1099511628211ull;
        hs ^= hs >> 29;
    }
    return hs;
}

// Argument agreement of a collective call (search / recommendation on a row-sharded ITEM_EMB).  Every rank all-gathers
// its header and its own validation verdict (code, message) before doing anything else, so a rank never leaves the
// others blocked in NCCL: headers that differ give CTR_EINVAL everywhere, else the verdict of the lowest failing rank,
// else CTR_EINVAL if the ranks' plans differ (hd.plan is read only when every rank is valid).  A failure after the
// agreement (out of memory for scratch, a failed publish) still leaves the peers waiting, as in the sharded train step.
static int comm_agree(ctr_handle* h, CommHdr hd, int verdict) {
    Comm& cm = h->comm;
    if (!cm.ready) return set_err(h, CTR_ESTATE, "world=%d but ctr_comm_init was not called", cm.world);
    hd.code = verdict;
    if (verdict != CTR_OK) snprintf(hd.msg, sizeof hd.msg, "%s", h->err.c_str());
    if (!cm.d_xchg) RET(dalloc(h, cm.d_xchg, 256 * (size_t)(kMaxPeers + 1), false));
    const int W = cm.world;
    std::vector<CommHdr> all((size_t)W);
    CommHdr* d_send = (CommHdr*)cm.d_xchg.get();
    CU(h, cudaMemcpyAsync(d_send, &hd, sizeof hd, cudaMemcpyHostToDevice, h->stream));
    NC(h, g_nccl.AllGather(d_send, d_send + 1, sizeof(CommHdr), kNcclChar, cm.nccl, h->stream));
    CU(h, cudaMemcpyAsync(all.data(), d_send + 1, sizeof(CommHdr) * (size_t)W, cudaMemcpyDeviceToHost, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    for (int j = 1; j < W; j++) {
        const CommHdr& a = all[0]; const CommHdr& b = all[(size_t)j];
        if (a.n != b.n || a.k != b.k || a.mode != b.mode || a.flag != b.flag || a.hash[0] != b.hash[0] || a.hash[1] != b.hash[1])
            return set_err(h, CTR_EINVAL, "ranks disagree on the arguments of this collective call: rank %d (n %lld, k %d) differs from rank 0 (n %lld, k %d) — every rank must pass the same arguments",
                           j, (long long)b.n, b.k, (long long)a.n, a.k);
    }
    for (int j = 0; j < W; j++)
        if (all[(size_t)j].code != CTR_OK) return set_err(h, all[(size_t)j].code, "%s", all[(size_t)j].msg);
    for (int j = 1; j < W; j++)          // every rank valid: their plans must give the same sequence of all-gathers
        if (all[(size_t)j].plan != all[0].plan)
            return set_err(h, CTR_EINVAL, "ranks disagree on the plan of this collective call: rank %d would exchange %lld entries per round, rank 0 %lld",
                           j, (long long)all[(size_t)j].plan, (long long)all[0].plan);
    return CTR_OK;
}

// The ranks' top-k lists, all-gathered on the engine stream (device buffers of the caller's scratch): send_s / send_r
// hold n entries, recv_s / recv_r receive [world][n].  Every rank's reads of the table are queued before its send, so
// the gather completes on a rank only after every rank has finished reading.
static int comm_gather_lists(ctr_handle* h, const void* send_s, void* recv_s, size_t score_bytes, const int* send_r, int* recv_r, size_t n) {
    Comm& cm = h->comm;
    NC(h, g_nccl.GroupStart());
    NC(h, g_nccl.AllGather(send_s, recv_s, n * score_bytes, kNcclChar, cm.nccl, h->stream));
    NC(h, g_nccl.AllGather(send_r, recv_r, n, kNcclInt32, cm.nccl, h->stream));
    NC(h, g_nccl.GroupEnd());
    h->launches += 1;
    return CTR_OK;
}

static int comm_barrier(ctr_handle* h) {
    Comm& cm = h->comm;
    BarArgs a{};
    a.mine = (unsigned long long*)cm.arena;
    for (int j = 0; j < cm.world; j++) a.peer[j] = (unsigned long long*)cm.peer_arena[j];
    a.world = cm.world; a.rank = cm.rank; a.epoch = ++cm.epoch; a.err = cm.d_err;
    return launch(h, "peer_barrier", [&] { k_peer_barrier<<<1, 32, 0, h->stream>>>(a); });
}

// dense gradients + the batch cost: sum over ranks (every rank then takes the identical Adam step)
static int comm_allreduce_grads(ctr_handle* h, float* extra, size_t extra_n) {
    Comm& cm = h->comm;
    if (!cm.ready) return set_err(h, CTR_ESTATE, "world=%d but ctr_comm_init was not called", cm.world);
    NC(h, g_nccl.GroupStart());
    if (extra && extra_n) NC(h, g_nccl.AllReduce(extra, extra, extra_n, kNcclFloat32, kNcclSum, cm.nccl, h->stream));
    NC(h, g_nccl.AllReduce(h->Gflat, h->Gflat, h->Gflat_n, kNcclFloat32, kNcclSum, cm.nccl, h->stream));     // all four gradient tensors, one buffer
    NC(h, g_nccl.AllReduce(h->d_cost, h->d_cost, 1, kNcclFloat64, kNcclSum, cm.nccl, h->stream));
    NC(h, g_nccl.GroupEnd());
    h->launches += 1;
    return CTR_OK;
}

// One train step with row-sharded tables.  Collective: every rank calls it with its own B samples; nvalid < B
// marks a zero-padded tail (model.go:357-371).
static int comm_train_step(ctr_handle* h, const int32_t* d_user, const int32_t* d_item, const int32_t* d_hist, const float* d_label, int32_t B, int32_t nvalid) {
    RET(comm_check(h));
    RET(comm_ensure(h, true));
    Comm& cm = h->comm;
    RET(comm_barrier(h));           // every rank's row updates of the previous step have landed
    RowSrc r = comm_src(h, d_user, d_item, d_hist, B, true);
    r.nvalid = nvalid;
    StepOpts o; o.training = true; o.update = true; o.d_label = d_label;
    o.comm = true; o.peer = true; o.grad_scale = 1.0f / (float)cm.world; o.adam_batch = B * cm.world;
    return step_core(h, r, B, o);
}

// Forward only: reads the owners' shards, no barrier (the caller keeps training and prediction apart: ctr_sync on
// every rank + a host barrier between them), any B <= Bmax per rank.
static int comm_predict(ctr_handle* h, const int32_t* d_user, const int32_t* d_item, const int32_t* d_hist, int32_t B, float* d_out) {
    RET(comm_check(h));
    RET(comm_ensure(h, false));
    RowSrc r = comm_src(h, d_user, d_item, d_hist, B, false);
    StepOpts o; o.peer = true;
    RET(step_core(h, r, B, o));
    if (d_out) CU(h, cudaMemcpyAsync(d_out, h->P, (size_t)B * sizeof(float), cudaMemcpyDeviceToDevice, h->stream));
    return CTR_OK;
}

static int comm_unique_id(void* id_out, int32_t* id_bytes) {
    std::string err;
    if (!id_out || !id_bytes || *id_bytes < 128) return CTR_EINVAL;
    if (!nccl_load(&err)) { g_create_error = err; return CTR_ECOMM; }
    Uid u;
    if (g_nccl.GetUniqueId(&u) != 0) return CTR_ECOMM;
    memcpy(id_out, &u, 128); *id_bytes = 128;
    return CTR_OK;
}

static int comm_init(ctr_handle* h, const void* id, int32_t id_bytes) {
    std::string err;
    Comm& cm = h->comm;
    if (id_bytes != 128) return set_err(h, CTR_EINVAL, "unique id must be 128 bytes");
    if (cm.world < 2) return set_err(h, CTR_EINVAL, "ctr_comm_init with world=%d", cm.world);
    if (cm.world > 64) return set_err(h, CTR_EINVAL, "world > 64 unsupported");
    if (cm.ready) return set_err(h, CTR_ESTATE, "ctr_comm_init called twice");
    if (!nccl_load(&err)) return set_err(h, CTR_ECOMM, "%s", err.c_str());
    Uid u; memcpy(&u, id, 128);
    NC(h, g_nccl.CommInitRank(&cm.nccl, cm.world, u, cm.rank));
    cm.wshift = 0; while ((1 << cm.wshift) < cm.world) cm.wshift++;
    // the shared arena (barrier flags) exists — zeroed — and this rank's descriptor socket listens before any peer can
    // reach the first publish (its all-gather is the rendezvous)
    unsigned long long hsh = 1469598103934665603ull;
    for (int i = 0; i < 128; i++) { hsh ^= (unsigned char)u.internal[i]; hsh *= 1099511628211ull; }
    cm.job_hash = hsh;
    if (!vmm_alloc(kArenaBytes, h->dev, &cm.arena_vmm, &err)) return set_err(h, CTR_ECUDA, "shared arena: %s", err.c_str());
    cm.arena = (unsigned char*)cm.arena_vmm.ptr;
    CU(h, cudaMemset(cm.arena, 0, kArenaBytes));
    char name[64]; comm_sock_name(cm, cm.rank, name, sizeof name);
    cm.lsock = uds_listen(name);
    if (cm.lsock < 0) return set_err(h, CTR_ECOMM, "cannot listen on the descriptor socket %s", name);
    timeval tv{60, 0};                                  // a rank that died must not hang the others in accept()
    setsockopt(cm.lsock, SOL_SOCKET, SO_RCVTIMEO, &tv, sizeof tv);
    CU(h, cm.h_err.alloc(1, cudaHostAllocMapped));
    *cm.h_err = 0;
    CU(h, cudaHostGetDevicePointer(&cm.d_err, cm.h_err, 0));
    cm.ready = true;
    return CTR_OK;
}

static void comm_destroy(ctr_handle* h) {
    Comm& cm = h->comm;
    comm_close_peers(h);
    vmm_free(&cm.adam_vmm);
    vmm_free(&cm.arena_vmm);
    cm.arena = nullptr;
    if (cm.lsock >= 0) { close(cm.lsock); cm.lsock = -1; }
    if (cm.nccl && g_nccl.CommDestroy) g_nccl.CommDestroy(cm.nccl);
    cm.nccl = nullptr; cm.ready = false;
}
