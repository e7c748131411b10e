// vmm.cuh — device memory that other PROCESSES of the box can map at full NVLink speed.
//
// The row-sharded placement needs every rank to read / red.add every other rank's table shard from inside its own
// kernels.  Legacy CUDA IPC (cudaIpcOpenMemHandle) maps the peer's memory with small pages: a random 256-byte-row
// gather over such a mapping is far slower than over in-process peer access (tests/cuda/peer_probe.cu, `ipc` vs
// in-process; the bigger the table the worse — TLB misses).  The VMM API keeps 2 MB pages on both sides: the owner
// creates the allocation with cuMemCreate (exportable as a POSIX file descriptor), the peers import the descriptor
// (passed over a Unix-domain socket, SCM_RIGHTS) and cuMemMap it into their own address space.
// GrowBuf (below) uses the same API in one process: tables that grow in place without a copy.
//
// Driver entry points are resolved through cudaGetDriverEntryPoint: the library links cudart only and still loads
// on a machine without libcuda (CPU-side ABI tests).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>
#include <sys/socket.h>
#include <sys/un.h>
#include <unistd.h>
#include <errno.h>
#include <algorithm>
#include <string>
#include <utility>
#include <vector>

namespace ctr {

struct DrvApi {
    bool ok = false;
    CUresult (*MemCreate)(CUmemGenericAllocationHandle*, size_t, const CUmemAllocationProp*, unsigned long long) = nullptr;
    CUresult (*MemRelease)(CUmemGenericAllocationHandle) = nullptr;
    CUresult (*MemAddressReserve)(CUdeviceptr*, size_t, size_t, CUdeviceptr, unsigned long long) = nullptr;
    CUresult (*MemAddressFree)(CUdeviceptr, size_t) = nullptr;
    CUresult (*MemMap)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long) = nullptr;
    CUresult (*MemUnmap)(CUdeviceptr, size_t) = nullptr;
    CUresult (*MemSetAccess)(CUdeviceptr, size_t, const CUmemAccessDesc*, size_t) = nullptr;
    CUresult (*MemGetAllocationGranularity)(size_t*, const CUmemAllocationProp*, CUmemAllocationGranularity_flags) = nullptr;
    CUresult (*MemExportToShareableHandle)(void*, CUmemGenericAllocationHandle, CUmemAllocationHandleType, unsigned long long) = nullptr;
    CUresult (*MemImportFromShareableHandle)(CUmemGenericAllocationHandle*, void*, CUmemAllocationHandleType) = nullptr;
};
inline DrvApi& drv() { static DrvApi d; return d; }

inline bool drv_load(std::string* err) {
    DrvApi& d = drv();
    if (d.ok) return true;
    auto get = [&](const char* name, void** out) {
        cudaDriverEntryPointQueryResult q; void* p = nullptr;
        if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q) != cudaSuccess || !p) { cudaGetLastError(); *err = std::string("driver entry point ") + name + " not available"; return false; }
        *out = p; return true;
    };
    if (!get("cuMemCreate", (void**)&d.MemCreate) || !get("cuMemRelease", (void**)&d.MemRelease) || !get("cuMemAddressReserve", (void**)&d.MemAddressReserve) ||
        !get("cuMemAddressFree", (void**)&d.MemAddressFree) || !get("cuMemMap", (void**)&d.MemMap) || !get("cuMemUnmap", (void**)&d.MemUnmap) ||
        !get("cuMemSetAccess", (void**)&d.MemSetAccess) || !get("cuMemGetAllocationGranularity", (void**)&d.MemGetAllocationGranularity) ||
        !get("cuMemExportToShareableHandle", (void**)&d.MemExportToShareableHandle) || !get("cuMemImportFromShareableHandle", (void**)&d.MemImportFromShareableHandle))
        return false;
    d.ok = true;
    return true;
}

struct VmmBuf {
    void* ptr = nullptr;
    size_t bytes = 0;                     // mapped size (granule multiple)
    CUmemGenericAllocationHandle h = 0;
    bool live = false;
};

inline CUmemAllocationProp vmm_prop(int dev) {
    CUmemAllocationProp prop; memset(&prop, 0, sizeof prop);
    prop.type = CU_MEM_ALLOCATION_TYPE_PINNED; prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE; prop.location.id = dev;
    prop.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    return prop;
}
// maps allocation b->h (b->bytes long) into this process for device dev
inline bool vmm_map(VmmBuf* b, int dev, std::string* err) {
    DrvApi& d = drv();
    CUdeviceptr va = 0;
    // big tables: a 512 MB-aligned virtual range lets the driver pick the largest page size it has for the mapping
    const size_t align = b->bytes >= ((size_t)512 << 20) ? ((size_t)512 << 20) : 0;
    if (d.MemAddressReserve(&va, b->bytes, align, 0, 0) != CUDA_SUCCESS) { *err = "cuMemAddressReserve failed"; return false; }
    if (d.MemMap(va, b->bytes, 0, b->h, 0) != CUDA_SUCCESS) { d.MemAddressFree(va, b->bytes); *err = "cuMemMap failed"; return false; }
    CUmemAccessDesc acc; memset(&acc, 0, sizeof acc);
    acc.location.type = CU_MEM_LOCATION_TYPE_DEVICE; acc.location.id = dev; acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    if (d.MemSetAccess(va, b->bytes, &acc, 1) != CUDA_SUCCESS) {
        d.MemUnmap(va, b->bytes); d.MemAddressFree(va, b->bytes);
        *err = "cuMemSetAccess failed (no peer access between the GPUs?)"; return false;
    }
    b->ptr = (void*)va; b->live = true;
    return true;
}
// owner side: at least `bytes` of device memory on dev, shareable with other processes
inline bool vmm_alloc(size_t bytes, int dev, VmmBuf* out, std::string* err) {
    if (!drv_load(err)) return false;
    DrvApi& d = drv();
    CUmemAllocationProp prop = vmm_prop(dev);
    size_t gran = 0;
    if (d.MemGetAllocationGranularity(&gran, &prop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED) != CUDA_SUCCESS || gran == 0) { *err = "cuMemGetAllocationGranularity failed"; return false; }
    if (bytes >= ((size_t)512 << 20)) gran = std::max(gran, (size_t)512 << 20);
    VmmBuf b; b.bytes = (bytes + gran - 1) / gran * gran;
    if (d.MemCreate(&b.h, b.bytes, &prop, 0) != CUDA_SUCCESS) { *err = "cuMemCreate failed (out of device memory?)"; return false; }
    if (!vmm_map(&b, dev, err)) { d.MemRelease(b.h); return false; }
    *out = b;
    return true;
}
inline void vmm_free(VmmBuf* b) {
    if (!b->live) return;
    DrvApi& d = drv();
    d.MemUnmap((CUdeviceptr)b->ptr, b->bytes); d.MemAddressFree((CUdeviceptr)b->ptr, b->bytes); d.MemRelease(b->h);
    *b = VmmBuf();
}
inline bool vmm_export_fd(const VmmBuf& b, int* fd, std::string* err) {
    int f = -1;
    if (drv().MemExportToShareableHandle(&f, b.h, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0) != CUDA_SUCCESS || f < 0) { *err = "cuMemExportToShareableHandle failed"; return false; }
    *fd = f; return true;
}
// peer side: takes ownership of fd (closed here)
inline bool vmm_import(int fd, size_t bytes, int dev, VmmBuf* out, std::string* err) {
    if (!drv_load(err)) { close(fd); return false; }
    VmmBuf b; b.bytes = bytes;
    CUresult r = drv().MemImportFromShareableHandle(&b.h, (void*)(uintptr_t)fd, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR);
    close(fd);
    if (r != CUDA_SUCCESS) { *err = "cuMemImportFromShareableHandle failed"; return false; }
    if (!vmm_map(&b, dev, err)) { drv().MemRelease(b.h); return false; }
    *out = b;
    return true;
}

// A row-sharded table's shard holding `rows` live rows of row_b bytes, grown to `want` rows.  The shard is an exportable
// allocation the peers map, which does not grow in place: when `want` rows exceed it, a new one of max(want, 2 x rows)
// rows (geometric, so a run of small growths reallocates O(log n) times) receives the live rows, the rest zeroed, and the
// old one is freed once the copy is done — old and new side by side at the peak.  Otherwise rows [rows, want) are
// zeroed in place.  Synchronises st when it reallocates.
inline bool vmm_grow_rows(VmmBuf* b, size_t rows, size_t want, size_t row_b, int dev, cudaStream_t st, std::string* err) {
    if (want <= rows) return true;
    if (want * row_b <= b->bytes) {
        if (cudaMemsetAsync((char*)b->ptr + rows * row_b, 0, (want - rows) * row_b, st) != cudaSuccess) { *err = "cudaMemsetAsync failed"; return false; }
        return true;
    }
    VmmBuf nb;
    if (!vmm_alloc(std::max(want, 2 * rows) * row_b, dev, &nb, err)) return false;
    if (cudaMemcpyAsync(nb.ptr, b->ptr, rows * row_b, cudaMemcpyDeviceToDevice, st) != cudaSuccess ||
        cudaMemsetAsync((char*)nb.ptr + rows * row_b, 0, nb.bytes - rows * row_b, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess) {
        *err = std::string("shard copy: ") + cudaGetErrorString(cudaGetLastError());
        vmm_free(&nb);
        return false;
    }
    vmm_free(b);
    *b = nb;
    return true;
}

// ---- growable device memory: the single-GPU tables and ITEM_EMB's row-Adam moments (ctr_table_write_rows) ------
// A virtual range reserved with headroom; physical chunks (non-shareable handles) are created and mapped at the end of
// what is mapped as the buffer grows, each about 1/8 of the mapped size and at least one granule, so a run of one-row
// growths maps O(log n) chunks.  When the reservation is full, a range twice the new size is reserved and the same
// chunks are mapped into it: no byte is copied, and the old and the new buffer never need memory side by side.  The old
// range is unmapped after `st` (the stream of every kernel that holds the old base) has passed them.
// One owner, like Buf (owner.cuh): destroyed or reset, it releases every chunk and range (after a device synchronise,
// which is what cudaFree does).
template <typename T>
class GrowBuf {
public:
    GrowBuf() = default;
    GrowBuf(GrowBuf&& o) noexcept { take(o); }
    GrowBuf& operator=(GrowBuf&& o) noexcept { if (this != &o) { reset(); take(o); } return *this; }
    ~GrowBuf() { reset(); }
    // at least n elements mapped; the contents of the part mapped here are undefined.  get() may change.
    bool grow(size_t n, int dev, cudaStream_t st, std::string* err) {
        const size_t need = n * sizeof(T);
        if (need <= mapped_) return true;
        if (!drv_load(err)) return false;
        DrvApi& d = drv();
        CUmemAllocationProp prop = vmm_prop(dev);
        prop.requestedHandleTypes = CU_MEM_HANDLE_TYPE_NONE;
        if (!gran_ && (d.MemGetAllocationGranularity(&gran_, &prop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED) != CUDA_SUCCESS || gran_ == 0)) {
            gran_ = 0; *err = "cuMemGetAllocationGranularity failed"; return false;
        }
        const size_t chunk = round(std::max(need - mapped_, mapped_ / 8));
        CUmemGenericAllocationHandle hnd = 0;
        if (d.MemCreate(&hnd, chunk, &prop, 0) != CUDA_SUCCESS) { *err = "cuMemCreate failed (out of device memory?)"; return false; }
        if (mapped_ + chunk > reserved_ && !move(2 * (mapped_ + chunk), dev, st, err)) { d.MemRelease(hnd); return false; }
        if (!map(va_ + mapped_, chunk, hnd, dev)) { d.MemRelease(hnd); *err = "cuMemMap / cuMemSetAccess failed"; return false; }
        chunks_.push_back({hnd, chunk});
        mapped_ += chunk;
        return true;
    }
    void reset() {
        if (!va_) return;
        cudaDeviceSynchronize();
        DrvApi& d = drv();
        unmap_all(va_);
        d.MemAddressFree(va_, reserved_);
        for (const Chunk& c : chunks_) d.MemRelease(c.h);
        chunks_.clear(); va_ = 0; reserved_ = mapped_ = 0;
    }
    T* get() const { return reinterpret_cast<T*>(va_); }
    operator T*() const { return get(); }
    size_t capacity() const { return mapped_ / sizeof(T); }     // elements mapped
    size_t chunks() const { return chunks_.size(); }
    int moves() const { return moves_; }                         // reservations replaced by a larger one
private:
    struct Chunk { CUmemGenericAllocationHandle h; size_t bytes; };
    size_t round(size_t b) const { return (std::max<size_t>(b, 1) + gran_ - 1) / gran_ * gran_; }
    static bool map(CUdeviceptr va, size_t bytes, CUmemGenericAllocationHandle hnd, int dev) {
        DrvApi& d = drv();
        if (d.MemMap(va, bytes, 0, hnd, 0) != CUDA_SUCCESS) return false;
        CUmemAccessDesc acc; memset(&acc, 0, sizeof acc);
        acc.location.type = CU_MEM_LOCATION_TYPE_DEVICE; acc.location.id = dev; acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
        if (d.MemSetAccess(va, bytes, &acc, 1) != CUDA_SUCCESS) { d.MemUnmap(va, bytes); return false; }
        return true;
    }
    void unmap_all(CUdeviceptr va) {
        size_t off = 0;
        for (const Chunk& c : chunks_) { drv().MemUnmap(va + off, c.bytes); off += c.bytes; }
    }
    // a new reservation of `bytes` holding the mapped chunks at the same offsets
    bool move(size_t bytes, int dev, cudaStream_t st, std::string* err) {
        DrvApi& d = drv();
        // big ranges: 512 MB alignment lets the driver pick its largest page size (as vmm_map does)
        const size_t align = bytes >= ((size_t)512 << 20) ? ((size_t)512 << 20) : 0;
        if (align) bytes = (bytes + align - 1) / align * align;
        CUdeviceptr va = 0;
        if (d.MemAddressReserve(&va, bytes, align, 0, 0) != CUDA_SUCCESS) { *err = "cuMemAddressReserve failed"; return false; }
        size_t off = 0;
        for (size_t i = 0; i < chunks_.size(); i++) {
            if (!map(va + off, chunks_[i].bytes, chunks_[i].h, dev)) {
                for (size_t j = 0, o = 0; j < i; o += chunks_[j].bytes, j++) d.MemUnmap(va + o, chunks_[j].bytes);
                d.MemAddressFree(va, bytes);
                *err = "cuMemMap / cuMemSetAccess failed"; return false;
            }
            off += chunks_[i].bytes;
        }
        if (va_) {
            cudaStreamSynchronize(st);
            unmap_all(va_);
            d.MemAddressFree(va_, reserved_);
            moves_++;
        }
        va_ = va; reserved_ = bytes;
        return true;
    }
    void take(GrowBuf& o) {
        va_ = std::exchange(o.va_, 0); reserved_ = std::exchange(o.reserved_, 0); mapped_ = std::exchange(o.mapped_, 0);
        gran_ = o.gran_; moves_ = o.moves_; chunks_ = std::move(o.chunks_); o.chunks_.clear();
    }
    CUdeviceptr va_ = 0;
    size_t reserved_ = 0, mapped_ = 0, gran_ = 0;
    int moves_ = 0;
    std::vector<Chunk> chunks_;
};

// ---- file descriptors between the rank processes: abstract Unix-domain sockets + SCM_RIGHTS -----------------
inline void uds_addr(const char* name, sockaddr_un* a, socklen_t* len) {
    memset(a, 0, sizeof *a); a->sun_family = AF_UNIX;
    const size_t n = strlen(name);
    memcpy(a->sun_path + 1, name, n);                    // sun_path[0] == 0: abstract namespace (no file, dies with the process)
    *len = (socklen_t)(offsetof(sockaddr_un, sun_path) + 1 + n);
}
inline int uds_listen(const char* name) {
    int s = socket(AF_UNIX, SOCK_STREAM, 0);
    if (s < 0) return -1;
    sockaddr_un a; socklen_t len; uds_addr(name, &a, &len);
    if (bind(s, (sockaddr*)&a, len) != 0 || listen(s, 64) != 0) { close(s); return -1; }
    return s;
}
inline int uds_connect(const char* name, int timeout_ms) {
    sockaddr_un a; socklen_t len; uds_addr(name, &a, &len);
    for (int waited = 0;; waited += 10) {
        int s = socket(AF_UNIX, SOCK_STREAM, 0);
        if (s < 0) return -1;
        if (connect(s, (sockaddr*)&a, len) == 0) return s;
        close(s);
        if (waited >= timeout_ms) return -1;
        usleep(10000);
    }
}
// one message: `hdr` (hdr_len bytes) + up to 4 descriptors
inline bool uds_send_fds(int s, const void* hdr, size_t hdr_len, const int* fds, int nfds) {
    iovec iov = {const_cast<void*>(hdr), hdr_len};
    char ctl[CMSG_SPACE(sizeof(int) * 4)]; memset(ctl, 0, sizeof ctl);
    msghdr msg; memset(&msg, 0, sizeof msg);
    msg.msg_iov = &iov; msg.msg_iovlen = 1;
    if (nfds > 0) {
        msg.msg_control = ctl; msg.msg_controllen = CMSG_SPACE(sizeof(int) * nfds);
        cmsghdr* c = CMSG_FIRSTHDR(&msg); c->cmsg_level = SOL_SOCKET; c->cmsg_type = SCM_RIGHTS; c->cmsg_len = CMSG_LEN(sizeof(int) * nfds);
        memcpy(CMSG_DATA(c), fds, sizeof(int) * nfds);
    }
    return sendmsg(s, &msg, 0) == (ssize_t)hdr_len;
}
inline bool uds_recv_fds(int s, void* hdr, size_t hdr_len, int* fds, int max_fds, int* nfds) {
    iovec iov = {hdr, hdr_len};
    char ctl[CMSG_SPACE(sizeof(int) * 4)]; memset(ctl, 0, sizeof ctl);
    msghdr msg; memset(&msg, 0, sizeof msg);
    msg.msg_iov = &iov; msg.msg_iovlen = 1; msg.msg_control = ctl; msg.msg_controllen = sizeof ctl;
    ssize_t r;
    do { r = recvmsg(s, &msg, MSG_WAITALL); } while (r < 0 && errno == EINTR);
    if (r != (ssize_t)hdr_len) return false;
    *nfds = 0;
    for (cmsghdr* c = CMSG_FIRSTHDR(&msg); c; c = CMSG_NXTHDR(&msg, c))
        if (c->cmsg_level == SOL_SOCKET && c->cmsg_type == SCM_RIGHTS) {
            const int n = (int)((c->cmsg_len - CMSG_LEN(0)) / sizeof(int));
            for (int i = 0; i < n && *nfds < max_fds; i++) memcpy(&fds[(*nfds)++], CMSG_DATA(c) + sizeof(int) * i, sizeof(int));
        }
    return true;
}

}  // namespace ctr
