// owner.cuh — single owners of the engine's CUDA allocations, events and streams (host code only).
// Each releases what it holds when it is destroyed or reassigned, so a struct member is freed with its struct and a
// function-local one on every return path.  A group of resources that must exist together is built into locals and
// moved into place once every member exists.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <utility>

namespace ctr {

// One cudaMalloc (Pinned: cudaHostAlloc) allocation of size() elements.  It converts to T*, so kernel launches and
// copies take it where they took the raw pointer.
template <typename T, bool Pinned = false>
class Buf {
public:
    Buf() = default;
    Buf(Buf&& o) noexcept : p_(std::exchange(o.p_, nullptr)), n_(std::exchange(o.n_, 0)) {}
    Buf& operator=(Buf&& o) noexcept {
        if (this != &o) { reset(); p_ = std::exchange(o.p_, nullptr); n_ = std::exchange(o.n_, 0); }
        return *this;
    }
    ~Buf() { reset(); }
    // frees the current allocation before it takes the new one; empty when the allocation fails
    cudaError_t alloc(size_t n, unsigned host_flags = cudaHostAllocDefault) {
        reset();
        void* p = nullptr;
        const cudaError_t e = Pinned ? cudaHostAlloc(&p, n * sizeof(T), host_flags) : cudaMalloc(&p, n * sizeof(T));
        if (e == cudaSuccess) { p_ = static_cast<T*>(p); n_ = n; }
        return e;
    }
    void reset() {
        if (p_) { if (Pinned) cudaFreeHost(p_); else cudaFree(p_); }
        p_ = nullptr; n_ = 0;
    }
    T* get() const { return p_; }
    operator T*() const { return p_; }
    size_t size() const { return n_; }
private:
    T* p_ = nullptr;
    size_t n_ = 0;
};
template <typename T> using DevBuf = Buf<T, false>;
template <typename T> using PinnedBuf = Buf<T, true>;

// An event or a stream the library created itself.
template <typename H, cudaError_t (*Destroy)(H)>
class Handle {
public:
    Handle() = default;
    Handle(Handle&& o) noexcept : h_(std::exchange(o.h_, nullptr)) {}
    Handle& operator=(Handle&& o) noexcept { if (this != &o) { reset(); h_ = std::exchange(o.h_, nullptr); } return *this; }
    ~Handle() { reset(); }
    void reset() { if (h_) Destroy(h_); h_ = nullptr; }
    operator H() const { return h_; }
protected:
    H h_ = nullptr;
};
struct Event : Handle<cudaEvent_t, cudaEventDestroy> {
    cudaError_t create(unsigned flags) { reset(); return cudaEventCreateWithFlags(&h_, flags); }
};
struct Stream : Handle<cudaStream_t, cudaStreamDestroy> {
    cudaError_t create() { reset(); return cudaStreamCreateWithFlags(&h_, cudaStreamNonBlocking); }
};

}  // namespace ctr
