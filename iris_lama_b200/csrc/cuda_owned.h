// cuda_owned.h -- move-only owners of the CUDA buffers, events and streams of the host code.  Plain C++17 on the runtime API, so
// both the nvcc and the g++ translation units include it.  Every other file allocates and releases CUDA resources through these.
#pragma once

#include <cuda_runtime_api.h>

#include <cstddef>
#include <memory>
#include <utility>

namespace lama_b200 {

namespace detail {
struct DeviceMem {
    static cudaError_t alloc(void** p, size_t bytes) { return cudaMalloc(p, bytes); }
    void operator()(void* p) const { cudaFree(p); }
};
struct PinnedMem {
    static cudaError_t alloc(void** p, size_t bytes) { return cudaMallocHost(p, bytes); }
    void operator()(void* p) const { cudaFreeHost(p); }
};

// n elements of T.  alloc and reserve return the runtime's error; on failure the owner is empty with size 0.
template <class T, class Mem>
class OwnedArray {
public:
    OwnedArray() = default;
    OwnedArray(OwnedArray&& o) noexcept : p_(std::move(o.p_)), n_(std::exchange(o.n_, 0)) {}
    OwnedArray& operator=(OwnedArray&& o) noexcept   // releases what it held after taking o's array
    {
        p_ = std::move(o.p_);
        n_ = std::exchange(o.n_, 0);
        return *this;
    }

    T* get() const { return p_.get(); }
    size_t size() const { return n_; }
    explicit operator bool() const { return p_ != nullptr; }
    void reset() { p_.reset(), n_ = 0; }
    cudaError_t alloc(size_t n)   // frees what it holds, then allocates n elements
    {
        reset();
        void* q = nullptr;
        const cudaError_t e = Mem::alloc(&q, n * sizeof(T));
        if (e == cudaSuccess) p_.reset(static_cast<T*>(q)), n_ = n;
        return e;
    }
    // at least n elements: grows (free before alloc, contents lost) only when it holds fewer
    cudaError_t reserve(size_t n) { return n <= n_ ? cudaSuccess : alloc(n); }

private:
    std::unique_ptr<T, Mem> p_;
    size_t n_ = 0;
};
}  // namespace detail

template <class T> using DeviceArray = detail::OwnedArray<T, detail::DeviceMem>;   // cudaMalloc / cudaFree
template <class T> using PinnedArray = detail::OwnedArray<T, detail::PinnedMem>;   // cudaMallocHost / cudaFreeHost

class Event {
public:
    cudaError_t create(unsigned flags)
    {
        cudaEvent_t ev = nullptr;
        const cudaError_t e = cudaEventCreateWithFlags(&ev, flags);
        e_.reset(e == cudaSuccess ? ev : nullptr);
        return e;
    }
    cudaEvent_t get() const { return e_.get(); }
    operator cudaEvent_t() const { return e_.get(); }

private:
    struct Destroy { void operator()(cudaEvent_t ev) const { cudaEventDestroy(ev); } };
    std::unique_ptr<CUevent_st, Destroy> e_;
};

// Either a non-blocking stream of its own (create) or the caller's stream (borrow), which it never destroys.
class Stream {
public:
    cudaError_t create()
    {
        cudaStream_t st = nullptr;
        const cudaError_t e = cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking);
        reset();
        own_.reset(e == cudaSuccess ? st : nullptr);
        return e;
    }
    void borrow(cudaStream_t st) { reset(), borrowed_ = st; }
    void reset() { own_.reset(), borrowed_ = nullptr; }
    cudaStream_t get() const { return own_ ? own_.get() : borrowed_; }
    operator cudaStream_t() const { return get(); }

private:
    struct Destroy { void operator()(cudaStream_t st) const { cudaStreamDestroy(st); } };
    std::unique_ptr<CUstream_st, Destroy> own_;
    cudaStream_t borrowed_ = nullptr;
};

}  // namespace lama_b200
