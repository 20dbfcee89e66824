// cuda_owned.h — owners of the engine's device and pinned allocations, events and streams.  Each frees what it holds when
// it is destroyed, so an error return never leaks and a teardown needs no list of frees.  Lazy buffers grow through
// reserve(): every buffer checks its own size, so a call after a failed allocation retries exactly what is missing.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>
#include <memory>
#include <string>
#include <type_traits>
#include <utility>

#include "host_math.h"

namespace gmm {

#define CUDA_TRY(expr)                                                                        \
    do {                                                                                      \
        cudaError_t e_ = (expr);                                                              \
        if (e_ != cudaSuccess)                                                                \
            return fail(GMM_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e_));    \
    } while (0)

enum class MemKind { Device, Pinned };

// One allocation of n elements of T in device memory (cudaMalloc) or pinned host memory (cudaMallocHost).  Converts to
// T*, so it is passed to kernels and copies, and indexed or offset, as the pointer it owns.
template <typename T, MemKind M>
class CudaArray {
public:
    CudaArray() = default;
    CudaArray(CudaArray&& o) noexcept : p_(std::exchange(o.p_, nullptr)), n_(std::exchange(o.n_, 0)) {}
    CudaArray& operator=(CudaArray&& o) noexcept {
        if (this != &o) {
            reset();
            p_ = std::exchange(o.p_, nullptr);
            n_ = std::exchange(o.n_, 0);
        }
        return *this;
    }
    CudaArray(const CudaArray&) = delete;
    CudaArray& operator=(const CudaArray&) = delete;
    ~CudaArray() { reset(); }

    operator T*() const { return p_; }
    T* get() const { return p_; }
    size_t size() const { return n_; }

    void reset() {
        if (p_) M == MemKind::Device ? cudaFree(p_) : cudaFreeHost(p_);
        p_ = nullptr;
        n_ = 0;
    }
    // At least n elements: nothing happens when the array already holds n, else the old allocation is freed and n are
    // allocated (never shrunk).  On failure the array is empty and the runtime's last error is cleared, so that a later
    // cudaGetLastError() after an unrelated launch does not report it.
    int reserve(size_t n) {
        if (n_ >= n) return GMM_OK;
        reset();
        const char* what = M == MemKind::Device ? "cudaMalloc" : "cudaMallocHost";
        if (n > SIZE_MAX / sizeof(T)) return fail(GMM_ERR_CUDA, std::string(what) + ": " + std::to_string(n) + " elements overflow size_t");
        void* p = nullptr;
        const size_t bytes = sizeof(T) * n;
        const cudaError_t e = M == MemKind::Device ? cudaMalloc(&p, bytes) : cudaMallocHost(&p, bytes);
        if (e != cudaSuccess) {
            cudaGetLastError();
            return fail(GMM_ERR_CUDA, std::string(what) + " of " + std::to_string(bytes) + " bytes: " + cudaGetErrorString(e));
        }
        p_ = static_cast<T*>(p);
        n_ = n;
        return GMM_OK;
    }

private:
    T* p_ = nullptr;
    size_t n_ = 0;
};
template <typename T> using DeviceArray = CudaArray<T, MemKind::Device>;
template <typename T> using PinnedArray = CudaArray<T, MemKind::Pinned>;

// An event or a stream, destroyed with its owner.  create() makes it once; later calls keep the existing one.
template <typename H, cudaError_t (*Create)(H*, unsigned), cudaError_t (*Destroy)(H)>
class CudaHandle {
public:
    operator H() const { return h_.get(); }
    int create(unsigned flags) {
        if (h_) return GMM_OK;
        H h = nullptr;
        const cudaError_t e = Create(&h, flags);
        if (e != cudaSuccess) {
            cudaGetLastError();
            return fail(GMM_ERR_CUDA, std::string("creating a CUDA event or stream: ") + cudaGetErrorString(e));
        }
        h_.reset(h);
        return GMM_OK;
    }

private:
    struct Deleter {
        void operator()(H h) const { Destroy(h); }
    };
    std::unique_ptr<std::remove_pointer_t<H>, Deleter> h_;
};
using Event = CudaHandle<cudaEvent_t, cudaEventCreateWithFlags, cudaEventDestroy>;
using Stream = CudaHandle<cudaStream_t, cudaStreamCreateWithFlags, cudaStreamDestroy>;

}  // namespace gmm
