// rl_cuda_host.h — host side of the CUDA units (rl_engine.cu, rl_maint.cu, rl_crdt.cu, rl_rls_dev.cu): the one owner of
// device and pinned memory, and the one path from a CUDA error to a status and a message.  Never included by a kernel
// header.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <algorithm>
#include <utility>

#include "../../include/rl_engine.h"
#include "rl_error.h"

// cudaErrorMemoryAllocation may pass (the caller can retry with less); any other CUDA error is fatal
inline int rl_cuda_status(cudaError_t r) { return r == cudaErrorMemoryAllocation ? RL_TRANSIENT : RL_FATAL; }

// Evaluates a CUDA call; on an error returns fail(owner, status, message) from the enclosing function.  Each unit
// declares fail for its owner type, which stores the message where that owner keeps its last error.
#define RL_CUDA(owner, call)                                                                                        \
    do {                                                                                                            \
        const cudaError_t _r = (call);                                                                              \
        if (_r != cudaSuccess)                                                                                      \
            return fail((owner), rl_cuda_status(_r), "CUDA error %s at %s:%d (%s)", cudaGetErrorName(_r), __FILE__, \
                        __LINE__, cudaGetErrorString(_r));                                                          \
    } while (0)

// plain cudaMalloc, never a stream-ordered pool: the shard slab is exported with cudaIpcGetMemHandle
struct RlDeviceMem {
    static cudaError_t alloc(void** p, size_t bytes) { return cudaMalloc(p, bytes); }
    static void release(void* p) { cudaFree(p); }
};
struct RlPinnedMem {
    static cudaError_t alloc(void** p, size_t bytes) { return cudaMallocHost(p, bytes); }
    static void release(void* p) { cudaFreeHost(p); }
};

// An array of n elements of T, owned by its holder: freed when the holder goes away, moved but never copied.  Every
// (re)allocation drops the old contents; the call site picks the policy (exact, reserve, grow, alloc).
template <class T, class Mem>
struct CudaArray {
    T* p = nullptr;
    size_t n = 0;
    CudaArray() = default;
    CudaArray(const CudaArray&) = delete;
    CudaArray& operator=(const CudaArray&) = delete;
    CudaArray(CudaArray&& o) noexcept { swap(o); }
    CudaArray& operator=(CudaArray&& o) noexcept {
        swap(o);
        return *this;
    }
    ~CudaArray() {
        if (p) Mem::release(p);
    }
    void swap(CudaArray& o) {
        std::swap(p, o.p);
        std::swap(n, o.n);
    }
    // exactly `want` elements (0: none)
    cudaError_t exact(size_t want) {
        if (p) Mem::release(p);
        p = nullptr;
        n = 0;
        if (want == 0) return cudaSuccess;
        const cudaError_t r = Mem::alloc((void**)&p, want * sizeof(T));
        if (r == cudaSuccess) n = want;
        return r;
    }
    // at least `want` elements: exactly `want` when it has fewer, never shrinks
    cudaError_t reserve(size_t want) { return want <= n ? cudaSuccess : exact(want); }
    // at least `want` elements, growing to 1.5 x `want` (64 at least): amortised over a per-batch path
    cudaError_t grow(size_t want) { return p && want <= n ? cudaSuccess : exact(std::max<size_t>(want + want / 2, 64)); }
    // `want` elements, one at least: for a pointer a kernel receives whatever the count
    cudaError_t alloc(size_t want) { return exact(want ? want : 1); }
};
template <class T>
using DevBuf = CudaArray<T, RlDeviceMem>;
template <class T>
using PinnedBuf = CudaArray<T, RlPinnedMem>;

// A call's input array on the device: the caller's pointer (RL_MEM_DEVICE), or a copy staged on stream `st` for the
// call and freed with this object.
template <class E>
struct In {
    const E* p = nullptr;
    DevBuf<E> staged;
    cudaError_t set(const E* src, uint64_t n, int mem, cudaStream_t st) {
        if (mem == RL_MEM_DEVICE || n == 0 || !src) {
            p = src;
            return cudaSuccess;
        }
        const cudaError_t r = staged.exact(n);
        if (r != cudaSuccess) return r;
        p = staged.p;
        return cudaMemcpyAsync(staged.p, src, n * sizeof(E), cudaMemcpyHostToDevice, st);
    }
};
