// ramp_owned.cuh -- owners of the library's device memory, pinned host memory, streams and events, and its error reporting.
// Every buffer the engine and the policy hold lives in an owner, so an early return frees what was allocated so far and a buffer
// that grows never points at freed memory.  The kernels keep taking raw pointers, filled from get().
#pragma once

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <memory>
#include <string>

#include <cuda_runtime.h>

#include "../../include/ramp_b200.h"

namespace ramp {

#pragma GCC visibility push(hidden)      // shared by the library's translation units, not exported next to the C ABI
inline thread_local std::string g_last_error;      // ramp_last_error

inline int set_error(int code, const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_last_error = buf;
    return code;
}

#define CUDA_TRY(expr)                                                                                   \
    do {                                                                                                 \
        cudaError_t _e = (expr);                                                                         \
        if (_e != cudaSuccess)                                                                           \
            return set_error(RAMP_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
    } while (0)

// raises a kernel's cudaFuncAttributeMaxDynamicSharedMemorySize to at least `bytes`, never lowers it (ramp_engine.cu)
cudaError_t reserve_dynamic_smem(const void* kern, size_t bytes);

// bytes the array owners below hold right now, over the whole process (ramp_debug_device_bytes)
inline std::atomic<int64_t> g_device_bytes{0}, g_pinned_bytes{0};
#pragma GCC visibility pop

// Frees ignore their return code, as at interpreter exit the runtime may already be unloading.
template <bool Pinned> struct ArrayFree {
    size_t bytes = 0;
    void operator()(void* p) const {
        if (Pinned) cudaFreeHost(p); else cudaFree(p);
        (Pinned ? g_pinned_bytes : g_device_bytes) -= (int64_t)bytes;
    }
};

// One cudaMalloc (Pinned: cudaMallocHost) of n elements of T, move-only.  alloc() frees the old buffer first and leaves the owner
// empty when the allocation fails; n = 0 allocates one element.
template <class T, bool Pinned> class OwnedArray {
public:
    cudaError_t alloc(size_t n) {
        p_.reset();
        const size_t bytes = sizeof(T) * (n > 0 ? n : 1);
        void* p = nullptr;
        const cudaError_t err = Pinned ? cudaMallocHost(&p, bytes) : cudaMalloc(&p, bytes);
        if (err != cudaSuccess) {
            // the runtime also keeps this error as the thread's last one: take it back, so that the launch check of a later call
            // does not report it again (an earlier, different error stays pending)
            if (cudaPeekAtLastError() == err) cudaGetLastError();
            return err;
        }
        p_ = std::unique_ptr<T, ArrayFree<Pinned>>(static_cast<T*>(p), ArrayFree<Pinned>{bytes});
        (Pinned ? g_pinned_bytes : g_device_bytes) += (int64_t)bytes;
        return cudaSuccess;
    }
    T* get() const { return p_.get(); }
    size_t size() const { return p_ ? p_.get_deleter().bytes / sizeof(T) : 0; }
private:
    std::unique_ptr<T, ArrayFree<Pinned>> p_;
};

template <class T> using DeviceArray = OwnedArray<T, false>;
template <class T> using PinnedArray = OwnedArray<T, true>;

// n elements in each of `arrays`, in order; stops at the first failure
template <class... Arrays> cudaError_t alloc_each(size_t n, Arrays&... arrays) {
    cudaError_t err = cudaSuccess;
    ((err = (err == cudaSuccess ? arrays.alloc(n) : err)), ...);
    return err;
}

// streams and events: create(owner, flags) makes one, the owner destroys it
struct CudaDestroy {
    void operator()(cudaStream_t s) const { cudaStreamDestroy(s); }
    void operator()(cudaEvent_t ev) const { cudaEventDestroy(ev); }
};
using Stream = std::unique_ptr<CUstream_st, CudaDestroy>;
using Event = std::unique_ptr<CUevent_st, CudaDestroy>;
inline cudaError_t create_raw(cudaStream_t* s, unsigned flags) { return cudaStreamCreateWithFlags(s, flags); }
inline cudaError_t create_raw(cudaEvent_t* ev, unsigned flags) { return cudaEventCreateWithFlags(ev, flags); }

template <class Owner> cudaError_t create(Owner& o, unsigned flags) {
    typename Owner::pointer raw = nullptr;
    const cudaError_t err = create_raw(&raw, flags);
    o.reset(raw);
    return err;
}

}  // namespace ramp
