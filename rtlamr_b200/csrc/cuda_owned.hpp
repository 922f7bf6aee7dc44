// cuda_owned.hpp -- what libertgpu's host code shares: error messages (fail, CUDA_TRY), the dynamic shared-memory
// limit, and move-only owners of CUDA resources.  An owner releases what it holds when it is cleared (`= {}`), given
// something new or destroyed, so a resource is listed once, where it is declared.  Owners convert to the raw pointer or
// handle, which launches and argument structs take.  Host code only.
#pragma once

#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdio>
#include <memory>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/ertgpu.h"

namespace ert {

// The message goes to err; returns code.
inline int fail(std::string& err, int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    err = buf;
    return code;
}

// `sink`: whatever fail() takes (a handle, an error string)
#define CUDA_TRY(sink, expr)                                                                    \
    do {                                                                                        \
        cudaError_t e__ = (expr);                                                               \
        if (e__ != cudaSuccess) {                                                               \
            cudaGetLastError();                                                                 \
            return fail(sink, e__ == cudaErrorMemoryAllocation ? ERTGPU_ENOMEM : ERTGPU_ECUDA,  \
                        "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
        }                                                                                       \
    } while (0)

// A kernel whose launches request `bytes` of dynamic shared memory may take the whole 227 KiB of a CTA: set on each kernel
// a handle may launch, when the handle is allocated.  `what` names the kernel when it needs more.
inline int allow_dynamic_smem(std::string& err, const void* kernel, size_t bytes, const char* what) {
    if (bytes > 227 * 1024) return fail(err, ERTGPU_EINVAL, "%s needs %zu B of shared memory", what, bytes);
    CUDA_TRY(err, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    return ERTGPU_OK;
}

template <class P, cudaError_t (*Release)(P)>
struct Releaser {
    void operator()(P p) const { Release(p); }
};

// n elements of T on the device (cudaMalloc), or in pinned host memory (cudaHostAlloc) when Pinned.
template <class T, bool Pinned = false>
struct CudaArray : std::unique_ptr<T, std::conditional_t<Pinned, Releaser<void*, cudaFreeHost>, Releaser<void*, cudaFree>>> {
    operator T*() const { return this->get(); }
    cudaError_t alloc(size_t n) {  // what it held is freed first
        this->reset();
        void* p = nullptr;
        const cudaError_t e = Pinned ? cudaHostAlloc(&p, n * sizeof(T), cudaHostAllocDefault) : cudaMalloc(&p, n * sizeof(T));
        this->reset(e == cudaSuccess ? static_cast<T*>(p) : nullptr);
        return e;
    }
    cudaError_t upload(const std::vector<T>& v) {  // a device copy of v
        const cudaError_t e = alloc(v.size());
        return e != cudaSuccess ? e : cudaMemcpy(this->get(), v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice);
    }
};
template <class T>
using DeviceArray = CudaArray<T, false>;
template <class T>
using PinnedArray = CudaArray<T, true>;

// A stream or an event: create(flags) as cudaStreamCreateWithFlags or cudaEventCreateWithFlags.
template <class H, cudaError_t (*Create)(H*, unsigned), cudaError_t (*Destroy)(H)>
struct CudaHandle : std::unique_ptr<std::remove_pointer_t<H>, Releaser<H, Destroy>> {
    operator H() const { return this->get(); }
    cudaError_t create(unsigned flags) {
        H x = nullptr;
        const cudaError_t e = Create(&x, flags);
        this->reset(e == cudaSuccess ? x : nullptr);
        return e;
    }
};
using Stream = CudaHandle<cudaStream_t, cudaStreamCreateWithFlags, cudaStreamDestroy>;
using Event = CudaHandle<cudaEvent_t, cudaEventCreateWithFlags, cudaEventDestroy>;

}  // namespace ert
