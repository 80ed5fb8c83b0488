// common.cuh -- host-side plumbing shared by the C-ABI translation units: error reporting,
// CUDA call checking, device buffers, TMA (cp.async.bulk) staging helper for kernels.
#pragma once
#include <exception>
#include <new>
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdio>
#include <mutex>
#include <string>

#include "../../include/cpb200.h"
#include "ptx.cuh"

namespace cpb {

std::string& last_error_ref();
cpb_status fail(cpb_status st, const char* fmt, ...);

// Every extern "C" entry point runs its body through this: no C++ exception (std::bad_alloc from a host vector,
// std::system_error from a mutex) crosses the C ABI.
template <class Fn> cpb_status guarded(Fn&& fn) noexcept {
    try {
        return fn();
    } catch (const std::bad_alloc&) {
        return fail(CPB_INTERNAL_ERROR, "out of host memory");
    } catch (const std::exception& e) {
        return fail(CPB_INTERNAL_ERROR, "unexpected exception: %s", e.what());
    } catch (...) {
        return fail(CPB_INTERNAL_ERROR, "unexpected exception");
    }
}

#define CPB_CUDA(call)                                                                           \
    do {                                                                                         \
        cudaError_t e__ = (call);                                                                \
        if (e__ != cudaSuccess)                                                                  \
            return cpb::fail(e__ == cudaErrorNoDevice || e__ == cudaErrorInsufficientDriver      \
                                 ? CPB_NO_DEVICE                                                 \
                                 : CPB_CUDA_ERROR,                                               \
                             "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__,  \
                             __LINE__);                                                          \
    } while (0)

#define CPB_TRY(expr)                       \
    do {                                    \
        cpb_status s__ = (expr);            \
        if (s__ != CPB_OK) return s__;      \
    } while (0)

struct DeviceGuard {
    int prev = -1;
    bool ok = false;
    explicit DeviceGuard(int dev) {
        if (cudaGetDevice(&prev) != cudaSuccess) { prev = -1; }
        ok = cudaSetDevice(dev) == cudaSuccess;
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

// Number of SMs of a device (cached per device id).
int sm_count(int device);

// The library carries sm_90a code only, which loads on compute capability 9.0 (H100) and nothing else.
bool device_is_sm90(int device);
cpb_status check_device_arch(int device);

// Stream-ordered scratch (cudaMallocAsync) is used per call; by default the driver's pool returns memory to the OS at
// every synchronisation, which makes the next cudaMallocAsync re-map (and serialise) each time: keep it cached in the pool.
void keep_pool_memory(int device);

// Grow-only device scratch buffer owned by a context (guarded by the context mutex).
struct Scratch {
    void* ptr = nullptr;
    size_t cap = 0;
    cpb_status reserve(size_t bytes) {
        if (bytes <= cap) return CPB_OK;
        if (ptr) cudaFree(ptr);
        ptr = nullptr;
        cap = 0;
        cudaError_t e = cudaMalloc(&ptr, bytes);
        if (e != cudaSuccess) return fail(CPB_CUDA_ERROR, "cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
        cap = bytes;
        return CPB_OK;
    }
    void release() {
        if (ptr) cudaFree(ptr);
        ptr = nullptr;
        cap = 0;
    }
};

#if defined(__CUDACC__)
// Stage `bytes` (multiple of 16, 16-byte aligned both sides) from global to shared memory with
// one bulk asynchronous copy (TMA, SASS UBLKCP) completing on an mbarrier; every thread of the
// CTA returns once the data is visible.  Used for round constants / MDS rows / window tables.
__device__ __forceinline__ void tma_stage_to_smem(void* smem_dst, const void* gmem_src, unsigned bytes,
                                                  unsigned long long* mbar) {
    unsigned mbar_s = (unsigned)__cvta_generic_to_shared(mbar);
    unsigned dst_s = (unsigned)__cvta_generic_to_shared(smem_dst);
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(mbar_s));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mbar_s), "r"(bytes) : "memory");
        asm volatile(
            "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_s),
            "l"(gmem_src), "r"(bytes), "r"(mbar_s)
            : "memory");
    }
    unsigned done = 0;
    while (!done) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(mbar_s)
            : "memory");
    }
}
#endif

}  // namespace cpb
