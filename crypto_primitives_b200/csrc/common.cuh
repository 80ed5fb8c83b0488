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

inline size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

// Grow-only device scratch buffer: one per context (guarded by the context mutex), or a local one freed on scope exit.
struct Scratch {
    void* ptr = nullptr;
    size_t cap = 0;
    Scratch() = default;
    Scratch(const Scratch&) = delete;
    Scratch& operator=(const Scratch&) = delete;
    ~Scratch() { release(); }
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

// How a host-pointer entry point stages its arrays through a Scratch arena on one stream.  Declare every region first (in: copied
// up, out: copied back, inout: both, dev: device only; each call returns the region's offset), then upload() reserves the
// 256-byte-aligned regions once and queues the uploads, at<T>(offset) gives the device pointers, and download() queues the copies
// back and synchronises.  The destructor synchronises too, so no return path, errors included, leaves a copy from or to a caller's
// buffer queued once the call (and the context mutex) is left.  A zero-byte region gets its own pointer and no copy.
class HostStage {
  public:
    HostStage(Scratch& arena, cudaStream_t st) : arena_(arena), st_(st) {}
    HostStage(const HostStage&) = delete;
    HostStage& operator=(const HostStage&) = delete;
    ~HostStage() {
        if (!synced_) cudaStreamSynchronize(st_);
    }
    size_t in(const void* h, size_t bytes) { return add(const_cast<void*>(h), bytes, kIn); }
    size_t out(void* h, size_t bytes) { return add(h, bytes, kOut); }
    size_t inout(void* h, size_t bytes) { return add(h, bytes, kIn | kOut); }
    size_t dev(size_t bytes) { return add(nullptr, bytes, 0); }
    template <class T> T* at(size_t off) const { return (T*)((char*)arena_.ptr + off); }

    cpb_status upload() {
        if (n_ > kMax) return fail(CPB_INTERNAL_ERROR, "more than %d staged regions", kMax);
        CPB_TRY(arena_.reserve(total_));
        for (int i = 0; i < n_; i++)
            if ((r_[i].dir & kIn) && r_[i].bytes)
                CPB_CUDA(cudaMemcpyAsync(at<char>(r_[i].off), r_[i].host, r_[i].bytes, cudaMemcpyHostToDevice, st_));
        return CPB_OK;
    }
    cpb_status download() {
        for (int i = 0; i < n_; i++)
            if ((r_[i].dir & kOut) && r_[i].bytes)
                CPB_CUDA(cudaMemcpyAsync(r_[i].host, at<char>(r_[i].off), r_[i].bytes, cudaMemcpyDeviceToHost, st_));
        synced_ = true;
        CPB_CUDA(cudaStreamSynchronize(st_));
        return CPB_OK;
    }

  private:
    enum { kIn = 1, kOut = 2, kMax = 10 };
    struct Region {
        void* host;
        size_t bytes, off;
        int dir;
    };
    size_t add(void* h, size_t bytes, int dir) {
        const size_t off = total_;
        total_ += align256(bytes ? bytes : 1);
        if (n_ < kMax) r_[n_] = Region{h, bytes, off, dir};
        n_++;
        return off;
    }
    Scratch& arena_;
    cudaStream_t st_;
    Region r_[kMax];
    int n_ = 0;
    size_t total_ = 0;
    bool synced_ = false;
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
