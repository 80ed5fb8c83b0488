// tc_probe.cu -- the tensor-core pieces of the BN254 Fr hash kernel (crypto_primitives_b200/csrc/poseidon_tc.cuh: tc_redc,
// tc_partial_round, tc_full_round, tc_finish; poseidon.cuh: pos_sbox5_tc) run on the device one piece at a time, on operands the
// caller chooses per lane, for tests/test_gpu_poseidon_tc_crafted.py.  Test-only: not linked into the product.
//
// Each launch is CTAs of kWarps whole, converged warps.  The tables the product keeps in shared memory (the R^-1 table, a partial
// round's table) are copied there with plain loads and __syncthreads -- no TMA, no mbarrier, no ring: the ring is covered by the
// hash kernel's own tests -- and the full rounds' row tables stay in global memory, where tc_full_round reads them.  Every
// launcher takes and returns host arrays of 32-bit limbs, one record per thread, and returns a cudaError_t (0 on success).
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../crypto_primitives_b200/csrc/poseidon.cuh"
using namespace cpb;
using F = Bn254_Fr;

namespace {
constexpr int kWarps = 4;
constexpr int kThreads = 32 * kWarps;

__device__ void stage_table(u32* dst, const u32* src, int words) {
    for (int i = threadIdx.x; i < words; i += blockDim.x) dst[i] = src[i];
    __syncthreads();
}

__global__ void __launch_bounds__(kThreads) k_redc(const u32* __restrict__ T, const u32* __restrict__ rinv_g, u32* __restrict__ out) {
    __shared__ __align__(16) u32 rinv[kTcRinvWords];
    __shared__ __align__(16) u32 buf[kWarps * kTcWarpWords];
    stage_table(rinv, rinv_g, kTcRinvWords);
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    u32 t[16], r[8], pm[8];
    fp_modulus<F>(pm);
    for (int j = 0; j < 16; j++) t[j] = T[16 * i + j];
#if defined(__CUDA_ARCH__)      // device-only pieces (poseidon_tc.cuh)
    tc_redc<F>(r, t, rinv, buf + (threadIdx.x >> 5) * kTcWarpWords, pm);
#endif
    for (int j = 0; j < 8; j++) out[8 * i + j] = r[j];
}

__global__ void __launch_bounds__(kThreads) k_sbox5(const u32* __restrict__ x, const u32* __restrict__ rinv_g, u32* __restrict__ out) {
    __shared__ __align__(16) u32 rinv[kTcRinvWords];
    __shared__ __align__(16) u32 buf[kWarps * kTcWarpWords];
    stage_table(rinv, rinv_g, kTcRinvWords);
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    u32 v[8], pm[8];
    fp_modulus<F>(pm);
    for (int j = 0; j < 8; j++) v[j] = x[8 * i + j];
    pos_sbox5_tc<F>(v, rinv, buf + (threadIdx.x >> 5) * kTcWarpWords, pm);
    for (int j = 0; j < 8; j++) out[8 * i + j] = v[j];
}

// s: (y, a, s2) per thread; out: an, then s2 after the column update, per thread.
__global__ void __launch_bounds__(kThreads) k_partial_round(const u32* __restrict__ s_in, const u32* __restrict__ tab_g, u32* __restrict__ out) {
    __shared__ __align__(16) u32 tab[kTcRoundWords];
    __shared__ __align__(16) u32 buf[kWarps * kTcWarpWords];
    stage_table(tab, tab_g, kTcRoundWords);
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    u32 s[3][8], an[8], pm[8];
    fp_modulus<F>(pm);
    for (int l = 0; l < 3; l++)
        for (int j = 0; j < 8; j++) s[l][j] = s_in[24 * i + 8 * l + j];
#if defined(__CUDA_ARCH__)      // device-only pieces (poseidon_tc.cuh)
    tc_partial_round<F>(an, s, tab, buf + (threadIdx.x >> 5) * kTcWarpWords, pm);
#endif
    for (int j = 0; j < 8; j++) {
        out[16 * i + j] = an[j];
        out[16 * i + 8 + j] = s[2][j];
    }
}

// s: three S-box outputs per thread, replaced by the round's rows (zero where need has no bit).  rows: three row tables, row1 the
// table row 1 reads (global memory).
__global__ void __launch_bounds__(kThreads) k_full_round(const u32* __restrict__ s_in, const u32* __restrict__ rows, const u32* __restrict__ row1,
                                                         unsigned need, u32* __restrict__ out) {
    __shared__ __align__(16) u32 buf[kWarps * kTcWarpWords];
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    u32 s[3][8], pm[8];
    fp_modulus<F>(pm);
    for (int l = 0; l < 3; l++)
        for (int j = 0; j < 8; j++) s[l][j] = s_in[24 * i + 8 * l + j];
#if defined(__CUDA_ARCH__)      // device-only pieces (poseidon_tc.cuh)
    tc_full_round<F>(s, rows, row1, need, buf + (threadIdx.x >> 5) * kTcWarpWords, pm);
#endif
    for (int l = 0; l < 3; l++)
        for (int j = 0; j < 8; j++) out[24 * i + 8 * l + j] = s[l][j];
}

// hy: h[16] then y[8] per thread.
template <bool U> __global__ void __launch_bounds__(kThreads) k_finish(const u32* __restrict__ hy, u32* __restrict__ out) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    u32 h[16], y[8], r[8], pm[8];
    fp_modulus<F>(pm);
    for (int j = 0; j < 16; j++) h[j] = hy[24 * i + j];
    for (int j = 0; j < 8; j++) y[j] = hy[24 * i + 16 + j];
    tc_finish<F, U>(r, h, y, pm);
    for (int j = 0; j < 8; j++) out[8 * i + j] = r[j];
}

// Device copies of the launch's arrays, freed on every return path.
struct Buffers {
    void* p[4] = {nullptr, nullptr, nullptr, nullptr};
    int n = 0;
    ~Buffers() {
        for (int i = 0; i < n; i++) cudaFree(p[i]);
    }
    cudaError_t up(u32** d, const void* h, size_t bytes) {
        cudaError_t e = cudaMalloc(&p[n], bytes);
        if (e != cudaSuccess) return e;
        *d = (u32*)p[n++];
        return h ? cudaMemcpy(*d, h, bytes, cudaMemcpyHostToDevice) : cudaSuccess;
    }
};

#define PROBE_TRY(x)                                 \
    do {                                             \
        const cudaError_t e_ = (x);                  \
        if (e_ != cudaSuccess) return (int)e_;       \
    } while (0)

// n threads (a multiple of kThreads); a: the per-thread input (in_words each), b: a table (b_words), out: out_words per thread.
template <class Launch>
int run(int n, const void* a, size_t in_words, const void* b, size_t b_words, void* out, size_t out_words, Launch launch) {
    if (n <= 0 || n % kThreads) return (int)cudaErrorInvalidValue;
    Buffers B;
    u32 *da = nullptr, *db = nullptr, *dout = nullptr;
    PROBE_TRY(B.up(&da, a, (size_t)n * in_words * 4));
    if (b) PROBE_TRY(B.up(&db, b, b_words * 4));
    PROBE_TRY(B.up(&dout, nullptr, (size_t)n * out_words * 4));
    launch(n / kThreads, da, db, dout);
    PROBE_TRY(cudaGetLastError());
    PROBE_TRY(cudaDeviceSynchronize());
    PROBE_TRY(cudaMemcpy(out, dout, (size_t)n * out_words * 4, cudaMemcpyDeviceToHost));
    return 0;
}
}  // namespace

extern "C" int probe_threads_per_cta() { return kThreads; }

// T: 16 limbs per thread; rinv: kTcRinvWords; out: 8 limbs per thread (tc_redc's unreduced result).
extern "C" int probe_redc(const uint32_t* T, const uint32_t* rinv, uint32_t* out, int n) {
    return run(n, T, 16, rinv, kTcRinvWords, out, 8, [](int g, u32* a, u32* b, u32* o) { k_redc<<<g, kThreads>>>(a, b, o); });
}

// x: 8 limbs per thread; out: pos_sbox5_tc's unreduced x^5.
extern "C" int probe_sbox5(const uint32_t* x, const uint32_t* rinv, uint32_t* out, int n) {
    return run(n, x, 8, rinv, kTcRinvWords, out, 8, [](int g, u32* a, u32* b, u32* o) { k_sbox5<<<g, kThreads>>>(a, b, o); });
}

// s: (y, a, s2) per thread, 24 limbs; tab: one partial round's kTcRoundWords; out: an then the updated s2, 16 limbs per thread.
extern "C" int probe_partial_round(const uint32_t* s, const uint32_t* tab, uint32_t* out, int n) {
    return run(n, s, 24, tab, kTcRoundWords, out, 16, [](int g, u32* a, u32* b, u32* o) { k_partial_round<<<g, kThreads>>>(a, b, o); });
}

// s: 24 limbs per thread; rows: the four tables [row 0, row 1, row 2, the table row 1 reads], kTcRowWords each; out: 24 limbs.
extern "C" int probe_full_round(const uint32_t* s, const uint32_t* rows, unsigned need, uint32_t* out, int n) {
    return run(n, s, 24, rows, 4 * kTcRowWords, out, 24, [need](int g, u32* a, u32* b, u32* o) {
        k_full_round<<<g, kThreads>>>(a, b, b + 3 * kTcRowWords, need, o);
    });
}

// hy: h[16] then y[8] per thread, 24 words; u != 0: y is the unit addend; out: 8 limbs.
extern "C" int probe_finish(const uint32_t* hy, int u, uint32_t* out, int n) {
    return run(n, hy, 24, nullptr, 0, out, 8, [u](int g, u32* a, u32*, u32* o) {
        if (u) k_finish<true><<<g, kThreads>>>(a, o);
        else k_finish<false><<<g, kThreads>>>(a, o);
    });
}
