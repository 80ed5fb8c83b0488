// ubench_modmul.cu -- 256-bit Montgomery multiplication throughput on an H100: the IMAD.WIDE path of csrc/fp.cuh against
// the FP64-pipe path of tools/fp52.cuh, same dependent chain per thread (x <- x*y, x <- x^2 alternating), and a
// bit-for-bit check of the GPU results against the host build of the very same functions (exact emulation).
// BN254 Fr also runs a third arm at the shape of k_poseidon_crh_tc (128-thread CTAs, 5 CTAs/SM, converged warps): the
// 512-bit product on the integer pipe (fp_sqr_wide, fp_mul_wide) and its Montgomery reduction on the tensor cores (tc_redc,
// the 1 KB R^-1 table in shared memory), against the lazy IMAD products at the same shape, for squarings and multiplications
// separately; its canonical results are checked against the IMAD arm's.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xptxas -v -o ubench_modmul ubench_modmul.cu
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <cuda_runtime.h>
#include "fp52.cuh"
#include "../crypto_primitives_b200/csrc/poseidon_host.hpp"
using namespace cpb;

template <class F> CPB_HD void chain_imad(u32* x, const u32* y, int n) {
    u32 pm[8];
    fp_modulus<F>(pm);
    for (int k = 0; k < n; k++) {
        if (k & 1) fp_sqr<F>(x, x, pm);
        else fp_mul<F>(x, x, y, pm);
    }
}
template <class F> CPB_HD void chain_f52(u32* xw, const u32* yw, int n) {
    double pd[5], yd[5];
    f52::load_modulus<F>(pd);
    u64 x[5], y[5];
    f52::from_words(x, xw);
    f52::from_words(y, yw);
    f52::to_dbl5(yd, y);
    for (int k = 0; k < n; k++) {
        double xd[5];
        f52::to_dbl5(xd, x);
        if (k & 1) f52::sqr<F>(x, xd, pd);
        else f52::mul<F>(x, xd, yd, pd);
    }
    f52::canon<F>(x);
    f52::to_words(xw, x);
}

template <class F, int WHICH> __global__ void __launch_bounds__(128) k_chain(const u32* in, u32* out, int n, long total) {
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    u32 x[8], y[8];
    for (int j = 0; j < 8; j++) { x[j] = in[16 * i + j]; y[j] = in[16 * i + 8 + j]; }
    if (WHICH == 0) chain_imad<F>(x, y, n);
    else chain_f52<F>(x, y, n);
    for (int j = 0; j < 8; j++) out[8 * i + j] = x[j];
}

template <class F> void run(const char* name, int sms) {
    const int n = 1000;
    const long total = (long)sms * 128 * 16;                 // 16 CTAs of 128 threads per SM: several waves
    std::vector<u32> h(16 * total);
    u64 s = 12345;
    for (auto& v : h) { s = s * 6364136223846793005ull + 1442695040888963407ull; v = (u32)(s >> 33); }
    for (long i = 0; i < 2 * total; i++) h[8 * i + 7] &= 0x0fffffffu;   // < 2^252 < p: valid operands for both paths
    u32 *din, *dout;
    cudaMalloc(&din, h.size() * 4);
    cudaMalloc(&dout, 8 * total * 4);
    cudaMemcpy(din, h.data(), h.size() * 4, cudaMemcpyHostToDevice);
    std::vector<u32> g0(8 * total), g1(8 * total);
    float ms[2];
    for (int which = 0; which < 2; which++) {
        cudaEvent_t e0, e1;
        cudaEventCreate(&e0); cudaEventCreate(&e1);
        for (int rep = 0; rep < 2; rep++) {
            cudaEventRecord(e0);
            if (which == 0) k_chain<F, 0><<<(int)(total / 128), 128>>>(din, dout, n, total);
            else k_chain<F, 1><<<(int)(total / 128), 128>>>(din, dout, n, total);
            cudaEventRecord(e1);
            cudaEventSynchronize(e1);
        }
        cudaEventElapsedTime(&ms[which], e0, e1);
        cudaMemcpy((which ? g1 : g0).data(), dout, 8 * total * 4, cudaMemcpyDeviceToHost);
        cudaError_t err = cudaGetLastError();
        if (err != cudaSuccess) printf("CUDA error: %s\n", cudaGetErrorString(err));
    }
    // host check of the first and last 64 chains: same functions, exact emulation
    long bad0 = 0, bad1 = 0;
    for (long t = 0; t < 128; t++) {
        long i = t < 64 ? t : total - 128 + t;
        u32 x[8], y[8];
        for (int j = 0; j < 8; j++) { x[j] = h[16 * i + j]; y[j] = h[16 * i + 8 + j]; }
        u32 a[8], b[8];
        for (int j = 0; j < 8; j++) { a[j] = x[j]; b[j] = x[j]; }
        chain_imad<F>(a, y, n);
        chain_f52<F>(b, y, n);
        for (int j = 0; j < 8; j++) { bad0 += a[j] != g0[8 * i + j]; bad1 += b[j] != g1[8 * i + j]; }
    }
    const double muls = (double)total * n;
    printf("%-14s IMAD.WIDE path %8.3f ms  %7.2f G modmul/s | FP64 path %8.3f ms  %7.2f G modmul/s | speed-up %.2fx | host mismatches: imad %ld, f52 %ld\n",
           name, ms[0], muls / ms[0] / 1e6, ms[1], muls / ms[1] / 1e6, ms[0] / ms[1], bad0, bad1);
    cudaFree(din); cudaFree(dout);
}

// The tensor-core arm and its IMAD reference at the hash kernel's shape.  OP 0: x <- x^2 and x <- x*y alternating, 1: squarings
// only, 2: multiplications only.  TC: tc_redc, else the LAZY IMAD products.  Operands stay below 2p (< 1.4p), so one conditional
// subtraction makes the result canonical.
constexpr int kTcSmem = 4 * kTcWarpWords * 4 + kTcRinvWords * 4;
template <int OP, bool TC> __global__ void __launch_bounds__(128, 5) k_chain_shape(const u32* in, const u32* rinv_g, u32* out, int n) {
    extern __shared__ __align__(16) u32 sm[];
    u32* rinv = sm + 4 * kTcWarpWords;
    for (int j = threadIdx.x; j < kTcRinvWords; j += blockDim.x) rinv[j] = rinv_g[j];
    __syncthreads();
    u32* buf = sm + (threadIdx.x >> 5) * kTcWarpWords;
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;      // the grid covers the batch exactly: warps stay converged
    u32 x[8], y[8], pm[8];
    fp_modulus<Bn254_Fr>(pm);
    for (int j = 0; j < 8; j++) { x[j] = in[16 * i + j]; y[j] = in[16 * i + 8 + j]; }
    for (int k = 0; k < n; k++) {
        const bool sqr = OP == 1 || (OP == 0 && (k & 1));
        if constexpr (TC) {
#if defined(__CUDA_ARCH__)
            u32 T[16];
            if (sqr) fp_sqr_wide(T, x);
            else fp_mul_wide(T, x, y);
            tc_redc<Bn254_Fr>(x, T, rinv, buf, pm);
#endif
        } else if (sqr) {
            fp_sqr<Bn254_Fr, true>(x, x, pm);
        } else {
            fp_mul<Bn254_Fr, true>(x, x, y, pm);
        }
    }
    fp_final_sub<Bn254_Fr>(x);
    for (int j = 0; j < 8; j++) out[8 * i + j] = x[j];
}

template <int OP, bool TC> float time_shape(const u32* din, const u32* drinv, u32* dout, int n, long total) {
    cudaFuncSetAttribute(k_chain_shape<OP, TC>, cudaFuncAttributeMaxDynamicSharedMemorySize, kTcSmem);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    float ms = 0;
    for (int rep = 0; rep < 2; rep++) {                     // the second launch is timed
        cudaEventRecord(e0);
        k_chain_shape<OP, TC><<<(int)(total / 128), 128, kTcSmem>>>(din, drinv, dout, n);
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
    }
    cudaEventElapsedTime(&ms, e0, e1);
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    return ms;
}

void run_tc(int sms) {
    const int n = 1000;
    const long total = (long)sms * 128 * 5 * 4;              // 4 waves of 5 CTAs per SM
    std::vector<u32> h(16 * total);
    u64 s = 6789;
    for (auto& v : h) { s = s * 6364136223846793005ull + 1442695040888963407ull; v = (u32)(s >> 33); }
    for (long i = 0; i < 2 * total; i++) h[8 * i + 7] &= 0x0fffffffu;   // < 2^252 < p
    const std::vector<u32> rinv = host::tc_rinv_table(host::Field(host::field_modulus(Bn254_Fr::ID)));
    u32 *din, *drinv, *dout;
    cudaMalloc(&din, h.size() * 4);
    cudaMalloc(&drinv, rinv.size() * 4);
    cudaMalloc(&dout, 8 * total * 4);
    cudaMemcpy(din, h.data(), h.size() * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(drinv, rinv.data(), rinv.size() * 4, cudaMemcpyHostToDevice);
    const char* names[3] = {"sqr/mul alternating", "sqr only", "mul only"};
    for (int op = 0; op < 3; op++) {
        std::vector<u32> g[2];
        float ms[2];
        for (int tc = 0; tc < 2; tc++) {
            if (op == 0) ms[tc] = tc ? time_shape<0, true>(din, drinv, dout, n, total) : time_shape<0, false>(din, drinv, dout, n, total);
            if (op == 1) ms[tc] = tc ? time_shape<1, true>(din, drinv, dout, n, total) : time_shape<1, false>(din, drinv, dout, n, total);
            if (op == 2) ms[tc] = tc ? time_shape<2, true>(din, drinv, dout, n, total) : time_shape<2, false>(din, drinv, dout, n, total);
            g[tc].resize(8 * total);
            cudaMemcpy(g[tc].data(), dout, 8 * total * 4, cudaMemcpyDeviceToHost);
        }
        cudaError_t err = cudaGetLastError();
        if (err != cudaSuccess) printf("CUDA error: %s\n", cudaGetErrorString(err));
        long bad = 0;
        for (long j = 0; j < 8 * total; j++) bad += g[0][j] != g[1][j];
        // host check of the IMAD arm on the first 64 chains: the same functions, exact emulation
        long bad_host = 0;
        for (long i = 0; i < 64; i++) {
            u32 x[8], y[8], pm[8];
            fp_modulus<Bn254_Fr>(pm);
            for (int j = 0; j < 8; j++) { x[j] = h[16 * i + j]; y[j] = h[16 * i + 8 + j]; }
            for (int k = 0; k < n; k++) {
                if (op == 1 || (op == 0 && (k & 1))) fp_sqr<Bn254_Fr>(x, x, pm);
                else fp_mul<Bn254_Fr>(x, x, y, pm);
            }
            for (int j = 0; j < 8; j++) bad_host += x[j] != g[0][8 * i + j];
        }
        const double prod = (double)total * n;
        printf("BN254 Fr %-20s IMAD %8.3f ms %6.3f ns/product/SM | IMAD + TC reduction %8.3f ms %6.3f ns/product/SM | TC/IMAD %.3f | "
               "mismatches: TC vs IMAD %ld, IMAD vs host %ld\n",
               names[op], ms[0], ms[0] * 1e6 * sms / prod, ms[1], ms[1] * 1e6 * sms / prod, ms[1] / ms[0], bad, bad_host);
    }
    cudaFree(din); cudaFree(drinv); cudaFree(dout);
}

int main() {
    cudaDeviceProp p;
    cudaGetDeviceProperties(&p, 0);
    printf("device %s, %d SMs; chain of 1000 dependent mul/sqr per thread, %d threads\n", p.name, p.multiProcessorCount, p.multiProcessorCount * 128 * 16);
    run<Bls12_381_Fr>("BLS12-381 Fr", p.multiProcessorCount);
    run<Bn254_Fr>("BN254 Fr", p.multiProcessorCount);
    int occ[2] = {0, 0};
    cudaFuncSetAttribute(k_chain_shape<0, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kTcSmem);
    cudaFuncSetAttribute(k_chain_shape<0, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kTcSmem);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ[0], k_chain_shape<0, false>, 128, kTcSmem);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ[1], k_chain_shape<0, true>, 128, kTcSmem);
    printf("hash-kernel shape: 128-thread CTAs, %d B shared memory, resident CTAs/SM: IMAD %d, TC %d\n", kTcSmem, occ[0], occ[1]);
    run_tc(p.multiProcessorCount);
    return 0;
}
