// ubench_modmul.cu -- 256-bit Montgomery multiplication throughput on an H100: the IMAD.WIDE path of csrc/fp.cuh against
// the FP64-pipe path of tools/fp52.cuh, same dependent chain per thread (x <- x*y, x <- x^2 alternating), and a
// bit-for-bit check of the GPU results against the host build of the very same functions (exact emulation).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xptxas -v -o ubench_modmul ubench_modmul.cu
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <cuda_runtime.h>
#include "fp52.cuh"
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

int main() {
    cudaDeviceProp p;
    cudaGetDeviceProperties(&p, 0);
    printf("device %s, %d SMs; chain of 1000 dependent mul/sqr per thread, %d threads\n", p.name, p.multiProcessorCount, p.multiProcessorCount * 128 * 16);
    run<Bls12_381_Fr>("BLS12-381 Fr", p.multiProcessorCount);
    run<Bn254_Fr>("BN254 Fr", p.multiProcessorCount);
    return 0;
}
