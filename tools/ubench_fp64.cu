// ubench_fp64.cu -- is the FP64 pipe of an H100 a second multiplier for big-integer arithmetic?
// Measures DFMA / DADD / 64-bit integer add issue rates and whether DFMA overlaps with IMAD.WIDE and with ALU work.
// (Background: 52-bit-limb Montgomery multiplication on the FP64 pipe -- two round-toward-zero FMAs give the high and
// low halves of a 104-bit product, column sums are 64-bit integer adds on the raw bit patterns.)
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o ubench_fp64 ubench_fp64.cu
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>
typedef uint32_t u32;
typedef uint64_t u64;
#define ITERS 4096
#define NACC 8

// MODE 0: fma.rz.f64            1: add.rz.f64           2: add.u64 (integer)
// MODE 3: DFMA + IMAD.WIDE 1:1  4: DFMA + 32-bit IADD3 1:1
// MODE 5: the DPF inner step: 2 DFMA + 1 DADD + 2 integer 64-bit adds
// MODE 6: 2 DFMA + 1 DADD + 2 x add.u64 + 1 IMAD.WIDE (hybrid)
template <int MODE> __global__ void k(u64* out, u32 seed, double mulv) {
    double f[NACC], g[NACC], h[NACC];
    u64 w[NACC], v[NACC];
    u32 b[NACC];
    u32 x = seed + threadIdx.x;
#pragma unroll
    for (int i = 0; i < NACC; i++) { f[i] = (double)(x * (i + 3)); g[i] = (double)(x ^ (i * 77)) + 0.5; h[i] = 4503599627370496.0 + i; w[i] = ((u64)x << 32) | (x * i); v[i] = x + i; b[i] = x - i; }
    const u32 y = (u32)mulv | 1;
#pragma unroll 1
    for (int it = 0; it < ITERS; it++) {
#pragma unroll
        for (int i = 0; i < NACC; i++) {
            if (MODE == 0) asm volatile("fma.rz.f64 %0, %0, %1, %2;" : "+d"(f[i]) : "d"(mulv), "d"(g[i]));
            if (MODE == 1) asm volatile("add.rz.f64 %0, %0, %1;" : "+d"(f[i]) : "d"(g[i]));
            if (MODE == 2) asm volatile("add.u64 %0, %0, %1;" : "+l"(w[i]) : "l"(v[i]));
            if (MODE == 3) {
                asm volatile("fma.rz.f64 %0, %0, %1, %2;" : "+d"(f[i]) : "d"(mulv), "d"(g[i]));
                asm volatile("{.reg .u32 lo, hi; mov.b64 {lo, hi}, %0; mad.lo.cc.u32 lo, %1, %2, lo; madc.hi.u32 hi, %1, %2, hi; mov.b64 %0, {lo, hi};}" : "+l"(w[i]) : "r"(b[i]), "r"(y));
            }
            if (MODE == 4) {
                asm volatile("fma.rz.f64 %0, %0, %1, %2;" : "+d"(f[i]) : "d"(mulv), "d"(g[i]));
                asm volatile("{.reg .u32 t; add.u32 t, %0, %1; add.u32 %0, t, %2;}" : "+r"(b[i]) : "r"(x), "r"(y));
            }
            if (MODE == 5 || MODE == 6) {
                double hi, lo, sub;
                asm volatile("fma.rz.f64 %0, %1, %2, %3;" : "=d"(hi) : "d"(f[i]), "d"(mulv), "d"(h[i]));
                asm volatile("sub.rz.f64 %0, %1, %2;" : "=d"(sub) : "d"(g[i]), "d"(hi));
                asm volatile("fma.rz.f64 %0, %1, %2, %3;" : "=d"(lo) : "d"(f[i]), "d"(mulv), "d"(sub));
                asm volatile("add.u64 %0, %0, %1;" : "+l"(w[i]) : "l"(__double_as_longlong(hi)));
                asm volatile("add.u64 %0, %0, %1;" : "+l"(v[i]) : "l"(__double_as_longlong(lo)));
                if (MODE == 6)
                    asm volatile("{.reg .u32 lo, hi; mov.b64 {lo, hi}, %0; mad.lo.cc.u32 lo, %1, %2, lo; madc.hi.u32 hi, %1, %2, hi; mov.b64 %0, {lo, hi};}" : "+l"(w[i]) : "r"(b[i]), "r"(y));
            }
        }
    }
    u64 r = 0;
#pragma unroll
    for (int i = 0; i < NACC; i++) r ^= (u64)__double_as_longlong(f[i]) ^ w[i] ^ v[i] ^ b[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = r;
}

template <int MODE> void run(const char* name, double ops_per_iter, int sms, int khz, u64* d) {
    for (int warps_per_smsp = 2; warps_per_smsp <= 8; warps_per_smsp *= 2) {
        int threads = 128 * warps_per_smsp > 1024 ? 1024 : 128 * warps_per_smsp;
        int grid = sms * ((128 * warps_per_smsp) / threads);
        cudaEvent_t e0, e1;
        cudaEventCreate(&e0); cudaEventCreate(&e1);
        k<MODE><<<grid, threads>>>(d, 1, 3.0);
        cudaDeviceSynchronize();
        cudaEventRecord(e0);
        k<MODE><<<grid, threads>>>(d, 1, 3.0);
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        float ms = 0;
        cudaEventElapsedTime(&ms, e0, e1);
        double groups = (double)grid * (threads / 32) * ITERS * NACC;
        double cyc_per_group_smsp = (ms * 1e-3) * (khz * 1e3) / (groups / (sms * 4));
        printf("%-44s warps/SMSP=%d  %.3f ms  %.2f cycles per group per SMSP (%g PTX ops/group)\n", name, warps_per_smsp, ms, cyc_per_group_smsp, ops_per_iter);
    }
}

int main() {
    cudaDeviceProp p;
    cudaGetDeviceProperties(&p, 0);
    int khz = 0;
    cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
    printf("device %s  SMs %d  clock %d kHz; a 'group' is one warp-wide execution of the listed PTX ops\n", p.name, p.multiProcessorCount, khz);
    u64* d;
    cudaMalloc(&d, 1 << 26);
    int sms = p.multiProcessorCount;
    run<0>("DFMA", 1, sms, khz, d);
    run<1>("DADD", 1, sms, khz, d);
    run<2>("add.u64", 1, sms, khz, d);
    run<3>("DFMA + IMAD.WIDE", 2, sms, khz, d);
    run<4>("DFMA + 2x add.u32 (IADD3)", 2, sms, khz, d);
    run<5>("2 DFMA + DSUB + 2 add.u64 (DPF step)", 5, sms, khz, d);
    run<6>("2 DFMA + DSUB + 2 add.u64 + IMAD.WIDE", 6, sms, khz, d);
    return 0;
}
