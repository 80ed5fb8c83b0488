// ubench_imad_wide.cu -- the denominator of the integer roofline: how many IMAD.WIDE.U32 (32x32+64 -> 64 multiply-add)
// thread-operations per clock does one SM of an H100 issue?  NACC independent 64-bit accumulators per thread (no dependent
// chain shorter than NACC instructions), nothing else in the loop (cuobjdump -sass: the body is NACC x UNROLL IMAD.WIDE.U32
// plus the loop counter), long enough that launch overhead is < 0.1 %.  Also the carry-chained form the field code uses
// (IMAD.WIDE.U32.X with predicate carry-in / carry-out).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o ubench_imad_wide ubench_imad_wide.cu
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>
typedef uint32_t u32;
typedef uint64_t u64;

#define ITERS (1 << 14)
#define UNROLL 4

template <int NACC, int MODE> __global__ void __launch_bounds__(1024) k(u64* out, u32 seed, u32 mulv) {
    u64 w[NACC];
    u32 b[NACC];
    const u32 y = mulv | 1u;
#pragma unroll
    for (int i = 0; i < NACC; i++) { w[i] = ((u64)(seed + threadIdx.x) << 32) | (u32)(i * 77u + blockIdx.x); b[i] = seed * (2 * i + 3) + threadIdx.x; }
#pragma unroll 1
    for (int it = 0; it < ITERS; it++) {
#pragma unroll
        for (int u = 0; u < UNROLL; u++) {
            if (MODE == 2) {               // pure products: the loop body is IMAD.WIDE.U32 Rd, Ra, Rb, RZ only
#pragma unroll
                for (int i = 0; i < NACC; i++) {
                    u32 lo, hi, lo2, hi2;          // factors: low word of accumulator i+1, high word of accumulator i+2
                    asm volatile("mov.b64 {%0, %1}, %2;" : "=r"(lo), "=r"(hi) : "l"(w[(i + 1) % NACC]));
                    asm volatile("mov.b64 {%0, %1}, %2;" : "=r"(lo2), "=r"(hi2) : "l"(w[(i + 2) % NACC]));
                    asm volatile("mul.wide.u32 %0, %1, %2;" : "=l"(w[i]) : "r"(lo), "r"(hi2));
                }
            } else if (MODE == 0) {
#pragma unroll
                for (int i = 0; i < NACC; i++) {       // one factor is the low word of the NEXT accumulator: nothing is loop-invariant,
                    u32 lo, hi;                        // and every instruction depends only on results NACC-1 instructions old
                    asm volatile("mov.b64 {%0, %1}, %2;" : "=r"(lo), "=r"(hi) : "l"(w[(i + 1) % NACC]));
                    asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(w[i]) : "r"(lo), "r"(b[i]));
                }
            } else {
                // one carry chain through all NACC accumulators, as a CIOS row does: lo.cc / madc.hi.cc pairs
                u32 lo[NACC], hi[NACC];
#pragma unroll
                for (int i = 0; i < NACC; i++) { lo[i] = (u32)w[i]; hi[i] = (u32)(w[i] >> 32); }
                const u32 m = lo[0] ^ y;           // the row's multiplier depends on the running value, as in CIOS
                asm volatile("mad.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;" : "+r"(lo[0]), "+r"(hi[0]) : "r"(b[0]), "r"(m));
#pragma unroll
                for (int i = 1; i < NACC; i++)
                    asm volatile("madc.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;" : "+r"(lo[i]), "+r"(hi[i]) : "r"(b[i]), "r"(m));
#pragma unroll
                for (int i = 0; i < NACC; i++) w[i] = ((u64)hi[i] << 32) | lo[i];
            }
        }
    }
    u64 r = 0;
#pragma unroll
    for (int i = 0; i < NACC; i++) r ^= w[i];
    out[(size_t)blockIdx.x * blockDim.x + threadIdx.x] = r;
}

template <int NACC, int MODE> void run(const char* name, int sms, int khz, u64* d) {
    for (int warps_per_smsp = 1; warps_per_smsp <= 8; warps_per_smsp *= 2) {
        int threads = 128 * warps_per_smsp > 1024 ? 1024 : 128 * warps_per_smsp;
        int grid = sms * ((128 * warps_per_smsp) / threads);
        cudaEvent_t e0, e1;
        cudaEventCreate(&e0); cudaEventCreate(&e1);
        k<NACC, MODE><<<grid, threads>>>(d, 1, 3);
        cudaDeviceSynchronize();
        float best = 1e30f;
        for (int rep = 0; rep < 3; rep++) {
            cudaEventRecord(e0);
            k<NACC, MODE><<<grid, threads>>>(d, 1 + rep, 3);
            cudaEventRecord(e1);
            cudaEventSynchronize(e1);
            float ms = 0;
            cudaEventElapsedTime(&ms, e0, e1);
            if (ms < best) best = ms;
        }
        double thread_ops = (double)grid * threads * (double)ITERS * UNROLL * NACC;
        double per_clk_sm = thread_ops / (best * 1e-3) / sms / (khz * 1e3);
        printf("%-34s acc/thread=%2d warps/SMSP=%d  %8.3f ms  %6.2f thread-ops/clk/SM at %d MHz\n", name, NACC, warps_per_smsp, best, per_clk_sm, khz / 1000);
    }
}

int main() {
    cudaDeviceProp p;
    cudaGetDeviceProperties(&p, 0);
    int khz = 0;
    cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
    printf("device %s  SMs %d  max SM clock %d kHz (rates below assume the max clock; nvidia-smi during the run confirms it)\n", p.name, p.multiProcessorCount, khz);
    u64* d;
    cudaMalloc(&d, (size_t)1 << 26);
    int sms = p.multiProcessorCount;
    run<8, 2>("IMAD.WIDE.U32 products only", sms, khz, d);
    run<16, 2>("IMAD.WIDE.U32 products only", sms, khz, d);
    run<8, 0>("mad.wide (IMAD.WIDE + 64-bit add)", sms, khz, d);
    run<8, 1>("IMAD.WIDE.U32.X carry chain of 8", sms, khz, d);
    return 0;
}
