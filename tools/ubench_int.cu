// ubench_int.cu -- integer-pipe microbenchmark for sm_90a: how many IMAD / IMAD.WIDE /
// IADD3 warp-instructions per clock per SM does an H100 sustain?  These are the denominators of
// the integer roofline in DESIGN.md (the Poseidon/Pedersen kernels are IMAD-bound, not HBM-bound).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o ubench_int ubench_int.cu
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>
typedef uint32_t u32;
typedef uint64_t u64;

#define ITERS 4096
#define NACC 8

// MODE 0: mad.lo.u32 (IMAD)            1: mad.wide.u32 64-bit accumulate (IMAD.WIDE.U32)
// MODE 2: mad.lo.cc/madc.hi.cc chains  (IMAD.WIDE.U32.X with predicate carry)
// MODE 3: add.u32 x3 (IADD3)           4: IMAD.WIDE + IADD3 interleaved 1:1
// MODE 5: split pair IMAD.X-like: mad.lo + mad.hi separately (2 x 32-bit IMAD per product)
template <int MODE> __global__ void k(u32* out, u32 seed, u32 mulv) {
    u32 a[NACC], b[NACC], c[NACC];
    u64 w[NACC];
    u32 w32[NACC];
    u32 x = seed + threadIdx.x, y = mulv | 1;
#pragma unroll
    for (int i = 0; i < NACC; i++) { a[i] = x * (i + 3); b[i] = x ^ (i * 77); c[i] = x + i; w32[i] = x - i; w[i] = ((u64)a[i] << 32) | b[i]; }
#pragma unroll 1
    for (int it = 0; it < ITERS; it++) {
        if (MODE == 0) {
#pragma unroll
            for (int i = 0; i < NACC; i++) asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(y), "r"(b[i]));
        } else if (MODE == 1) {
            asm volatile("{.reg .u32 lo, hi; mov.b64 {lo, hi}, %0; mad.lo.cc.u32 lo, %1, %2, lo; madc.hi.u32 hi, %1, %2, hi; mov.b64 %0, {lo, hi};}" : "+l"(w[0]) : "r"(b[0]), "r"(y));
            asm volatile("{.reg .u32 lo, hi; mov.b64 {lo, hi}, %0; mad.lo.cc.u32 lo, %1, %2, lo; madc.hi.u32 hi, %1, %2, hi; mov.b64 %0, {lo, hi};}" : "+l"(w[1]) : "r"(b[1]), "r"(y));
            asm volatile("{.reg .u32 lo, hi; mov.b64 {lo, hi}, %0; mad.lo.cc.u32 lo, %1, %2, lo; madc.hi.u32 hi, %1, %2, hi; mov.b64 %0, {lo, hi};}" : "+l"(w[2]) : "r"(b[2]), "r"(y));
            asm volatile("{.reg .u32 lo, hi; mov.b64 {lo, hi}, %0; mad.lo.cc.u32 lo, %1, %2, lo; madc.hi.u32 hi, %1, %2, hi; mov.b64 %0, {lo, hi};}" : "+l"(w[3]) : "r"(b[3]), "r"(y));
            asm volatile("{.reg .u32 lo, hi; mov.b64 {lo, hi}, %0; mad.lo.cc.u32 lo, %1, %2, lo; madc.hi.u32 hi, %1, %2, hi; mov.b64 %0, {lo, hi};}" : "+l"(w[4]) : "r"(b[4]), "r"(y));
            asm volatile("{.reg .u32 lo, hi; mov.b64 {lo, hi}, %0; mad.lo.cc.u32 lo, %1, %2, lo; madc.hi.u32 hi, %1, %2, hi; mov.b64 %0, {lo, hi};}" : "+l"(w[5]) : "r"(b[5]), "r"(y));
            asm volatile("{.reg .u32 lo, hi; mov.b64 {lo, hi}, %0; mad.lo.cc.u32 lo, %1, %2, lo; madc.hi.u32 hi, %1, %2, hi; mov.b64 %0, {lo, hi};}" : "+l"(w[6]) : "r"(b[6]), "r"(y));
            asm volatile("{.reg .u32 lo, hi; mov.b64 {lo, hi}, %0; mad.lo.cc.u32 lo, %1, %2, lo; madc.hi.u32 hi, %1, %2, hi; mov.b64 %0, {lo, hi};}" : "+l"(w[7]) : "r"(b[7]), "r"(y));
        } else if (MODE == 2) {
            asm volatile("{.reg .u32 lo, hi; mov.b64 {lo, hi}, %0; mad.lo.cc.u32 lo, %1, %2, lo; madc.hi.cc.u32 hi, %1, %2, hi; mov.b64 %0, {lo, hi};}" : "+l"(w[0]) : "r"(b[0]), "r"(y));
            asm volatile("{.reg .u32 lo, hi; mov.b64 {lo, hi}, %0; madc.lo.cc.u32 lo, %1, %2, lo; madc.hi.cc.u32 hi, %1, %2, hi; mov.b64 %0, {lo, hi};}" : "+l"(w[1]) : "r"(b[1]), "r"(y));
            asm volatile("{.reg .u32 lo, hi; mov.b64 {lo, hi}, %0; madc.lo.cc.u32 lo, %1, %2, lo; madc.hi.cc.u32 hi, %1, %2, hi; mov.b64 %0, {lo, hi};}" : "+l"(w[2]) : "r"(b[2]), "r"(y));
            asm volatile("{.reg .u32 lo, hi; mov.b64 {lo, hi}, %0; madc.lo.cc.u32 lo, %1, %2, lo; madc.hi.u32 hi, %1, %2, hi; mov.b64 %0, {lo, hi};}" : "+l"(w[3]) : "r"(b[3]), "r"(y));
            asm volatile("{.reg .u32 lo, hi; mov.b64 {lo, hi}, %0; mad.lo.cc.u32 lo, %1, %2, lo; madc.hi.cc.u32 hi, %1, %2, hi; mov.b64 %0, {lo, hi};}" : "+l"(w[4]) : "r"(b[4]), "r"(y));
            asm volatile("{.reg .u32 lo, hi; mov.b64 {lo, hi}, %0; madc.lo.cc.u32 lo, %1, %2, lo; madc.hi.cc.u32 hi, %1, %2, hi; mov.b64 %0, {lo, hi};}" : "+l"(w[5]) : "r"(b[5]), "r"(y));
            asm volatile("{.reg .u32 lo, hi; mov.b64 {lo, hi}, %0; madc.lo.cc.u32 lo, %1, %2, lo; madc.hi.cc.u32 hi, %1, %2, hi; mov.b64 %0, {lo, hi};}" : "+l"(w[6]) : "r"(b[6]), "r"(y));
            asm volatile("{.reg .u32 lo, hi; mov.b64 {lo, hi}, %0; madc.lo.cc.u32 lo, %1, %2, lo; madc.hi.u32 hi, %1, %2, hi; mov.b64 %0, {lo, hi};}" : "+l"(w[7]) : "r"(b[7]), "r"(y));
        } else if (MODE == 3) {
#pragma unroll
            for (int i = 0; i < NACC; i++) asm volatile("{.reg .u32 t; add.u32 t, %0, %1; add.u32 %0, t, %2;}" : "+r"(a[i]) : "r"(b[i]), "r"(y));
        } else if (MODE == 4) {
            asm volatile("{.reg .u32 lo, hi; mov.b64 {lo, hi}, %0; mad.lo.cc.u32 lo, %1, %2, lo; madc.hi.u32 hi, %1, %2, hi; mov.b64 %0, {lo, hi};}" : "+l"(w[0]) : "r"(b[0]), "r"(y));
            asm volatile("{.reg .u32 t; add.u32 t, %0, %1; add.u32 %0, t, %2;}" : "+r"(c[0]) : "r"(b[0]), "r"(y));
            asm volatile("{.reg .u32 lo, hi; mov.b64 {lo, hi}, %0; mad.lo.cc.u32 lo, %1, %2, lo; madc.hi.u32 hi, %1, %2, hi; mov.b64 %0, {lo, hi};}" : "+l"(w[1]) : "r"(b[1]), "r"(y));
            asm volatile("{.reg .u32 t; add.u32 t, %0, %1; add.u32 %0, t, %2;}" : "+r"(c[1]) : "r"(b[1]), "r"(y));
            asm volatile("{.reg .u32 lo, hi; mov.b64 {lo, hi}, %0; mad.lo.cc.u32 lo, %1, %2, lo; madc.hi.u32 hi, %1, %2, hi; mov.b64 %0, {lo, hi};}" : "+l"(w[2]) : "r"(b[2]), "r"(y));
            asm volatile("{.reg .u32 t; add.u32 t, %0, %1; add.u32 %0, t, %2;}" : "+r"(c[2]) : "r"(b[2]), "r"(y));
            asm volatile("{.reg .u32 lo, hi; mov.b64 {lo, hi}, %0; mad.lo.cc.u32 lo, %1, %2, lo; madc.hi.u32 hi, %1, %2, hi; mov.b64 %0, {lo, hi};}" : "+l"(w[3]) : "r"(b[3]), "r"(y));
            asm volatile("{.reg .u32 t; add.u32 t, %0, %1; add.u32 %0, t, %2;}" : "+r"(c[3]) : "r"(b[3]), "r"(y));
            asm volatile("{.reg .u32 lo, hi; mov.b64 {lo, hi}, %0; mad.lo.cc.u32 lo, %1, %2, lo; madc.hi.u32 hi, %1, %2, hi; mov.b64 %0, {lo, hi};}" : "+l"(w[4]) : "r"(b[4]), "r"(y));
            asm volatile("{.reg .u32 t; add.u32 t, %0, %1; add.u32 %0, t, %2;}" : "+r"(c[4]) : "r"(b[4]), "r"(y));
            asm volatile("{.reg .u32 lo, hi; mov.b64 {lo, hi}, %0; mad.lo.cc.u32 lo, %1, %2, lo; madc.hi.u32 hi, %1, %2, hi; mov.b64 %0, {lo, hi};}" : "+l"(w[5]) : "r"(b[5]), "r"(y));
            asm volatile("{.reg .u32 t; add.u32 t, %0, %1; add.u32 %0, t, %2;}" : "+r"(c[5]) : "r"(b[5]), "r"(y));
            asm volatile("{.reg .u32 lo, hi; mov.b64 {lo, hi}, %0; mad.lo.cc.u32 lo, %1, %2, lo; madc.hi.u32 hi, %1, %2, hi; mov.b64 %0, {lo, hi};}" : "+l"(w[6]) : "r"(b[6]), "r"(y));
            asm volatile("{.reg .u32 t; add.u32 t, %0, %1; add.u32 %0, t, %2;}" : "+r"(c[6]) : "r"(b[6]), "r"(y));
            asm volatile("{.reg .u32 lo, hi; mov.b64 {lo, hi}, %0; mad.lo.cc.u32 lo, %1, %2, lo; madc.hi.u32 hi, %1, %2, hi; mov.b64 %0, {lo, hi};}" : "+l"(w[7]) : "r"(b[7]), "r"(y));
            asm volatile("{.reg .u32 t; add.u32 t, %0, %1; add.u32 %0, t, %2;}" : "+r"(c[7]) : "r"(b[7]), "r"(y));
        } else if (MODE == 5) {
#pragma unroll
            for (int i = 0; i < NACC; i++) {
                asm volatile("mad.lo.u32 %0, %1, %2, %0;" : "+r"(a[i]) : "r"(b[i]), "r"(y));
                asm volatile("mad.hi.u32 %0, %1, %2, %0;" : "+r"(b[i]) : "r"(a[i]), "r"(y));
            }
        }
    }
    u32 r = 0;
#pragma unroll
    for (int i = 0; i < NACC; i++) r ^= a[i] ^ b[i] ^ c[i] ^ w32[i] ^ (u32)w[i] ^ (u32)(w[i] >> 32);
    out[blockIdx.x * blockDim.x + threadIdx.x] = r;
}

template <int MODE> void run(const char* name, double ops_per_iter, int sms, int khz, u32* d) {
    for (int warps_per_smsp = 1; warps_per_smsp <= 8; warps_per_smsp *= 2) {
        int threads = 128 * warps_per_smsp > 1024 ? 1024 : 128 * warps_per_smsp;
        int blocks_per_sm = (128 * warps_per_smsp) / threads;
        int grid = sms * blocks_per_sm;
        cudaEvent_t e0, e1;
        cudaEventCreate(&e0); cudaEventCreate(&e1);
        k<MODE><<<grid, threads>>>(d, 1, 3);
        cudaDeviceSynchronize();
        cudaEventRecord(e0);
        k<MODE><<<grid, threads>>>(d, 1, 3);
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        float ms = 0;
        cudaEventElapsedTime(&ms, e0, e1);
        double warp_instr = (double)grid * (threads / 32) * ITERS * ops_per_iter;
        double per_clk_sm = warp_instr / (ms * 1e-3) / sms / (khz * 1e3);
        printf("%-28s warps/SMSP=%d  %.3f ms  %.2f warp-instr/clk/SM (at max clock %d MHz) = %.1f thread-ops/clk/SM\n", name,
               warps_per_smsp, ms, per_clk_sm, khz / 1000, per_clk_sm * 32);
    }
}

int main() {
    cudaDeviceProp p;
    cudaGetDeviceProperties(&p, 0);
    int khz = 0;
    cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
    printf("device %s  SMs %d  clock %d kHz\n", p.name, p.multiProcessorCount, khz);
    u32* d;
    cudaMalloc(&d, 1 << 24);
    int sms = p.multiProcessorCount;
    run<0>("IMAD (mad.lo)", NACC, sms, khz, d);
    run<1>("IMAD.WIDE (lo.cc+hi)", NACC, sms, khz, d);
    run<2>("IMAD.WIDE.X (cc chain)", 8, sms, khz, d);
    run<3>("IADD3 (2 adds fused?)", NACC, sms, khz, d);
    run<4>("IMAD.WIDE + IADD3 1:1", NACC * 2, sms, khz, d);
    run<5>("IMAD lo + IMAD.HI pairs", NACC * 2, sms, khz, d);
    return 0;
}
