// ubench_modmul.cu -- 256-bit Montgomery multiplication throughput on an H100: the IMAD.WIDE path of csrc/fp.cuh against
// the FP64-pipe path of tools/fp52.cuh, same dependent chain per thread (x <- x*y, x <- x^2 alternating), and a
// bit-for-bit check of the GPU results against the host build of the very same functions (exact emulation).
// BN254 Fr also runs a third arm at the shape of k_poseidon_crh_tc (128-thread CTAs, 5 CTAs/SM, converged warps): the
// 512-bit product on the integer pipe (fp_sqr_wide, fp_mul_wide) and its Montgomery reduction on the tensor cores (tc_redc,
// the 1 KB R^-1 table in shared memory), against the lazy IMAD products at the same shape, for squarings and multiplications
// separately; its canonical results are checked against the IMAD arm's.  A fourth arm runs the same reduction as warpgroup MMAs
// (redc_wg below: wgmma.m64n32k32 with the R^-1 table read from shared memory through a matrix descriptor), checked the same way.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xptxas -v -o ubench_modmul ubench_modmul.cu
#include <algorithm>
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

// The wgmma arm.  B (32 k x 32 columns, the R^-1 table) as one 1 KB block, K-major without swizzle (PTX ISA, "Shared Memory Matrix
// Layout"): core matrices of 8 columns x 16 k bytes, 128 contiguous bytes each; core matrix (n >> 3, k >> 4) at 256 (n >> 3) +
// 128 (k >> 4), so the descriptor's leading byte offset (next 16 k) is 128 and its stride byte offset (next 8 columns) 256.
constexpr int kWgLbo = 128, kWgSbo = 256;
CPB_HD int wg_byte(int k, int n) { return (n >> 3) * kWgSbo + (k >> 4) * kWgLbo + (n & 7) * 16 + (k & 15); }
// tc_rinv_table (tc_tab_word's layout, one constant) rearranged into wg_byte's: the same bytes, permuted.
std::vector<u32> wg_image(const std::vector<u32>& tab) {
    std::vector<u32> out(tab.size(), 0u);
    unsigned char* o = reinterpret_cast<unsigned char*>(out.data());
    for (int nt = 0; nt < 4; nt++)
        for (int lane = 0; lane < 32; lane++)
            for (int r = 0; r < 2; r++)
                for (int q = 0; q < 4; q++)
                    o[wg_byte(tc_b_k(lane, r, q), 8 * nt + tc_b_col(lane))] = (unsigned char)(tab[tc_tab_word(nt, 0, lane, r, 1)] >> (8 * q));
    return out;
}
#if defined(__CUDA_ARCH__)
// d = A . B over the warpgroup's 64 x 32 tile: A in registers (this warp's 16 rows: the m16n8k32 A fragment), B through the
// descriptor of the block at smem (scale-d = 0).  D: register r holds row g + 8 ((r >> 1) & 1), column 8 (r >> 2) + 2t + (r & 1),
// i.e. the mma.m16n8k32 C fragment of n-tile r >> 2 in registers 4 (r >> 2) .. +3.
__device__ void wgmma_u8(u32 (&d)[16], const u32 (&a)[4], const u32* smem) {
    const unsigned lo = (((unsigned)__cvta_generic_to_shared(smem) & 0x3FFFFu) >> 4) | (unsigned)(kWgLbo >> 4) << 16;
    asm volatile("{\n\t.reg .b64 bd;\n\tmov.b64 bd, {%20, %21};\n\twgmma.fence.sync.aligned;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n32k32.s32.u8.u8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, "
                 "%15}, {%16, %17, %18, %19}, bd, 0;\n\twgmma.commit_group.sync.aligned;\n\twgmma.wait_group.sync.aligned 0;\n\t}"
                 : "=r"(d[0]), "=r"(d[1]), "=r"(d[2]), "=r"(d[3]), "=r"(d[4]), "=r"(d[5]), "=r"(d[6]), "=r"(d[7]), "=r"(d[8]),
                   "=r"(d[9]), "=r"(d[10]), "=r"(d[11]), "=r"(d[12]), "=r"(d[13]), "=r"(d[14]), "=r"(d[15])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(lo), "r"((unsigned)(kWgSbo >> 4))
                 : "memory");
}
// tc_redc with the product as warpgroup MMAs (every thread of the CTA calls it together): T_lo staged as tc_redc stages it, one
// wgmma per m-half of the warp's 32 rows, then tc_redc's packing, C buffer and tc_finish, so the result is bit-identical.  T_hi
// waits in the lane's stage row beside T_lo, which keeps the hash kernel at 96 registers without spills.
__device__ void redc_wg(u32* r, const u32 (&T)[16], const u32* rinv, u32* buf, const u32* pm) {
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    u32* row = buf + lane * kTcStageStride;
    u32* cbuf = buf + 32 * kTcStageStride;
    *reinterpret_cast<uint4*>(row) = make_uint4(T[0], T[1], T[2], T[3]);
    *reinterpret_cast<uint4*>(row + 4) = make_uint4(T[4], T[5], T[6], T[7]);
    *reinterpret_cast<uint4*>(row + 8) = make_uint4(T[8], T[9], T[10], T[11]);
    *reinterpret_cast<uint4*>(row + 12) = make_uint4(T[12], T[13], T[14], T[15]);
    __syncwarp();
    for (int mt = 0; mt < 2; mt++) {
        u32 a[4], d[16];
        tc_ldsm_x4(a, buf + (16 * mt + tc_ldsm_row(lane)) * kTcStageStride + 4 * tc_ldsm_half(lane));
        wgmma_u8(d, a, rinv);
        for (int u = 0; u < 2; u++) {
            const int rw = 16 * mt + 8 * u + g;
            u32 pk[4];
            for (int nt = 0; nt < 4; nt++) pk[nt] = d[4 * nt + 2 * u] + (d[4 * nt + 2 * u + 1] << 8);
            *reinterpret_cast<uint4*>(cbuf + 16 * rw + 4 * tc_cbuf_chunk(rw, t)) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
        }
    }
    __syncwarp();
    u32 h[16];
    for (int tt = 0; tt < 4; tt++) {
        const uint4 v = *reinterpret_cast<const uint4*>(cbuf + 16 * lane + 4 * tc_cbuf_chunk(lane, tt));
        h[tt] = v.x; h[4 + tt] = v.y; h[8 + tt] = v.z; h[12 + tt] = v.w;
    }
    __syncwarp();
    tc_finish<Bn254_Fr, true>(r, h, row + 8, pm);
}
#endif

// The tensor-core arms and their IMAD reference at the hash kernel's shape.  OP 0: x <- x^2 and x <- x*y alternating, 1: squarings
// only, 2: multiplications only.  ARM 0: the LAZY IMAD products, 1: tc_redc on mma.sync, 2: redc_wg (rinv_g in wg_byte's
// layout).  Operands stay below 2p (< 1.4p), so one conditional subtraction makes the result canonical.
// The arms use the four warps' buffers and the R^-1 table; every launch asks for kTcShapeSmem, so that exactly 5 CTAs fit on an
// SM (as the hash kernel's 96 registers allow) whatever the arm's register count.
constexpr int kTcShapeSmem = 40 * 1024;
static_assert(4 * kTcWarpWords * 4 + kTcRinvWords * 4 <= kTcShapeSmem, "the arms' shared memory");
template <int OP, int ARM> __global__ void __launch_bounds__(128, 5) k_chain_shape(const u32* in, const u32* rinv_g, u32* out, int n) {
    extern __shared__ __align__(16) u32 sm[];
    u32* rinv = sm + 4 * kTcWarpWords;
    for (int j = threadIdx.x; j < kTcRinvWords; j += blockDim.x) rinv[j] = rinv_g[j];
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");    // the table's stores, before the tensor cores' async reads
    __syncthreads();
    u32* buf = sm + (threadIdx.x >> 5) * kTcWarpWords;
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;      // the grid covers the batch exactly: warps stay converged
    u32 x[8], y[8], pm[8];
    fp_modulus<Bn254_Fr>(pm);
    for (int j = 0; j < 8; j++) { x[j] = in[16 * i + j]; y[j] = in[16 * i + 8 + j]; }
    for (int k = 0; k < n; k++) {
        const bool sqr = OP == 1 || (OP == 0 && (k & 1));
        if constexpr (ARM > 0) {
#if defined(__CUDA_ARCH__)
            u32 T[16];
            if (sqr) fp_sqr_wide(T, x);
            else fp_mul_wide(T, x, y);
            if (ARM == 2) redc_wg(x, T, rinv, buf, pm);
            else tc_redc<Bn254_Fr>(x, T, rinv, buf, pm);
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

template <int OP, int ARM> float time_shape(const u32* din, const u32* drinv, u32* dout, int n, long total) {
    cudaFuncSetAttribute(k_chain_shape<OP, ARM>, cudaFuncAttributeMaxDynamicSharedMemorySize, kTcShapeSmem);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    float ms[6];
    for (int rep = 0; rep < 6; rep++) {                     // the first launch warms up; the median of the other five is timed
        cudaEventRecord(e0);
        k_chain_shape<OP, ARM><<<(int)(total / 128), 128, kTcShapeSmem>>>(din, drinv, dout, n);
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        cudaEventElapsedTime(&ms[rep], e0, e1);
    }
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    std::sort(ms + 1, ms + 6);
    return ms[3];
}

void run_tc(int sms) {
    const int n = 1000;
    const long total = (long)sms * 128 * 5 * 4;              // 4 full waves of 5 CTAs per SM
    std::vector<u32> h(16 * total);
    u64 s = 6789;
    for (auto& v : h) { s = s * 6364136223846793005ull + 1442695040888963407ull; v = (u32)(s >> 33); }
    for (long i = 0; i < 2 * total; i++) h[8 * i + 7] &= 0x0fffffffu;   // < 2^252 < p
    const std::vector<u32> rinv = host::tc_rinv_table(host::Field(host::field_modulus(Bn254_Fr::ID)));
    const std::vector<u32> rinv_wg = wg_image(rinv);
    u32 *din, *drinv, *drinv_wg, *dout;
    cudaMalloc(&din, h.size() * 4);
    cudaMalloc(&drinv, rinv.size() * 4);
    cudaMalloc(&drinv_wg, rinv_wg.size() * 4);
    cudaMalloc(&dout, 8 * total * 4);
    cudaMemcpy(din, h.data(), h.size() * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(drinv, rinv.data(), rinv.size() * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(drinv_wg, rinv_wg.data(), rinv_wg.size() * 4, cudaMemcpyHostToDevice);
    const char* names[3] = {"sqr/mul alternating", "sqr only", "mul only"};
    for (int op = 0; op < 3; op++) {
        std::vector<u32> g[3];
        float ms[3];
        for (int arm = 0; arm < 3; arm++) {
            const u32* tab = arm == 2 ? drinv_wg : drinv;
            cudaMemset(dout, 0, 8 * total * 4);                  // no arm's results can pass for another's
            if (op == 0) ms[arm] = arm == 0 ? time_shape<0, 0>(din, tab, dout, n, total) : arm == 1 ? time_shape<0, 1>(din, tab, dout, n, total) : time_shape<0, 2>(din, tab, dout, n, total);
            if (op == 1) ms[arm] = arm == 0 ? time_shape<1, 0>(din, tab, dout, n, total) : arm == 1 ? time_shape<1, 1>(din, tab, dout, n, total) : time_shape<1, 2>(din, tab, dout, n, total);
            if (op == 2) ms[arm] = arm == 0 ? time_shape<2, 0>(din, tab, dout, n, total) : arm == 1 ? time_shape<2, 1>(din, tab, dout, n, total) : time_shape<2, 2>(din, tab, dout, n, total);
            g[arm].resize(8 * total);
            cudaMemcpy(g[arm].data(), dout, 8 * total * 4, cudaMemcpyDeviceToHost);
        }
        cudaError_t err = cudaGetLastError();
        if (err != cudaSuccess) printf("CUDA error: %s\n", cudaGetErrorString(err));
        long bad = 0, bad_wg = 0;
        for (long j = 0; j < 8 * total; j++) { bad += g[0][j] != g[1][j]; bad_wg += g[0][j] != g[2][j]; }
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
               "IMAD + wgmma reduction %8.3f ms %6.3f ns/product/SM | wgmma/TC %.3f | mismatches: TC vs IMAD %ld, wgmma vs IMAD %ld, "
               "IMAD vs host %ld\n",
               names[op], ms[0], ms[0] * 1e6 * sms / prod, ms[1], ms[1] * 1e6 * sms / prod, ms[1] / ms[0], ms[2],
               ms[2] * 1e6 * sms / prod, ms[2] / ms[1], bad, bad_wg, bad_host);
    }
    cudaFree(din); cudaFree(drinv); cudaFree(drinv_wg); cudaFree(dout);
}

int main() {
    cudaDeviceProp p;
    cudaGetDeviceProperties(&p, 0);
    printf("device %s, %d SMs; chain of 1000 dependent mul/sqr per thread, %d threads\n", p.name, p.multiProcessorCount, p.multiProcessorCount * 128 * 16);
    run<Bls12_381_Fr>("BLS12-381 Fr", p.multiProcessorCount);
    run<Bn254_Fr>("BN254 Fr", p.multiProcessorCount);
    int occ[3] = {0, 0, 0};
    cudaFuncSetAttribute(k_chain_shape<0, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, kTcShapeSmem);
    cudaFuncSetAttribute(k_chain_shape<0, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, kTcShapeSmem);
    cudaFuncSetAttribute(k_chain_shape<0, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, kTcShapeSmem);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ[0], k_chain_shape<0, 0>, 128, kTcShapeSmem);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ[1], k_chain_shape<0, 1>, 128, kTcShapeSmem);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ[2], k_chain_shape<0, 2>, 128, kTcShapeSmem);
    printf("hash-kernel shape: 128-thread CTAs, %d B shared memory, resident CTAs/SM: IMAD %d, TC %d, wgmma %d\n", kTcShapeSmem, occ[0],
           occ[1], occ[2]);
    run_tc(p.multiProcessorCount);
    return 0;
}
