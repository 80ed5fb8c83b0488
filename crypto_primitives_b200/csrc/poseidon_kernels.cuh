// poseidon_kernels.cuh -- Poseidon kernel templates, the context struct and the launch wrappers.
// Included by cpb_poseidon.cu (C-ABI, dispatch) and by the per-field instantiation units
// poseidon_inst_*.cu and poseidon_ragged_*.cu, which exist only so that nvcc can compile the (field, width) grid in parallel.
#pragma once
#include <mutex>

#include "common.cuh"
#include "poseidon.cuh"
#include "poseidon_host.hpp"
#include "poseidon_team.cuh"

namespace cpb {

constexpr int kBlock = 128;
// resident CTAs per SM the register allocator must allow: 5 for the narrow states (96 registers), 1 for wide ones
#ifndef CPB_POS_MINB3
#define CPB_POS_MINB3 5
#endif
constexpr int pos_min_blocks(int t) { return t <= 3 ? CPB_POS_MINB3 : t <= 5 ? 3 : 1; }

// SINGLE: len <= rate, 1 <= n_out <= rate, capacity >= 1 (checked by launch_crh_ft): one permutation per hash, pos_hash_single.
// A5 (SINGLE only): alpha == 5 compiled in (pos_permute_split); launch_crh_ft picks it where pos_alpha5_kernel says it exists.
template <class F, int T, bool SINGLE, bool A5 = false>
__global__ void __launch_bounds__(kBlock, pos_min_blocks(T))
k_poseidon_crh(PoseidonDev P, const u32* __restrict__ consts, const u32* __restrict__ in, u32* __restrict__ out,
               long n, long len, long n_out) {
    extern __shared__ __align__(16) u32 cs[];
    __shared__ __align__(8) unsigned long long mbar;
    tma_stage_to_smem(cs, consts, (unsigned)P.n_elems * 32u, &mbar);
    const u32* ct = cs + (int)threadIdx.x * P.zero;   // == cs, but not provably warp-uniform
    u32 pm[8];
    ld_elem(pm, ct + 8 * P.off_mod);
    const long stride = (long)gridDim.x * blockDim.x;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        if constexpr (SINGLE) pos_hash_single<F, T, A5>(out + 8 * n_out * i, (int)n_out, in + 8 * len * i, (int)len, P, ct, pm);
        else pos_sponge<F, T>(out + 8 * n_out * i, n_out, in + 8 * len * i, len, P, ct, pm);
    }
}

// The (field, width) pairs with an alpha = 5 one-permutation kernel: BN254 Fr at t = 3, the configuration of the Merkle benchmark
// (2-element leaves and two-to-one nodes, alpha = 5).  Every other pair, and any other exponent, runs the generic kernel.
template <class F, int T> constexpr bool pos_alpha5_kernel() { return F::ID == Bn254_Fr::ID && T == 3; }

template <class F, int T>
__global__ void __launch_bounds__(kBlock, pos_min_blocks(T))
k_poseidon_permute(PoseidonDev P, const u32* __restrict__ consts, const u32* __restrict__ in, u32* __restrict__ out,
                   long n) {
    extern __shared__ __align__(16) u32 cs[];
    __shared__ __align__(8) unsigned long long mbar;
    tma_stage_to_smem(cs, consts, (unsigned)P.n_elems * 32u, &mbar);
    const u32* ct = cs + (int)threadIdx.x * P.zero;
    u32 pm[8];
    ld_elem(pm, ct + 8 * P.off_mod);
    const long stride = (long)gridDim.x * blockDim.x;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        u32 s[T][8];
#pragma unroll
        for (int j = 0; j < T; j++) ld_elem(s[j], in + 8 * (T * i + j));
        pos_permute<F, T>(s, P, ct, pm);
#pragma unroll
        for (int j = 0; j < T; j++) st_elem(out + 8 * (T * i + j), s[j]);
    }
}

}  // namespace cpb

struct cpb_poseidon_ctx {
    typedef cpb::u32 u32;
    int field_id = 0, device = 0, sms = 132;
    cpb::host::PoseidonSchedule sched;
    cpb::PoseidonDev dev{};
    u32* d_consts = nullptr;
    cudaStream_t stream = nullptr;
    std::mutex mu;
    cpb::Scratch s_in, s_out, s_aux;
    std::mutex side_mu;                 // guards creation of side[] only (mu may already be held by a host-pointer call)
    cudaStream_t side[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};   // subtree streams of the Merkle build
};


namespace cpb {

// cudaFuncAttributeMaxDynamicSharedMemorySize and the occupancy are properties of (kernel, device): the cache key holds the
// current device, so one host thread driving contexts on several GPUs re-configures the kernel on each of them.
template <class K> cpb_status configure_kernel(K kernel, size_t smem, int block, int& occ_out) {
    static thread_local const void* last = nullptr;
    static thread_local int last_occ = 0, last_dev = -1;
    static thread_local size_t last_smem = 0;
    int dev = -1;
    CPB_CUDA(cudaGetDevice(&dev));
    if (last != (const void*)kernel || last_smem != smem || last_dev != dev) {
        if (smem > 48 * 1024) CPB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        int occ = 0;
        CPB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, block, smem));
        if (occ < 1) return fail(CPB_CUDA_ERROR, "kernel does not fit on an SM (smem=%zu)", smem);
        last = (const void*)kernel; last_occ = occ; last_smem = smem; last_dev = dev;
    }
    occ_out = last_occ;
    return CPB_OK;
}

template <class K> cpb_status grid_for(K kernel, size_t smem, int sms, long n, int& grid) {
    int last_occ = 0;
    CPB_TRY(configure_kernel(kernel, smem, kBlock, last_occ));
    // One CTA per 128 hashes (capped; the kernels grid-stride).  Short-lived CTAs instead of one persistent
    // wave let the block scheduler interleave kernels from different streams: the latency-bound top
    // levels of one Merkle subtree then overlap with the bulk hashing of the next (merkle build).
    long need = (n + kBlock - 1) / kBlock;
    long cap = (long)sms * last_occ * 64;
    grid = (int)(need < cap ? need : cap);
    if (grid < 1) grid = 1;
    return CPB_OK;
}

template <class F, int T>
cpb_status launch_crh_ft(cpb_poseidon_ctx* c, const u32* in, size_t len, u32* out, size_t n_out, size_t n, cudaStream_t st) {
    size_t smem = (size_t)c->dev.n_elems * 32;
    int grid = 1;
    const bool single = len <= (size_t)c->dev.rate && n_out >= 1 && n_out <= (size_t)c->dev.rate && c->dev.cap >= 1;
    if constexpr (pos_alpha5_kernel<F, T>()) {
        if (single && c->dev.alpha == 5) {
            CPB_TRY(grid_for(k_poseidon_crh<F, T, true, true>, smem, c->sms, (long)n, grid));
            k_poseidon_crh<F, T, true, true><<<grid, kBlock, smem, st>>>(c->dev, c->d_consts, in, out, (long)n, (long)len, (long)n_out);
            CPB_CUDA(cudaGetLastError());
            return CPB_OK;
        }
    }
    if (single) {
        CPB_TRY(grid_for(k_poseidon_crh<F, T, true>, smem, c->sms, (long)n, grid));
        k_poseidon_crh<F, T, true><<<grid, kBlock, smem, st>>>(c->dev, c->d_consts, in, out, (long)n, (long)len, (long)n_out);
    } else {
        CPB_TRY(grid_for(k_poseidon_crh<F, T, false>, smem, c->sms, (long)n, grid));
        k_poseidon_crh<F, T, false><<<grid, kBlock, smem, st>>>(c->dev, c->d_consts, in, out, (long)n, (long)len, (long)n_out);
    }
    CPB_CUDA(cudaGetLastError());
    return CPB_OK;
}
template <class F, int T>
cpb_status launch_permute_ft(cpb_poseidon_ctx* c, const u32* in, u32* out, size_t n, cudaStream_t st) {
    size_t smem = (size_t)c->dev.n_elems * 32;
    int grid = 1;
    CPB_TRY(grid_for(k_poseidon_permute<F, T>, smem, c->sms, (long)n, grid));
    k_poseidon_permute<F, T><<<grid, kBlock, smem, st>>>(c->dev, c->d_consts, in, out, (long)n);
    CPB_CUDA(cudaGetLastError());
    return CPB_OK;
}


// One Path::verify per thread; both round schedules staged in shared memory.
template <class F, int T>
__global__ void __launch_bounds__(kBlock, pos_min_blocks(T))
k_poseidon_verify_paths(PoseidonDev PL, const u32* __restrict__ consts_l, PoseidonDev PN, const u32* __restrict__ consts_n,
                        const u32* __restrict__ root, const u32* __restrict__ leaves, long leaf_len,
                        const u32* __restrict__ siblings, const u32* __restrict__ paths, int plen,
                        const unsigned long long* __restrict__ indexes, unsigned char* __restrict__ ok, long n) {
    extern __shared__ __align__(16) u32 cs[];
    __shared__ __align__(8) unsigned long long mbar[2];
    u32* csn = cs + 8 * PL.n_elems;
    tma_stage_to_smem(cs, consts_l, (unsigned)PL.n_elems * 32u, &mbar[0]);
    tma_stage_to_smem(csn, consts_n, (unsigned)PN.n_elems * 32u, &mbar[1]);
    const int z = (int)threadIdx.x * PL.zero;
    u32 pm[8];
    ld_elem(pm, cs + z + 8 * PL.off_mod);
    const long stride = (long)gridDim.x * blockDim.x;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
        ok[i] = pos_verify_path<F, T>(leaves + 8 * leaf_len * i, leaf_len, siblings + 8 * i, paths + 8 * (long)plen * i, plen, indexes[i],
                                      root, PL, cs + z, PN, csn + z, pm) ? 1 : 0;
}

template <class F, int T>
cpb_status launch_verify_ft(cpb_poseidon_ctx* leaf, cpb_poseidon_ctx* node, const u32* root, const u32* leaves, size_t leaf_len,
                            const u32* siblings, const u32* paths, int plen, const unsigned long long* indexes,
                            unsigned char* ok, size_t n, cudaStream_t st) {
    size_t smem = ((size_t)leaf->dev.n_elems + node->dev.n_elems) * 32;
    if (smem > 200 * 1024) return fail(CPB_UNSUPPORTED, "round schedules (%zu B) exceed shared memory", smem);
    int grid = 1;
    CPB_TRY(grid_for(k_poseidon_verify_paths<F, T>, smem, leaf->sms, (long)n, grid));
    k_poseidon_verify_paths<F, T><<<grid, kBlock, smem, st>>>(leaf->dev, leaf->d_consts, node->dev, node->d_consts, root, leaves,
                                                              (long)leaf_len, siblings, paths, plen, indexes, ok, (long)n);
    CPB_CUDA(cudaGetLastError());
    return CPB_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Ragged batches (poseidon.cuh: ragged_span): item i hashes values[offsets[i] - vbase ..] at its own length and writes out[i].
// Slot j of [range[0], range[1]) is item order[j]; order == nullptr walks the items in input order and range == nullptr is
// [0, n).  The range lives in device memory (written by the ordering kernels), so the grid covers n slots and a CTA wholly past
// the end of its range exits before staging.  One item per thread, no grid-stride loop: nothing but the item's own pointers stays
// live across the hash, which keeps the t = 3 kernels at the uniform kernels' 96 registers.
// SINGLE: every item of the range is one permutation (len <= rate, n_out <= rate, capacity >= 1): pos_hash_single.
// ---------------------------------------------------------------------------------------------------------------
template <class F, int T, bool SINGLE>
__global__ void __launch_bounds__(kBlock, pos_min_blocks(T))
k_poseidon_crh_ragged(PoseidonDev P, const u32* __restrict__ consts, const u32* __restrict__ values, u64 vbase,
                      const u64* __restrict__ offsets, const unsigned* __restrict__ order, const unsigned* __restrict__ range,
                      u32* __restrict__ out, long n, long n_out) {
    extern __shared__ __align__(16) u32 cs[];
    __shared__ __align__(8) unsigned long long mbar;
    const long begin = range ? (long)range[0] : 0, end = range ? (long)range[1] : n;
    if (begin + (long)blockIdx.x * blockDim.x >= end) return;
    tma_stage_to_smem(cs, consts, (unsigned)P.n_elems * 32u, &mbar);
    const long j = begin + (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= end) return;
    const u32* ct = cs + (int)threadIdx.x * P.zero;
    u32 pm[8];
    ld_elem(pm, ct + 8 * P.off_mod);
    const long i = order ? (long)order[j] : j;
    const RaggedSpan sp = ragged_span(offsets, i, n);
    const u32* in = values + 8 * (sp.lo - vbase);
    if constexpr (SINGLE) pos_hash_single<F, T>(out + 8 * n_out * i, (int)n_out, in, (int)sp.len, P, ct, pm);
    else pos_sponge<F, T>(out + 8 * n_out * i, n_out, in, sp.len, P, ct, pm);
}

template <class K> cpb_status grid_ragged(K kernel, size_t smem, size_t n, int& grid) {
    int occ = 0;
    CPB_TRY(configure_kernel(kernel, smem, kBlock, occ));
    grid = (int)((n + kBlock - 1) / kBlock);          // n < 2^32 (checked by the caller)
    return CPB_OK;
}

// The two hash launches over the ordered items (or one sponge launch in input order when order == nullptr; range_* then unused).
template <class F, int T>
cpb_status launch_crh_ragged_ft(cpb_poseidon_ctx* c, const u32* values, u64 vbase, const u64* offsets, const unsigned* order,
                                const unsigned* ranges, u32* out, size_t n_out, size_t n, bool single, cudaStream_t st) {
    size_t smem = (size_t)c->dev.n_elems * 32;
    int grid = 1;
    if (order && single) {
        CPB_TRY(grid_ragged(k_poseidon_crh_ragged<F, T, true>, smem, n, grid));
        k_poseidon_crh_ragged<F, T, true><<<grid, kBlock, smem, st>>>(c->dev, c->d_consts, values, vbase, offsets, order, ranges, out,
                                                                      (long)n, (long)n_out);
        CPB_CUDA(cudaGetLastError());
    }
    CPB_TRY(grid_ragged(k_poseidon_crh_ragged<F, T, false>, smem, n, grid));
    k_poseidon_crh_ragged<F, T, false><<<grid, kBlock, smem, st>>>(c->dev, c->d_consts, values, vbase, offsets, order,
                                                                   order ? ranges + 2 : nullptr, out, (long)n, (long)n_out);
    CPB_CUDA(cudaGetLastError());
    return CPB_OK;
}

// Path::verify with each leaf at its own length; no ordering: a path's cost is dominated by its plen + 1 compressions.
template <class F, int T>
__global__ void __launch_bounds__(kBlock, pos_min_blocks(T))
k_poseidon_verify_paths_ragged(PoseidonDev PL, const u32* __restrict__ consts_l, PoseidonDev PN, const u32* __restrict__ consts_n,
                               const u32* __restrict__ root, const u32* __restrict__ values, u64 vbase, const u64* __restrict__ offsets,
                               const u32* __restrict__ siblings, const u32* __restrict__ paths, int plen,
                               const unsigned long long* __restrict__ indexes, unsigned char* __restrict__ ok, long n) {
    extern __shared__ __align__(16) u32 cs[];
    __shared__ __align__(8) unsigned long long mbar[2];
    u32* csn = cs + 8 * PL.n_elems;
    tma_stage_to_smem(cs, consts_l, (unsigned)PL.n_elems * 32u, &mbar[0]);
    tma_stage_to_smem(csn, consts_n, (unsigned)PN.n_elems * 32u, &mbar[1]);
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int z = (int)threadIdx.x * PL.zero;
    u32 pm[8];
    ld_elem(pm, cs + z + 8 * PL.off_mod);
    const RaggedSpan sp = ragged_span(offsets, i, n);
    ok[i] = pos_verify_path<F, T>(values + 8 * (sp.lo - vbase), sp.len, siblings + 8 * i, paths + 8 * (long)plen * i, plen, indexes[i],
                                  root, PL, cs + z, PN, csn + z, pm) ? 1 : 0;
}

template <class F, int T>
cpb_status launch_verify_ragged_ft(cpb_poseidon_ctx* leaf, cpb_poseidon_ctx* node, const u32* root, const u32* values, u64 vbase,
                                   const u64* offsets, const u32* siblings, const u32* paths, int plen, const unsigned long long* indexes,
                                   unsigned char* ok, size_t n, cudaStream_t st) {
    size_t smem = ((size_t)leaf->dev.n_elems + node->dev.n_elems) * 32;
    if (smem > 200 * 1024) return fail(CPB_UNSUPPORTED, "round schedules (%zu B) exceed shared memory", smem);
    int grid = 1;
    CPB_TRY(grid_ragged(k_poseidon_verify_paths_ragged<F, T>, smem, n, grid));
    k_poseidon_verify_paths_ragged<F, T><<<grid, kBlock, smem, st>>>(leaf->dev, leaf->d_consts, node->dev, node->d_consts, root, values,
                                                                     vbase, offsets, siblings, paths, plen, indexes, ok, (long)n);
    CPB_CUDA(cudaGetLastError());
    return CPB_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Tree-top kernel: ALL the small levels of a Merkle (sub)tree in one launch, four warps per 32 hashes
// (poseidon_team.cuh), and -- on a multi-GPU build -- the exchange of the subtree roots over NVLink peer memory and
// the replicated top levels in the same kernel.  t = 3, capacity 1 (poseidon::TwoToOneCRH) only.
//
// Level l of the job has cnt(l) hashes, 32 per CTA; CTA b needs the 64 children produced by CTAs 2b and 2b+1 of the
// level below, so levels are chained with per-CTA progress words (release store after the CTA's outputs, acquire spin by
// the consumer) instead of a grid-wide barrier: a CTA starts level l as soon as ITS inputs exist.  Children are read
// with ld.global.cg (L2): they were written by other SMs during this launch.  A CTA with no hashes left at a level has
// none at any later level and exits.  All CTAs of the grid (<= 128) must be resident for the spins to end; they are
// 128-thread CTAs with ≤ 29 KB of shared memory at t = 3 on a 132-SM H100, and every spin is bounded (trap after ~4 s).
// ---------------------------------------------------------------------------------------------------------------
constexpr int kMaxPeers = 16;
struct ExchangeDev {
    int world = 1, rank = 0;
    unsigned long long epoch = 0;                 // this call's number (> 0); slot parity = epoch & 1
    u32* slots[kMaxPeers] = {};                   // slots[p]: peer p's digest buffer  [2 parities][world] x 8 words
    unsigned long long* flags[kMaxPeers] = {};    // flags[p]: peer p's flag buffer    [2 parities][world]
    u32* top_out = nullptr;                       // (world - 1) x 8 words, heap order: the replicated top levels; root at 0
};
struct TopJob {
    const u32* leaf_digests = nullptr;   // children of level h-1
    u32* nodes = nullptr;                // heap-ordered inner nodes of the (local) tree
    int h = 0, lgS = 0;                  // log2(#leaf digests of the local tree); subtree k of 2^lgS
    long k = 0;
    int l_start = 0, l_end = 0;          // levels computed: l_start, l_start-1, ..., l_end
    const u32* flat_in = nullptr;        // flat mode (l_start == l_end == 0, one level): n_flat pairs -> n_flat digests
    u32* flat_out = nullptr;
    long n_flat = 0;
    unsigned* prog = nullptr;            // [gridDim.x] progress words, zero at launch
    ExchangeDev x;
};

__device__ __forceinline__ void ld_elem_cg(u32* r, const u32* p) {
    uint4 a = __ldcg(reinterpret_cast<const uint4*>(p));
    uint4 b = __ldcg(reinterpret_cast<const uint4*>(p + 4));
    r[0] = a.x; r[1] = a.y; r[2] = a.z; r[3] = a.w;
    r[4] = b.x; r[5] = b.y; r[6] = b.z; r[7] = b.w;
}
__device__ __forceinline__ unsigned ld_acquire_gpu(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_gpu(unsigned* p, unsigned v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}

// Leading-bit indexes of alpha and alpha - 1, the exponents of team_phase1.
__device__ __forceinline__ void team_top_bits(const PoseidonDev& P, int& tb_alpha, int& tb_e) {
    tb_alpha = 0;
    tb_e = 0;
    for (int i = 63; i > 0; i--)
        if ((P.alpha >> i) & 1) { tb_alpha = i; break; }
    for (int i = 63; i > 0; i--)
        if (((P.alpha - 1) >> i) & 1) { tb_e = i; break; }
}

// The permutation of 32 two-to-one states by the 128 threads of the CTA: thread (w, lane) enters with lane w of its state in s
// (zero for w = 0 and w = 3) and, for w = 1, leaves with the digest in s.
template <class F>
__device__ __forceinline__ void team_permute32(u32* s, int w, int lane, const PoseidonDev& P, const u32* ct, const u32* pm, u32* xb,
                                               int tb_alpha, int tb_e) {
    u32 t[8];
    fp_zero(t);
    const int total = P.rf + P.rp;
#pragma unroll 1
    for (int r = 0; r < total; r++) {
        team_phase1<F>(s, t, w, lane, r, P, ct, pm, xb, tb_alpha, tb_e);
        __syncthreads();
        team_phase2<F>(s, t, w, lane, r, P, ct, pm, xb);
        team_publish<F>(s, w, lane, r, P, ct, xb);
        __syncthreads();
    }
}

// 32 two-to-one hashes by the 128 threads of the CTA: thread (w, lane) -- pair/out are THIS lane's pointers.
template <class F>
__device__ __forceinline__ void team_compress32(const u32* pair, u32* out, bool active, int w, int lane, const PoseidonDev& P,
                                                const u32* ct, const u32* pm, u32* xb, int tb_alpha, int tb_e) {
    u32 s[8];
    if (w == 1 || w == 2) ld_elem_cg(s, pair + 8 * (w - 1));
    else fp_zero(s);
    team_permute32<F>(s, w, lane, P, ct, pm, xb, tb_alpha, tb_e);
    if (w == 1 && active) st_elem(out, s);
}

template <class F>
__global__ void __launch_bounds__(kTeamThreads)
k_poseidon_tree_top(PoseidonDev P, const u32* __restrict__ consts, TopJob J) {
    extern __shared__ __align__(16) u32 cs[];
    __shared__ __align__(8) unsigned long long mbar;
    __shared__ __align__(16) u32 rootbuf[8];
    tma_stage_to_smem(cs, consts, (unsigned)P.n_elems * 32u, &mbar);
    u32* xb = cs + 8 * P.n_elems;
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, b = blockIdx.x;
    const u32* ct = cs + (int)threadIdx.x * P.zero;
    u32 pm[8];
    ld_elem(pm, ct + 8 * P.off_mod);
    int tb_alpha, tb_e;
    team_top_bits(P, tb_alpha, tb_e);

    const bool flat = J.flat_in != nullptr;
    unsigned done = 0;
    for (int l = J.l_start; l >= J.l_end; l--, done++) {
        const long cnt = flat ? J.n_flat : ((1L << l) >> J.lgS);
        if ((long)b * 32 >= cnt) return;                    // no hashes here => none at any later level
        if (done > 0) {
            if (threadIdx.x == 0) {
                const long nblk_prev = (2 * cnt + 31) / 32;
                const unsigned long long t0 = globaltimer_ns();
                for (long q = 2L * b; q <= 2L * b + 1 && q < nblk_prev; q++)
                    while (ld_acquire_gpu(J.prog + q) < done)
                        if (globaltimer_ns() - t0 > 4000000000ull) __trap();
            }
            __syncthreads();
        }
        const long i = (long)b * 32 + lane;
        const bool active = i < cnt;
        const long ii = active ? i : cnt - 1;
        const u32 *in;
        u32* out;
        if (flat) {
            in = J.flat_in;
            out = J.flat_out;
        } else {
            in = (l == J.h - 1) ? J.leaf_digests + 8 * (2 * J.k * cnt) : J.nodes + 8 * (((2L << l) - 1) + 2 * J.k * cnt);
            out = J.nodes + 8 * (((1L << l) - 1) + J.k * cnt);
        }
        team_compress32<F>(in + 16 * ii, out + 8 * ii, active, w, lane, P, ct, pm, xb, tb_alpha, tb_e);
        __syncthreads();                                    // every output store of the CTA has been issued
        if (threadIdx.x == 0) {
            __threadfence();
            st_release_gpu(J.prog + b, done + 1);
        }
    }
    if (J.x.world <= 1 || b != 0) return;

    // ---- fused exchange: push this rank's root into every peer's slot over NVLink, wait for theirs, replicated top
    const ExchangeDev& X = J.x;
    const int par = (int)(X.epoch & 1ull);
    if (threadIdx.x < 8) rootbuf[threadIdx.x] = __ldcg(J.nodes + threadIdx.x);      // the local root: nodes[0]
    __syncthreads();
    if ((int)threadIdx.x < X.world) {
        const int p = threadIdx.x;
        u32* dst = X.slots[p] + 8 * (par * X.world + X.rank);
        asm volatile("st.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "r"(rootbuf[0]), "r"(rootbuf[1]), "r"(rootbuf[2]), "r"(rootbuf[3]) : "memory");
        asm volatile("st.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(dst + 4), "r"(rootbuf[4]), "r"(rootbuf[5]), "r"(rootbuf[6]), "r"(rootbuf[7]) : "memory");
        __threadfence_system();
        st_release_sys(X.flags[p] + (par * X.world + X.rank), X.epoch);
        const unsigned long long t0 = globaltimer_ns();
        while (ld_acquire_sys(X.flags[X.rank] + (par * X.world + p)) != X.epoch)
            if (globaltimer_ns() - t0 > 20000000000ull) __trap();
    }
    __syncthreads();
    int lgW = 0;
    while ((1 << lgW) < X.world) lgW++;
    const u32* gathered = X.slots[X.rank] + 8 * (par * X.world);
    for (int j = lgW - 1; j >= 0; j--) {
        const long cnt = 1L << j;
        const bool active = lane < cnt;
        const long ii = active ? lane : cnt - 1;
        const u32* in = (j == lgW - 1) ? gathered : X.top_out + 8 * ((2L << j) - 1);
        u32* out = X.top_out + 8 * ((1L << j) - 1);
        team_compress32<F>(in + 16 * ii, out + 8 * ii, active, w, lane, P, ct, pm, xb, tb_alpha, tb_e);
        __syncthreads();
        __threadfence_block();
    }
}

// Launch: `prog` is a stream-ordered, zeroed scratch of grid words.
template <class F>
cpb_status launch_tree_top_f(cpb_poseidon_ctx* c, TopJob J, cudaStream_t st) {
    size_t smem = (size_t)c->dev.n_elems * 32 + (size_t)kTeamXbWords * 4;
    int occ = 0;
    CPB_TRY(configure_kernel(k_poseidon_tree_top<F>, smem, kTeamThreads, occ));
    const long cnt0 = J.flat_in ? J.n_flat : ((1L << J.l_start) >> J.lgS);
    const long grid = (cnt0 + 31) / 32;
    if (grid < 1 || grid > 128) return fail(CPB_INTERNAL_ERROR, "tree-top grid %ld out of range", grid);
    unsigned* prog = nullptr;
    CPB_CUDA(cudaMallocAsync((void**)&prog, (size_t)grid * sizeof(unsigned), st));
    CPB_CUDA(cudaMemsetAsync(prog, 0, (size_t)grid * sizeof(unsigned), st));
    J.prog = prog;
    k_poseidon_tree_top<F><<<(int)grid, kTeamThreads, smem, st>>>(c->dev, c->d_consts, J);
    cudaError_t e = cudaGetLastError();
    cudaFreeAsync(prog, st);
    if (e != cudaSuccess) return fail(CPB_CUDA_ERROR, "tree-top launch failed: %s", cudaGetErrorString(e));
    return CPB_OK;
}

// ---- Merkle build internals shared by the C-ABI translation units (defined in cpb_poseidon.cu)
// Optional host mirrors (host-pointer entry points): when given, each subtree's stream also copies its slice of the
// leaves in before hashing and its slices of leaf_nodes / of every level out afterwards, so PCIe transfers of one
// subtree overlap the hashing of the others (copy engines + side streams).  The local tree may be shard `rank` of a
// tree 2^g times larger (multi-GPU build into the reference's full arrays): local level l is then the rank-th slice of
// global level l + g, and `nodes` points at the GLOBAL heap-ordered array.
struct MerkleHost {
    const u32* leaves = nullptr;   // this shard's n * leaf_len elements
    u32* leaf_nodes = nullptr;     // this shard's n digests
    u32* nodes = nullptr;          // heap-ordered inner nodes (of the global tree when g > 0)
    int g = 0;
    size_t rank = 0;
    u32* node_ptr(int local_level, size_t first) const {
        return nodes + 8 * ((((size_t)1 << (local_level + g)) - 1) + (rank << local_level) + first);
    }
};
cpb_status check_ctx(const cpb_poseidon_ctx* c);
bool pow2_gt1(size_t n);
size_t team_max();
size_t team_max_for(size_t S);
bool team_capable(const cpb_poseidon_ctx* c);
cpb_status launch_crh(cpb_poseidon_ctx* c, const u32* in, size_t len, u32* out, size_t n, cudaStream_t st, size_t n_out = 1);
cpb_status merkle_subtree_levels(cpb_poseidon_ctx* node, const u32* leaf_digests, size_t n, u32* nodes, size_t S, size_t k,
                                 cudaStream_t st, const MerkleHost* H = nullptr, const ExchangeDev* X = nullptr, int* small_from = nullptr);
cpb_status merkle_build_streams(cpb_poseidon_ctx* leaf, cpb_poseidon_ctx* node, const u32* leaves, size_t leaf_len, size_t n,
                                u32* leaf_nodes, u32* nodes, cudaStream_t st, const MerkleHost* H = nullptr,
                                const ExchangeDev* X = nullptr);

// explicit instantiations live in poseidon_inst_<field>.cu
#define CPB_POS_WIDTHS(M, F) M(F, 2) M(F, 3) M(F, 4) M(F, 5) M(F, 6) M(F, 7) M(F, 8) M(F, 9)
#define CPB_POS_INSTANTIATE(F, T)                                                                                        \
    template cpb_status launch_crh_ft<F, T>(cpb_poseidon_ctx*, const u32*, size_t, u32*, size_t, size_t, cudaStream_t);            \
    template cpb_status launch_permute_ft<F, T>(cpb_poseidon_ctx*, const u32*, u32*, size_t, cudaStream_t);             \
    template cpb_status launch_verify_ft<F, T>(cpb_poseidon_ctx*, cpb_poseidon_ctx*, const u32*, const u32*, size_t, const u32*, \
                                               const u32*, int, const unsigned long long*, unsigned char*, size_t, cudaStream_t);
// the ragged kernels live in translation units of their own (poseidon_ragged_<field>.cu), so adding them leaves the code of the
// uniform kernels exactly as it was
#define CPB_POS_INSTANTIATE_RAGGED(F, T)                                                                                 \
    template cpb_status launch_crh_ragged_ft<F, T>(cpb_poseidon_ctx*, const u32*, u64, const u64*, const unsigned*, const unsigned*, \
                                                   u32*, size_t, size_t, bool, cudaStream_t);                            \
    template cpb_status launch_verify_ragged_ft<F, T>(cpb_poseidon_ctx*, cpb_poseidon_ctx*, const u32*, const u32*, u64, const u64*, \
                                                      const u32*, const u32*, int, const unsigned long long*, unsigned char*, size_t, \
                                                      cudaStream_t);
#define CPB_POS_INSTANTIATE_TEAM(F) template cpb_status launch_tree_top_f<F>(cpb_poseidon_ctx*, TopJob, cudaStream_t);
#define CPB_POS_EXTERN_TEAM(F) extern template cpb_status launch_tree_top_f<F>(cpb_poseidon_ctx*, TopJob, cudaStream_t);
#define CPB_POS_EXTERN(F, T)                                                                                             \
    extern template cpb_status launch_crh_ft<F, T>(cpb_poseidon_ctx*, const u32*, size_t, u32*, size_t, size_t, cudaStream_t);     \
    extern template cpb_status launch_permute_ft<F, T>(cpb_poseidon_ctx*, const u32*, u32*, size_t, cudaStream_t);      \
    extern template cpb_status launch_verify_ft<F, T>(cpb_poseidon_ctx*, cpb_poseidon_ctx*, const u32*, const u32*, size_t, const u32*, \
                                                      const u32*, int, const unsigned long long*, unsigned char*, size_t, cudaStream_t);
#define CPB_POS_EXTERN_RAGGED(F, T)                                                                                      \
    extern template cpb_status launch_crh_ragged_ft<F, T>(cpb_poseidon_ctx*, const u32*, u64, const u64*, const unsigned*,       \
                                                          const unsigned*, u32*, size_t, size_t, bool, cudaStream_t);           \
    extern template cpb_status launch_verify_ragged_ft<F, T>(cpb_poseidon_ctx*, cpb_poseidon_ctx*, const u32*, const u32*, u64,  \
                                                             const u64*, const u32*, const u32*, int, const unsigned long long*, \
                                                             unsigned char*, size_t, cudaStream_t);

}  // namespace cpb
