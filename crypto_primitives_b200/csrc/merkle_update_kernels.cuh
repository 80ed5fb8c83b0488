// merkle_update_kernels.cuh -- the device side of the update plan (merkle_update.cuh) shared by the Poseidon-node update
// (cpb_merkle_update.cu, 8-word field digests) and the Pedersen-node update (cpb_merkle_update_pedersen.cu, 16-word affine points):
// the sort keys and run-tail flags, the compaction that builds U and places the leaf digests, the predicated commit, the element
// moves of the host forms, and the host-side steps around them.  W is the digest width in 32-bit words (a multiple of 8).
#pragma once
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cstring>
#include <mutex>
#include <vector>

#include "common.cuh"
#include "fp.cuh"
#include "merkle_update.cuh"

namespace cpb {
namespace {

constexpr int kUpdBlock = 256;

inline unsigned upd_grid(u64 items, int block) { return (unsigned)((items + block - 1) / block); }

template <int W> __device__ __forceinline__ void upd_ld(u32* e, const u32* p) {
#pragma unroll
    for (int i = 0; i < W; i += 8) ld_elem(e + i, p + i);
}
template <int W> __device__ __forceinline__ void upd_st(u32* p, const u32* e) {
#pragma unroll
    for (int i = 0; i < W; i += 8) st_elem(p + i, e + i);
}

__global__ void k_upd_keys(const u64* __restrict__ idx, u64 k, u64 n, u64* __restrict__ keys, unsigned* __restrict__ pos) {
    const u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= k) return;
    const u64 v = idx[j];
    keys[j] = v < n ? v : n;                                   // out of range: sorts last, dropped by k_upd_flags
    pos[j] = (unsigned)j;
}

// Keep the last occurrence of every in-range index.
__global__ void k_upd_flags(const u64* __restrict__ K, u64 k, u64 n, unsigned* __restrict__ flag) {
    const u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= k) return;
    flag[j] = K[j] < n && (j + 1 == k || K[j + 1] != K[j]) ? 1u : 0u;
}

// U[scan[j]] = K[j] for the kept j, the digest of input pos[j] into the leaf level of the scratch, m = the number kept.
template <int W>
__global__ void k_upd_compact(const u64* __restrict__ K, const unsigned* __restrict__ pos, const unsigned* __restrict__ flag,
                              const unsigned* __restrict__ scan, u64 k, int h, const u32* __restrict__ digests, u64* __restrict__ U,
                              u64* __restrict__ m, u32* __restrict__ leaf_scratch) {
    const u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= k) return;
    if (j + 1 == k) *m = (u64)scan[j] + flag[j];
    if (!flag[j]) return;
    const u64 i = scan[j];
    U[i] = K[j];
    u32 e[W];
    upd_ld<W>(e, digests + W * (u64)pos[j]);
    upd_st<W>(leaf_scratch + W * (upd_dense(h, k) ? K[j] : i), e);
}

// applied = (asserted == NULL or new root == asserted, all W words); when applied, every touched node's new value goes into the tree.
// X.m == NULL: nothing is touched (k == 0), the new root is the current one.
template <int W>
__global__ void k_upd_commit(UpdPlan X, const u32* __restrict__ scratch, u32* leaf_nodes, u32* nodes, const u32* __restrict__ asserted,
                             unsigned char* __restrict__ applied) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const u64 m = X.m ? *X.m : 0;
    bool ok = true;
    if (asserted) {
        const u32* r = m ? scratch + W * X.off[0] : nodes;
#pragma unroll
        for (int i = 0; i < W; i += 8) {
            u32 a[8], b[8];
            ld_elem(a, r + i);
            ld_elem(b, asserted + i);
            ok = ok && fp_eq(a, b);
        }
    }
    if (t == 0 && applied) *applied = ok ? 1 : 0;
    if (!ok || m == 0 || t >= X.off[X.h + 1]) return;
    const int l = upd_level_of(X.off, X.h, t);
    const UpdSite S = upd_site(X.U, m, X.h, l, X.k, t - X.off[l]);
    if (!S.touched) return;
    u32 e[W];
    upd_ld<W>(e, scratch + W * t);                             // slot t - off[l] of level l
    upd_st<W>(l == X.h ? leaf_nodes + W * S.node : nodes + W * (((1ull << l) - 1) + S.node), e);
}

// dst[pos[i]] = src[i] (scatter) or dst[i] = src[pos[i]] (gather), elements of W words.
template <int W>
__global__ void k_upd_move(const u32* __restrict__ src, u32* __restrict__ dst, const u64* __restrict__ pos, u64 cnt, int gather) {
    const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= cnt) return;
    u32 e[W];
    upd_ld<W>(e, src + W * (gather ? pos[i] : i));
    upd_st<W>(dst + W * (gather ? i : pos[i]), e);
}

inline int log2_exact(size_t n) {
    int h = 0;
    while (((size_t)1 << h) < n) h++;
    return h;
}

// Shape rules shared by every update entry point, checked before any context or pointer is used.
inline cpb_status check_update_shape(size_t n, size_t k) {
    if (n < 2 || (n & (n - 1))) return fail(CPB_NOT_POW2, "leaves.len() should be power of two and greater than one (got %zu)", n);
    if (k >= ((size_t)1 << 32)) return fail(CPB_BAD_LENGTH, "an update holds fewer than 2^32 leaves (got %zu)", k);
    return CPB_OK;
}

// One pool allocation per update call: the plan's arrays, `extra` bytes for the node hash, then the scratch of new values
// (off[h + 1] elements of W words).
struct UpdBuffers {
    size_t tmp_b = 0, o_kin = 0, o_kout = 0, o_pin = 0, o_pout = 0, o_flag = 0, o_scan = 0, o_U = 0, o_m = 0, o_tmp = 0, o_extra = 0,
           o_scr = 0, total = 0;
    char* b = nullptr;
    u32* scratch() const { return (u32*)(b + o_scr); }
    void* extra() const { return b + o_extra; }
};

// Plan offsets of an n-leaf tree and k updates (k > 0) into X; the buffer sizes into B.
inline cpb_status upd_layout(UpdPlan& X, size_t n, size_t k, size_t extra, int W, cudaStream_t st, UpdBuffers& B) {
    X.h = log2_exact(n);
    X.k = k;
    upd_offsets(X.h, k, X.off);
    const unsigned uk = (unsigned)k;
    size_t sort_b = 0, scan_b = 0;
    CPB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_b, (const u64*)nullptr, (u64*)nullptr, (const unsigned*)nullptr, (unsigned*)nullptr,
                                             uk, 0, X.h + 1, st));
    CPB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan_b, (const unsigned*)nullptr, (unsigned*)nullptr, uk, st));
    B.tmp_b = sort_b > scan_b ? sort_b : scan_b;
    size_t o = 0;
    B.o_kin = o; o += align256(8 * k);
    B.o_kout = o; o += align256(8 * k);
    B.o_pin = o; o += align256(4 * k);
    B.o_pout = o; o += align256(4 * k);
    B.o_flag = o; o += align256(4 * k);
    B.o_scan = o; o += align256(4 * k);
    B.o_U = o; o += align256(8 * k);
    B.o_m = o; o += 256;
    B.o_tmp = o; o += align256(B.tmp_b);
    B.o_extra = o; o += align256(extra);
    B.o_scr = o; o += 4 * (size_t)W * (size_t)X.off[X.h + 1];
    B.total = o;
    return CPB_OK;
}

// The plan on the device: sort (index, position) pairs, keep the last occurrence of each in-range index, build U and m and place
// the kept digests in the leaf level of the scratch.  Four launches plus the CUB sort and scan.
template <int W>
cpb_status upd_run_plan(const UpdBuffers& B, UpdPlan& X, const u64* idx, size_t n, const u32* digests, cudaStream_t st) {
    const u64 k = X.k;
    const unsigned uk = (unsigned)k;
    char* b = B.b;
    u64* kin = (u64*)(b + B.o_kin);
    u64* kout = (u64*)(b + B.o_kout);
    unsigned* pin = (unsigned*)(b + B.o_pin);
    unsigned* pout = (unsigned*)(b + B.o_pout);
    unsigned* flag = (unsigned*)(b + B.o_flag);
    unsigned* scan = (unsigned*)(b + B.o_scan);
    X.U = (const u64*)(b + B.o_U);
    X.m = (const u64*)(b + B.o_m);
    const unsigned g = upd_grid(k, kUpdBlock);
    k_upd_keys<<<g, kUpdBlock, 0, st>>>(idx, k, n, kin, pin);
    CPB_CUDA(cudaGetLastError());
    size_t tb = B.tmp_b;
    CPB_CUDA(cub::DeviceRadixSort::SortPairs(b + B.o_tmp, tb, (const u64*)kin, kout, (const unsigned*)pin, pout, uk, 0, X.h + 1, st));
    k_upd_flags<<<g, kUpdBlock, 0, st>>>(kout, k, n, flag);
    CPB_CUDA(cudaGetLastError());
    tb = B.tmp_b;
    CPB_CUDA(cub::DeviceScan::ExclusiveSum(b + B.o_tmp, tb, (const unsigned*)flag, scan, uk, st));
    k_upd_compact<W><<<g, kUpdBlock, 0, st>>>(kout, pout, flag, scan, k, X.h, digests, (u64*)(b + B.o_U), (u64*)(b + B.o_m),
                                              B.scratch() + W * X.off[X.h]);
    CPB_CUDA(cudaGetLastError());
    return CPB_OK;
}

// Host arrays (leaf_nodes: n elements, non_leaf_nodes: n - 1, W words each; arguments already checked, k > 0): only the siblings
// the touched nodes read go up, only the touched nodes come back.  The device mirror of the tree (2n - 1 elements in the node context's
// arena: leaves, then inner nodes) is allocated but never filled beyond those siblings.  `in` (in_bytes) is uploaded as it is;
// run(mirror_leaves, mirror_nodes, d_idx, d_in, d_root or NULL, d_applied, stream) is the _dev form on the mirror.
template <int W, class Ctx, class Run>
cpb_status upd_host_form(Ctx* node, uint64_t* leaf_nodes, uint64_t* non_leaf_nodes, size_t n, const uint64_t* indexes, const void* in,
                         size_t in_bytes, size_t k, const uint64_t* asserted_root, int* applied, Run&& run) {
    constexpr size_t EB = 4 * W;                               // bytes per element
    const int h = log2_exact(n);
    std::vector<u64> uniq(indexes, indexes + k), reads, writes;
    std::sort(uniq.begin(), uniq.end());
    uniq.erase(std::unique(uniq.begin(), uniq.end()), uniq.end());
    upd_host_sets(uniq, h, reads, writes);
    auto host_elem = [&](u64 pos) -> uint64_t* { return pos < n ? leaf_nodes + (W / 2) * pos : non_leaf_nodes + (W / 2) * (pos - n); };
    std::vector<uint64_t> read_vals((W / 2) * reads.size());
    for (size_t i = 0; i < reads.size(); i++) memcpy(&read_vals[(W / 2) * i], host_elem(reads[i]), EB);

    const size_t nr = reads.size(), nw = writes.size();
    std::vector<uint64_t> write_vals((W / 2) * nw);
    unsigned char ok = 0;
    std::lock_guard<std::mutex> lk(node->mu);
    DeviceGuard g(node->device);
    cudaStream_t st = node->stream;
    HostStage S(node->arena, st);
    const size_t o_idx = S.in(indexes, 8 * k), o_in = S.in(in, in_bytes), o_root = S.in(asserted_root, asserted_root ? EB : 0),
                 o_rpos = S.in(reads.data(), 8 * nr), o_rval = S.in(read_vals.data(), EB * nr), o_wpos = S.in(writes.data(), 8 * nw),
                 o_out = S.out(write_vals.data(), EB * nw), o_applied = S.out(&ok, 1), o_mirror = S.dev(EB * (2 * n - 1));
    CPB_TRY(S.upload());
    u32* mirror = S.at<u32>(o_mirror);
    if (nr) {
        k_upd_move<W><<<upd_grid(nr, kUpdBlock), kUpdBlock, 0, st>>>(S.at<const u32>(o_rval), mirror, S.at<const u64>(o_rpos), nr, 0);
        CPB_CUDA(cudaGetLastError());
    }
    CPB_TRY(run((uint64_t*)mirror, (uint64_t*)(mirror + W * n), S.at<const uint64_t>(o_idx), S.at<const void>(o_in),
                asserted_root ? S.at<const uint64_t>(o_root) : nullptr, S.at<unsigned char>(o_applied), st));
    k_upd_move<W><<<upd_grid(nw, kUpdBlock), kUpdBlock, 0, st>>>(mirror, S.at<u32>(o_out), S.at<const u64>(o_wpos), nw, 1);
    CPB_CUDA(cudaGetLastError());
    CPB_TRY(S.download());
    if (ok)
        for (size_t i = 0; i < nw; i++) memcpy(host_elem(writes[i]), &write_vals[(W / 2) * i], EB);
    if (applied) *applied = ok;
    return CPB_OK;
}

}  // namespace
}  // namespace cpb
