// cpb_merkle_update_pedersen.cu -- k x MerkleTree::update / check_update (R/merkle_tree/mod.rs:627-725) for byte trees whose inner
// nodes are pedersen::TwoToOneCRH (JubJubMerkleTreeParams, R/merkle_tree/tests/mod.rs:19-33), on the device and in place
// (include/cpb200.h, "Merkle tree update (Pedersen inner nodes)").
//
// The plan, the scratch layout and the commit are those of the Poseidon-node update (merkle_update.cuh, merkle_update_kernels.cuh)
// with 16-word digests: affine (x, y) in Montgomery form, as the build stores them.  Levels bottom-up; one grid per level while a
// level has more than ped_warp_max() candidate slots:
//   rows      one thread per candidate slot of the level (k_ped_upd_rows): a touched candidate's children, read through upd_kids
//             from the scratch (touched child) or the caller's tree, serialised as TwoToOneCRH::compress does (te_node_row);
//             an untouched candidate's row is zero
//   hash      the node context's own hash launch over the level's rows (launch_hash: k_pedersen_hash for 8-bit chunks,
//             k_pedersen_hash_gather for wider ones, then k_pedersen_normalise), two_to_one_len bytes of each row, into the
//             level's scratch slots.  Untouched candidates are hashed too; their slots are never committed (DESIGN.md §4.4)
//   narrow    ONE launch of k_ped_upd_top for all the levels above: one warp per node, the table lookups split over the lanes,
//             levels chained by per-parent arrival counters as in the Poseidon team launch
//   commit    k_upd_commit<16>, predicated on the 16-word device-side comparison with asserted_root
// The launch count depends on the tree height only.  Scratch comes from the stream-ordered pool; nothing synchronises the host.
#include "merkle_update.cuh"
#include "merkle_update_kernels.cuh"
#include "pedersen_internal.cuh"
#include "te_ops.cuh"

#include <cstdlib>

namespace cpb {
namespace {

constexpr int kPedW = 16;                                      // digest words: affine (x, y)
constexpr int kPedEntryWords = 24;                             // table entry: affine Niels (y + x, y - x, 2d x y)
constexpr int kWarpBlock = 128;                                // k_ped_upd_top: four independent warps per CTA

// Widest level (in candidate slots) the warp launch starts at; wider levels get the per-level grids.  Level widths shrink towards
// the root, so every level above fits too.  CPB_PED_UPD_WARP_MAX overrides it for measurement (0: per-level grids only).
size_t ped_warp_max() {
    static long v = -1;
    if (v < 0) {
        const char* e = getenv("CPB_PED_UPD_WARP_MAX");
        v = e ? atol(e) : 4096;
        if (v < 0) v = 0;
    }
    return (size_t)v;
}
int warp_start_level(int h, u64 k) {
    const size_t mx = ped_warp_max();
    if (mx == 0) return -1;
    for (int l = h - 1; l >= 0; l--)
        if (upd_width(l, k) <= mx) return l;
    return -1;
}

__device__ __forceinline__ void ld_elem_l2(u32* r, const u32* p) {      // through L2: other SMs wrote it during this launch
    uint4 a = __ldcg(reinterpret_cast<const uint4*>(p));
    uint4 b = __ldcg(reinterpret_cast<const uint4*>(p + 4));
    r[0] = a.x; r[1] = a.y; r[2] = a.z; r[3] = a.w;
    r[4] = b.x; r[5] = b.y; r[6] = b.z; r[7] = b.w;
}

// Levels l_start .. 0 in one launch, one warp per node.  Warp w of the grid starts on candidate w of level l_start.  Lanes 0-3
// serialise the node's four child coordinates into the warp's 128-byte row in shared memory; every lane then adds its share of
// the table lookups (te_lane_sum: lookups lane, lane + 32, ...), the 32 partial sums are reduced with five shuffle rounds of
// te_add (lane i takes lane i + 16, then i + 8, ...), and lane 0 normalises with one inversion and stores the affine digest.  It
// then arrives at the parent's counter; the warp continues with the parent only when it was the last of the parent's touched
// children to arrive, so no warp waits for another.
template <class F>
__global__ void __launch_bounds__(kWarpBlock)
k_ped_upd_top(PedersenDev P, const u32* __restrict__ consts, const u32* __restrict__ table, UpdPlan X, int l_start, int row_len, u32* scratch,
              const u32* leaf_nodes, const u32* nodes, unsigned* arrivals) {
    __shared__ __align__(16) u32 rows[kWarpBlock / 32][32];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    u32* row = rows[wib];
    u32 pm[8], d2[8];
    ld_elem(pm, consts);
    ld_elem(d2, consts + 8);
    const u64 m = *X.m;
    int l = l_start;
    const u64 c0 = (u64)blockIdx.x * (kWarpBlock / 32) + wib;
    UpdSite S;
    if (c0 < upd_width(l, X.k)) S = upd_site(X.U, m, X.h, l, X.k, c0);
    bool active = S.touched;                                   // warp-uniform
    const int cb = P.chunk_bits;
    while (active) {
        if (lane < 4) {
            const UpdKids K = upd_kids(X.U, m, X.h, l, X.k, S);
            const bool right = lane >= 2;
            const u32* src = upd_child_at<kPedW>(X, l, right ? K.rt : K.lt, right ? K.rslot : K.lslot, 2 * S.node + (right ? 1 : 0), (const u32*)scratch,
                                                 leaf_nodes, nodes) + 8 * (lane & 1);
            u32 a[8], one[8];
            ld_elem_l2(a, src);
            fp_zero(one);
            one[0] = 1;
            fp_mul<F>(a, a, one, pm);                          // canonical, as te_node_row
            st_elem(row + 8 * lane, a);
        }
        __syncwarp();
        TePoint acc;
        te_lane_sum<F>(acc, reinterpret_cast<const uint8_t*>(row), row_len, cb, P.n_in_chunks, lane, 32,
                       [&](int c, u32 v, u32* yp, u32* ym, u32* t2d) {
                           const u32* e = table + (((long)c << cb) + v) * kPedEntryWords;
                           ld_elem(yp, e);
                           ld_elem(ym, e + 8);
                           ld_elem(t2d, e + 16);
                       }, pm);
#pragma unroll 1
        for (int off = 16; off > 0; off >>= 1) {
            TePoint o;
#pragma unroll
            for (int i = 0; i < 8; i++) {
                o.X[i] = __shfl_down_sync(0xffffffffu, acc.X[i], off);
                o.Y[i] = __shfl_down_sync(0xffffffffu, acc.Y[i], off);
                o.Z[i] = __shfl_down_sync(0xffffffffu, acc.Z[i], off);
                o.T[i] = __shfl_down_sync(0xffffffffu, acc.T[i], off);
            }
            te_add<F>(acc, o, d2, pm);                         // lanes >= off add a copy of themselves; only lane 0's sum is used
        }
        bool next = false;
        u64 pc = 0;
        if (lane == 0) {
            u32 x[8], y[8];
            te_to_affine<F>(x, y, acc, pm);
            u32* o = scratch + kPedW * (X.off[l] + S.slot);
            st_elem(o, x);
            st_elem(o + 8, y);
            if (l > 0) {
                pc = upd_parent_cand(X.U, m, X.h, l, X.k, S.node);
                const UpdSite PS = upd_site(X.U, m, X.h, l - 1, X.k, pc);
                const UpdKids PK = upd_kids(X.U, m, X.h, l - 1, X.k, PS);
                const unsigned need = (PK.lt ? 1u : 0u) + (PK.rt ? 1u : 0u);
                __threadfence();                               // the digest is visible before the arrival
                next = atomicAdd(arrivals + X.off[l - 1] + PS.slot, 1u) + 1u == need;
                if (next) __threadfence();
            }
        }
        active = __shfl_sync(0xffffffffu, next ? 1 : 0, 0) != 0;
        pc = __shfl_sync(0xffffffffu, pc, 0);
        __syncwarp();                                          // the row is free again
        if (active) {
            l--;
            S = upd_site(X.U, m, X.h, l, X.k, pc);
        }
    }
}

cpb_status launch_top(cpb_pedersen_ctx* node, const UpdPlan& X, int l, int row_len, u32* scratch, const u32* leaf_nodes, const u32* nodes,
                      unsigned* arrivals, cudaStream_t st) {
    const unsigned grid = upd_grid(upd_width(l, X.k), kWarpBlock / 32);
#define ARGS node->dev, node->d_consts, node->d_table, X, l, row_len, scratch, leaf_nodes, nodes, arrivals
    switch (node->field_id) {
        case CPB_BLS12_381_FR: k_ped_upd_top<Bls12_381_Fr><<<grid, kWarpBlock, 0, st>>>(ARGS); break;
        case CPB_BLS12_377_FR: k_ped_upd_top<Bls12_377_Fr><<<grid, kWarpBlock, 0, st>>>(ARGS); break;
        default: return fail(CPB_UNSUPPORTED, "no kernel for base field %d", node->field_id);
    }
#undef ARGS
    CPB_CUDA(cudaGetLastError());
    return CPB_OK;
}

template <class F>
__global__ void k_ped_upd_rows(UpdPlan X, int l, const u32* scratch, const u32* leaf_nodes, const u32* nodes, u32* __restrict__ rows) {
    const u64 c = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= upd_width(l, X.k)) return;
    const u64 m = *X.m;
    const UpdSite S = upd_site(X.U, m, X.h, l, X.k, c);
    u32* o = rows + 32 * c;
    if (!S.touched) {
        u32 z[8];
        fp_zero(z);
#pragma unroll
        for (int i = 0; i < 32; i += 8) st_elem(o + i, z);
        return;
    }
    const UpdKids K = upd_kids(X.U, m, X.h, l, X.k, S);
    te_node_row<F>(o, upd_child_at<kPedW>(X, l, K.lt, K.lslot, 2 * S.node, scratch, leaf_nodes, nodes),
                   upd_child_at<kPedW>(X, l, K.rt, K.rslot, 2 * S.node + 1, scratch, leaf_nodes, nodes));
}

cpb_status launch_rows(const cpb_pedersen_ctx* node, const UpdPlan& X, int l, const u32* scratch, const u32* leaf_nodes, const u32* nodes,
                       u32* rows, cudaStream_t st) {
    const unsigned grid = upd_grid(upd_width(l, X.k), kUpdBlock);
    switch (node->field_id) {
        case CPB_BLS12_381_FR: k_ped_upd_rows<Bls12_381_Fr><<<grid, kUpdBlock, 0, st>>>(X, l, scratch, leaf_nodes, nodes, rows); break;
        case CPB_BLS12_377_FR: k_ped_upd_rows<Bls12_377_Fr><<<grid, kUpdBlock, 0, st>>>(X, l, scratch, leaf_nodes, nodes, rows); break;
        default: return fail(CPB_UNSUPPORTED, "no kernel for base field %d", node->field_id);
    }
    CPB_CUDA(cudaGetLastError());
    return CPB_OK;
}

// The whole update on device arrays (tree in place; idx, digests, asserted, applied in device memory; the last two nullable).
cpb_status update_digests_dev(cpb_pedersen_ctx* node, u32* leaf_nodes, u32* nodes, size_t n, const u64* idx, const u32* digests, size_t k,
                              const u32* asserted, unsigned char* applied, cudaStream_t st) {
    UpdPlan X;
    X.h = log2_exact(n);
    X.k = k;
    upd_offsets(X.h, k, X.off);
    if (k == 0) {
        if (applied) {
            k_upd_commit<kPedW><<<1, 32, 0, st>>>(X, nullptr, leaf_nodes, nodes, asserted, applied);
            CPB_CUDA(cudaGetLastError());
        }
        return CPB_OK;
    }
    const int lt = warp_start_level(X.h, k);
    const size_t n_arr = lt >= 0 ? (size_t)X.off[lt] : 0;      // arrival counters of the levels above the warp launch's start
    const size_t rows_b = align256(128 * (size_t)upd_width(X.h - 1, k));   // the widest inner level's rows
    const size_t row_len = two_to_one_len(node);
    UpdBuffers B;
    CPB_TRY(upd_layout(X, n, k, rows_b + 4 * n_arr + 4, kPedW, st, B));
    CPB_CUDA(cudaMallocAsync((void**)&B.b, B.total, st));
    auto run = [&]() -> cpb_status {
        u32* scratch = B.scratch();
        u32* rows = (u32*)B.extra();
        CPB_TRY(upd_run_plan<kPedW>(B, X, idx, n, digests, st));
        const int l_grid_end = lt >= 0 ? lt + 1 : 0;
        for (int l = X.h - 1; l >= l_grid_end; l--) {
            CPB_TRY(launch_rows(node, X, l, scratch, leaf_nodes, nodes, rows, st));
            CPB_TRY(launch_hash(node, (const uint8_t*)rows, row_len, 128, nullptr, scratch + kPedW * X.off[l], upd_width(l, k), 0, st));
        }
        if (lt >= 0) {
            unsigned* arr = (unsigned*)((char*)B.extra() + rows_b);
            CPB_CUDA(cudaMemsetAsync(arr, 0, 4 * n_arr + 4, st));
            CPB_TRY(launch_top(node, X, lt, (int)row_len, scratch, leaf_nodes, nodes, arr, st));
        }
        k_upd_commit<kPedW><<<upd_grid(X.off[X.h + 1], kUpdBlock), kUpdBlock, 0, st>>>(X, scratch, leaf_nodes, nodes, asserted, applied);
        CPB_CUDA(cudaGetLastError());
        return CPB_OK;
    };
    const cpb_status rc = run();
    cudaFreeAsync(B.b, st);
    return rc;
}

// The leaf form hashes the k new leaves (pedersen::CRH with the leaf context) into pool scratch first.
cpb_status update_dev(cpb_pedersen_ctx* leaf, cpb_pedersen_ctx* node, uint64_t* leaf_nodes, uint64_t* non_leaf_nodes, size_t n,
                      const uint64_t* indexes, const void* in, size_t leaf_len, size_t leaf_stride, size_t k, const uint64_t* asserted_root,
                      uint8_t* applied, cudaStream_t st) {
    if (!leaf || k == 0)
        return update_digests_dev(node, (u32*)leaf_nodes, (u32*)non_leaf_nodes, n, indexes, k ? (const u32*)in : nullptr, k,
                                  (const u32*)asserted_root, applied, st);
    u32* d = nullptr;
    CPB_CUDA(cudaMallocAsync((void**)&d, 64 * k, st));
    cpb_status rc = launch_hash(leaf, (const uint8_t*)in, leaf_len, leaf_stride, nullptr, d, k, 0, st);
    if (rc == CPB_OK)
        rc = update_digests_dev(node, (u32*)leaf_nodes, (u32*)non_leaf_nodes, n, indexes, d, k, (const u32*)asserted_root, applied, st);
    cudaFreeAsync(d, st);
    return rc;
}

// Argument rules of all four forms: the shape first, then the buffers (in_len == 0: the new leaves are empty, `in` is not read), then
// the contexts and the leaf length (check_ctxs).
cpb_status check_args(uint64_t* leaf_nodes, uint64_t* non_leaf_nodes, size_t n, const uint64_t* indexes, const void* in, size_t in_len,
                      size_t k) {
    CPB_TRY(check_update_shape(n, k));
    if (!leaf_nodes || !non_leaf_nodes || (k && !indexes) || (k && in_len && !in)) return fail(CPB_NULL_POINTER, "null buffer");
    return CPB_OK;
}
cpb_status check_ctxs(cpb_pedersen_ctx* leaf, cpb_pedersen_ctx* node, size_t leaf_len) {
    if (!node) return fail(CPB_NULL_POINTER, "null context");
    if (leaf) {
        if (leaf->device != node->device || leaf->field_id != node->field_id)
            return fail(CPB_BAD_PARAMS, "leaf and node contexts must share device and curve");
        CPB_TRY(check_len(leaf, leaf_len, false));
    }
    return CPB_OK;
}

cpb_status update_dev_checked(cpb_pedersen_ctx* leaf, cpb_pedersen_ctx* node, uint64_t* leaf_nodes, uint64_t* non_leaf_nodes, size_t n,
                              const uint64_t* indexes, const void* in, size_t leaf_len, size_t leaf_stride, size_t k,
                              const uint64_t* asserted_root, uint8_t* applied, void* stream) {
    CPB_TRY(check_args(leaf_nodes, non_leaf_nodes, n, indexes, in, leaf ? leaf_len : 1, k));
    CPB_TRY(check_ctxs(leaf, node, leaf_len));
    if (leaf && k > 1 && leaf_stride < leaf_len) return fail(CPB_BAD_PARAMS, "leaf_stride < leaf_len");
    DeviceGuard g(node->device);
    return update_dev(leaf, node, leaf_nodes, non_leaf_nodes, n, indexes, in, leaf_len, leaf_stride, k, asserted_root, applied,
                      (cudaStream_t)stream);
}

// Host arrays: upd_host_form (merkle_update_kernels.cuh) around the _dev form; byte leaves are n x leaf_len, packed.
cpb_status update_host(cpb_pedersen_ctx* leaf, cpb_pedersen_ctx* node, uint64_t* leaf_nodes, uint64_t* non_leaf_nodes, size_t n,
                       const uint64_t* indexes, const void* in, size_t leaf_len, size_t k, const uint64_t* asserted_root, int* applied) {
    const size_t in_bytes = leaf ? k * leaf_len : 64 * k;
    CPB_TRY(check_args(leaf_nodes, non_leaf_nodes, n, indexes, in, leaf ? leaf_len : 1, k));
    for (size_t j = 0; j < k; j++)
        if (indexes[j] >= n) return fail(CPB_BAD_PARAMS, "index %llu out of range (%zu leaves)", (unsigned long long)indexes[j], n);
    CPB_TRY(check_ctxs(leaf, node, leaf_len));
    if (k == 0) {
        if (applied) *applied = !asserted_root || memcmp(non_leaf_nodes, asserted_root, 64) == 0;
        return CPB_OK;
    }
    return upd_host_form<kPedW>(node, leaf_nodes, non_leaf_nodes, n, indexes, in, in_bytes, k, asserted_root, applied,
                                [&](uint64_t* ml, uint64_t* mn, const uint64_t* d_idx, const void* d_in, const uint64_t* d_root,
                                    uint8_t* d_applied, cudaStream_t st) {
                                    return update_dev(leaf, node, ml, mn, n, d_idx, d_in, leaf_len, leaf_len, k, d_root, d_applied, st);
                                });
}

}  // namespace
}  // namespace cpb

using namespace cpb;

extern "C" {

cpb_status cpb_merkle_pedersen_update_digests_dev(cpb_pedersen_ctx* node_ctx, uint64_t* leaf_nodes_xy, uint64_t* non_leaf_nodes_xy, size_t n,
                                                  const uint64_t* indexes, const uint64_t* new_leaf_digests_xy, size_t k,
                                                  const uint64_t* asserted_root_xy, uint8_t* applied, void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    return update_dev_checked(nullptr, node_ctx, leaf_nodes_xy, non_leaf_nodes_xy, n, indexes, new_leaf_digests_xy, 0, 0, k, asserted_root_xy,
                              applied, stream);
    });
}

cpb_status cpb_merkle_pedersen_update_dev(cpb_pedersen_ctx* leaf_ctx, cpb_pedersen_ctx* node_ctx, uint64_t* leaf_nodes_xy,
                                          uint64_t* non_leaf_nodes_xy, size_t n, const uint64_t* indexes, const uint8_t* new_leaves,
                                          size_t leaf_len, size_t leaf_stride, size_t k, const uint64_t* asserted_root_xy, uint8_t* applied,
                                          void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    if (!leaf_ctx) return fail(CPB_NULL_POINTER, "null context");
    return update_dev_checked(leaf_ctx, node_ctx, leaf_nodes_xy, non_leaf_nodes_xy, n, indexes, new_leaves, leaf_len, leaf_stride, k,
                              asserted_root_xy, applied, stream);
    });
}

cpb_status cpb_merkle_pedersen_update_digests(cpb_pedersen_ctx* node_ctx, uint64_t* leaf_nodes_xy, uint64_t* non_leaf_nodes_xy, size_t n,
                                              const uint64_t* indexes, const uint64_t* new_leaf_digests_xy, size_t k,
                                              const uint64_t* asserted_root_xy, int* applied) {
    return cpb::guarded([&]() -> cpb_status {
    return update_host(nullptr, node_ctx, leaf_nodes_xy, non_leaf_nodes_xy, n, indexes, new_leaf_digests_xy, 0, k, asserted_root_xy, applied);
    });
}

cpb_status cpb_merkle_pedersen_update(cpb_pedersen_ctx* leaf_ctx, cpb_pedersen_ctx* node_ctx, uint64_t* leaf_nodes_xy, uint64_t* non_leaf_nodes_xy,
                                      size_t n, const uint64_t* indexes, const uint8_t* new_leaves, size_t leaf_len, size_t k,
                                      const uint64_t* asserted_root_xy, int* applied) {
    return cpb::guarded([&]() -> cpb_status {
    if (!leaf_ctx) return fail(CPB_NULL_POINTER, "null context");
    return update_host(leaf_ctx, node_ctx, leaf_nodes_xy, non_leaf_nodes_xy, n, indexes, new_leaves, leaf_len, k, asserted_root_xy, applied);
    });
}

}  // extern "C"
