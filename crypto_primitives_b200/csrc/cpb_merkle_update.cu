// cpb_merkle_update.cu -- k x MerkleTree::update / check_update (R/merkle_tree/mod.rs:627-725) for trees whose inner nodes are
// poseidon::TwoToOneCRH, on the device and in place (include/cpb200.h, "Merkle tree update").
//
// One call, any k:
//   plan      the (index, position) pairs sorted by index (cub radix sort, stable, so the last occurrence of an index comes
//             last in its run); run tails that are in range become U, the distinct updated leaves, and their digests go to
//             the leaf level of the scratch (merkle_update.cuh describes the layout)
//   levels    bottom-up, one grid per level over that level's candidates (one hash per thread, pos_hash_single) while a level
//             may hold more than team_max_for(1) touched nodes; then ONE launch of the four-warp team round for every level
//             above, chained on the device: the last child to arrive at a parent (an atomic counter per parent) hashes it,
//             so no CTA ever waits for another
//   commit    one grid scatters the scratch into the tree, predicated on the device-side comparison with asserted_root
// The launch count depends on the tree height only.  Scratch comes from the stream-ordered pool; nothing synchronises the host.
#include "merkle_update.cuh"
#include "merkle_update_kernels.cuh"
#include "poseidon_kernels.cuh"

namespace cpb {
namespace {

// Where the current value of child `node` (level l + 1) of a touched node of level l is (merkle_update.cuh, upd_child_at).
__device__ __forceinline__ const u32* upd_child(const UpdPlan& X, int l, bool touched, u64 slot, u64 node, const u32* scratch,
                                                const u32* leaf_nodes, const u32* nodes) {
    return upd_child_at<8>(X, l, touched, slot, node, scratch, leaf_nodes, nodes);
}

// One level, one candidate per thread; only touched candidates hash.
template <class F, int T, bool A5>
__global__ void __launch_bounds__(kBlock, pos_min_blocks(T))
k_merkle_update_level(PoseidonDev P, const u32* __restrict__ consts, UpdPlan X, int l, u32* scratch, const u32* leaf_nodes,
                      const u32* nodes) {
    extern __shared__ __align__(16) u32 cs[];
    __shared__ __align__(8) unsigned long long mbar;
    tma_stage_to_smem(cs, consts, (unsigned)P.n_elems * 32u, &mbar);
    const u64 c = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= upd_width(l, X.k)) return;
    const u64 m = *X.m;
    const UpdSite S = upd_site(X.U, m, X.h, l, X.k, c);
    if (!S.touched) return;
    const UpdKids K = upd_kids(X.U, m, X.h, l, X.k, S);
    const u32* ct = cs + (int)threadIdx.x * P.zero;
    u32 pm[8];
    ld_elem(pm, ct + 8 * P.off_mod);
    alignas(16) u32 pair[16];
    ld_elem(pair, upd_child(X, l, K.lt, K.lslot, 2 * S.node, scratch, leaf_nodes, nodes));
    ld_elem(pair + 8, upd_child(X, l, K.rt, K.rslot, 2 * S.node + 1, scratch, leaf_nodes, nodes));
    pos_hash_single<F, T, A5>(scratch + 8 * (X.off[l] + S.slot), 1, pair, 2, P, ct, pm);
}

// Levels l_start .. 0 in one launch, 32 hashes per CTA with the four-warp team round (poseidon_team.cuh).  Lane j of a CTA starts
// on candidate 32 b + j of level l_start; after hashing a node it arrives at the parent's counter and continues with the parent
// only when it is the last of the parent's touched children to arrive (the other child's digest is then in memory: it was
// stored and fenced before its arrival).  Lanes that do not continue idle; a CTA ends when none of its lanes continues.
// Children are read through L2 (ld.global.cg): other SMs wrote them during this launch.
template <class F>
__global__ void __launch_bounds__(kTeamThreads)
k_merkle_update_top(PoseidonDev P, const u32* __restrict__ consts, UpdPlan X, int l_start, u32* scratch, const u32* leaf_nodes,
                    const u32* nodes, unsigned* arrivals) {
    extern __shared__ __align__(16) u32 cs[];
    __shared__ __align__(8) unsigned long long mbar;
    __shared__ u64 next_cand[32];
    __shared__ int next_active[32];
    tma_stage_to_smem(cs, consts, (unsigned)P.n_elems * 32u, &mbar);
    u32* xb = cs + 8 * P.n_elems;
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const u32* ct = cs + (int)threadIdx.x * P.zero;
    u32 pm[8];
    ld_elem(pm, ct + 8 * P.off_mod);
    int tb_alpha, tb_e;
    team_top_bits(P, tb_alpha, tb_e);
    const u64 m = *X.m;
    int l = l_start;
    const u64 c0 = (u64)blockIdx.x * 32 + lane;
    UpdSite S;
    if (c0 < upd_width(l, X.k)) S = upd_site(X.U, m, X.h, l, X.k, c0);
    bool active = S.touched;
    while (__syncthreads_or(active)) {
        u32 s[8];
        fp_zero(s);
        if (active && (w == 1 || w == 2)) {
            const UpdKids K = upd_kids(X.U, m, X.h, l, X.k, S);
            const u32* src = w == 1 ? upd_child(X, l, K.lt, K.lslot, 2 * S.node, scratch, leaf_nodes, nodes)
                                    : upd_child(X, l, K.rt, K.rslot, 2 * S.node + 1, scratch, leaf_nodes, nodes);
            ld_elem_cg(s, src);
        }
        team_permute32<F>(s, w, lane, P, ct, pm, xb, tb_alpha, tb_e);
        if (w == 1) {
            bool next = false;
            u64 pc = 0;
            if (active) {
                st_elem(scratch + 8 * (X.off[l] + S.slot), s);
                if (l > 0) {
                    pc = upd_parent_cand(X.U, m, X.h, l, X.k, S.node);
                    const UpdSite PS = upd_site(X.U, m, X.h, l - 1, X.k, pc);
                    const UpdKids PK = upd_kids(X.U, m, X.h, l - 1, X.k, PS);
                    const unsigned need = (PK.lt ? 1u : 0u) + (PK.rt ? 1u : 0u);
                    __threadfence();                           // the digest is visible before the arrival
                    next = atomicAdd(arrivals + X.off[l - 1] + PS.slot, 1u) + 1u == need;
                    if (next) __threadfence();
                }
            }
            next_active[lane] = next ? 1 : 0;
            next_cand[lane] = pc;
        }
        __syncthreads();
        active = next_active[lane] != 0;
        if (active) S = upd_site(X.U, m, X.h, l - 1, X.k, next_cand[lane]);
        l--;
    }
}

template <class F, int T>
cpb_status launch_level_ft(cpb_poseidon_ctx* c, const UpdPlan& X, int l, u32* scratch, const u32* leaf_nodes, const u32* nodes,
                           cudaStream_t st) {
    const size_t smem = (size_t)c->dev.n_elems * 32;
    const unsigned grid = upd_grid(upd_width(l, X.k), kBlock);
    int occ = 0;
    if constexpr (pos_alpha5_kernel<F, T>()) {
        if (c->dev.alpha == 5) {
            CPB_TRY(configure_kernel(k_merkle_update_level<F, T, true>, smem, kBlock, occ));
            k_merkle_update_level<F, T, true><<<grid, kBlock, smem, st>>>(c->dev, c->d_consts, X, l, scratch, leaf_nodes, nodes);
            CPB_CUDA(cudaGetLastError());
            return CPB_OK;
        }
    }
    CPB_TRY(configure_kernel(k_merkle_update_level<F, T, false>, smem, kBlock, occ));
    k_merkle_update_level<F, T, false><<<grid, kBlock, smem, st>>>(c->dev, c->d_consts, X, l, scratch, leaf_nodes, nodes);
    CPB_CUDA(cudaGetLastError());
    return CPB_OK;
}

template <class F>
cpb_status launch_level_f(cpb_poseidon_ctx* c, const UpdPlan& X, int l, u32* scratch, const u32* leaf_nodes, const u32* nodes,
                          cudaStream_t st) {
    switch (c->dev.t) {           // rate >= 2 and capacity >= 1: t >= 3
        case 3: return launch_level_ft<F, 3>(c, X, l, scratch, leaf_nodes, nodes, st);
        case 4: return launch_level_ft<F, 4>(c, X, l, scratch, leaf_nodes, nodes, st);
        case 5: return launch_level_ft<F, 5>(c, X, l, scratch, leaf_nodes, nodes, st);
        case 6: return launch_level_ft<F, 6>(c, X, l, scratch, leaf_nodes, nodes, st);
        case 7: return launch_level_ft<F, 7>(c, X, l, scratch, leaf_nodes, nodes, st);
        case 8: return launch_level_ft<F, 8>(c, X, l, scratch, leaf_nodes, nodes, st);
        case 9: return launch_level_ft<F, 9>(c, X, l, scratch, leaf_nodes, nodes, st);
    }
    return fail(CPB_UNSUPPORTED, "state width t=%d is not built for the Merkle update (t = 3..9)", c->dev.t);
}

template <class F>
cpb_status launch_top_f(cpb_poseidon_ctx* c, const UpdPlan& X, int l, u32* scratch, const u32* leaf_nodes, const u32* nodes,
                        unsigned* arrivals, cudaStream_t st) {
    const size_t smem = (size_t)c->dev.n_elems * 32 + (size_t)kTeamXbWords * 4;
    int occ = 0;
    CPB_TRY(configure_kernel(k_merkle_update_top<F>, smem, kTeamThreads, occ));
    k_merkle_update_top<F><<<upd_grid(upd_width(l, X.k), 32), kTeamThreads, smem, st>>>(c->dev, c->d_consts, X, l, scratch, leaf_nodes,
                                                                                        nodes, arrivals);
    CPB_CUDA(cudaGetLastError());
    return CPB_OK;
}

cpb_status launch_level(cpb_poseidon_ctx* c, const UpdPlan& X, int l, u32* scratch, const u32* leaf_nodes, const u32* nodes, cudaStream_t st) {
#define CALL(F) launch_level_f<F>(c, X, l, scratch, leaf_nodes, nodes, st)
    switch (c->field_id) {
        case CPB_BLS12_381_FR: return CALL(Bls12_381_Fr);
        case CPB_BN254_FR: return CALL(Bn254_Fr);
        case CPB_JUBJUB_FR: return CALL(Jubjub_Fr);
        case CPB_BLS12_377_FR: return CALL(Bls12_377_Fr);
    }
#undef CALL
    return fail(CPB_BAD_PARAMS, "unknown field id %d", c->field_id);
}
cpb_status launch_top(cpb_poseidon_ctx* c, const UpdPlan& X, int l, u32* scratch, const u32* leaf_nodes, const u32* nodes, unsigned* arrivals,
                      cudaStream_t st) {
#define CALL(F) launch_top_f<F>(c, X, l, scratch, leaf_nodes, nodes, arrivals, st)
    switch (c->field_id) {
        case CPB_BLS12_381_FR: return CALL(Bls12_381_Fr);
        case CPB_BN254_FR: return CALL(Bn254_Fr);
        case CPB_JUBJUB_FR: return CALL(Jubjub_Fr);
        case CPB_BLS12_377_FR: return CALL(Bls12_377_Fr);
    }
#undef CALL
    return fail(CPB_BAD_PARAMS, "unknown field id %d", c->field_id);
}

// Highest level the team launch starts at (-1: every level gets a grid of its own).  Level widths shrink towards the root, so
// every level above it fits too.
int team_start_level(const cpb_poseidon_ctx* node, int h, u64 k) {
    if (!team_capable(node) || team_max() == 0) return -1;
    for (int l = h - 1; l >= 0; l--)
        if (upd_width(l, k) <= team_max_for(1)) return l;
    return -1;
}

// The whole update on device arrays (tree in place; idx, digests, asserted, applied in device memory; the last two nullable).
cpb_status update_digests_dev(cpb_poseidon_ctx* node, u32* leaf_nodes, u32* nodes, size_t n, const u64* idx, const u32* digests, size_t k,
                              const u32* asserted, unsigned char* applied, cudaStream_t st) {
    UpdPlan X;
    X.h = log2_exact(n);
    X.k = k;
    upd_offsets(X.h, k, X.off);
    if (k == 0) {
        if (applied) {
            k_upd_commit<8><<<1, 32, 0, st>>>(X, nullptr, leaf_nodes, nodes, asserted, applied);
            CPB_CUDA(cudaGetLastError());
        }
        return CPB_OK;
    }
    const int lt = team_start_level(node, X.h, k);
    const size_t n_arr = lt >= 0 ? (size_t)X.off[lt] : 0;      // arrival counters of the levels above the team start
    UpdBuffers B;
    CPB_TRY(upd_layout(X, n, k, 4 * n_arr + 4, 8, st, B));
    CPB_CUDA(cudaMallocAsync((void**)&B.b, B.total, st));
    auto run = [&]() -> cpb_status {
        u32* scratch = B.scratch();
        CPB_TRY(upd_run_plan<8>(B, X, idx, n, digests, st));
        const int l_grid_end = lt >= 0 ? lt + 1 : 0;
        for (int l = X.h - 1; l >= l_grid_end; l--) CPB_TRY(launch_level(node, X, l, scratch, leaf_nodes, nodes, st));
        if (lt >= 0) {
            unsigned* arr = (unsigned*)B.extra();
            CPB_CUDA(cudaMemsetAsync(arr, 0, 4 * n_arr + 4, st));
            CPB_TRY(launch_top(node, X, lt, scratch, leaf_nodes, nodes, arr, st));
        }
        k_upd_commit<8><<<upd_grid(X.off[X.h + 1], kUpdBlock), kUpdBlock, 0, st>>>(X, scratch, leaf_nodes, nodes, asserted, applied);
        CPB_CUDA(cudaGetLastError());
        return CPB_OK;
    };
    const cpb_status rc = run();
    cudaFreeAsync(B.b, st);
    return rc;
}

cpb_status check_update_ctxs(cpb_poseidon_ctx* leaf, cpb_poseidon_ctx* node) {
    if (leaf) CPB_TRY(check_ctx(leaf));
    CPB_TRY(check_ctx(node));
    if (leaf && (leaf->device != node->device || leaf->field_id != node->field_id))
        return fail(CPB_BAD_PARAMS, "leaf and node contexts must share device and field");
    if (node->dev.rate < 2) return fail(CPB_UNSUPPORTED, "two-to-one with rate < 2 not supported");
    return CPB_OK;
}

// The leaf form hashes the k new leaves (poseidon::CRH) into pool scratch first.
cpb_status update_dev(cpb_poseidon_ctx* leaf, cpb_poseidon_ctx* node, uint64_t* leaf_nodes, uint64_t* non_leaf_nodes, size_t n,
                      const uint64_t* indexes, const uint64_t* in, size_t leaf_len, size_t k, const uint64_t* asserted_root,
                      uint8_t* applied, cudaStream_t st) {
    if (!leaf) return update_digests_dev(node, (u32*)leaf_nodes, (u32*)non_leaf_nodes, n, indexes, (const u32*)in, k, (const u32*)asserted_root,
                                         applied, st);
    if (k == 0) return update_digests_dev(node, (u32*)leaf_nodes, (u32*)non_leaf_nodes, n, indexes, nullptr, 0, (const u32*)asserted_root,
                                          applied, st);
    u32* d = nullptr;
    CPB_CUDA(cudaMallocAsync((void**)&d, 32 * k, st));
    cpb_status rc = launch_crh(leaf, (const u32*)in, leaf_len, d, k, st);
    if (rc == CPB_OK)
        rc = update_digests_dev(node, (u32*)leaf_nodes, (u32*)non_leaf_nodes, n, indexes, d, k, (const u32*)asserted_root, applied, st);
    cudaFreeAsync(d, st);
    return rc;
}

cpb_status check_dev_args(cpb_poseidon_ctx* leaf, cpb_poseidon_ctx* node, uint64_t* leaf_nodes, uint64_t* non_leaf_nodes, size_t n,
                          const uint64_t* indexes, const uint64_t* in, size_t in_elems, size_t k) {
    CPB_TRY(check_update_shape(n, k));
    if (!leaf_nodes || !non_leaf_nodes || (k && !indexes) || (k && in_elems && !in)) return fail(CPB_NULL_POINTER, "null buffer");
    return check_update_ctxs(leaf, node);
}

// Host arrays: upd_host_form (merkle_update_kernels.cuh) around the _dev form.
cpb_status update_host(cpb_poseidon_ctx* leaf, cpb_poseidon_ctx* node, uint64_t* leaf_nodes, uint64_t* non_leaf_nodes, size_t n,
                       const uint64_t* indexes, const uint64_t* in, size_t leaf_len, size_t k, const uint64_t* asserted_root, int* applied) {
    const size_t in_elems = leaf ? leaf_len : 1;
    CPB_TRY(check_update_shape(n, k));
    if (!leaf_nodes || !non_leaf_nodes || (k && !indexes) || (k && in_elems && !in)) return fail(CPB_NULL_POINTER, "null buffer");
    for (size_t j = 0; j < k; j++)
        if (indexes[j] >= n) return fail(CPB_BAD_PARAMS, "index %llu out of range (%zu leaves)", (unsigned long long)indexes[j], n);
    CPB_TRY(check_update_ctxs(leaf, node));
    if (k == 0) {
        if (applied) *applied = !asserted_root || memcmp(non_leaf_nodes, asserted_root, 32) == 0;
        return CPB_OK;
    }
    return upd_host_form<8>(node, leaf_nodes, non_leaf_nodes, n, indexes, in, 32 * k * in_elems, k, asserted_root, applied,
                            [&](uint64_t* ml, uint64_t* mn, const uint64_t* d_idx, const void* d_in, const uint64_t* d_root, uint8_t* d_applied,
                                cudaStream_t st) {
                                return update_dev(leaf, node, ml, mn, n, d_idx, (const uint64_t*)d_in, leaf_len, k, d_root, d_applied, st);
                            });
}

}  // namespace
}  // namespace cpb

using namespace cpb;

extern "C" {

cpb_status cpb_merkle_poseidon_update_digests_dev(cpb_poseidon_ctx* node_ctx, uint64_t* leaf_nodes, uint64_t* non_leaf_nodes, size_t n,
                                                  const uint64_t* indexes, const uint64_t* new_leaf_digests, size_t k,
                                                  const uint64_t* asserted_root, uint8_t* applied, void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_dev_args(nullptr, node_ctx, leaf_nodes, non_leaf_nodes, n, indexes, new_leaf_digests, 1, k));
    DeviceGuard g(node_ctx->device);
    return update_dev(nullptr, node_ctx, leaf_nodes, non_leaf_nodes, n, indexes, new_leaf_digests, 0, k, asserted_root, applied,
                      (cudaStream_t)stream);
    });
}

cpb_status cpb_merkle_poseidon_update_dev(cpb_poseidon_ctx* leaf_ctx, cpb_poseidon_ctx* node_ctx, uint64_t* leaf_nodes, uint64_t* non_leaf_nodes,
                                          size_t n, const uint64_t* indexes, const uint64_t* new_leaves, size_t leaf_len, size_t k,
                                          const uint64_t* asserted_root, uint8_t* applied, void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    if (!leaf_ctx) return fail(CPB_NULL_POINTER, "null context");
    CPB_TRY(check_dev_args(leaf_ctx, node_ctx, leaf_nodes, non_leaf_nodes, n, indexes, new_leaves, leaf_len, k));
    DeviceGuard g(node_ctx->device);
    return update_dev(leaf_ctx, node_ctx, leaf_nodes, non_leaf_nodes, n, indexes, new_leaves, leaf_len, k, asserted_root, applied,
                      (cudaStream_t)stream);
    });
}

cpb_status cpb_merkle_poseidon_update_digests(cpb_poseidon_ctx* node_ctx, uint64_t* leaf_nodes, uint64_t* non_leaf_nodes, size_t n,
                                              const uint64_t* indexes, const uint64_t* new_leaf_digests, size_t k, const uint64_t* asserted_root,
                                              int* applied) {
    return cpb::guarded([&]() -> cpb_status {
    return update_host(nullptr, node_ctx, leaf_nodes, non_leaf_nodes, n, indexes, new_leaf_digests, 0, k, asserted_root, applied);
    });
}

cpb_status cpb_merkle_poseidon_update(cpb_poseidon_ctx* leaf_ctx, cpb_poseidon_ctx* node_ctx, uint64_t* leaf_nodes, uint64_t* non_leaf_nodes,
                                      size_t n, const uint64_t* indexes, const uint64_t* new_leaves, size_t leaf_len, size_t k,
                                      const uint64_t* asserted_root, int* applied) {
    return cpb::guarded([&]() -> cpb_status {
    if (!leaf_ctx) return fail(CPB_NULL_POINTER, "null context");
    return update_host(leaf_ctx, node_ctx, leaf_nodes, non_leaf_nodes, n, indexes, new_leaves, leaf_len, k, asserted_root, applied);
    });
}

}  // extern "C"
