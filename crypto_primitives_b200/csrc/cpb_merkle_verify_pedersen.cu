// cpb_merkle_verify_pedersen.cu -- n x Path::verify (R/merkle_tree/mod.rs:172-212) against one root for the two trees with a Pedersen
// leaf hash (include/cpb200.h, "Merkle path verification (Pedersen leaves)"):
//   byte tree  (cpb_merkle_pedersen_build: pedersen::CRH leaves, ByteDigestConverter, pedersen::TwoToOneCRH nodes)
//     leaf     the leaf context's hash launch (launch_hash, mode 0) writes every claimed leaf digest, affine (x, y), into pool scratch
//     level j  for j = 0 .. path_len: k_ped_verify_rows, one thread per proof, writes the 128-byte TwoToOneCRH row of the current
//              digest and the level's sibling (ped_verify_row), then the node context's hash launch over the rows
//              (two_to_one_len bytes of each, as the build hashes them) overwrites the current digests
//     compare  k_ped_verify_cmp: ok[i] = both coordinates equal the root's
//   mixed tree (cpb_merkle_mixed_build: PedersenCRHCompressor leaves, poseidon::TwoToOneCRH nodes)
//     leaf     the leaf context's hash launch, mode 1 (x-coordinates), into pool scratch
//     fold     ONE launch of k_poseidon_verify_digests (poseidon_kernels.cuh), one thread per proof
// Every level of a batch has width n, so the byte tree takes one grid per level: 3 path_len + 6 launches, the mixed tree 3, for
// any n.  Scratch comes from the stream-ordered pool; nothing synchronises the host.
#include "merkle_verify_pedersen.cuh"
#include "pedersen_internal.cuh"
#include "poseidon_kernels.cuh"

namespace cpb {

CPB_POS_WIDTHS(CPB_POS_EXTERN_DIGESTS, Bls12_381_Fr)
CPB_POS_WIDTHS(CPB_POS_EXTERN_DIGESTS, Bls12_377_Fr)

namespace {

constexpr int kVerBlock = 256;

unsigned ver_grid(size_t n) { return (unsigned)((n + kVerBlock - 1) / kVerBlock); }

template <class F>
__global__ void __launch_bounds__(kVerBlock)
k_ped_verify_rows(const u32* __restrict__ cur, const u32* __restrict__ leaf_sibs, const u32* __restrict__ paths, int plen, int j,
                  const unsigned long long* __restrict__ indexes, u32* __restrict__ rows, long n) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ped_verify_row<F>(rows + 32 * i, cur + 16 * i, leaf_sibs, paths, (u64)i, plen, j, indexes[i]);
}

__global__ void __launch_bounds__(kVerBlock)
k_ped_verify_cmp(const u32* __restrict__ cur, const u32* __restrict__ root, unsigned char* __restrict__ ok, long n) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    u32 d = 0;
#pragma unroll
    for (int w = 0; w < 16; w++) d |= cur[16 * i + w] ^ root[w];
    ok[i] = d == 0 ? 1 : 0;
}

cpb_status launch_rows(const cpb_pedersen_ctx* node, const u32* cur, const u32* leaf_sibs, const u32* paths, int plen, int j,
                       const unsigned long long* indexes, u32* rows, size_t n, cudaStream_t st) {
    switch (node->field_id) {
        case CPB_BLS12_381_FR:
            k_ped_verify_rows<Bls12_381_Fr><<<ver_grid(n), kVerBlock, 0, st>>>(cur, leaf_sibs, paths, plen, j, indexes, rows, (long)n);
            break;
        case CPB_BLS12_377_FR:
            k_ped_verify_rows<Bls12_377_Fr><<<ver_grid(n), kVerBlock, 0, st>>>(cur, leaf_sibs, paths, plen, j, indexes, rows, (long)n);
            break;
        default: return fail(CPB_UNSUPPORTED, "no kernel for base field %d", node->field_id);
    }
    CPB_CUDA(cudaGetLastError());
    return CPB_OK;
}

#define CPB_DIGESTS_T(F)                                                                                                  \
    switch (node->dev.t) {                                                                                                \
        case 2: return launch_verify_digests_ft<F, 2>(node, root, digests, sibs, paths, plen, indexes, ok, n, st);        \
        case 3: return launch_verify_digests_ft<F, 3>(node, root, digests, sibs, paths, plen, indexes, ok, n, st);        \
        case 4: return launch_verify_digests_ft<F, 4>(node, root, digests, sibs, paths, plen, indexes, ok, n, st);        \
        case 5: return launch_verify_digests_ft<F, 5>(node, root, digests, sibs, paths, plen, indexes, ok, n, st);        \
        case 6: return launch_verify_digests_ft<F, 6>(node, root, digests, sibs, paths, plen, indexes, ok, n, st);        \
        case 7: return launch_verify_digests_ft<F, 7>(node, root, digests, sibs, paths, plen, indexes, ok, n, st);        \
        case 8: return launch_verify_digests_ft<F, 8>(node, root, digests, sibs, paths, plen, indexes, ok, n, st);        \
        case 9: return launch_verify_digests_ft<F, 9>(node, root, digests, sibs, paths, plen, indexes, ok, n, st);        \
    }                                                                                                                     \
    break;

cpb_status launch_verify_digests(cpb_poseidon_ctx* node, const u32* root, const u32* digests, const u32* sibs, const u32* paths, int plen,
                                 const unsigned long long* indexes, unsigned char* ok, size_t n, cudaStream_t st) {
    switch (node->field_id) {
        case CPB_BLS12_381_FR: CPB_DIGESTS_T(Bls12_381_Fr)
        case CPB_BLS12_377_FR: CPB_DIGESTS_T(Bls12_377_Fr)
        default: return fail(CPB_UNSUPPORTED, "no kernel for base field %d", node->field_id);
    }
    return fail(CPB_UNSUPPORTED, "state width t=%d is not built (this library: t = 2..9)", node->dev.t);
}
#undef CPB_DIGESTS_T

// ---- device code of both trees (every pointer device memory; arguments already checked, n > 0)
cpb_status verify_bytes_dev(cpb_pedersen_ctx* leaf, cpb_pedersen_ctx* node, const u32* root, const uint8_t* leaves, size_t leaf_len,
                            size_t leaf_stride, const u32* leaf_sibs, const u32* paths, int plen, const unsigned long long* indexes,
                            unsigned char* ok, size_t n, cudaStream_t st) {
    const size_t row_len = two_to_one_len(node);
    u32* cur = nullptr;
    CPB_CUDA(cudaMallocAsync((void**)&cur, 64 * n + 128 * n, st));          // n digests (x, y), then n rows of 128 bytes
    u32* rows = cur + 16 * n;
    auto run = [&]() -> cpb_status {
        CPB_TRY(launch_hash(leaf, leaves, leaf_len, leaf_stride, nullptr, cur, n, 0, st));
        for (int j = 0; j <= plen; j++) {
            CPB_TRY(launch_rows(node, cur, leaf_sibs, paths, plen, j, indexes, rows, n, st));
            CPB_TRY(launch_hash(node, (const uint8_t*)rows, row_len, 128, nullptr, cur, n, 0, st));
        }
        k_ped_verify_cmp<<<ver_grid(n), kVerBlock, 0, st>>>(cur, root, ok, (long)n);
        CPB_CUDA(cudaGetLastError());
        return CPB_OK;
    };
    const cpb_status rc = run();
    cudaFreeAsync(cur, st);
    return rc;
}

cpb_status verify_mixed_dev(cpb_pedersen_ctx* leaf, cpb_poseidon_ctx* node, const u32* root, const uint8_t* leaves, size_t leaf_len,
                            size_t leaf_stride, const u32* leaf_sibs, const u32* paths, int plen, const unsigned long long* indexes,
                            unsigned char* ok, size_t n, cudaStream_t st) {
    u32* d = nullptr;
    CPB_CUDA(cudaMallocAsync((void**)&d, 32 * n, st));
    cpb_status rc = launch_hash(leaf, leaves, leaf_len, leaf_stride, nullptr, d, n, 1, st);
    if (rc == CPB_OK) rc = launch_verify_digests(node, root, d, leaf_sibs, paths, plen, indexes, ok, n, st);
    cudaFreeAsync(d, st);
    return rc;
}

// ---- argument rules, in the order include/cpb200.h states: shape, buffers, contexts, lengths
cpb_status check_shape(size_t path_len, size_t leaf_len, size_t leaf_stride, size_t n, bool strided) {
    if (path_len > 62) return fail(CPB_BAD_PARAMS, "path too long (%zu > 62)", path_len);
    if (strided && n > 1 && leaf_stride < leaf_len) return fail(CPB_BAD_PARAMS, "leaf_stride < leaf_len");
    return CPB_OK;
}
cpb_status check_buffers(const void* root, const void* leaves, size_t leaf_len, const void* leaf_sibs, const void* paths, size_t path_len,
                         const void* indexes, const void* ok, size_t n) {
    if (n && (!root || (!leaves && leaf_len) || !leaf_sibs || (!paths && path_len) || !indexes || !ok))
        return fail(CPB_NULL_POINTER, "null buffer");
    return CPB_OK;
}
cpb_status check_bytes_ctxs(cpb_pedersen_ctx* leaf, cpb_pedersen_ctx* node, size_t leaf_len) {
    if (!leaf || !node) return fail(CPB_NULL_POINTER, "null context");
    if (leaf->device != node->device || leaf->field_id != node->field_id)
        return fail(CPB_BAD_PARAMS, "leaf and node contexts must share device and curve");
    CPB_TRY(check_len(leaf, leaf_len, false));
    return check_len(node, two_to_one_len(node), false);
}
cpb_status check_mixed_ctxs(cpb_pedersen_ctx* leaf, cpb_poseidon_ctx* node, size_t leaf_len) {
    if (!leaf || !node) return fail(CPB_NULL_POINTER, "null context");
    if (node->field_id != leaf->field_id || node->device != leaf->device)
        return fail(CPB_BAD_PARAMS, "the Poseidon field must be the curve's base field, on the same device");
    if (node->dev.rate < 2) return fail(CPB_UNSUPPORTED, "two-to-one with rate < 2 not supported");
    return check_len(leaf, leaf_len, false);
}

// Host forms: the proofs go up through the leaf context's arena, on its stream under its mutex, the device code runs there, ok comes back.  `dw`: words of
// one digest (16: affine point, 8: field element).
template <class Dev>
cpb_status verify_host(cpb_pedersen_ctx* leaf, size_t dw, const uint64_t* root, const uint8_t* leaves, size_t leaf_len,
                       const uint64_t* leaf_sibs, const uint64_t* paths, size_t path_len, const uint64_t* indexes, uint8_t* ok, size_t n,
                       Dev&& dev) {
    std::lock_guard<std::mutex> lk(leaf->mu);
    DeviceGuard g(leaf->device);
    HostStage S(leaf->arena, leaf->stream);
    const size_t db = 4 * dw;
    const size_t o_root = S.in(root, db), o_leaves = S.in(leaves, n * leaf_len), o_sib = S.in(leaf_sibs, n * db),
                 o_path = S.in(paths, n * path_len * db), o_idx = S.in(indexes, n * 8), o_ok = S.out(ok, n);
    CPB_TRY(S.upload());
    CPB_TRY(dev(S.at<u32>(o_root), S.at<uint8_t>(o_leaves), S.at<u32>(o_sib), S.at<u32>(o_path), S.at<unsigned long long>(o_idx),
                S.at<unsigned char>(o_ok), leaf->stream));
    return S.download();
}

}  // namespace
}  // namespace cpb

using namespace cpb;

extern "C" {

cpb_status cpb_merkle_pedersen_verify_batch_dev(cpb_pedersen_ctx* leaf_ctx, cpb_pedersen_ctx* node_ctx, const uint64_t* root_xy,
                                                const uint8_t* leaves, size_t leaf_len, size_t leaf_stride,
                                                const uint64_t* leaf_sibling_hashes_xy, const uint64_t* auth_paths_xy, size_t path_len,
                                                const uint64_t* leaf_indexes, uint8_t* ok, size_t n, void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_shape(path_len, leaf_len, leaf_stride, n, true));
    CPB_TRY(check_buffers(root_xy, leaves, leaf_len, leaf_sibling_hashes_xy, auth_paths_xy, path_len, leaf_indexes, ok, n));
    CPB_TRY(check_bytes_ctxs(leaf_ctx, node_ctx, leaf_len));
    if (n == 0) return CPB_OK;
    DeviceGuard g(leaf_ctx->device);
    return verify_bytes_dev(leaf_ctx, node_ctx, (const u32*)root_xy, leaves, leaf_len, leaf_stride, (const u32*)leaf_sibling_hashes_xy,
                            (const u32*)auth_paths_xy, (int)path_len, (const unsigned long long*)leaf_indexes, ok, n, (cudaStream_t)stream);
    });
}

cpb_status cpb_merkle_pedersen_verify_batch(cpb_pedersen_ctx* leaf_ctx, cpb_pedersen_ctx* node_ctx, const uint64_t* root_xy,
                                            const uint8_t* leaves, size_t leaf_len, const uint64_t* leaf_sibling_hashes_xy,
                                            const uint64_t* auth_paths_xy, size_t path_len, const uint64_t* leaf_indexes, uint8_t* ok,
                                            size_t n) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_shape(path_len, leaf_len, leaf_len, n, false));
    CPB_TRY(check_buffers(root_xy, leaves, leaf_len, leaf_sibling_hashes_xy, auth_paths_xy, path_len, leaf_indexes, ok, n));
    CPB_TRY(check_bytes_ctxs(leaf_ctx, node_ctx, leaf_len));
    if (n == 0) return CPB_OK;
    return verify_host(leaf_ctx, 16, root_xy, leaves, leaf_len, leaf_sibling_hashes_xy, auth_paths_xy, path_len, leaf_indexes, ok, n,
                       [&](const u32* root, const uint8_t* lv, const u32* sib, const u32* paths, const unsigned long long* idx,
                           unsigned char* d_ok, cudaStream_t st) {
                           return verify_bytes_dev(leaf_ctx, node_ctx, root, lv, leaf_len, leaf_len, sib, paths, (int)path_len, idx, d_ok,
                                                   n, st);
                       });
    });
}

cpb_status cpb_merkle_mixed_verify_batch_dev(cpb_pedersen_ctx* leaf_ctx, cpb_poseidon_ctx* node_ctx, const uint64_t* root,
                                             const uint8_t* leaves, size_t leaf_len, size_t leaf_stride, const uint64_t* leaf_sibling_hashes,
                                             const uint64_t* auth_paths, size_t path_len, const uint64_t* leaf_indexes, uint8_t* ok, size_t n,
                                             void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_shape(path_len, leaf_len, leaf_stride, n, true));
    CPB_TRY(check_buffers(root, leaves, leaf_len, leaf_sibling_hashes, auth_paths, path_len, leaf_indexes, ok, n));
    CPB_TRY(check_mixed_ctxs(leaf_ctx, node_ctx, leaf_len));
    if (n == 0) return CPB_OK;
    DeviceGuard g(leaf_ctx->device);
    return verify_mixed_dev(leaf_ctx, node_ctx, (const u32*)root, leaves, leaf_len, leaf_stride, (const u32*)leaf_sibling_hashes,
                            (const u32*)auth_paths, (int)path_len, (const unsigned long long*)leaf_indexes, ok, n, (cudaStream_t)stream);
    });
}

cpb_status cpb_merkle_mixed_verify_batch(cpb_pedersen_ctx* leaf_ctx, cpb_poseidon_ctx* node_ctx, const uint64_t* root,
                                         const uint8_t* leaves, size_t leaf_len, const uint64_t* leaf_sibling_hashes,
                                         const uint64_t* auth_paths, size_t path_len, const uint64_t* leaf_indexes, uint8_t* ok, size_t n) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_shape(path_len, leaf_len, leaf_len, n, false));
    CPB_TRY(check_buffers(root, leaves, leaf_len, leaf_sibling_hashes, auth_paths, path_len, leaf_indexes, ok, n));
    CPB_TRY(check_mixed_ctxs(leaf_ctx, node_ctx, leaf_len));
    if (n == 0) return CPB_OK;
    return verify_host(leaf_ctx, 8, root, leaves, leaf_len, leaf_sibling_hashes, auth_paths, path_len, leaf_indexes, ok, n,
                       [&](const u32* r, const uint8_t* lv, const u32* sib, const u32* paths, const unsigned long long* idx,
                           unsigned char* d_ok, cudaStream_t st) {
                           return verify_mixed_dev(leaf_ctx, node_ctx, r, lv, leaf_len, leaf_len, sib, paths, (int)path_len, idx, d_ok, n,
                                                   st);
                       });
    });
}

}  // extern "C"
