// cpb_multi.cu -- multi-GPU Merkle build behind the C-ABI (include/cpb200.h, "Merkle tree across several GPUs").
//
// A tree over N leaves on G = 2^g GPUs is G independent subtrees over contiguous leaf ranges plus a g-level top
// (the reference has no distributed path: MerkleTree::new, R/merkle_tree/mod.rs:411-523, is one process).  Two ways to
// drive it, same kernels:
//
//   * one process per GPU (torchrun): cpb_exchange_* + cpb_merkle_*_build_sharded*.  Every rank owns a small device
//     buffer (`cpb_exchange`) that its peers map through CUDA IPC; the last kernel of the local build
//     (k_poseidon_tree_top) pushes the local root into every peer's buffer over NVLink, waits for the peers' roots
//     and computes the g replicated top levels -- compute, exchange and top in ONE launch, no host round trip.
//   * one process, several GPUs (a Rust host): cpb_multi_create + cpb_merkle_poseidon_build_multi.  The exchange is
//     the same fused kernel over peer-enabled pointers, or -- CPB_MULTI_EXCHANGE=nccl, or when peer access is not
//     available -- one ncclAllGather of the G roots (ncclCommInitAll; libnccl is dlopen'ed on first use so the library
//     itself has no link-time NCCL dependency), followed by the same top-level code.
#include <dlfcn.h>

#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include "poseidon_kernels.cuh"

using namespace cpb;

// ------------------------------------------------------------------------------ NCCL, resolved at run time
namespace {

typedef struct ncclComm* nccl_comm_t;
struct NcclApi {
    void* handle = nullptr;
    int (*CommInitAll)(nccl_comm_t*, int, const int*) = nullptr;
    int (*CommDestroy)(nccl_comm_t) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, nccl_comm_t, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
    bool ok = false;
};
NcclApi& nccl() {
    static NcclApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        for (const char* name : {"libnccl.so.2", "libnccl.so"}) {
            api.handle = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
            if (api.handle) break;
        }
        if (!api.handle) return;
#define CPB_NCCL_SYM(field, sym) *(void**)(&api.field) = dlsym(api.handle, sym)
        CPB_NCCL_SYM(CommInitAll, "ncclCommInitAll");
        CPB_NCCL_SYM(CommDestroy, "ncclCommDestroy");
        CPB_NCCL_SYM(GroupStart, "ncclGroupStart");
        CPB_NCCL_SYM(GroupEnd, "ncclGroupEnd");
        CPB_NCCL_SYM(AllGather, "ncclAllGather");
        CPB_NCCL_SYM(GetErrorString, "ncclGetErrorString");
#undef CPB_NCCL_SYM
        api.ok = api.CommInitAll && api.CommDestroy && api.GroupStart && api.GroupEnd && api.AllGather && api.GetErrorString;
    });
    return api;
}
#define CPB_NCCL(call)                                                                                              \
    do {                                                                                                            \
        int r__ = (call);                                                                                           \
        if (r__ != 0) return cpb::fail(CPB_NCCL_ERROR, "%s failed: %s", #call, nccl().GetErrorString(r__));         \
    } while (0)

int log2_exact(size_t n) {
    int l = 0;
    while (((size_t)1 << l) < n) l++;
    return ((size_t)1 << l) == n ? l : -1;
}

}  // namespace

// ------------------------------------------------------------------------------ exchange object
struct cpb_exchange {
    int device = 0, world = 1, rank = 0;
    void* base = nullptr;                       // [2][world] digests (32 B) | [2][world] flags (8 B)
    size_t bytes = 0;
    u32* peer_slots[kMaxPeers] = {};
    unsigned long long* peer_flags[kMaxPeers] = {};
    void* ipc_opened[kMaxPeers] = {};           // bases opened with cudaIpcOpenMemHandle (closed on destroy)
    bool connected = false;
    unsigned long long epoch = 0;               // calls so far; every rank issues its calls in the same order
    std::mutex mu;

    size_t flags_offset() const { return (size_t)2 * world * 32; }
    void set_peer(int p, void* peer_base) {
        peer_slots[p] = (u32*)peer_base;
        peer_flags[p] = (unsigned long long*)((char*)peer_base + flags_offset());
    }
    // Device-side view for the next call (advances the epoch).  top_out: (world - 1) digests on this device.
    ExchangeDev next(u32* top_out) {
        std::lock_guard<std::mutex> lk(mu);
        ExchangeDev X;
        X.world = world; X.rank = rank; X.epoch = ++epoch; X.top_out = top_out;
        for (int p = 0; p < world; p++) { X.slots[p] = peer_slots[p]; X.flags[p] = peer_flags[p]; }
        return X;
    }
};

namespace {
cpb_status check_exchange(const cpb_exchange* ex, const cpb_poseidon_ctx* node) {
    if (!ex) return fail(CPB_NULL_POINTER, "null exchange");
    if (!ex->connected) return fail(CPB_BAD_PARAMS, "exchange is not connected (cpb_exchange_connect_ipc / _local)");
    if (node && node->device != ex->device) return fail(CPB_BAD_PARAMS, "context and exchange live on different devices");
    return CPB_OK;
}
}  // namespace

extern "C" {

cpb_status cpb_exchange_create(int device, int world, int rank, cpb_exchange** out) {
    return cpb::guarded([&]() -> cpb_status {
    if (!out) return fail(CPB_NULL_POINTER, "null out");
    *out = nullptr;
    if (world < 1 || world > kMaxPeers || (world & (world - 1)) || rank < 0 || rank >= world)
        return fail(CPB_BAD_PARAMS, "world must be a power of two <= %d and 0 <= rank < world (got %d, %d)", kMaxPeers, world, rank);
    DeviceGuard g(device);
    if (!g.ok) { cudaGetLastError(); return fail(CPB_NO_DEVICE, "cudaSetDevice(%d) failed", device); }
    cpb_exchange* ex = new cpb_exchange();
    ex->device = device; ex->world = world; ex->rank = rank;
    ex->bytes = (size_t)2 * world * 32 + (size_t)2 * world * 8;
    cudaError_t e = cudaMalloc(&ex->base, ex->bytes);
    if (e == cudaSuccess) e = cudaMemset(ex->base, 0, ex->bytes);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) {
        if (ex->base) cudaFree(ex->base);
        delete ex;
        return fail(CPB_CUDA_ERROR, "exchange buffer: %s", cudaGetErrorString(e));
    }
    ex->set_peer(rank, ex->base);
    ex->connected = world == 1;
    *out = ex;
    return CPB_OK;
    });
}

void cpb_exchange_destroy(cpb_exchange* ex) {
    if (!ex) return;
    DeviceGuard g(ex->device);
    cudaDeviceSynchronize();
    for (int p = 0; p < ex->world; p++)
        if (ex->ipc_opened[p]) cudaIpcCloseMemHandle(ex->ipc_opened[p]);
    if (ex->base) cudaFree(ex->base);
    delete ex;
}

int cpb_exchange_world(const cpb_exchange* ex) { return ex ? ex->world : 0; }
int cpb_exchange_rank(const cpb_exchange* ex) { return ex ? ex->rank : -1; }

cpb_status cpb_exchange_ipc_handle(cpb_exchange* ex, uint8_t handle_out[64]) {
    return cpb::guarded([&]() -> cpb_status {
    if (!ex || !handle_out) return fail(CPB_NULL_POINTER, "null argument");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handles are 64 bytes");
    DeviceGuard g(ex->device);
    cudaIpcMemHandle_t h;
    CPB_CUDA(cudaIpcGetMemHandle(&h, ex->base));
    memcpy(handle_out, &h, 64);
    return CPB_OK;
    });
}

cpb_status cpb_exchange_connect_ipc(cpb_exchange* ex, const uint8_t* handles) {
    return cpb::guarded([&]() -> cpb_status {
    if (!ex || !handles) return fail(CPB_NULL_POINTER, "null argument");
    DeviceGuard g(ex->device);
    for (int p = 0; p < ex->world; p++) {
        if (p == ex->rank || ex->ipc_opened[p]) continue;
        cudaIpcMemHandle_t h;
        memcpy(&h, handles + 64 * p, 64);
        void* ptr = nullptr;
        CPB_CUDA(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
        ex->ipc_opened[p] = ptr;
        ex->set_peer(p, ptr);
    }
    ex->connected = true;
    return CPB_OK;
    });
}

cpb_status cpb_exchange_connect_local(cpb_exchange** all, int world) {
    return cpb::guarded([&]() -> cpb_status {
    if (!all) return fail(CPB_NULL_POINTER, "null argument");
    for (int r = 0; r < world; r++)
        if (!all[r] || all[r]->world != world || all[r]->rank != r) return fail(CPB_BAD_PARAMS, "exchange %d does not belong to this group", r);
    for (int r = 0; r < world; r++) {
        DeviceGuard g(all[r]->device);
        for (int p = 0; p < world; p++) {
            if (p == r) continue;
            if (all[p]->device != all[r]->device) {
                int can = 0;
                CPB_CUDA(cudaDeviceCanAccessPeer(&can, all[r]->device, all[p]->device));
                if (!can) return fail(CPB_UNSUPPORTED, "device %d cannot access device %d (no peer access)", all[r]->device, all[p]->device);
                cudaError_t e = cudaDeviceEnablePeerAccess(all[p]->device, 0);
                if (e == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
                else if (e != cudaSuccess) return fail(CPB_CUDA_ERROR, "cudaDeviceEnablePeerAccess: %s", cudaGetErrorString(e));
            }
            all[r]->set_peer(p, all[p]->base);
        }
        all[r]->connected = true;
    }
    return CPB_OK;
    });
}

// ---- sharded builds: this rank's subtree + fused root exchange + replicated top
cpb_status cpb_merkle_poseidon_from_digests_sharded_dev(cpb_poseidon_ctx* node, cpb_exchange* ex, const uint64_t* leaf_digests, size_t n_local,
                                                        uint64_t* non_leaf_nodes, uint64_t* top_nodes, void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_ctx(node));
    CPB_TRY(check_exchange(ex, node));
    if (!pow2_gt1(n_local)) return fail(CPB_NOT_POW2, "the local leaf count should be a power of two greater than one (got %zu)", n_local);
    if (node->dev.rate < 2) return fail(CPB_UNSUPPORTED, "two-to-one with rate < 2 not supported");
    if (ex->world > 1 && !top_nodes) return fail(CPB_NULL_POINTER, "null top_nodes");
    DeviceGuard g(node->device);
    if (ex->world == 1) return merkle_build_streams(node, node, nullptr, 0, n_local, (u32*)leaf_digests, (u32*)non_leaf_nodes, (cudaStream_t)stream);
    ExchangeDev X = ex->next((u32*)top_nodes);
    return merkle_build_streams(node, node, nullptr, 0, n_local, (u32*)leaf_digests, (u32*)non_leaf_nodes, (cudaStream_t)stream, nullptr, &X);
    });
}

cpb_status cpb_merkle_poseidon_build_sharded_dev(cpb_poseidon_ctx* leaf, cpb_poseidon_ctx* node, cpb_exchange* ex, const uint64_t* leaves,
                                                 size_t leaf_len, size_t n_local, uint64_t* leaf_nodes, uint64_t* non_leaf_nodes,
                                                 uint64_t* top_nodes, void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_ctx(leaf));
    CPB_TRY(check_ctx(node));
    CPB_TRY(check_exchange(ex, node));
    if (leaf->device != node->device || leaf->field_id != node->field_id) return fail(CPB_BAD_PARAMS, "leaf and node contexts must share device and field");
    if (!pow2_gt1(n_local)) return fail(CPB_NOT_POW2, "the local leaf count should be a power of two greater than one (got %zu)", n_local);
    if (node->dev.rate < 2) return fail(CPB_UNSUPPORTED, "two-to-one with rate < 2 not supported");
    if (ex->world > 1 && !top_nodes) return fail(CPB_NULL_POINTER, "null top_nodes");
    DeviceGuard g(leaf->device);
    if (ex->world == 1)
        return merkle_build_streams(leaf, node, (const u32*)leaves, leaf_len, n_local, (u32*)leaf_nodes, (u32*)non_leaf_nodes, (cudaStream_t)stream);
    ExchangeDev X = ex->next((u32*)top_nodes);
    return merkle_build_streams(leaf, node, (const u32*)leaves, leaf_len, n_local, (u32*)leaf_nodes, (u32*)non_leaf_nodes, (cudaStream_t)stream,
                                nullptr, &X);
    });
}

// Host-pointer form: this rank's leaves in, its leaf digests / subtree nodes (local heap order) / the replicated top out.
cpb_status cpb_merkle_poseidon_build_sharded(cpb_poseidon_ctx* leaf, cpb_poseidon_ctx* node, cpb_exchange* ex, const uint64_t* leaves,
                                             size_t leaf_len, size_t n_local, uint64_t* leaf_nodes, uint64_t* non_leaf_nodes,
                                             uint64_t* top_nodes) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_ctx(leaf));
    CPB_TRY(check_ctx(node));
    CPB_TRY(check_exchange(ex, node));
    if (leaf->device != node->device || leaf->field_id != node->field_id) return fail(CPB_BAD_PARAMS, "leaf and node contexts must share device and field");
    if (!pow2_gt1(n_local)) return fail(CPB_NOT_POW2, "the local leaf count should be a power of two greater than one (got %zu)", n_local);
    if (node->dev.rate < 2) return fail(CPB_UNSUPPORTED, "two-to-one with rate < 2 not supported");
    if ((!leaves && leaf_len) || !leaf_nodes || !non_leaf_nodes || (ex->world > 1 && !top_nodes)) return fail(CPB_NULL_POINTER, "null buffer");
    std::lock_guard<std::mutex> lk(leaf->mu);
    DeviceGuard g(leaf->device);
    cudaStream_t st = leaf->stream;
    HostStage S(leaf->arena, st);        // the leaves and levels move through MerkleHost; only the replicated top comes back here
    const size_t o_in = S.dev(n_local * leaf_len * 32), o_leaf = S.dev(n_local * 32), o_nodes = S.dev((n_local - 1) * 32),
                 o_top = S.out(top_nodes, (size_t)(ex->world - 1) * 32);
    CPB_TRY(S.upload());
    MerkleHost H;
    H.leaves = (const u32*)leaves; H.leaf_nodes = (u32*)leaf_nodes; H.nodes = (u32*)non_leaf_nodes;
    if (ex->world == 1) {
        CPB_TRY(merkle_build_streams(leaf, node, S.at<u32>(o_in), leaf_len, n_local, S.at<u32>(o_leaf), S.at<u32>(o_nodes), st, &H));
    } else {
        ExchangeDev X = ex->next(S.at<u32>(o_top));
        CPB_TRY(merkle_build_streams(leaf, node, S.at<u32>(o_in), leaf_len, n_local, S.at<u32>(o_leaf), S.at<u32>(o_nodes), st, &H, &X));
    }
    return S.download();
    });
}

}  // extern "C"

// ------------------------------------------------------------------------------ one process, several GPUs
struct cpb_multi {
    int ndev = 0;
    std::vector<int> devices;
    std::vector<cpb_exchange*> ex;
    bool use_nccl = false;
    std::vector<nccl_comm_t> comms;
    std::vector<u32*> d_top;            // per device: (ndev - 1) digests
    std::mutex mu;
};

extern "C" {

cpb_status cpb_multi_create(int ndev, const int* devices, cpb_multi** out) {
    return cpb::guarded([&]() -> cpb_status {
    if (!out || !devices) return fail(CPB_NULL_POINTER, "null argument");
    *out = nullptr;
    if (ndev < 1 || ndev > kMaxPeers || (ndev & (ndev - 1))) return fail(CPB_BAD_PARAMS, "the number of devices must be a power of two <= %d (got %d)", kMaxPeers, ndev);
    for (int i = 0; i < ndev; i++)
        for (int j = 0; j < i; j++)
            if (devices[i] == devices[j]) return fail(CPB_BAD_PARAMS, "device %d listed twice", devices[i]);
    cpb_multi* m = new cpb_multi();
    m->ndev = ndev;
    m->devices.assign(devices, devices + ndev);
    m->ex.assign(ndev, nullptr);
    m->d_top.assign(ndev, nullptr);
    auto cleanup = [&](cpb_status rc) {
        for (int i = 0; i < ndev; i++) {
            if (m->d_top[i]) { DeviceGuard g(devices[i]); cudaFree(m->d_top[i]); }
            if (m->ex[i]) cpb_exchange_destroy(m->ex[i]);
        }
        delete m;
        return rc;
    };
    for (int i = 0; i < ndev; i++) {
        cpb_status rc = cpb_exchange_create(devices[i], ndev, i, &m->ex[i]);
        if (rc != CPB_OK) return cleanup(rc);
        DeviceGuard g(devices[i]);
        if (cudaMalloc((void**)&m->d_top[i], (size_t)(ndev > 1 ? ndev - 1 : 1) * 32) != cudaSuccess) return cleanup(fail(CPB_CUDA_ERROR, "cudaMalloc failed"));
    }
    const char* force = getenv("CPB_MULTI_EXCHANGE");
    bool want_nccl = force && !strcmp(force, "nccl");
    if (ndev > 1 && !want_nccl) {
        cpb_status rc = cpb_exchange_connect_local(m->ex.data(), ndev);
        if (rc == CPB_UNSUPPORTED && !(force && !strcmp(force, "p2p"))) want_nccl = true;     // no peer access: fall back to NCCL
        else if (rc != CPB_OK) return cleanup(rc);
    }
    if (ndev > 1 && want_nccl) {
        if (!nccl().ok) return cleanup(fail(CPB_NCCL_ERROR, "libnccl.so.2 could not be loaded"));
        m->comms.assign(ndev, nullptr);
        int r = nccl().CommInitAll(m->comms.data(), ndev, devices);
        if (r != 0) return cleanup(fail(CPB_NCCL_ERROR, "ncclCommInitAll failed: %s", nccl().GetErrorString(r)));
        for (int i = 0; i < ndev; i++) m->ex[i]->connected = true;      // slots are filled by ncclAllGather, not by peers
        m->use_nccl = true;
    }
    *out = m;
    return CPB_OK;
    });
}

void cpb_multi_destroy(cpb_multi* m) {
    if (!m) return;
    for (int i = 0; i < m->ndev; i++) {
        DeviceGuard g(m->devices[i]);
        cudaDeviceSynchronize();
        if (m->use_nccl && m->comms[i]) nccl().CommDestroy(m->comms[i]);
        if (m->d_top[i]) cudaFree(m->d_top[i]);
        if (m->ex[i]) cpb_exchange_destroy(m->ex[i]);
    }
    delete m;
}

int cpb_multi_uses_nccl(const cpb_multi* m) { return m && m->use_nccl ? 1 : 0; }

// MerkleTree::new over HOST arrays in the reference's layout, leaves sharded contiguously over the devices of `m`.
cpb_status cpb_merkle_poseidon_build_multi(cpb_multi* m, cpb_poseidon_ctx* const* leaf_ctxs, cpb_poseidon_ctx* const* node_ctxs,
                                           const uint64_t* leaves, size_t leaf_len, size_t n, uint64_t* leaf_nodes, uint64_t* non_leaf_nodes) {
    return cpb::guarded([&]() -> cpb_status {
    if (!m || !leaf_ctxs || !node_ctxs) return fail(CPB_NULL_POINTER, "null argument");
    if (!pow2_gt1(n)) return fail(CPB_NOT_POW2, "leaves.len() should be power of two and greater than one (got %zu)", n);
    if ((!leaves && leaf_len) || !leaf_nodes || !non_leaf_nodes) return fail(CPB_NULL_POINTER, "null buffer");
    const int G = m->ndev;
    const int g = log2_exact((size_t)G);
    if (n / G < 2) return fail(CPB_BAD_PARAMS, "%zu leaves are too few for %d devices (need >= 2 per device)", n, G);
    for (int d = 0; d < G; d++) {
        CPB_TRY(check_ctx(leaf_ctxs[d]));
        CPB_TRY(check_ctx(node_ctxs[d]));
        if (leaf_ctxs[d]->device != m->devices[d] || node_ctxs[d]->device != m->devices[d])
            return fail(CPB_BAD_PARAMS, "contexts of slot %d must live on device %d", d, m->devices[d]);
        if (leaf_ctxs[d]->field_id != node_ctxs[d]->field_id) return fail(CPB_BAD_PARAMS, "leaf and node contexts must share the field");
        if (node_ctxs[d]->dev.rate < 2) return fail(CPB_UNSUPPORTED, "two-to-one with rate < 2 not supported");
    }
    std::lock_guard<std::mutex> lk(m->mu);
    const size_t per = n / G;
    // One host thread per device: copies from / to pageable host memory block the issuing thread, and device d's last
    // kernel waits for the roots of all the others -- every device must be fed independently.
    std::vector<cpb_status> rcs((size_t)G, CPB_OK);
    std::vector<std::string> errs((size_t)G);
    auto work = [&](int d) -> cpb_status {
        cpb_poseidon_ctx* L = leaf_ctxs[d];
        std::lock_guard<std::mutex> lkd(L->mu);
        DeviceGuard gd(m->devices[d]);
        HostStage S(L->arena, L->stream);
        const size_t o_in = S.dev(per * leaf_len * 32), o_leaf = S.dev(per * 32), o_nodes = S.dev((per - 1) * 32);
        CPB_TRY(S.upload());
        MerkleHost H;
        H.leaves = (const u32*)leaves + 8 * leaf_len * (per * d);
        H.leaf_nodes = (u32*)leaf_nodes + 8 * (per * d);
        H.nodes = (u32*)non_leaf_nodes;
        H.g = g; H.rank = (size_t)d;
        const u32* d_leaves = S.at<u32>(o_in);
        u32 *d_ln = S.at<u32>(o_leaf), *d_nodes = S.at<u32>(o_nodes);
        if (G == 1 || m->use_nccl) {
            CPB_TRY(merkle_build_streams(L, node_ctxs[d], d_leaves, leaf_len, per, d_ln, d_nodes, L->stream, &H));
        } else {
            ExchangeDev X = m->ex[d]->next(m->d_top[d]);
            CPB_TRY(merkle_build_streams(L, node_ctxs[d], d_leaves, leaf_len, per, d_ln, d_nodes, L->stream, &H, &X));
        }
        if (G > 1 && m->use_nccl) {
            // one all-gather of the G subtree roots (32 B each) over NCCL, then the replicated top on this device
            CPB_NCCL(nccl().AllGather(d_nodes, m->ex[d]->base, 32, /*ncclChar*/ 0, m->comms[d], L->stream));
            CPB_TRY(merkle_build_streams(node_ctxs[d], node_ctxs[d], nullptr, 0, (size_t)G, (u32*)m->ex[d]->base, m->d_top[d], L->stream));
        }
        if (G > 1 && d == 0) CPB_CUDA(cudaMemcpyAsync(non_leaf_nodes, m->d_top[0], (size_t)(G - 1) * 32, cudaMemcpyDeviceToHost, L->stream));
        return S.download();
    };
    std::vector<std::thread> threads;
    for (int d = 0; d < G; d++)
        threads.emplace_back([&, d] {
            rcs[d] = cpb::guarded([&]() -> cpb_status { return work(d); });
            if (rcs[d] != CPB_OK) errs[d] = cpb_last_error();          // the message is thread-local: carry it over
        });
    for (auto& t : threads) t.join();
    for (int d = 0; d < G; d++)
        if (rcs[d] != CPB_OK) return fail(rcs[d], "device %d: %s", m->devices[d], errs[d].c_str());
    return CPB_OK;
    });
}

}  // extern "C"
