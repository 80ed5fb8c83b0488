"""Leaf-sharded Merkle build across the GPUs of one node (SURVEY.md §8e).

The reference has no distributed path: MerkleTree::new (R/merkle_tree/mod.rs:411-523) runs in one
process with one rayon barrier per level.  A height-h tree over N leaves on G = 2^g ranks is G
independent subtrees over contiguous leaf ranges plus a g-level top, so:

  1. rank k hashes leaves [k*N/G, (k+1)*N/G) and builds its whole local subtree on its own GPU
     (no communication);
  2. ONE all-gather of the G subtree roots (32 B each) over NCCL / NVLink;
  3. every rank computes the top g levels (G-1 hashes) redundantly -- cheaper than a second collective.

`gather="levels"` additionally all-gathers every level (and the leaf digests) so that each rank
holds the reference's complete `leaf_nodes` / `non_leaf_nodes` arrays: because the node array is
heap-ordered by level, rank k's nodes of global level l >= g are the k-th contiguous slice of
that level, so each level is one in-place all_gather_into_tensor -- no repacking.

Two exchanges for step 2.  `Exchange` (default on GPUs): every rank owns a small device buffer that its
peers map through CUDA IPC; the last kernel of the local build pushes the local root into every peer's buffer
over NVLink, waits for theirs and computes the top levels -- steps 1-3 are one chain of launches inside
libcpb200.so, with no host round trip and no collective call (csrc/cpb_multi.cu, k_poseidon_tree_top).
Without an Exchange the roots go through one torch.distributed all_gather (NCCL or gloo).

One process per GPU (torchrun); torch.distributed is plumbing only (rendezvous, IPC-handle exchange, the
optional level gather).  The hashing backend is injected so the sharding / collective logic can be
exercised on CPU with gloo (tests/test_dist_cpu.py).
"""
from __future__ import annotations

from dataclasses import dataclass

import torch
import torch.distributed as dist


class Exchange:
    """This rank's end of the fused root exchange (cpb_exchange, include/cpb200.h): created collectively by all ranks of
    `group`; the 64-byte CUDA-IPC handles travel through one all_gather."""

    def __init__(self, device_index: int, group=None):
        import ctypes as C
        from . import _native as N
        self.N = N
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.device = device_index
        h = N.vp()
        N.check(N.lib.cpb_exchange_create(device_index, self.world, self.rank, C.byref(h)))
        self.handle = h.value
        if self.world > 1:
            mine = (C.c_uint8 * 64)()
            N.check(N.lib.cpb_exchange_ipc_handle(self.handle, mine))
            dev = torch.device("cuda", device_index)
            src = torch.tensor(list(mine), dtype=torch.uint8, device=dev)
            allh = torch.empty(64 * self.world, dtype=torch.uint8, device=dev)
            dist.all_gather_into_tensor(allh, src, group=group)
            buf = (C.c_uint8 * (64 * self.world))(*allh.cpu().tolist())
            N.check(N.lib.cpb_exchange_connect_ipc(self.handle, buf))
            dist.barrier(group=group)

    def close(self):
        if getattr(self, "handle", None):
            self.N.lib.cpb_exchange_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _log2(n: int) -> int:
    assert n > 0 and n & (n - 1) == 0, "must be a power of two"
    return n.bit_length() - 1


class CudaPoseidonBackend:
    """Field-leaf tree: poseidon::CRH leaves + poseidon::TwoToOneCRH nodes on the current CUDA device.
    The returned tensors are workspaces owned by the backend: a later build with the same shape
    overwrites them (clone what must outlive the next call)."""

    digest_words = 4

    def __init__(self, leaf_params, node_params, device_index: int):
        from . import _native as N
        self.N = N
        self.dev = device_index
        self.leaf_ctx = leaf_params.context(device_index)
        self.node_ctx = node_params.context(device_index)
        self._ws = {}                      # output workspaces reused across builds (no allocator traffic per step)

    def _buf(self, key, shape, device):
        t = self._ws.get(key)
        if t is None or tuple(t.shape) != tuple(shape) or t.device != device:
            t = torch.empty(shape, dtype=torch.int64, device=device)
            self._ws[key] = t
        return t

    def _stream(self):
        return torch.cuda.current_stream().cuda_stream

    def build_local(self, leaves: torch.Tensor):
        """leaves (n, L, 4) int64 on the GPU -> (leaf_nodes (n,4), nodes (n-1,4)) heap order."""
        n, L = leaves.shape[0], leaves.shape[1]
        leaf_nodes = self._buf("leaf", (n, 4), leaves.device)
        nodes = self._buf("nodes", (n - 1, 4), leaves.device)
        self.N.check(self.N.lib.cpb_merkle_poseidon_build_dev(self.leaf_ctx, self.node_ctx, leaves.data_ptr(), L, n,
                                                              leaf_nodes.data_ptr(), nodes.data_ptr(), self._stream()))
        return leaf_nodes, nodes

    def build_sharded(self, leaves: torch.Tensor, ex: "Exchange"):
        """Local subtree + fused root exchange + replicated top in one chain of launches:
        -> (leaf_nodes (n,4), nodes (n-1,4) local heap order, top (world-1, 4))."""
        n, L = leaves.shape[0], leaves.shape[1]
        leaf_nodes = self._buf("leaf", (n, 4), leaves.device)
        nodes = self._buf("nodes", (n - 1, 4), leaves.device)
        top = self._buf("top", (max(ex.world - 1, 1), 4), leaves.device)
        self.N.check(self.N.lib.cpb_merkle_poseidon_build_sharded_dev(self.leaf_ctx, self.node_ctx, ex.handle, leaves.data_ptr(), L, n,
                                                                      leaf_nodes.data_ptr(), nodes.data_ptr(), top.data_ptr(), self._stream()))
        return leaf_nodes, nodes, top

    def hash_leaves(self, leaves: torch.Tensor):
        n, L = leaves.shape[0], leaves.shape[1]
        out = self._buf("leaf", (n, 4), leaves.device)
        self.N.check(self.N.lib.cpb_poseidon_crh_batch_dev(self.leaf_ctx, leaves.data_ptr(), L, out.data_ptr(), n, self._stream()))
        return out

    def from_digests(self, digests: torch.Tensor):
        """digests (m, 4), m a power of two >= 2 -> (m-1, 4) heap-ordered inner nodes."""
        m = digests.shape[0]
        nodes = self._buf("top", (m - 1, 4), digests.device)
        self.N.check(self.N.lib.cpb_merkle_poseidon_from_digests_dev(self.node_ctx, digests.data_ptr(), m, nodes.data_ptr(),
                                                                     self._stream()))
        return nodes

    def _update_args(self, leaf_nodes, nodes, indexes, asserted_root):
        n = leaf_nodes.shape[0]
        assert leaf_nodes.is_contiguous() and nodes.is_contiguous() and tuple(nodes.shape) == (n - 1, 4) and leaf_nodes.shape[1] == 4
        idx = indexes.to(device=leaf_nodes.device, dtype=torch.int64).contiguous()
        root = None if asserted_root is None else asserted_root.to(device=leaf_nodes.device, dtype=torch.int64).contiguous().clone()
        applied = torch.empty(1, dtype=torch.uint8, device=leaf_nodes.device)
        return n, idx, root, applied

    def update(self, leaf_nodes: torch.Tensor, nodes: torch.Tensor, indexes: torch.Tensor, new_leaves: torch.Tensor, asserted_root=None):
        """k x MerkleTree::update -- or check_update when `asserted_root` (4,) is given -- on a tree built on this device, in place and
        on the current stream: leaf_nodes (n, 4), nodes (n-1, 4) heap order, indexes (k,) (the last occurrence of a repeated index
        wins; an index >= n is skipped), new_leaves (k, L, 4).  Returns the device flag `applied` (uint8, (1,)); no synchronisation."""
        n, idx, root, applied = self._update_args(leaf_nodes, nodes, indexes, asserted_root)
        lv = new_leaves.contiguous()
        k, L = lv.shape[0], lv.shape[1] if lv.dim() > 1 else 0
        assert idx.shape[0] == k, "one new leaf per index"
        self.N.check(self.N.lib.cpb_merkle_poseidon_update_dev(self.leaf_ctx, self.node_ctx, leaf_nodes.data_ptr(), nodes.data_ptr(), n,
                                                               idx.data_ptr(), lv.data_ptr(), L, k, None if root is None else root.data_ptr(),
                                                               applied.data_ptr(), self._stream()))
        return applied

    def _update_digests(self, leaf_nodes, nodes, idx, digests, root, applied):
        self.N.check(self.N.lib.cpb_merkle_poseidon_update_digests_dev(self.node_ctx, leaf_nodes.data_ptr(), nodes.data_ptr(), leaf_nodes.shape[0],
                                                                       idx.data_ptr(), digests.data_ptr(), idx.shape[0],
                                                                       None if root is None else root.data_ptr(), applied.data_ptr(),
                                                                       self._stream()))
        return applied


class CudaMixedBackend(CudaPoseidonBackend):
    """BASELINE config 5: byte leaves hashed with PedersenCRHCompressor (x-coordinate, R/crh/injective_map/mod.rs:22-62),
    inner nodes with poseidon::TwoToOneCRH over the curve's base field.  local_leaves: (n, leaf_len) uint8 on the GPU."""

    def __init__(self, pedersen_params, node_params, device_index: int):
        from . import _native as N
        self.N = N
        self.dev = device_index
        self.leaf_ctx = pedersen_params.context(device_index)
        self.node_ctx = node_params.context(device_index)
        self._ws = {}

    def build_local(self, leaves: torch.Tensor):
        n, ln = leaves.shape
        leaf_nodes = self._buf("leaf", (n, 4), leaves.device)
        nodes = self._buf("nodes", (n - 1, 4), leaves.device)
        self.N.check(self.N.lib.cpb_merkle_mixed_build_dev(self.leaf_ctx, self.node_ctx, leaves.data_ptr(), ln, leaves.stride(0), n,
                                                           leaf_nodes.data_ptr(), nodes.data_ptr(), self._stream()))
        return leaf_nodes, nodes

    def build_sharded(self, leaves: torch.Tensor, ex: "Exchange"):
        n, ln = leaves.shape
        leaf_nodes = self._buf("leaf", (n, 4), leaves.device)
        nodes = self._buf("nodes", (n - 1, 4), leaves.device)
        top = self._buf("top", (max(ex.world - 1, 1), 4), leaves.device)
        self.N.check(self.N.lib.cpb_merkle_mixed_build_sharded_dev(self.leaf_ctx, self.node_ctx, ex.handle, leaves.data_ptr(), ln, leaves.stride(0), n,
                                                                   leaf_nodes.data_ptr(), nodes.data_ptr(), top.data_ptr(), self._stream()))
        return leaf_nodes, nodes, top

    def hash_leaves(self, leaves: torch.Tensor):
        n, ln = leaves.shape
        out = self._buf("leaf", (n, 4), leaves.device)
        self.N.check(self.N.lib.cpb_pedersen_crh_x_batch_dev(self.leaf_ctx, leaves.data_ptr(), ln, leaves.stride(0), out.data_ptr(), n,
                                                             self._stream()))
        return out

    def update(self, leaf_nodes: torch.Tensor, nodes: torch.Tensor, indexes: torch.Tensor, new_leaves: torch.Tensor, asserted_root=None):
        """CudaPoseidonBackend.update with byte leaves new_leaves (k, leaf_len) uint8: their Pedersen x-coordinate digests go to a
        workspace of their own (the "leaf" workspace may hold this tree's leaf digests), then the digest form of the update."""
        n, idx, root, applied = self._update_args(leaf_nodes, nodes, indexes, asserted_root)
        k, ln = new_leaves.shape
        assert idx.shape[0] == k, "one new leaf per index"
        digests = self._buf("update_leaf", (k, 4), leaf_nodes.device)
        if k:
            self.N.check(self.N.lib.cpb_pedersen_crh_x_batch_dev(self.leaf_ctx, new_leaves.data_ptr(), ln, new_leaves.stride(0), digests.data_ptr(),
                                                                 k, self._stream()))
        return self._update_digests(leaf_nodes, nodes, idx, digests, root, applied)


class CudaPedersenBackend(CudaPoseidonBackend):
    """Byte tree of JubJubMerkleTreeParams (R/merkle_tree/tests/mod.rs:19-33): byte leaves hashed with pedersen::CRH, inner nodes
    with pedersen::TwoToOneCRH.  Digests are affine points, (2, 4) words; leaves: (n, leaf_len) uint8 on the GPU.  There is no
    sharded build for byte trees."""

    digest_words = 8

    def __init__(self, leaf_params, node_params, device_index: int):
        from . import _native as N
        self.N = N
        self.dev = device_index
        self.leaf_ctx = leaf_params.context(device_index)
        self.node_ctx = node_params.context(device_index)
        self._ws = {}

    def build_local(self, leaves: torch.Tensor):
        """leaves (n, leaf_len) uint8 -> (leaf_nodes (n, 2, 4), nodes (n-1, 2, 4)) heap order."""
        n, ln = leaves.shape
        leaf_nodes = self._buf("leaf", (n, 2, 4), leaves.device)
        nodes = self._buf("nodes", (n - 1, 2, 4), leaves.device)
        scratch = self._buf("scratch", (n, 8), leaves.device)            # 64 bytes per leaf
        self.N.check(self.N.lib.cpb_merkle_pedersen_build_dev(self.leaf_ctx, self.node_ctx, leaves.data_ptr(), ln, leaves.stride(0), n,
                                                              leaf_nodes.data_ptr(), nodes.data_ptr(), scratch.data_ptr(), self._stream()))
        return leaf_nodes, nodes

    def build_sharded(self, leaves, ex):
        raise NotImplementedError("byte trees have no sharded build")

    def hash_leaves(self, leaves: torch.Tensor):
        n, ln = leaves.shape
        out = self._buf("leaf", (n, 2, 4), leaves.device)
        self.N.check(self.N.lib.cpb_pedersen_crh_batch_dev(self.leaf_ctx, leaves.data_ptr(), ln, leaves.stride(0), out.data_ptr(), n,
                                                           self._stream()))
        return out

    def from_digests(self, digests):
        raise NotImplementedError("use build_local")

    def update(self, leaf_nodes: torch.Tensor, nodes: torch.Tensor, indexes: torch.Tensor, new_leaves: torch.Tensor, asserted_root=None):
        """k x MerkleTree::update -- or check_update when `asserted_root` (2, 4) is given -- on a tree built on this device, in place
        and on the current stream: leaf_nodes (n, 2, 4), nodes (n-1, 2, 4) heap order, indexes (k,) (the last occurrence of a repeated
        index wins; an index >= n is skipped), new_leaves (k, leaf_len) uint8, rows any stride apart.  Returns the device flag
        `applied` (uint8, (1,)); no synchronisation."""
        n = leaf_nodes.shape[0]
        assert leaf_nodes.is_contiguous() and nodes.is_contiguous() and tuple(nodes.shape[1:]) == (2, 4) and nodes.shape[0] == n - 1
        assert tuple(leaf_nodes.shape[1:]) == (2, 4)
        idx = indexes.to(device=leaf_nodes.device, dtype=torch.int64).contiguous()
        root = None if asserted_root is None else asserted_root.to(device=leaf_nodes.device, dtype=torch.int64).contiguous().clone()
        applied = torch.empty(1, dtype=torch.uint8, device=leaf_nodes.device)
        k, ln = new_leaves.shape
        assert idx.shape[0] == k, "one new leaf per index"
        assert new_leaves.dtype == torch.uint8 and (k == 0 or new_leaves.stride(1) == 1)
        self.N.check(self.N.lib.cpb_merkle_pedersen_update_dev(self.leaf_ctx, self.node_ctx, leaf_nodes.data_ptr(), nodes.data_ptr(), n,
                                                               idx.data_ptr(), new_leaves.data_ptr(), ln, new_leaves.stride(0), k,
                                                               None if root is None else root.data_ptr(), applied.data_ptr(), self._stream()))
        return applied


@dataclass
class ShardedTree:
    """Result of a sharded build on this rank."""
    root: torch.Tensor                    # (digest_words,)
    n_leaves: int                         # global
    world: int
    rank: int
    local_leaf_nodes: torch.Tensor        # this rank's leaf digests (n/G, w)
    local_nodes: torch.Tensor | None      # this rank's subtree inner nodes, heap order (n/G - 1, w); None when n/G == 1
    top_nodes: torch.Tensor | None        # the replicated top g levels, heap order (G - 1, w); None when G == 1
    leaf_nodes: torch.Tensor | None = None       # gather="levels": the reference's full arrays on every rank
    non_leaf_nodes: torch.Tensor | None = None

    def height(self) -> int:
        return _log2(self.n_leaves) + 1


def level_slices(n_leaves: int, world: int, rank: int):
    """For every global inner level l in [g, log2 n): (global_start, count_per_rank, local_start) describing
    where rank's nodes of that level live in the global and in the local heap-ordered arrays."""
    g, h = _log2(world), _log2(n_leaves)
    out = []
    for l in range(g, h):
        width = 1 << l                     # nodes at global level l
        per = width // world
        out.append(((1 << l) - 1 + rank * per, per, (1 << (l - g)) - 1))
    return out


def sharded_merkle_build(backend, local_leaves: torch.Tensor, gather: str = "roots", group=None, exchange: Exchange | None = None) -> ShardedTree:
    """Build the tree whose leaves are the concatenation over ranks of `local_leaves` (rank order).  With `exchange` (and
    at least two leaves per rank) the root exchange and the top levels run fused inside the library; otherwise the roots
    go through one all_gather of torch.distributed."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    g = _log2(world)
    n_local = local_leaves.shape[0]
    _log2(n_local)
    n = n_local * world
    if n < 2:
        raise ValueError("`leaves.len() should be power of two and greater than one")
    w = backend.digest_words

    if exchange is not None and world > 1 and n_local >= 2:
        assert exchange.world == world and exchange.rank == rank
        leaf_nodes, nodes, top = backend.build_sharded(local_leaves, exchange)
        tree = ShardedTree(top[0], n, world, rank, leaf_nodes, nodes, top)
        return _gather_levels(tree, gather, group, w)
    if n_local >= 2:
        leaf_nodes, nodes = backend.build_local(local_leaves)
        local_root = nodes[0]
    else:
        leaf_nodes, nodes = backend.hash_leaves(local_leaves), None
        local_root = leaf_nodes[0]

    top = None
    if world > 1:
        roots = torch.empty((world, w), dtype=local_root.dtype, device=local_root.device)
        dist.all_gather_into_tensor(roots, local_root.reshape(1, w).contiguous(), group=group)   # the one collective
        top = backend.from_digests(roots)
        root = top[0]
    else:
        root = local_root

    tree = ShardedTree(root, n, world, rank, leaf_nodes, nodes, top)
    return _gather_levels(tree, gather, group, w)


def _gather_levels(tree: ShardedTree, gather: str, group, w: int) -> ShardedTree:
    n, world, rank = tree.n_leaves, tree.world, tree.rank
    leaf_nodes, nodes, top = tree.local_leaf_nodes, tree.local_nodes, tree.top_nodes
    if gather == "levels":
        full_leaf = torch.empty((n, w), dtype=leaf_nodes.dtype, device=leaf_nodes.device)
        full_nodes = torch.empty((n - 1, w), dtype=leaf_nodes.dtype, device=leaf_nodes.device)
        if world > 1:
            dist.all_gather_into_tensor(full_leaf, leaf_nodes.contiguous(), group=group)
            full_nodes[: world - 1] = top
            for gstart, per, lstart in level_slices(n, world, rank):
                seg = full_nodes[gstart - rank * per: gstart - rank * per + per * world]
                dist.all_gather_into_tensor(seg, nodes[lstart: lstart + per].contiguous(), group=group)
        else:
            full_leaf.copy_(leaf_nodes)
            full_nodes.copy_(nodes)
        tree.leaf_nodes, tree.non_leaf_nodes = full_leaf, full_nodes
    elif gather != "roots":
        raise ValueError("gather must be 'roots' or 'levels'")
    return tree
