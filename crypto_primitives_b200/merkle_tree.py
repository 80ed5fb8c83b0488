"""merkle_tree::{Config, MerkleTree, Path, MultiPath} -- host mirror of R/merkle_tree/mod.rs over
the CUDA library (R = /root/reference/crypto-primitives/src).

The build (MerkleTree::new, mod.rs:411-523) runs on the GPU: one kernel hashes all leaves, then one
launch per level compresses contiguous child pairs of the heap-ordered node array.  The tree object
keeps the reference's two arrays -- leaf_nodes[n] and non_leaf_nodes[n-1] (root at 0, children of i
at 2i+1 / 2i+2, mod.rs:383-395) -- on the host, so proofs are index arithmetic exactly as in
mod.rs:547-623.  Verification and update are LEVEL-SYNCHRONOUS device batches for every Config: all paths
(or all touched nodes) of one tree level go through ONE two-to-one batch call, so k proofs / k updated
leaves cost height launches, not k * height (`verify_paths_batch`, `MultiPath.verify`, `update_batch`);
the Poseidon field-leaf Config additionally has a single-launch kernel that recomputes one root per
thread (`cpb_merkle_poseidon_verify_batch`), and Configs whose inner hash is Poseidon update in ONE library
call (`cpb_merkle_poseidon_update_digests`, and `cpb_merkle_pedersen_update` for the Pedersen byte tree: every level on the
device, only touched nodes cross PCIe).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import _native as N
from . import ragged as R
from .crh import pedersen as pedersen_crh
from .crh import poseidon as poseidon_crh


def _p(a):
    return a.ctypes.data_as(N.u64p)


def _leaf_batch(leaves):
    """Leaves as one array -- or, for leaves of different lengths, which no array holds, the sequence itself: the field-leaf
    Config's leaf hash takes it as a ragged batch (each leaf hashed at its own length, as MerkleTree::new does)."""
    return leaves if R.is_ragged(leaves) else np.asarray(leaves)


class Config:
    """merkle_tree::Config (mod.rs:83-122) as a value: which leaf hash, converter and two-to-one hash.
    Subclasses provide batched GPU evaluation of the three associated functions."""

    digest_words = 4            # uint64 words per inner digest

    def leaf_hash_batch(self, leaf_param, leaves, device):
        raise NotImplementedError

    def two_to_one_batch(self, param, pairs, device):
        """pairs: (n, 2, digest_words) of already converted digests -> (n, digest_words)."""
        raise NotImplementedError

    def build(self, leaf_param, two_to_one_param, leaves, device):
        """Generic build (mod.rs:411-523): all leaves in one GPU batch, then one GPU batch per level.  Configs with a
        fused device-side build (`cpb_merkle_*_build`) override this; the generic form round-trips each level
        through the host."""
        leaf_nodes = self.leaf_hash_batch(leaf_param, leaves, device)
        return leaf_nodes, self.build_from_digests(two_to_one_param, leaf_nodes, device)

    def _pairs(self, nodes):
        return np.ascontiguousarray(nodes).reshape((-1, 2) + tuple(nodes.shape[1:]))

    def build_from_digests(self, two_to_one_param, leaf_digests, device):
        d = np.ascontiguousarray(leaf_digests, dtype=np.uint64)
        n = d.shape[0]
        if n < 2 or n & (n - 1):
            raise ValueError("`leaves.len() should be power of two and greater than one")
        nodes = np.empty((n - 1,) + d.shape[1:], dtype=np.uint64)
        start = n // 2 - 1
        nodes[start:] = self.two_to_one_batch(two_to_one_param, self._pairs(d), device)
        while start > 0:
            upper, start = start, (start - 1) // 2
            nodes[start:upper] = self.two_to_one_batch(two_to_one_param, self._pairs(nodes[upper:2 * upper + 1]), device)
        return nodes

    def default_leaf_digest(self, leaf_param=None):
        return np.zeros(self.digest_words, dtype=np.uint64)


class PoseidonFieldConfig(Config):
    """Config{Leaf=[F], LeafDigest=InnerDigest=F, IdentityDigestConverter, LeafHash=poseidon::CRH,
    TwoToOneHash=poseidon::TwoToOneCRH} -- FieldMTConfig of R/merkle_tree/tests/mod.rs:198-206."""

    def leaf_hash_batch(self, leaf_param, leaves, device):
        return poseidon_crh.CRH.evaluate_batch(leaf_param, leaves, device)

    def two_to_one_batch(self, param, pairs, device):
        return poseidon_crh.TwoToOneCRH.compress_batch(param, pairs, device)

    def build(self, leaf_param, two_to_one_param, leaves, device):
        if R.is_ragged(leaves):
            return self.build_ragged(leaf_param, two_to_one_param, *R.pack(leaves), device)
        lv = np.ascontiguousarray(leaves, dtype=np.uint64)
        assert lv.ndim == 3 and lv.shape[2] == 4, "leaves must be (n, leaf_len, 4) or a list of (leaf_len_i, 4)"
        n, ln = lv.shape[0], lv.shape[1]
        leaf_nodes = np.empty((n, 4), dtype=np.uint64)
        non_leaf = np.empty((max(n - 1, 0), 4), dtype=np.uint64)
        N.check(N.lib.cpb_merkle_poseidon_build(leaf_param.context(device), two_to_one_param.context(device),
                                                _p(lv), ln, n, _p(leaf_nodes), _p(non_leaf)))
        return leaf_nodes, non_leaf

    def build_ragged(self, leaf_param, two_to_one_param, values, offsets, device):
        """MerkleTree::new over leaves of different lengths: leaf i = values[offsets[i] .. offsets[i+1])."""
        vals, off = R.as_arrays(values, offsets)
        n = off.shape[0] - 1
        leaf_nodes = np.empty((max(n, 0), 4), dtype=np.uint64)
        non_leaf = np.empty((max(n - 1, 0), 4), dtype=np.uint64)
        R.check(N.lib.cpb_merkle_poseidon_build_ragged(leaf_param.context(device), two_to_one_param.context(device), _p(vals), _p(off), n,
                                                       _p(leaf_nodes), _p(non_leaf)))
        return leaf_nodes, non_leaf

    def build_from_digests(self, two_to_one_param, leaf_digests, device):
        d = np.ascontiguousarray(leaf_digests, dtype=np.uint64).reshape(-1, 4)
        n = d.shape[0]
        non_leaf = np.empty((max(n - 1, 0), 4), dtype=np.uint64)
        N.check(N.lib.cpb_merkle_poseidon_from_digests(two_to_one_param.context(device), _p(d), n, _p(non_leaf)))
        return non_leaf


class PedersenByteConfig(Config):
    """Config{Leaf=[u8], LeafDigest=InnerDigest=C::Affine, ByteDigestConverter, LeafHash=pedersen::CRH,
    TwoToOneHash=pedersen::TwoToOneCRH} -- JubJubMerkleTreeParams of R/merkle_tree/tests/mod.rs:19-33.
    Digests are affine points, (2, 4) words."""

    digest_words = 8

    def leaf_hash_batch(self, leaf_param, leaves, device):
        return pedersen_crh.CRH.evaluate_batch(leaf_param, leaves, device)

    def two_to_one_batch(self, param, pairs, device):
        return pedersen_crh.TwoToOneCRH.compress_batch(param, np.asarray(pairs).reshape(-1, 2, 2, 4), device)

    def build(self, leaf_param, two_to_one_param, leaves, device):
        lv = np.ascontiguousarray(leaves, dtype=np.uint8)
        assert lv.ndim == 2, "leaves must be (n, leaf_len) bytes"
        n, ln = lv.shape
        leaf_nodes = np.empty((n, 2, 4), dtype=np.uint64)
        non_leaf = np.empty((max(n - 1, 0), 2, 4), dtype=np.uint64)
        try:
            N.check(N.lib.cpb_merkle_pedersen_build(leaf_param.context(device), two_to_one_param.context(device),
                                                    lv.ctypes.data_as(N.u8p), ln, n, _p(leaf_nodes), _p(non_leaf)))
        except N.CpbError as e:
            if e.status == N.CPB_BAD_LENGTH:
                raise ValueError("incorrect input length") from e
            raise
        return leaf_nodes, non_leaf

    def build_from_digests(self, two_to_one_param, leaf_digests, device):
        return Config.build_from_digests(self, two_to_one_param, np.asarray(leaf_digests, dtype=np.uint64).reshape(-1, 2, 4), device)

    def default_leaf_digest(self, leaf_param=None):
        """C::Affine::default() -- the identity (0, 1) of the twisted-Edwards curve (ark-ec `Affine::zero()`, dep), which the
        ByteDigestConverter serialises like any other point (mod.rs:71-78): MerkleTree::blank works for byte-digest Configs."""
        from .curves import JUBJUB
        curve = leaf_param.curve if leaf_param is not None else JUBJUB
        return curve.base_field.elements([0, 1]).reshape(2, 4)


class PedersenPoseidonConfig(Config):
    """Config{Leaf=[u8], LeafHash=PedersenCRHCompressor<C,TECompressor,W>, LeafDigest=InnerDigest=Fq,
    IdentityDigestConverter, TwoToOneHash=poseidon::TwoToOneCRH<Fq>} (BASELINE config 5)."""

    def leaf_hash_batch(self, leaf_param, leaves, device):
        return pedersen_crh.PedersenCRHCompressor.evaluate_batch(leaf_param, leaves, device)

    def two_to_one_batch(self, param, pairs, device):
        return poseidon_crh.TwoToOneCRH.compress_batch(param, pairs, device)

    def build(self, leaf_param, two_to_one_param, leaves, device):
        lv = np.ascontiguousarray(leaves, dtype=np.uint8)
        n, ln = lv.shape
        leaf_nodes = np.empty((n, 4), dtype=np.uint64)
        non_leaf = np.empty((max(n - 1, 0), 4), dtype=np.uint64)
        try:
            N.check(N.lib.cpb_merkle_mixed_build(leaf_param.context(device), two_to_one_param.context(device),
                                                 lv.ctypes.data_as(N.u8p), ln, n, _p(leaf_nodes), _p(non_leaf)))
        except N.CpbError as e:
            if e.status == N.CPB_BAD_LENGTH:
                raise ValueError("incorrect input length") from e
            raise
        return leaf_nodes, non_leaf

    def build_from_digests(self, two_to_one_param, leaf_digests, device):
        return PoseidonFieldConfig().build_from_digests(two_to_one_param, leaf_digests, device)


class BoweHopwoodByteConfig(Config):
    """Config{Leaf=[u8], LeafHash=bowe_hopwood::CRH, LeafDigest=InnerDigest=Fq (the x-coordinate),
    IdentityDigestConverter, TwoToOneHash=bowe_hopwood::TwoToOneCRH} -- the Zcash-style tree (R/crh/bowe_hopwood/mod.rs:
    112-241).  Hashing runs on the GPU (one batch per level); the level loop is the generic host one."""

    def leaf_hash_batch(self, leaf_param, leaves, device):
        from .crh import bowe_hopwood as bh
        return bh.CRH.evaluate_batch(leaf_param, np.ascontiguousarray(leaves, dtype=np.uint8), device)

    def two_to_one_batch(self, param, pairs, device):
        from .crh import bowe_hopwood as bh
        return bh.TwoToOneCRH.compress_batch(param, np.asarray(pairs, dtype=np.uint64).reshape(-1, 2, 4), device)


# ---- index helpers, mod.rs:728-786
def tree_height(num_leaves: int) -> int:
    return 1 if num_leaves == 1 else num_leaves.bit_length()


def is_root(i):
    return i == 0


def left_child(i):
    return 2 * i + 1


def right_child(i):
    return 2 * i + 2


def sibling(i):
    if i == 0:
        return None
    return i + 1 if is_left_child(i) else i - 1


def is_left_child(i):
    return i % 2 == 1


def parent(i):
    return (i - 1) >> 1 if i > 0 else None


def convert_index_to_last_level(index, height):
    return index + (1 << (height - 1)) - 1


def _select_and_hash(cfg: Config, two_to_one_params, cur, sib, on_right, device):
    """select_left_right_child (mod.rs:214-228) for a whole batch, then ONE two-to-one call: row i hashes (cur_i, sib_i),
    swapped where on_right[i] (the computed node is the right child)."""
    cur = np.asarray(cur, dtype=np.uint64)
    sib = np.asarray(sib, dtype=np.uint64)
    flag = np.asarray(on_right, dtype=bool).reshape((-1,) + (1,) * (cur.ndim - 1))
    pairs = np.stack([np.where(flag, sib, cur), np.where(flag, cur, sib)], axis=1)
    return cfg.two_to_one_batch(two_to_one_params, np.ascontiguousarray(pairs), device)


def verify_paths_batch(leaf_hash_params, two_to_one_params, root_hash, leaves, proofs, config: Config = None, device: int = 0) -> np.ndarray:
    """n x Path::verify (mod.rs:172-212) for any Config as device batches: one leaf-hash batch, then one two-to-one batch
    per tree level for ALL n paths (height launches in total).  `proofs`: Paths of one tree; returns a bool array."""
    cfg = config or PoseidonFieldConfig()
    n = len(proofs)
    if n == 0:
        return np.zeros(0, dtype=bool)
    plen = len(proofs[0].auth_path)
    assert all(len(p.auth_path) == plen for p in proofs), "paths of different heights"
    claimed = cfg.leaf_hash_batch(leaf_hash_params, _leaf_batch(leaves), device)
    idx = np.array([p.leaf_index for p in proofs], dtype=np.int64)
    cur = _select_and_hash(cfg, two_to_one_params, claimed, np.stack([p.leaf_sibling_hash for p in proofs]), idx & 1, device)
    idx >>= 1
    for level in range(plen - 1, -1, -1):
        cur = _select_and_hash(cfg, two_to_one_params, cur, np.stack([p.auth_path[level] for p in proofs]), idx & 1, device)
        idx >>= 1
    root = np.asarray(root_hash, dtype=np.uint64).reshape(1, -1)
    return np.all(np.asarray(cur).reshape(n, -1) == root, axis=1)


@dataclass
class Path:
    """mod.rs:139-152."""
    leaf_sibling_hash: np.ndarray
    auth_path: list
    leaf_index: int

    def verify(self, leaf_hash_params, two_to_one_params, root_hash, leaf, config: Config = None, device: int = 0) -> bool:
        """Path::verify, mod.rs:172-212.  Field-leaf Poseidon Config: ONE kernel launch recomputes the root
        (cpb_merkle_poseidon_verify_batch with n = 1); other Configs: the level-synchronous batch with n = 1."""
        cfg = config or PoseidonFieldConfig()
        if type(cfg) is PoseidonFieldConfig:
            lv = np.ascontiguousarray(np.asarray(leaf, dtype=np.uint64).reshape(1, -1, 4))
            plen = len(self.auth_path)
            sib = np.ascontiguousarray(np.asarray(self.leaf_sibling_hash, dtype=np.uint64).reshape(1, 4))
            paths = np.ascontiguousarray(np.stack(self.auth_path).astype(np.uint64).reshape(1, plen, 4)) if plen else np.zeros((1, 0, 4), dtype=np.uint64)
            idx = np.array([self.leaf_index], dtype=np.uint64)
            root = np.ascontiguousarray(root_hash, dtype=np.uint64)
            ok = np.zeros(1, dtype=np.uint8)
            N.check(N.lib.cpb_merkle_poseidon_verify_batch(leaf_hash_params.context(device), two_to_one_params.context(device), _p(root), _p(lv),
                                                           lv.shape[1], _p(sib), _p(paths), plen, _p(idx), ok.ctypes.data_as(N.u8p), 1))
            return bool(ok[0])
        return bool(verify_paths_batch(leaf_hash_params, two_to_one_params, root_hash, np.asarray(leaf)[None], [self], cfg, device)[0])


@dataclass
class MultiPath:
    """mod.rs:239-254 (field names as in the reference, including its spelling)."""
    leaf_siblings_hashes: list
    auth_paths_prefix_lenghts: list
    auth_paths_suffixes: list
    leaf_indexes: list

    def verify(self, leaf_hash_params, two_to_one_params, root_hash, leaves, config: Config = None, device: int = 0) -> bool:
        """MultiPath::verify, mod.rs:262-331 (with the same lookup table of already hashed nodes)."""
        cfg = config or PoseidonFieldConfig()
        n = len(self.leaf_indexes)
        if n == 0:
            return True
        plen = len(self.auth_paths_suffixes[0])
        # decode the front-incremental auth paths (prefix_decode_path, mod.rs:289-297); host index work only
        paths, prev = [], list(self.auth_paths_suffixes[0])
        for i in range(n):
            k = self.auth_paths_prefix_lenghts[i]
            auth = list(self.auth_paths_suffixes[i]) if k == 0 else prev[:k] + list(self.auth_paths_suffixes[i])
            assert len(auth) == plen, "auth paths of different lengths"
            paths.append(auth)
            prev = auth
        idx = np.array(self.leaf_indexes, dtype=np.int64)
        claimed = cfg.leaf_hash_batch(leaf_hash_params, _leaf_batch(leaves), device)
        # Level-synchronous form of the reference's loop with its look-up table of already hashed nodes (mod.rs:272-322):
        # at every level each tree node is hashed ONCE, from the first path (in order) that reaches it -- exactly the
        # `hash_lut.entry(..).or_insert_with(..)` semantics -- and all distinct nodes of a level are one device batch.
        node = idx >> 1                                        # position of the path's node within its level
        uniq, first, inverse = np.unique(node, return_index=True, return_inverse=True)
        vals = _select_and_hash(cfg, two_to_one_params, np.asarray(claimed)[first], np.stack(self.leaf_siblings_hashes)[first], idx[first] & 1, device)
        cur = np.asarray(vals)[inverse]
        for level in range(plen - 1, -1, -1):
            sib = np.stack([p[level] for p in paths])
            on_right = node & 1
            node = node >> 1
            uniq, first, inverse = np.unique(node, return_index=True, return_inverse=True)
            vals = _select_and_hash(cfg, two_to_one_params, cur[first], sib[first], on_right[first], device)
            cur = np.asarray(vals)[inverse]
        root = np.asarray(root_hash, dtype=np.uint64).reshape(1, -1)
        return bool(np.all(cur.reshape(n, -1) == root))


class MerkleTree:
    """mod.rs:381-395."""

    def __init__(self, config, leaf_nodes, non_leaf_nodes, leaf_hash_param, two_to_one_hash_param, device):
        self.config = config
        self.leaf_nodes = leaf_nodes
        self.non_leaf_nodes = non_leaf_nodes
        self.leaf_hash_param = leaf_hash_param
        self.two_to_one_hash_param = two_to_one_hash_param
        self._height = tree_height(leaf_nodes.shape[0])
        self.device = device

    @classmethod
    def blank(cls, leaf_hash_param, two_to_one_hash_param, height: int, config: Config = None, device: int = 0):
        """mod.rs:400-408: all leaf digests = LeafDigest::default()."""
        cfg = config or PoseidonFieldConfig()
        one = np.asarray(cfg.default_leaf_digest(leaf_hash_param), dtype=np.uint64)
        d = np.ascontiguousarray(np.broadcast_to(one, (1 << (height - 1),) + one.shape))
        return cls.new_with_leaf_digest(leaf_hash_param, two_to_one_hash_param, d, cfg, device)

    @classmethod
    def new(cls, leaf_hash_param, two_to_one_hash_param, leaves, config: Config = None, device: int = 0):
        """mod.rs:411-422.  Raises ValueError where the reference asserts (:430-433)."""
        cfg = config or PoseidonFieldConfig()
        try:
            leaf_nodes, non_leaf = cfg.build(leaf_hash_param, two_to_one_hash_param, leaves, device)
        except N.CpbError as e:
            if e.status == N.CPB_NOT_POW2:
                raise ValueError("`leaves.len() should be power of two and greater than one") from e
            raise
        return cls(cfg, leaf_nodes, non_leaf, leaf_hash_param, two_to_one_hash_param, device)

    @classmethod
    def new_with_leaf_digest(cls, leaf_hash_param, two_to_one_hash_param, leaf_digests, config: Config = None, device: int = 0):
        """mod.rs:424-523."""
        cfg = config or PoseidonFieldConfig()
        d = np.ascontiguousarray(leaf_digests, dtype=np.uint64)
        try:
            non_leaf = cfg.build_from_digests(two_to_one_hash_param, d, device)
        except N.CpbError as e:
            if e.status == N.CPB_NOT_POW2:
                raise ValueError("`leaves.len() should be power of two and greater than one") from e
            raise
        return cls(cfg, d, non_leaf, leaf_hash_param, two_to_one_hash_param, device)

    def root(self):
        return self.non_leaf_nodes[0].copy()

    def height(self) -> int:
        return self._height

    def get_leaf_sibling_hash(self, index: int):
        return self.leaf_nodes[index ^ 1].copy()

    def _compute_auth_path(self, index: int):
        """mod.rs:548-573."""
        path = []
        cur = parent(convert_index_to_last_level(index, self._height))
        while not is_root(cur):
            path.append(self.non_leaf_nodes[sibling(cur)].copy())
            cur = parent(cur)
        path.reverse()
        return path

    def generate_proof(self, index: int) -> Path:
        return Path(self.get_leaf_sibling_hash(index), self._compute_auth_path(index), index)

    def generate_multi_proof(self, indexes) -> MultiPath:
        """mod.rs:589-623: sorted, de-duplicated indexes; every auth path is stored as the length of the prefix it shares with
        the previous one plus its own suffix.  The paths come from the vectorised index arithmetic of generate_proofs_batch;
        the shared-prefix lengths are one array comparison."""
        idx = sorted(set(int(i) for i in indexes))
        if not idx:
            return MultiPath([], [], [], [])
        sib, paths, _ = self.generate_proofs_batch(idx)
        k, plen = paths.shape[0], paths.shape[1]
        if plen and k > 1:
            flat = paths.reshape(k, plen, -1)
            same = np.all(flat[1:] == flat[:-1], axis=2)                                          # (k-1, plen)
            # length of the common prefix with the previous path = index of the first differing node (plen when all agree)
            lead = np.where(same.all(axis=1), plen, np.argmin(same, axis=1))
        else:                                   # a two-leaf tree has empty auth paths (height 2); one leaf has no predecessor
            lead = np.zeros(max(k - 1, 0), dtype=np.int64)
        prefix = [0] + [int(x) for x in lead]
        suffixes = [[paths[i, j].copy() for j in range(prefix[i], plen)] for i in range(k)]
        return MultiPath([sib[i].copy() for i in range(k)], prefix, suffixes, idx)

    def generate_proofs_batch(self, indexes):
        """generate_proof (mod.rs:547-575) for many leaves at once as arrays: (leaf_sibling_hashes (k, ...), auth_paths
        (k, height-2, ...) root side first, leaf_indexes (k,)).  Pure index arithmetic on the heap-ordered arrays, vectorised:
        the sibling of the path node at depth d is node ((2^d - 1) + ((i >> (h-1-d)) ^ 1))."""
        idx = np.asarray(indexes, dtype=np.int64).reshape(-1)
        h1 = self._height - 1                                      # depth of the leaf level
        sib = self.leaf_nodes[idx ^ 1]
        cols = [self.non_leaf_nodes[((1 << d) - 1) + ((idx >> (h1 - d)) ^ 1)] for d in range(1, h1)]
        paths = np.stack(cols, axis=1) if cols else np.zeros((idx.size, 0) + self.non_leaf_nodes.shape[1:], dtype=np.uint64)
        return sib, paths, idx.astype(np.uint64)

    def verify_proofs_batch(self, proofs, leaves, root_hash=None) -> np.ndarray:
        """Many Path::verify (mod.rs:172-212) in one kernel launch (field-leaf Config): proofs = list of Path for
        `leaves[i]`, or the (siblings, paths, indexes) arrays of generate_proofs_batch; returns a bool array.
        One GPU thread recomputes one root."""
        if not isinstance(self.config, PoseidonFieldConfig):
            raise NotImplementedError("the one-launch kernel is for the Poseidon field-leaf Config; use verify_paths_batch")
        if R.is_ragged(leaves):                # leaves of different lengths: (values, offsets)
            lv, n_leaves = R.pack(leaves), len(leaves)
        else:
            lv = np.ascontiguousarray(leaves, dtype=np.uint64)
            assert lv.ndim == 3
            n_leaves = lv.shape[0]
        plen = self._height - 2
        if isinstance(proofs, tuple):
            sib, paths, idx = (np.ascontiguousarray(a, dtype=np.uint64) for a in proofs)
            n = idx.shape[0]
            assert n_leaves == n and paths.shape == (n, plen, 4)
            return self._verify_arrays(lv, sib, paths, idx, root_hash)
        n = len(proofs)
        assert n_leaves == n
        sib = np.ascontiguousarray(np.stack([p.leaf_sibling_hash for p in proofs]), dtype=np.uint64)
        paths = np.ascontiguousarray(np.stack([np.stack(p.auth_path) if plen else np.zeros((0, 4), dtype=np.uint64) for p in proofs]),
                                     dtype=np.uint64).reshape(n, plen, 4)
        idx = np.array([p.leaf_index for p in proofs], dtype=np.uint64)
        return self._verify_arrays(lv, sib, paths, idx, root_hash)

    def _verify_arrays(self, lv, sib, paths, idx, root_hash):
        n, plen = idx.shape[0], self._height - 2
        root = np.ascontiguousarray(self.root() if root_hash is None else root_hash, dtype=np.uint64)
        ok = np.zeros(n, dtype=np.uint8)
        lctx, nctx = self.leaf_hash_param.context(self.device), self.two_to_one_hash_param.context(self.device)
        if isinstance(lv, tuple):
            vals, off = lv
            R.check(N.lib.cpb_merkle_poseidon_verify_ragged_batch(lctx, nctx, _p(root), _p(vals), _p(off), _p(sib), _p(paths), plen, _p(idx),
                                                                  ok.ctypes.data_as(N.u8p), n))
            return ok.astype(bool)
        N.check(N.lib.cpb_merkle_poseidon_verify_batch(lctx, nctx, _p(root), _p(lv), lv.shape[1], _p(sib), _p(paths), plen, _p(idx),
                                                       ok.ctypes.data_as(N.u8p), n))
        return ok.astype(bool)

    def _check_indexes(self, indexes):
        idx = np.asarray(indexes, dtype=np.int64).reshape(-1)
        assert idx.size and idx.min() >= 0 and idx.max() < self.leaf_nodes.shape[0], "index out of range"
        assert np.unique(idx).size == idx.size, "indexes must be distinct"
        return idx

    def _updates_on_device(self) -> bool:
        """Configs whose inner hash is poseidon::TwoToOneCRH update through cpb_merkle_poseidon_update_digests, the Pedersen byte tree
        through cpb_merkle_pedersen_update: the touched nodes of every level are hashed on the device in one call, and only they and
        the siblings they read cross PCIe."""
        return type(self.config) in (PoseidonFieldConfig, PedersenPoseidonConfig, PedersenByteConfig)

    def _update_digests(self, idx, new_leaves, asserted_new_root=None) -> bool:
        """The Config's leaf hash of `new_leaves`, then one update call on the tree's arrays in place; True when applied."""
        cfg, dev = self.config, self.device
        if type(cfg) is PedersenByteConfig:
            return self._update_pedersen(idx, new_leaves, asserted_new_root)
        new_hash = np.ascontiguousarray(cfg.leaf_hash_batch(self.leaf_hash_param, _leaf_batch(new_leaves), dev), dtype=np.uint64).reshape(-1, 4)
        assert new_hash.shape[0] == idx.size, "one new leaf per index"
        self.leaf_nodes = np.ascontiguousarray(self.leaf_nodes, dtype=np.uint64)
        self.non_leaf_nodes = np.ascontiguousarray(self.non_leaf_nodes, dtype=np.uint64)
        ix = np.ascontiguousarray(idx, dtype=np.uint64)
        root = None if asserted_new_root is None else np.ascontiguousarray(asserted_new_root, dtype=np.uint64).reshape(4)
        ok = C.c_int(0)
        N.check(N.lib.cpb_merkle_poseidon_update_digests(self.two_to_one_hash_param.context(dev), _p(self.leaf_nodes), _p(self.non_leaf_nodes),
                                                         self.leaf_nodes.shape[0], _p(ix), _p(new_hash), ix.size,
                                                         None if root is None else _p(root), C.byref(ok)))
        return bool(ok.value)

    def _update_pedersen(self, idx, new_leaves, asserted_new_root=None) -> bool:
        """Byte tree with Pedersen inner nodes: the byte leaves and the indexes go to cpb_merkle_pedersen_update, which hashes the
        leaves and every touched node on the device in one call."""
        lv = np.ascontiguousarray(new_leaves, dtype=np.uint8)
        assert lv.ndim == 2 and lv.shape[0] == idx.size, "one new leaf (bytes) per index"
        self.leaf_nodes = np.ascontiguousarray(self.leaf_nodes, dtype=np.uint64)
        self.non_leaf_nodes = np.ascontiguousarray(self.non_leaf_nodes, dtype=np.uint64)
        ix = np.ascontiguousarray(idx, dtype=np.uint64)
        root = None if asserted_new_root is None else np.ascontiguousarray(asserted_new_root, dtype=np.uint64).reshape(8)
        ok = C.c_int(0)
        try:
            N.check(N.lib.cpb_merkle_pedersen_update(self.leaf_hash_param.context(self.device), self.two_to_one_hash_param.context(self.device),
                                                     _p(self.leaf_nodes), _p(self.non_leaf_nodes), self.leaf_nodes.shape[0], _p(ix),
                                                     lv.ctypes.data_as(N.u8p), lv.shape[1], ix.size, None if root is None else _p(root),
                                                     C.byref(ok)))
        except N.CpbError as e:
            if e.status == N.CPB_BAD_LENGTH:
                raise ValueError("incorrect input length") from e
            raise
        return bool(ok.value)

    def _updated_nodes(self, indexes, new_leaves):
        """The nodes that change when leaves `indexes` (distinct) are replaced by `new_leaves` (mod.rs:627-677 for one leaf):
        -> (new leaf digests, [(heap indexes, new values)] bottom level first).  Level-synchronous: the new leaves are one
        leaf-hash batch and all touched nodes of a level one two-to-one batch -- height launches for any number of leaves.
        The path of the Configs without a one-call device update (Bowe-Hopwood nodes, toy Configs)."""
        cfg, dev = self.config, self.device
        idx = self._check_indexes(indexes)
        n = self.leaf_nodes.shape[0]
        new_hash = np.asarray(cfg.leaf_hash_batch(self.leaf_hash_param, _leaf_batch(new_leaves), dev))
        par = np.unique(idx >> 1)                                  # touched leaf pairs
        pairs = np.stack([self.leaf_nodes[2 * par], self.leaf_nodes[2 * par + 1]], axis=1)     # gathers only the touched rows
        pairs[np.searchsorted(par, idx >> 1), idx & 1] = new_hash                              # ... with the new digests patched in
        vals = np.asarray(cfg.two_to_one_batch(self.two_to_one_hash_param, np.ascontiguousarray(pairs), dev))
        ids = par + (n // 2 - 1)                                   # heap indexes of the bottom inner level
        changes = [(ids, vals)]
        while ids[0] != 0:
            par = np.unique((ids - 1) >> 1)
            pairs = np.stack([self.non_leaf_nodes[2 * par + 1], self.non_leaf_nodes[2 * par + 2]], axis=1)
            pairs[np.searchsorted(par, (ids - 1) >> 1), (ids - 1) & 1] = vals
            vals = np.asarray(cfg.two_to_one_batch(self.two_to_one_hash_param, np.ascontiguousarray(pairs), dev))
            ids = par
            changes.append((ids, vals))
        return idx, new_hash, changes

    def _apply(self, idx, new_hash, changes):
        self.leaf_nodes[idx] = new_hash
        for ids, vals in changes:
            self.non_leaf_nodes[ids] = vals

    def update_batch(self, indexes, new_leaves):
        """k x MerkleTree::update (mod.rs:690-701) for distinct leaves as one level-synchronous pass: the resulting tree is
        the one k sequential updates produce, for height device launches instead of k * height."""
        if self._updates_on_device():
            self._update_digests(self._check_indexes(indexes), new_leaves)
            return
        self._apply(*self._updated_nodes(indexes, new_leaves))

    def update(self, index: int, new_leaf):
        """mod.rs:690-701."""
        assert index < self.leaf_nodes.shape[0], "index out of range"
        self.update_batch([index], np.asarray(new_leaf)[None])

    def check_update(self, index: int, new_leaf, asserted_new_root) -> bool:
        """mod.rs:706-725: the tree is modified only when the recomputed root equals `asserted_new_root`."""
        assert index < self.leaf_nodes.shape[0], "index out of range"
        return self.check_update_batch([index], np.asarray(new_leaf)[None], asserted_new_root)

    def check_update_batch(self, indexes, new_leaves, asserted_new_root) -> bool:
        """check_update for k distinct leaves at once (same acceptance rule, one level-synchronous pass)."""
        if self._updates_on_device():
            return self._update_digests(self._check_indexes(indexes), new_leaves, asserted_new_root)
        idx, new_hash, changes = self._updated_nodes(indexes, new_leaves)
        if not np.array_equal(changes[-1][1][0], np.asarray(asserted_new_root, dtype=np.uint64)):
            return False
        self._apply(idx, new_hash, changes)
        return True
