"""Pedersen-leaf path verification without a GPU: the per-level operand choice of csrc/merkle_verify_pedersen.cuh (which sibling, which
side, the TwoToOneCRH row of the byte tree) runs on the CPU through a host shim against the ordering of oracle/merkle.py::verify_path,
and the argument rules of cpb_merkle_pedersen_verify_batch[_dev] and cpb_merkle_mixed_verify_batch[_dev] that need no context."""
import ctypes as C

import numpy as np
import pytest

from helpers import build_host_shim
from crypto_primitives_b200 import _native as N
from oracle import cref, fields as OF, jubjub as jj, merkle as OM, pedersen as OPD

u64p = C.POINTER(C.c_uint64)
u32p = C.POINTER(C.c_uint32)


@pytest.fixture(scope="module")
def shim():
    lib = build_host_shim("merkle_verify_shim")
    lib.host_verify_step.argtypes = [C.c_uint64, C.c_int, C.c_int, C.c_uint64, u64p]
    lib.host_ped_verify_row.argtypes = [C.c_int, u32p, u32p, u32p, C.c_uint64, C.c_int, C.c_int, C.c_uint64, u32p]
    return lib


def _p32(a):
    return a.ctypes.data_as(u32p)


def oracle_pairs(plen, index):
    """The (left, right) pairs oracle/merkle.py::verify_path hashes, bottom-up, over symbolic digests: ("C",) the claimed leaf digest,
    ("S",) the leaf sibling, ("P", k) auth_path[k] (root side first), ("H", j) the digest level j computed."""
    pairs = []

    def h(left, right):
        pairs.append((left, right))
        return ("H", len(pairs) - 1)

    OM.verify_path((("S",), [("P", k) for k in range(plen)], index), ("C",), None, h, h)
    return pairs


def shim_pairs(shim, i, plen, index):
    out = np.zeros(3, dtype=np.uint64)
    pairs = []
    for j in range(plen + 1):
        shim.host_verify_step(i, plen, j, index, out.ctypes.data_as(u64p))
        from_path, elem, right = (int(x) for x in out)
        if from_path:
            assert i * plen <= elem < (i + 1) * plen, (i, plen, j)
            sib = ("P", elem - i * plen)
        else:
            assert elem == i
            sib = ("S",)
        cur = ("C",) if j == 0 else ("H", j - 1)
        pairs.append((sib, cur) if right else (cur, sib))
    return pairs


@pytest.mark.parametrize("plen", range(7))
def test_operand_choice_follows_the_oracle(shim, plen):
    rng = np.random.default_rng(plen)
    indexes = [0, (1 << (plen + 1)) - 1] + [int(x) for x in rng.integers(0, 1 << (plen + 1), size=24)]
    # bits above path_len + 1 (and the top bit of a u64) are ignored, as in the reference
    indexes += [x | (int(rng.integers(1, 1 << 20)) << (plen + 1)) for x in indexes[:8]] + [(1 << 64) - 1, 1 << 63]
    for index in indexes:
        i = int(rng.integers(0, 1 << 20))
        assert shim_pairs(shim, i, plen, index) == oracle_pairs(plen, index), (plen, index)


def _mont(vals, p):
    return cref.ints_to_mont(vals, p).reshape(-1, 2, 4)


@pytest.mark.parametrize("field,p", [(0, OF.BLS12_381_FR), (1, OF.BLS12_377_FR)])
@pytest.mark.parametrize("plen", [0, 1, 5])
def test_rows_are_the_oracle_serialisation(shim, field, p, plen):
    """Level j's row is the canonical x_l || y_l || x_r || y_r of the pair verify_path hashes there (TwoToOneCRH::compress input)."""
    rng = OF.SplitMix64(100 * field + plen)
    n = 3
    ints = lambda k: [rng.field(p) for _ in range(2 * k)]                 # noqa: E731
    sib_i, path_i, cur_i = ints(n), ints(n * plen), ints(n)
    sib_i[0], cur_i[0] = 0, p - 1                                        # both ends of the field
    sibs = np.ascontiguousarray(_mont(sib_i, p))
    paths = np.ascontiguousarray(_mont(path_i, p)) if plen else np.zeros((1, 2, 4), dtype=np.uint64)
    curs = np.ascontiguousarray(_mont(cur_i, p))
    pt = lambda a, k: (a[2 * k], a[2 * k + 1])                            # noqa: E731
    for i in range(n):
        for index in (0, (1 << (plen + 1)) - 1, int(rng.next() >> 1)):
            exp = {"S": pt(sib_i, i)}
            for k in range(plen):
                exp[("P", k)] = pt(path_i, i * plen + k)
            for j, (left, right) in enumerate(oracle_pairs(plen, index)):
                val = lambda s: pt(cur_i, i) if s[0] in ("C", "H") else (exp["S"] if s == ("S",) else exp[s])   # noqa: E731
                row = np.zeros(32, dtype=np.uint32)
                shim.host_ped_verify_row(field, _p32(np.ascontiguousarray(curs[i]).view(np.uint32)), _p32(sibs.view(np.uint32)),
                                         _p32(paths.view(np.uint32)), i, plen, j, index, _p32(row))
                assert row.tobytes() == jj.serialize_uncompressed(val(left)) + jj.serialize_uncompressed(val(right)), (i, index, j)


# ---------------------------------------------------------------------------------------------------- ABI argument rules
def test_verify_entry_points_validate_before_touching_a_device():
    root, sib, paths = np.zeros(8, dtype=np.uint64), np.zeros((2, 8), dtype=np.uint64), np.zeros((2, 3, 8), dtype=np.uint64)
    idx, ok = np.array([1, 2], dtype=np.uint64), np.full(2, 7, dtype=np.uint8)
    leaves = np.zeros((2, 32), dtype=np.uint8)
    u8 = lambda a: a.ctypes.data_as(N.u8p)                                # noqa: E731
    p = lambda a: a.ctypes.data_as(N.u64p)                                # noqa: E731
    hosts = (N.lib.cpb_merkle_pedersen_verify_batch, N.lib.cpb_merkle_mixed_verify_batch)
    devs = (N.lib.cpb_merkle_pedersen_verify_batch_dev, N.lib.cpb_merkle_mixed_verify_batch_dev)
    for H in hosts:
        # shape first: path_len 63 with null contexts and null buffers
        assert H(None, None, None, None, 32, None, None, 63, None, None, 2) == N.CPB_BAD_PARAMS
        assert H(None, None, None, None, 32, None, None, 63, None, None, 0) == N.CPB_BAD_PARAMS
        # then the buffers (n > 0), before the contexts
        assert H(None, None, None, u8(leaves), 32, p(sib), p(paths), 3, p(idx), u8(ok), 2) == N.CPB_NULL_POINTER
        assert H(None, None, p(root), None, 32, p(sib), p(paths), 3, p(idx), u8(ok), 2) == N.CPB_NULL_POINTER
        assert H(None, None, p(root), u8(leaves), 32, p(sib), None, 3, p(idx), u8(ok), 2) == N.CPB_NULL_POINTER
        assert H(None, None, p(root), u8(leaves), 32, p(sib), p(paths), 3, p(idx), None, 2) == N.CPB_NULL_POINTER
        # then the contexts: null contexts with valid buffers, and with n == 0
        assert H(None, None, p(root), u8(leaves), 32, p(sib), p(paths), 3, p(idx), u8(ok), 2) == N.CPB_NULL_POINTER
        assert H(None, None, None, None, 32, None, None, 3, None, None, 0) == N.CPB_NULL_POINTER
    for D in devs:
        assert D(None, None, None, None, 32, 32, None, None, 63, None, None, 2, None) == N.CPB_BAD_PARAMS
        assert D(None, None, None, None, 32, 16, None, None, 3, None, None, 2, None) == N.CPB_BAD_PARAMS     # leaf_stride < leaf_len
        assert D(None, None, None, None, 32, 16, None, None, 3, None, None, 1, None) == N.CPB_NULL_POINTER   # n == 1: no stride rule
        assert D(None, None, root.ctypes.data, leaves.ctypes.data, 32, 32, None, paths.ctypes.data, 3, idx.ctypes.data, ok.ctypes.data, 2,
                 None) == N.CPB_NULL_POINTER
        assert D(None, None, root.ctypes.data, leaves.ctypes.data, 32, 32, sib.ctypes.data, paths.ctypes.data, 3, idx.ctypes.data,
                 ok.ctypes.data, 2, None) == N.CPB_NULL_POINTER
    assert (ok == 7).all()
    assert N.lib.cpb_abi_version() == 5


# The context rules (curves, devices, Poseidon field and rate), the leaf-length rule and n == 0 need contexts, which need a device:
# tests/test_gpu_merkle_verify_pedersen.py covers them through the C-ABI.


@pytest.mark.skipif(N.lib.cpb_device_count() > 0, reason="an H100 is present")
def test_verify_has_no_cpu_fallback():
    import crypto_primitives_b200 as cp
    from crypto_primitives_b200.crh.pedersen import Parameters, Window
    from crypto_primitives_b200.merkle_tree import MerkleTree, PedersenByteConfig
    w = OPD.Window(4, 8)
    oprm = OPD.setup(w, 3)
    g = cp.BLS12_381_FR.elements([c for ws in oprm.generators for pt in ws for c in pt]).reshape(8, 4, 2, 4)
    prm = Parameters(cp.curves.JUBJUB, Window(4, 8), g)
    tree = MerkleTree(PedersenByteConfig(), np.zeros((4, 2, 4), dtype=np.uint64), np.zeros((3, 2, 4), dtype=np.uint64), prm, prm, 0)
    with pytest.raises(N.CpbError) as e:
        tree.verify_proofs_batch(tree.generate_proofs_batch([1]), np.zeros((1, 4), dtype=np.uint8))
    assert e.value.status in (N.CPB_NO_DEVICE, N.CPB_CUDA_ERROR)
