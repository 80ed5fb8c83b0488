"""Merkle update without a GPU: the plan of the device code (csrc/merkle_update.cuh) run on the CPU through a host shim against a
Python model of k sequential MerkleTree::update calls (R/merkle_tree/mod.rs:690-701), the sibling / touched sets of the host-pointer
forms, and the argument rules of the four update entry points of include/cpb200.h."""
import ctypes as C

import numpy as np
import pytest

from helpers import build_host_shim
import crypto_primitives_b200 as cp
from crypto_primitives_b200 import _native as N
from crypto_primitives_b200.merkle_tree import MerkleTree, PoseidonFieldConfig

u64p = C.POINTER(C.c_uint64)
MASK = (1 << 64) - 1


@pytest.fixture(scope="module")
def shim():
    lib = build_host_shim("merkle_update_shim")
    lib.host_upd_toy_hash.restype = C.c_uint64
    lib.host_upd_toy_hash.argtypes = [C.c_uint64, C.c_uint64]
    lib.host_upd_offsets.argtypes = [C.c_int, C.c_uint64, u64p]
    lib.host_upd_run.restype = C.c_int
    lib.host_upd_run.argtypes = [u64p, u64p, C.c_uint64, C.c_int, C.c_int, u64p, u64p, u64p, C.c_uint64, u64p, u64p]
    lib.host_upd_sets.argtypes = [u64p, C.c_uint64, C.c_int, u64p, u64p, u64p, u64p]
    return lib


def _p(a):
    return a.ctypes.data_as(u64p)


def toy(a, b):
    return (a * 0x9E3779B97F4A7C15 + b * 0xC2B2AE3D27D4EB4F + 1) & MASK


def model_tree(leaves):
    """(leaf_nodes, non_leaf_nodes heap order) of one-word digests under the toy hash."""
    n = len(leaves)
    full = [0] * (n - 1) + [int(x) for x in leaves]
    for q in range(n - 2, -1, -1):
        full[q] = toy(full[2 * q + 1], full[2 * q + 2])
    return full[n - 1:], full[:n - 1]


def model_update(leaf_nodes, nodes, idx, digests):
    """k sequential updates in input order; indexes >= n skipped (the _dev rule)."""
    leaves = list(leaf_nodes)
    for i, d in zip(idx, digests):
        if i < len(leaves):
            leaves[int(i)] = int(d)
    return model_tree(leaves)


def run(shim, leaf_nodes, nodes, idx, digests, lt, asserted=None, seed=1):
    h = len(leaf_nodes).bit_length() - 1
    ln = np.array(leaf_nodes, dtype=np.uint64)
    nn = np.array(nodes, dtype=np.uint64)
    ix = np.ascontiguousarray(idx, dtype=np.uint64)
    dg = np.ascontiguousarray(digests, dtype=np.uint64)
    hashes, scratch = C.c_uint64(), C.c_uint64()
    a = None if asserted is None else np.array([asserted], dtype=np.uint64)
    ok = shim.host_upd_run(_p(ix) if ix.size else None, _p(dg) if dg.size else None, ix.size, h, lt, _p(ln), _p(nn),
                           None if a is None else _p(a), seed, C.byref(hashes), C.byref(scratch))
    return ok, [int(x) for x in ln], [int(x) for x in nn], hashes.value, scratch.value


def expected_hashes(n, idx):
    u = {int(i) for i in idx if i < n}
    total = 0
    while u and n > 1:
        u = {i >> 1 for i in u}
        total += len(u)
        n >>= 1
    return total


def index_cases(n, rng):
    cases = {"k1_first": [0], "k1_last": [n - 1], "all": list(range(n)), "all_reversed": list(range(n))[::-1],
             "siblings": [0, 1] if n >= 2 else [0], "dup_last_wins": [n - 1, 0, n - 1, 0, n // 2]}
    cases["random"] = list(rng.integers(0, n, size=min(17, 2 * n)))
    cases["random_dups"] = list(rng.integers(0, max(n // 4, 1), size=min(3 * n, 64)))
    cases["out_of_range"] = [n, 0, n + 5, n - 1, 2 ** 40]
    cases["only_out_of_range"] = [n, n + 1]
    return cases


@pytest.mark.parametrize("n", [2, 4, 8, 64, 1024])
def test_plan_equals_sequential_updates(shim, n):
    rng = np.random.default_rng(n)
    h = n.bit_length() - 1
    leaves = [int(x) for x in rng.integers(0, 2 ** 63, size=n)]
    ln0, nn0 = model_tree(leaves)
    for name, idx in index_cases(n, rng).items():
        idx = [int(i) for i in idx]
        dg = [int(x) for x in rng.integers(0, 2 ** 63, size=len(idx))]
        exp_ln, exp_nn = model_update(ln0, nn0, idx, dg)
        for lt in sorted({-1, h - 1, h // 2, 0}):
            for seed in (1, 2):
                ok, got_ln, got_nn, hashes, scratch = run(shim, ln0, nn0, idx, dg, lt, seed=seed)
                assert ok == 1, (name, lt)
                assert got_ln == exp_ln and got_nn == exp_nn, (name, lt, seed)
                assert hashes == expected_hashes(n, idx), (name, lt)             # every touched node exactly once
                assert scratch <= 2 * n - 1 and scratch == sum(min(len(idx), 1 << l) for l in range(h + 1))


def test_check_update_rule(shim):
    n, rng = 32, np.random.default_rng(5)
    leaves = [int(x) for x in rng.integers(0, 2 ** 63, size=n)]
    ln0, nn0 = model_tree(leaves)
    idx, dg = [3, 9, 3], [11, 12, 13]
    exp_ln, exp_nn = model_update(ln0, nn0, idx, dg)
    ok, got_ln, got_nn, _, _ = run(shim, ln0, nn0, idx, dg, 2, asserted=(exp_nn[0] + 1) & MASK)
    assert ok == 0 and got_ln == ln0 and got_nn == nn0                              # wrong root: untouched
    ok, got_ln, got_nn, _, _ = run(shim, ln0, nn0, idx, dg, 2, asserted=exp_nn[0])
    assert ok == 1 and got_ln == exp_ln and got_nn == exp_nn
    ok, got_ln, got_nn, _, _ = run(shim, ln0, nn0, [], [], 2, asserted=nn0[0])      # k = 0: the current root
    assert ok == 1 and got_ln == ln0 and got_nn == nn0
    ok, _, _, _, _ = run(shim, ln0, nn0, [], [], 2, asserted=nn0[0] ^ 1)
    assert ok == 0


def test_offsets(shim):
    for h, k in ((1, 1), (3, 2), (10, 17), (10, 1024), (10, 5000), (24, 1 << 16)):
        off = np.zeros(66, dtype=np.uint64)
        shim.host_upd_offsets(h, k, _p(off))
        widths = [min(k, 1 << l) for l in range(h + 1)]
        assert [int(x) for x in off[:h + 2]] == [sum(widths[:l]) for l in range(h + 2)]


def model_sets(uniq, h):
    n = 1 << h
    reads, writes, cur = [], [], sorted(set(uniq))
    for l in range(h, -1, -1):
        base = 0 if l == h else n + (1 << l) - 1
        s = set(cur)
        for c in cur:
            writes.append(base + c)
            if l > 0 and (c ^ 1) not in s:
                reads.append(base + (c ^ 1))
        cur = sorted({c >> 1 for c in cur})
    return reads, writes


@pytest.mark.parametrize("n", [2, 4, 256])
def test_host_form_sets(shim, n):
    rng = np.random.default_rng(n + 7)
    h = n.bit_length() - 1
    for uniq in ([0], [n - 1], [0, 1], list(range(n)), sorted(set(int(x) for x in rng.integers(0, n, size=9)))):
        u = np.array(uniq, dtype=np.uint64)
        nr, nw = C.c_uint64(), C.c_uint64()
        shim.host_upd_sets(_p(u), u.size, h, None, C.byref(nr), None, C.byref(nw))
        r = np.zeros(max(nr.value, 1), dtype=np.uint64)
        w = np.zeros(max(nw.value, 1), dtype=np.uint64)
        shim.host_upd_sets(_p(u), u.size, h, _p(r), C.byref(nr), _p(w), C.byref(nw))
        er, ew = model_sets(uniq, h)
        assert [int(x) for x in r[:nr.value]] == er and [int(x) for x in w[:nw.value]] == ew
        assert not set(er) & set(ew)                             # a sibling that is read is never also written


# ---------------------------------------------------------------------------------------------------- ABI argument rules
def _arr(n):
    return np.zeros((max(n, 1), 4), dtype=np.uint64)


def test_update_entry_points_validate_before_touching_a_device():
    ln, nn, idx, dg = _arr(8), _arr(7), np.array([1, 2], dtype=np.uint64), _arr(2)
    ok = C.c_int(7)
    H, HL = N.lib.cpb_merkle_poseidon_update_digests, N.lib.cpb_merkle_poseidon_update
    # null context, otherwise valid
    assert H(None, _p(ln), _p(nn), 8, _p(idx), _p(dg), 2, None, C.byref(ok)) == N.CPB_NULL_POINTER
    assert HL(None, None, _p(ln), _p(nn), 8, _p(idx), _p(dg), 1, 2, None, C.byref(ok)) == N.CPB_NULL_POINTER
    # n not a power of two > 1
    for n in (0, 1, 3, 6):
        assert H(None, _p(ln), _p(nn), n, _p(idx), _p(dg), 2, None, None) == N.CPB_NOT_POW2
        assert N.lib.cpb_merkle_poseidon_update_digests_dev(None, ln.ctypes.data, nn.ctypes.data, n, idx.ctypes.data, dg.ctypes.data, 2,
                                                            None, None, None) == N.CPB_NOT_POW2
    # k >= 2^32, checked before any array is read
    assert H(None, _p(ln), _p(nn), 8, _p(idx), _p(dg), 1 << 32, None, None) == N.CPB_BAD_LENGTH
    assert N.lib.cpb_merkle_poseidon_update_dev(None, None, ln.ctypes.data, nn.ctypes.data, 8, idx.ctypes.data, dg.ctypes.data, 1, 1 << 32,
                                                None, None, None) in (N.CPB_NULL_POINTER, N.CPB_BAD_LENGTH)
    assert N.lib.cpb_merkle_poseidon_update_digests_dev(None, ln.ctypes.data, nn.ctypes.data, 8, idx.ctypes.data, dg.ctypes.data, 1 << 32,
                                                        None, None, None) == N.CPB_BAD_LENGTH
    # host forms: an index >= n is rejected before any copy
    bad = np.array([1, 8], dtype=np.uint64)
    assert H(None, _p(ln), _p(nn), 8, _p(bad), _p(dg), 2, None, C.byref(ok)) == N.CPB_BAD_PARAMS
    assert HL(None, None, _p(ln), _p(nn), 8, _p(bad), _p(dg), 1, 2, None, C.byref(ok)) in (N.CPB_NULL_POINTER, N.CPB_BAD_PARAMS)
    # null arrays
    assert H(None, None, _p(nn), 8, _p(idx), _p(dg), 2, None, None) == N.CPB_NULL_POINTER
    assert H(None, _p(ln), _p(nn), 8, None, _p(dg), 2, None, None) == N.CPB_NULL_POINTER
    assert N.lib.cpb_merkle_poseidon_update_digests_dev(None, ln.ctypes.data, None, 8, idx.ctypes.data, dg.ctypes.data, 2, None, None,
                                                        None) == N.CPB_NULL_POINTER
    assert N.lib.cpb_abi_version() == 5


@pytest.mark.skipif(N.lib.cpb_device_count() > 0, reason="an H100 is present")
def test_update_has_no_cpu_fallback():
    cfg = cp.get_default_poseidon_parameters(cp.BLS12_381_FR, 2, False)
    tree = MerkleTree(PoseidonFieldConfig(), np.zeros((4, 4), dtype=np.uint64), np.zeros((3, 4), dtype=np.uint64), cfg, cfg, 0)
    with pytest.raises(N.CpbError) as e:
        tree.update_batch([1], np.zeros((1, 2, 4), dtype=np.uint64))
    assert e.value.status in (N.CPB_NO_DEVICE, N.CPB_CUDA_ERROR)
