"""Merkle update / check_update on the GPU (cpb_merkle_poseidon_update*, include/cpb200.h) against the oracle: host and _dev forms
on random trees of every Poseidon setup, the check_update rule, the _dev bounds rule, the Pedersen-leaf tree, ragged leaves, the
2^24 bench tree, the C++ mirror and CUDA-graph capture of the _dev form."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from helpers import ROOT, oracle_config, product_config, synth_elems
import crypto_primitives_b200 as cp
from crypto_primitives_b200 import _native as N
from crypto_primitives_b200.merkle_tree import MerkleTree, PedersenPoseidonConfig
from oracle import cref, poseidon as OP

pytestmark = pytest.mark.gpu

SETUPS = {"bn254_r2": 2, "bls_default_r2": 2, "jubjub_merkle_fixture": 3, "bls_sponge_fixture": 4}


def _p(a):
    return a.ctypes.data_as(N.u64p)


def _torch():
    import torch
    return torch


def to_dev(a):
    torch = _torch()
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64)).cuda()


def to_np(t):
    return t.cpu().numpy().view(np.uint64)


def sequential(leaves, idx, new):
    out = leaves.copy()
    for j, i in enumerate(idx):
        if i < out.shape[0]:
            out[i] = new[j]
    return out


def update_host(cfg, ln, nn, idx, new, asserted=None):
    ok = C.c_int(-1)
    ix = np.ascontiguousarray(idx, dtype=np.uint64)
    a = None if asserted is None else np.ascontiguousarray(asserted, dtype=np.uint64)
    N.check(N.lib.cpb_merkle_poseidon_update(cfg.context(0), cfg.context(0), _p(ln), _p(nn), ln.shape[0], _p(ix), _p(new), new.shape[1],
                                             ix.size, None if a is None else _p(a), C.byref(ok)))
    return ok.value


def update_dev(cfg, ln, nn, idx, new, asserted=None):
    torch = _torch()
    ix, nv = to_dev(np.asarray(idx, dtype=np.uint64)), to_dev(new)
    a = None if asserted is None else to_dev(asserted)
    applied = torch.full((1,), 7, dtype=torch.uint8, device="cuda")
    N.check(N.lib.cpb_merkle_poseidon_update_dev(cfg.context(0), cfg.context(0), ln.data_ptr(), nn.data_ptr(), ln.shape[0], ix.data_ptr(),
                                                 nv.data_ptr(), new.shape[1], ix.shape[0], None if a is None else a.data_ptr(),
                                                 applied.data_ptr(), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return int(applied.item())


@pytest.mark.parametrize("which", list(SETUPS))
@pytest.mark.parametrize("n", [2, 4, 1 << 10, 1 << 16])
def test_random_updates_match_oracle(which, n):
    _, ocfg = oracle_config(which)
    cfg = product_config(which)
    L = SETUPS[which]
    O = cref.Poseidon(ocfg)
    leaves = synth_elems(40 + n, (n, L), ocfg.p)
    t0 = MerkleTree.new(cfg, cfg, leaves)
    rng = np.random.default_rng(n + L)
    for k in sorted({1, 2, 17, n // 2, n}):
        idx = rng.integers(0, n, size=k).astype(np.uint64)
        if k >= 2:
            idx[-1] = idx[0]                                              # a repeated index: the last occurrence wins
        new = synth_elems(int(rng.integers(1 << 30)), (k, L), ocfg.p)
        exp_leaf, exp_nodes = cref.poseidon_merkle(O, O, sequential(leaves, idx, new), threads=8)
        ln, nn = t0.leaf_nodes.copy(), t0.non_leaf_nodes.copy()
        assert update_host(cfg, ln, nn, idx, new) == 1
        assert np.array_equal(ln, exp_leaf) and np.array_equal(nn, exp_nodes), ("host", k)
        dl, dn = to_dev(t0.leaf_nodes), to_dev(t0.non_leaf_nodes)
        assert update_dev(cfg, dl, dn, idx, new) == 1
        assert np.array_equal(to_np(dl), exp_leaf) and np.array_equal(to_np(dn), exp_nodes), ("dev", k)


def test_check_update_rule():
    _, ocfg = oracle_config("bn254_r2")
    cfg = product_config("bn254_r2")
    O = cref.Poseidon(ocfg)
    n = 1 << 10
    leaves = synth_elems(7, (n, 2), ocfg.p)
    t0 = MerkleTree.new(cfg, cfg, leaves)
    idx = np.array([5, 900, 5, 1023, 0], dtype=np.uint64)
    new = synth_elems(8, (5, 2), ocfg.p)
    exp_leaf, exp_nodes = cref.poseidon_merkle(O, O, sequential(leaves, idx, new), threads=8)
    wrong = exp_nodes[0].copy()
    wrong[0] ^= np.uint64(1)
    for fn, mk, back in ((update_host, lambda a: a.copy(), lambda a: a), (update_dev, to_dev, to_np)):
        ln, nn = mk(t0.leaf_nodes), mk(t0.non_leaf_nodes)
        assert fn(cfg, ln, nn, idx, new, asserted=wrong) == 0
        assert np.array_equal(back(ln), t0.leaf_nodes) and np.array_equal(back(nn), t0.non_leaf_nodes)      # bit for bit untouched
        assert fn(cfg, ln, nn, idx, new, asserted=exp_nodes[0]) == 1
        assert np.array_equal(back(ln), exp_leaf) and np.array_equal(back(nn), exp_nodes)
        empty = np.zeros((0, 2, 4), dtype=np.uint64)
        assert fn(cfg, ln, nn, np.zeros(0, dtype=np.uint64), empty, asserted=exp_nodes[0]) == 1        # k = 0, current root
        assert fn(cfg, ln, nn, np.zeros(0, dtype=np.uint64), empty, asserted=wrong) == 0
    # the Python mirror keeps its contract: distinct indexes, False on a wrong root
    tree = MerkleTree.new(cfg, cfg, leaves)
    assert tree.check_update_batch([3, 4], new[:2], wrong) is False
    assert np.array_equal(tree.non_leaf_nodes, t0.non_leaf_nodes)
    with pytest.raises(AssertionError):
        tree.update_batch([3, 3], new[:2])


def test_dev_bounds_guard_regions():
    torch = _torch()
    _, ocfg = oracle_config("bls_default_r2")
    cfg = product_config("bls_default_r2")
    O = cref.Poseidon(ocfg)
    n, G = 256, 64
    leaves = synth_elems(11, (n, 2), ocfg.p)
    t0 = MerkleTree.new(cfg, cfg, leaves)
    sentinel = np.full((G, 4), 0x5A5A5A5A5A5A5A5A, dtype=np.uint64)
    buf = to_dev(np.concatenate([sentinel, t0.leaf_nodes, sentinel, t0.non_leaf_nodes, sentinel]))
    ln, nn = buf[G:G + n], buf[2 * G + n:2 * G + 2 * n - 1]
    idx = np.array([n, 3, n + 1, 1 << 40, n - 1, (1 << 64) - 1], dtype=np.uint64)
    new = synth_elems(12, (idx.size, 2), ocfg.p)
    assert update_dev(cfg, ln, nn, idx, new) == 1
    exp_leaf, exp_nodes = cref.poseidon_merkle(O, O, sequential(leaves, idx, new), threads=8)
    got = to_np(buf)
    for g in (got[:G], got[G + n:2 * G + n], got[2 * G + 2 * n - 1:]):
        assert np.array_equal(g, sentinel)
    assert np.array_equal(got[G:G + n], exp_leaf) and np.array_equal(got[2 * G + n:2 * G + 2 * n - 1], exp_nodes)
    torch.cuda.synchronize()


def _mixed_setup():
    from test_gpu_pedersen import setup
    ow, oprm, oc, prm = setup(4, 256, 5)
    _, ocfg = oracle_config("bls_default_r2")
    return oc, prm, ocfg, product_config("bls_default_r2")


def test_mixed_tree_update():
    torch = _torch()
    from crypto_primitives_b200.distributed import CudaMixedBackend
    oc, prm, ocfg, pcfg = _mixed_setup()
    n = 512
    leaves = np.ascontiguousarray(cref.synth_bytes(88, n * 128).reshape(n, 128))
    idx = np.array([7, 300, 7, 511, 0, 1], dtype=np.uint64)
    new = np.ascontiguousarray(cref.synth_bytes(89, idx.size * 128).reshape(idx.size, 128))
    final = leaves.copy()
    for j, i in enumerate(idx):
        final[i] = new[j]
    exp_leaf, exp_nodes = cref.mixed_merkle(oc, cref.Poseidon(ocfg), final, threads=8)
    be = CudaMixedBackend(prm, pcfg, 0)
    dl, dn = be.build_local(torch.from_numpy(leaves).cuda())
    dl, dn = dl.clone(), dn.clone()
    applied = be.update(dl, dn, torch.from_numpy(idx.view(np.int64)).cuda(), torch.from_numpy(new).cuda())
    torch.cuda.synchronize()
    assert int(applied.item()) == 1
    assert np.array_equal(to_np(dl), exp_leaf) and np.array_equal(to_np(dn), exp_nodes)
    # the Python mirror (distinct indexes): the Config's Pedersen leaf hash, then the host-pointer digest form
    tree = MerkleTree.new(prm, pcfg, leaves, config=PedersenPoseidonConfig())
    uniq = [7, 300, 511, 0, 1]
    rows = np.stack([final[i] for i in uniq])
    tree.update_batch(uniq, rows)
    assert np.array_equal(tree.leaf_nodes, exp_leaf) and np.array_equal(tree.non_leaf_nodes, exp_nodes)


def test_ragged_tree_update_with_new_lengths():
    _, ocfg = oracle_config("bls_default_r2")
    cfg = product_config("bls_default_r2")
    n = 64
    rng = np.random.default_rng(3)
    leaves = [synth_elems(500 + i, (int(rng.integers(0, 7)),), ocfg.p) for i in range(n)]
    tree = MerkleTree.new(cfg, cfg, leaves)
    idx = [2, 3, 40, 63]
    new = [synth_elems(600 + j, (L,), ocfg.p) for j, L in enumerate((0, 9, 1, 4))]
    tree.update_batch(idx, new)
    for j, i in enumerate(idx):
        leaves[i] = new[j]
    from oracle import merkle as OM
    ints = [cref.mont_to_ints(x, ocfg.p) if x.shape[0] else [] for x in leaves]
    comp = lambda a, b: OP.two_to_one_compress(ocfg, a, b)                  # noqa: E731
    otree = OM.MerkleTree.new(ints, lambda x: OP.crh_evaluate(ocfg, x), comp, comp)
    assert cref.mont_to_ints(tree.leaf_nodes, ocfg.p) == otree.leaf_nodes
    assert cref.mont_to_ints(tree.non_leaf_nodes, ocfg.p) == otree.non_leaf_nodes


def test_full_size_bench_tree_update():
    torch = _torch()
    sys.path.insert(0, ROOT)
    import bench
    import bench_inputs as BI
    from crypto_primitives_b200.distributed import CudaPoseidonBackend
    prm = bench.poseidon_params(cp, "bn254")
    n = 1 << 24
    leaves = BI.field_elements_torch(torch, N, prm.field.id, BI.SEED_CONFIG4, 0, 2 * n, 0).view(n, 2, 4)
    be = CudaPoseidonBackend(prm, prm, 0)
    ln, nn = be.build_local(leaves)
    ln, nn = ln.clone(), nn.clone()
    g = torch.Generator(device="cuda").manual_seed(5)
    for k in (1 << 16, 1):
        idx = torch.randint(0, n, (k,), device="cuda", generator=g)
        new = BI.field_elements_torch(torch, N, prm.field.id, 1000 + k, 0, 2 * k, 0).view(k, 2, 4)
        applied = be.update(ln, nn, idx, new)
        uniq, inv = torch.unique(idx, return_inverse=True)         # a repeated index takes its last new leaf
        last = torch.full((uniq.shape[0],), -1, dtype=torch.int64, device="cuda").scatter_reduce(
            0, inv, torch.arange(k, device="cuda"), reduce="amax")
        leaves[uniq] = new[last]
        rl, rn = CudaPoseidonBackend(prm, prm, 0).build_local(leaves)
        torch.cuda.synchronize()
        assert int(applied.item()) == 1
        assert torch.equal(ln, rl) and torch.equal(nn, rn), k


def test_cpp_update_mirror():
    out_dir = os.path.join(ROOT, "tests", "host", "_build")
    os.makedirs(out_dir, exist_ok=True)
    exe = os.path.join(out_dir, "test_update")
    lib_dir = os.path.join(ROOT, "crypto_primitives_b200")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "test_update.cpp"),
                           "-L", lib_dir, "-l:libcpb200.so", f"-Wl,-rpath,{lib_dir}", "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "cpp update ok" in r.stdout


def test_dev_update_is_graph_capturable():
    """No host synchronisation in the _dev form: one update captured in a CUDA graph and replayed equals the eager update."""
    torch = _torch()
    from crypto_primitives_b200.distributed import CudaPoseidonBackend
    _, ocfg = oracle_config("bn254_r2")
    cfg = product_config("bn254_r2")
    n = 1 << 12
    leaves = synth_elems(21, (n, 2), ocfg.p)
    t0 = MerkleTree.new(cfg, cfg, leaves)
    be = CudaPoseidonBackend(cfg, cfg, 0)
    idx = torch.tensor([4, 4000, 17, 4], dtype=torch.int64, device="cuda")
    new = to_dev(synth_elems(22, (4, 2), ocfg.p)).view(4, 2, 4)
    el, en = to_dev(t0.leaf_nodes), to_dev(t0.non_leaf_nodes)
    be.update(el, en, idx, new)                                   # eager (also warms the kernels up)
    gl, gn = to_dev(t0.leaf_nodes), to_dev(t0.non_leaf_nodes)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            applied = be.update(gl, gn, idx, new)
    torch.cuda.synchronize()
    assert np.array_equal(to_np(gl), t0.leaf_nodes)              # capture ran nothing
    graph.replay()
    torch.cuda.synchronize()
    assert int(applied.item()) == 1
    assert torch.equal(gl, el) and torch.equal(gn, en)
    exp_leaf, exp_nodes = cref.poseidon_merkle(cref.Poseidon(ocfg), cref.Poseidon(ocfg), sequential(leaves, idx.cpu().numpy(), to_np(new)),
                                               threads=8)
    assert np.array_equal(to_np(gn), exp_nodes) and np.array_equal(to_np(gl), exp_leaf)
