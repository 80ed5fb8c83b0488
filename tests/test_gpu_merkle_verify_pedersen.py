"""Path verification on the GPU for the byte tree (cpb_merkle_pedersen_verify_batch[_dev]) and the Pedersen-leaf / Poseidon-node tree
(cpb_merkle_mixed_verify_batch[_dev]), include/cpb200.h: every proof of trees built by the C oracle verifies; a tamper matrix makes
exactly the tampered rows false, as oracle/merkle.py::verify_path and the level loop (verify_paths_batch) say; the _dev forms' stride,
bounds, n == 0 and CUDA-graph rules; the context and length rules; a 2^20-leaf tree; the Python and C++ mirrors."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from helpers import ROOT, oracle_config, product_config
import crypto_primitives_b200 as cp
from crypto_primitives_b200 import _native as N
from crypto_primitives_b200.crh.pedersen import CRH, Parameters, Window
from crypto_primitives_b200.merkle_tree import MerkleTree, PedersenByteConfig, PedersenPoseidonConfig, Path, verify_paths_batch
from oracle import cref, fields as OF, merkle as OM, pedersen as OPD

pytestmark = pytest.mark.gpu

_cache = {}


def _p(a):
    return a.ctypes.data_as(N.u64p)


def _torch():
    import torch
    return torch


def setup(chunk_bits=8):
    """Jubjub, window 4 x 256 (R/merkle_tree/tests/mod.rs:12-17): (oracle window, oracle parameters, C oracle, product parameters)."""
    if chunk_bits not in _cache:
        ow = OPD.Window(4, 256)
        oprm = OPD.setup(ow, 5)
        g = cp.BLS12_381_FR.elements([c for w in oprm.generators for pt in w for c in pt]).reshape(256, 4, 2, 4)
        _cache[chunk_bits] = (ow, oprm, cref.Pedersen(oprm, ow), Parameters(cp.curves.JUBJUB, Window(4, 256), g, chunk_bits=chunk_bits))
    return _cache[chunk_bits]


def byte_tree(prm, oc, n, L, seed):
    leaves = np.ascontiguousarray(cref.synth_bytes(seed, n * L).reshape(n, L))
    exp_leaf, exp_nodes = cref.pedersen_merkle(oc, oc, leaves, threads=8)
    return leaves, MerkleTree(PedersenByteConfig(), exp_leaf, exp_nodes, prm, prm, 0)


def to_dev(a):
    torch = _torch()
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.int64) if a.dtype == np.uint64 else a).cuda()


def as_paths(sib, paths, idx):
    return [Path(sib[i], list(paths[i]), int(idx[i])) for i in range(idx.shape[0])]


def level_loop(tree, leaves, proofs, root):
    sib, paths, idx = proofs
    cfg = PedersenByteConfig() if type(tree.config) is PedersenByteConfig else PedersenPoseidonConfig()
    return verify_paths_batch(tree.leaf_hash_param, tree.two_to_one_hash_param, root, leaves, as_paths(sib, paths, idx), cfg)


def tamper(leaves, proofs, plen):
    """One tampered row per case: a leaf byte, the leaf sibling's first coordinate (and, for points, its second), one auth-path node
    at every level, one index bit at every level (bit j = the side of level j).  -> (leaves, proofs, tampered rows)."""
    sib, paths, idx = (a.copy() for a in proofs)
    lv = leaves.copy()
    rows, r = [], 0
    lv[r, r % lv.shape[1]] ^= 0x10
    rows.append(r); r += 1
    for c in range(sib.shape[1] if sib.ndim == 3 else 1):               # x, then y
        s = sib[r].reshape(-1, 4)
        s[c, 0] ^= np.uint64(2)
        rows.append(r); r += 1
    for k in range(plen):
        paths[r].reshape(plen, -1)[k, 0] ^= np.uint64(2)
        rows.append(r); r += 1
    for j in range(plen + 1):
        idx[r] ^= np.uint64(1 << j)
        rows.append(r); r += 1
    assert r <= idx.shape[0]
    return lv, (sib, paths, idx), rows


def check_tamper_matrix(tree, leaves, oracle_verify=None):
    """All proofs of `leaves` (one per leaf, in order), tampered as `tamper` says: exactly the tampered rows are false, and the level
    loop agrees row for row; a tampered root's x or y fails every row.  oracle_verify(i, leaf, proof_i) -> bool for a few rows."""
    n, plen = leaves.shape[0], tree.height() - 2
    proofs = tree.generate_proofs_batch(np.arange(n) % tree.leaf_nodes.shape[0])
    lv, tp, rows = tamper(leaves, proofs, plen)
    got = tree.verify_proofs_batch(tp, lv)
    exp = np.ones(n, dtype=bool)
    exp[rows] = False
    assert np.array_equal(got, exp), np.nonzero(got != exp)
    assert np.array_equal(level_loop(tree, lv, tp, tree.root()), got)
    if oracle_verify is not None:
        for i in rows[:4] + [n - 1]:
            assert oracle_verify(lv[i], (tp[0][i], tp[1][i], int(tp[2][i]))) == bool(got[i]), i
    for c in range(tree.root().reshape(-1, 4).shape[0]):
        bad = tree.root().copy()
        bad.reshape(-1, 4)[c, 0] ^= np.uint64(2)
        assert not tree.verify_proofs_batch(proofs, leaves, root_hash=bad).any()
        assert not level_loop(tree, leaves, proofs, bad).any()


def oracle_byte_verify(ow, oprm, root_mont):
    """oracle/merkle.py::verify_path with the Python Pedersen oracle, on Montgomery-form arrays."""
    p = OF.BLS12_381_FR
    pt = lambda a: tuple(cref.mont_to_ints(np.asarray(a, dtype=np.uint64).reshape(2, 4), p))    # noqa: E731
    h = lambda l, r: OPD.two_to_one_compress(oprm, ow, l, r)                                      # noqa: E731

    def f(leaf, proof):
        sib, paths, idx = proof
        return OM.verify_path((pt(sib), [pt(x) for x in paths], idx), OPD.crh_evaluate(oprm, ow, bytes(leaf)), pt(root_mont), h, h)
    return f


@pytest.mark.parametrize("L", [32, 128])
@pytest.mark.parametrize("n", [1 << 6, 1 << 10])
@pytest.mark.parametrize("chunk_bits", [8, 12, 0])
def test_every_proof_verifies(n, L, chunk_bits):
    _, _, oc, prm = setup(chunk_bits)
    leaves, tree = byte_tree(prm, oc, n, L, 1000 + n + L)
    assert tree.verify_proofs_batch(tree.generate_proofs_batch(np.arange(n)), leaves).all()
    assert tree.verify_proofs_batch([tree.generate_proof(i) for i in (0, 5, n - 1)], leaves[[0, 5, n - 1]]).all()


@pytest.mark.parametrize("chunk_bits", [8, 0])
def test_byte_tree_tamper_matrix(chunk_bits):
    ow, oprm, oc, prm = setup(chunk_bits)
    leaves, tree = byte_tree(prm, oc, 1 << 6, 32, 61)
    check_tamper_matrix(tree, leaves, oracle_byte_verify(ow, oprm, tree.root()))


def test_height_two_and_high_index_bits():
    _, _, oc, prm = setup(8)
    leaves, tree = byte_tree(prm, oc, 2, 32, 2)
    proofs = tree.generate_proofs_batch([0, 1])
    assert tree.verify_proofs_batch(proofs, leaves).all()                 # path_len 0
    check_tamper_matrix(tree, np.concatenate([leaves] * 2))
    leaves, tree = byte_tree(prm, oc, 16, 32, 3)
    sib, paths, idx = tree.generate_proofs_batch(np.arange(16))
    hi = idx | np.uint64(0xABCD << 4) | np.uint64(1 << 63)                  # bits above path_len + 1 are ignored
    assert tree.verify_proofs_batch((sib, paths, hi), leaves).all()


def test_ed_on_bls12_377_against_level_loop():
    prm = CRH.setup(OF.SplitMix64(42), Window(4, 256), cp.curves.ED_ON_BLS12_377)
    n, L = 1 << 6, 64
    leaves = np.ascontiguousarray(cref.synth_bytes(377, n * L).reshape(n, L))
    tree = MerkleTree.new(prm, prm, leaves, config=PedersenByteConfig())
    assert tree.verify_proofs_batch(tree.generate_proofs_batch(np.arange(n)), leaves).all()
    check_tamper_matrix(tree, leaves)


def mixed_setup(curve):
    if curve == "jubjub":
        _, _, oc, prm = setup(0)
        _, ocfg = oracle_config("bls_default_r2")
        return prm, product_config("bls_default_r2"), (oc, cref.Poseidon(ocfg))
    return CRH.setup(OF.SplitMix64(43), Window(4, 256), cp.curves.ED_ON_BLS12_377), product_config("bls377_random"), None


@pytest.mark.parametrize("curve", ["jubjub", "ed_on_bls12_377"])
def test_mixed_tree(curve):
    prm, pcfg, oracles = mixed_setup(curve)
    n, L = 1 << 8, 128
    leaves = np.ascontiguousarray(cref.synth_bytes(88, n * L).reshape(n, L))
    tree = MerkleTree.new(prm, pcfg, leaves, config=PedersenPoseidonConfig())
    if oracles is not None:
        exp_leaf, exp_nodes = cref.mixed_merkle(oracles[0], oracles[1], leaves, threads=8)
        assert np.array_equal(tree.leaf_nodes, exp_leaf) and np.array_equal(tree.non_leaf_nodes, exp_nodes)
    assert tree.verify_proofs_batch(tree.generate_proofs_batch(np.arange(n)), leaves).all()
    check_tamper_matrix(tree, leaves)
    cfg = PedersenPoseidonConfig()
    for i in (0, 77, n - 1):
        pr = tree.generate_proof(i)
        assert pr.verify(prm, pcfg, tree.root(), leaves[i], config=cfg)
        assert not pr.verify(prm, pcfg, tree.root(), leaves[i ^ 1], config=cfg)
        assert not Path(pr.leaf_sibling_hash, pr.auth_path, i ^ 2).verify(prm, pcfg, tree.root(), leaves[i], config=cfg)
    with pytest.raises(ValueError):
        tree.verify_proofs_batch(tree.generate_proofs_batch([0]), np.zeros((1, 129), dtype=np.uint8))


def test_path_verify_byte_tree_is_one_call():
    _, _, oc, prm = setup(8)
    leaves, tree = byte_tree(prm, oc, 1 << 6, 32, 9)
    cfg = PedersenByteConfig()
    for i in (0, 33, 63):
        pr = tree.generate_proof(i)
        assert pr.verify(prm, prm, tree.root(), leaves[i], config=cfg)
        assert not pr.verify(prm, prm, tree.root(), leaves[i ^ 1], config=cfg)
    with pytest.raises(ValueError):
        tree.generate_proof(0).verify(prm, prm, tree.root(), np.zeros(129, dtype=np.uint8), config=cfg)
    other = MerkleTree(cp.merkle_tree.BoweHopwoodByteConfig(), tree.leaf_nodes, tree.non_leaf_nodes, prm, prm, 0)
    with pytest.raises(NotImplementedError):                              # Bowe-Hopwood trees keep the level loop
        other.verify_proofs_batch(tree.generate_proofs_batch([0]), leaves[:1])


# ---------------------------------------------------------------------------------------------------- _dev forms
def dev_call(kind, leaf_ctx, node_ctx, root, lv, L, S, sib, paths, plen, idx, ok, n):
    torch = _torch()
    fn = N.lib.cpb_merkle_pedersen_verify_batch_dev if kind == "byte" else N.lib.cpb_merkle_mixed_verify_batch_dev
    return fn(leaf_ctx, node_ctx, root.data_ptr(), lv.data_ptr(), L, S, sib.data_ptr(), paths.data_ptr() if plen else None, plen,
              idx.data_ptr(), ok.data_ptr(), n, torch.cuda.current_stream().cuda_stream)


@pytest.mark.parametrize("kind", ["byte", "mixed"])
def test_dev_stride_guards_and_empty_batch(kind):
    torch = _torch()
    if kind == "byte":
        _, _, oc, prm = setup(0)
        n, L, S = 1 << 6, 32, 48
        leaves = np.ascontiguousarray(cref.synth_bytes(71, n * L).reshape(n, L))
        tree = MerkleTree.new(prm, prm, leaves, config=PedersenByteConfig())
        lctx, nctx = prm.context(0), prm.context(0)
    else:
        prm, pcfg, _ = mixed_setup("jubjub")
        n, L, S = 1 << 6, 32, 48
        leaves = np.ascontiguousarray(cref.synth_bytes(72, n * L).reshape(n, L))
        tree = MerkleTree.new(prm, pcfg, leaves, config=PedersenPoseidonConfig())
        lctx, nctx = prm.context(0), pcfg.context(0)
    plen = tree.height() - 2
    sib, paths, idx = tree.generate_proofs_batch(np.arange(n))
    lv, tp, rows = tamper(leaves, (sib, paths, idx), plen)
    wide = np.zeros((n, S), dtype=np.uint8)
    wide[:, :L] = lv
    wide[:, L:] = 0xEE                                                     # bytes past leaf_len are not read
    G = 64
    okbuf = torch.full((G + n + G,), 0x5A, dtype=torch.uint8, device="cuda")
    ok = okbuf[G:G + n]
    args = (to_dev(tree.root()), to_dev(wide), L, S, to_dev(tp[0]), to_dev(tp[1]), plen, to_dev(tp[2]))
    N.check(dev_call(kind, lctx, nctx, *args, ok, n))
    torch.cuda.synchronize()
    got = okbuf.cpu().numpy()
    assert (got[:G] == 0x5A).all() and (got[G + n:] == 0x5A).all()
    exp = np.ones(n, dtype=np.uint8)
    exp[rows] = 0
    assert np.array_equal(got[G:G + n], exp)
    okbuf.fill_(0x5A)
    N.check(dev_call(kind, lctx, nctx, *args, ok, 0))                     # n == 0 writes nothing
    torch.cuda.synchronize()
    assert (okbuf.cpu().numpy() == 0x5A).all()


@pytest.mark.parametrize("kind", ["byte", "mixed"])
def test_dev_graph_replay(kind):
    torch = _torch()
    n, L = 1 << 10, 128
    if kind == "byte":
        _, _, oc, prm = setup(0)
        leaves, tree = byte_tree(prm, oc, n, L, 81)
        lctx, nctx = prm.context(0), prm.context(0)
    else:
        prm, pcfg, _ = mixed_setup("jubjub")
        leaves = np.ascontiguousarray(cref.synth_bytes(82, n * L).reshape(n, L))
        tree = MerkleTree.new(prm, pcfg, leaves, config=PedersenPoseidonConfig())
        lctx, nctx = prm.context(0), pcfg.context(0)
    plen = tree.height() - 2
    lv, tp, rows = tamper(leaves, tree.generate_proofs_batch(np.arange(n)), plen)
    args = (to_dev(tree.root()), to_dev(lv), L, L, to_dev(tp[0]), to_dev(tp[1]), plen, to_dev(tp[2]))
    ok = torch.zeros(n, dtype=torch.uint8, device="cuda")
    N.check(dev_call(kind, lctx, nctx, *args, ok, n))                     # eager, also warms up
    torch.cuda.synchronize()
    eager = ok.clone()
    ok.zero_()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            N.check(dev_call(kind, lctx, nctx, *args, ok, n))
    torch.cuda.synchronize()
    assert not ok.any()                                                   # capture ran nothing
    for _ in range(2):
        ok.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(ok, eager)
    exp = np.ones(n, dtype=np.uint8)
    exp[rows] = 0
    assert np.array_equal(eager.cpu().numpy(), exp)


# ---------------------------------------------------------------------------------------------------- context and length rules
def test_host_form_rules():
    _, _, oc, prm = setup(8)
    leaves, tree = byte_tree(prm, oc, 8, 32, 5)
    sib, paths, idx = tree.generate_proofs_batch([1, 2])
    plen = tree.height() - 2
    root, ok = np.ascontiguousarray(tree.root()), np.full(2, 7, dtype=np.uint8)
    u8 = lambda a: np.ascontiguousarray(a).ctypes.data_as(N.u8p)          # noqa: E731
    sib, paths = np.ascontiguousarray(sib), np.ascontiguousarray(paths)
    H, M = N.lib.cpb_merkle_pedersen_verify_batch, N.lib.cpb_merkle_mixed_verify_batch
    ctx = prm.context(0)
    long_leaves = np.zeros((2, 129), dtype=np.uint8)
    assert H(ctx, ctx, _p(root), u8(long_leaves), 129, _p(sib), _p(paths), plen, _p(idx), u8(ok), 2) == N.CPB_BAD_LENGTH
    ed = CRH.setup(OF.SplitMix64(42), Window(4, 256), cp.curves.ED_ON_BLS12_377)
    assert H(ctx, ed.context(0), _p(root), u8(leaves[:2]), 32, _p(sib), _p(paths), plen, _p(idx), u8(ok), 2) == N.CPB_BAD_PARAMS
    assert H(ctx, ctx, _p(root), u8(leaves[:2]), 32, _p(sib), _p(paths), plen, _p(idx), u8(ok), 0) == N.CPB_OK
    assert (ok == 7).all()                                                # n == 0 writes nothing
    # mixed tree: the Poseidon field must be the curve's base field; rate >= 2
    xs, xp = np.ascontiguousarray(sib.reshape(2, 2, 4)[:, 0]), np.ascontiguousarray(paths.reshape(2, plen, 2, 4)[:, :, 0])
    xr = np.ascontiguousarray(root.reshape(2, 4)[0])
    bn = product_config("bn254_r2")
    assert M(ctx, bn.context(0), _p(xr), u8(leaves[:2]), 32, _p(xs), _p(xp), plen, _p(idx), u8(ok), 2) == N.CPB_BAD_PARAMS
    from crypto_primitives_b200.sponge.poseidon import PoseidonConfig, find_poseidon_ark_and_mds
    ark, mds = find_poseidon_ark_and_mds(cp.BLS12_381_FR, 255, 1, 8, 31, 0)
    r1 = PoseidonConfig(cp.BLS12_381_FR, 8, 31, 17, mds, ark, 1, 1)
    assert M(ctx, r1.context(0), _p(xr), u8(leaves[:2]), 32, _p(xs), _p(xp), plen, _p(idx), u8(ok), 2) == N.CPB_UNSUPPORTED
    pcfg = product_config("bls_default_r2")
    assert M(ctx, pcfg.context(0), _p(xr), u8(long_leaves), 129, _p(xs), _p(xp), plen, _p(idx), u8(ok), 2) == N.CPB_BAD_LENGTH
    assert M(ctx, pcfg.context(0), _p(xr), u8(leaves[:2]), 32, _p(xs), _p(xp), plen, _p(idx), u8(ok), 0) == N.CPB_OK
    assert (ok == 7).all()


def test_large_tree_against_level_loop():
    """2^20 leaves of 128 bytes, 18-bit tables: 2^16 random valid proofs plus 2^16 tampered ones, verdicts equal to the level loop."""
    _, _, _, prm = setup(0)
    n, L, k = 1 << 20, 128, 1 << 16
    rng = np.random.default_rng(20)
    leaves = rng.integers(0, 256, size=(n, L), dtype=np.uint8)
    tree = MerkleTree.new(prm, prm, leaves, config=PedersenByteConfig())
    ix = rng.integers(0, n, size=2 * k).astype(np.int64)
    sib, paths, idx = tree.generate_proofs_batch(ix)
    lv = leaves[ix].copy()
    plen = tree.height() - 2
    t = np.arange(k, 2 * k)
    kind = rng.integers(0, 4, size=k)
    lv[t[kind == 0], 7] ^= 1
    sib[t[kind == 1], 1, 2] ^= np.uint64(4)
    lev = rng.integers(0, plen, size=k)
    paths[t[kind == 2], lev[kind == 2], 0, 0] ^= np.uint64(8)
    idx[t[kind == 3]] ^= np.uint64(1) << rng.integers(0, plen + 1, size=int((kind == 3).sum())).astype(np.uint64)
    got = tree.verify_proofs_batch((sib, paths, idx), lv)
    assert got[:k].all() and not got[k:].any()
    assert np.array_equal(got, level_loop(tree, lv, (sib, paths, idx), tree.root()))


def test_cpp_verify_mirror(tmp_path):
    _, _, _, prm = setup(8)
    gens = tmp_path / "gens.bin"
    gens.write_bytes(np.ascontiguousarray(prm.generators, dtype=np.uint64).tobytes())
    out_dir = os.path.join(ROOT, "tests", "host", "_build")
    os.makedirs(out_dir, exist_ok=True)
    exe = os.path.join(out_dir, "test_verify_pedersen")
    lib_dir = os.path.join(ROOT, "crypto_primitives_b200")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "test_verify_pedersen.cpp"), "-L", lib_dir, "-l:libcpb200.so",
                           f"-Wl,-rpath,{lib_dir}", "-o", exe])
    r = subprocess.run([exe, str(gens)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "cpp pedersen verify ok" in r.stdout
