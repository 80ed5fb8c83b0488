"""Ragged Poseidon batches on the GPU: CRH, sponge, Merkle build and path verification over inputs of different lengths
(include/cpb200.h, "Poseidon over inputs of different lengths"), against the oracles, through the C-ABI, the Python API and the
C++ header."""
import os
import random
import subprocess

import numpy as np
import pytest

from helpers import ALL_CONFIGS, ROOT, oracle_config, product_config
import crypto_primitives_b200 as cp
from crypto_primitives_b200 import _native as N
from crypto_primitives_b200 import ragged as R
from crypto_primitives_b200.crh.poseidon import CRH
from crypto_primitives_b200.merkle_tree import MerkleTree
from oracle import cref, fields as OF, merkle as OM, poseidon as OP
from test_poseidon_lane1_basis import random_config

pytestmark = pytest.mark.gpu


def _batch(p, lens, seed, front=3):
    """Inputs of the given lengths behind `front` other elements: (values, offsets with offsets[0] = front, per-input arrays)."""
    vals = cref.synth_field_mont(seed, front + int(sum(lens)), p).reshape(-1, 4)
    offsets = np.array(np.cumsum([front] + list(lens)), dtype=np.uint64)
    parts = [vals[offsets[i]:offsets[i + 1]] for i in range(len(lens))]
    return vals, offsets, parts


def _oracle_crh(O, parts, threads=os.cpu_count() or 8):
    """The C oracle's uniform crh_batch, one call per length."""
    vals, off = R.pack(parts)
    return _oracle_crh_flat(O, vals, off, threads)


def _oracle_crh_flat(O, vals, off, threads=os.cpu_count() or 8):
    off = off.astype(np.int64)
    lens = np.diff(off)
    out = np.empty((lens.size, 4), dtype=np.uint64)
    for L in np.unique(lens):
        idx = np.nonzero(lens == L)[0]
        out[idx] = O.crh_batch(vals[off[idx][:, None] + np.arange(L)[None, :]], threads=threads)
    return out


def _interleaved_lengths(r, n, seed):
    rnd = random.Random(seed)
    return [rnd.choice([0, 1, r - 1, r, r + 1, 2 * r, 2 * r + 1, 17]) for _ in range(n)]


@pytest.mark.parametrize("which", ALL_CONFIGS)
def test_ragged_crh_matches_oracle(which):
    _, ocfg = oracle_config(which)
    cfg = product_config(which)
    vals, off, parts = _batch(ocfg.p, _interleaved_lengths(ocfg.rate, 1000, 5), 40)
    want = _oracle_crh(cref.Poseidon(ocfg), parts)
    assert np.array_equal(CRH.evaluate_ragged(cfg, vals, off), want)
    assert np.array_equal(CRH.evaluate_batch(cfg, parts), want)                # a list of different lengths packs itself


@pytest.mark.parametrize("fname,t", [("bls12_381_fr", 2), ("bn254_fr", 5), ("jubjub_fr", 9)])
def test_ragged_crh_other_widths(fname, t):
    p = OF.MODULI[fname]
    ocfg = random_config(p, t, 8, 21, 5, 7 * t)
    cfg = cp.PoseidonConfig.from_ints(cp.FIELDS[fname], 8, 21, 5, ocfg.mds, ocfg.ark, ocfg.rate, 1)
    vals, off, parts = _batch(p, _interleaved_lengths(ocfg.rate, 1000, t), 50 + t)
    assert np.array_equal(CRH.evaluate_ragged(cfg, vals, off), _oracle_crh(cref.Poseidon(ocfg), parts))


@pytest.mark.parametrize("L", [2, 5])
def test_equal_lengths_match_the_uniform_call(L):
    import torch
    import bench_inputs as BI
    cfg = cp.PoseidonConfig.from_ints(cp.BN254_FR, *_bn254_shape())
    n = 1 << 20
    x = BI.field_elements_torch(torch, N, cp.BN254_FR.id, BI.SEED_CONFIG4, 0, n * L, 0).view(n, L, 4)
    uni = CRH.evaluate_batch_dev(cfg, x)
    off = torch.arange(0, n + 1, dtype=torch.int64, device=x.device) * L
    rag = CRH.evaluate_ragged_dev(cfg, x.view(-1, 4), off)
    torch.cuda.synchronize()
    assert torch.equal(uni, rag)


def _bn254_shape():
    _, o = oracle_config("bn254_r2")
    return o.full_rounds, o.partial_rounds, o.alpha, o.mds, o.ark, o.rate, o.capacity


@pytest.mark.parametrize("which", ["bn254_r2", "bls_sponge_fixture"])
def test_ragged_sponge_matches_oracle(which):
    _, ocfg = oracle_config(which)
    cfg = product_config(which)
    r = ocfg.rate
    vals, off, parts = _batch(ocfg.p, _interleaved_lengths(r, 48, 9), 60)
    ints = [cref.mont_to_ints(x, ocfg.p) if x.shape[0] else [] for x in parts]
    for n_sq in (1, r, r + 1, 3 * r):
        got = cp.absorb_squeeze_ragged(cfg, vals, off, n_sq)
        assert np.array_equal(cp.absorb_squeeze_batch(cfg, parts, n_sq), got)
        for i, x in enumerate(ints):
            s = OP.PoseidonSponge(ocfg)
            s.absorb(x)
            assert cref.mont_to_ints(got[i], ocfg.p) == s.squeeze_native_field_elements(n_sq), (n_sq, i)


# ---------------------------------------------------------------------------------------------------- trees
def _build_dev(cfg, vals, off, stream):
    import torch
    n = off.shape[0] - 1
    with torch.cuda.stream(stream):
        v = torch.from_numpy(vals.view(np.int64)).cuda()
        o = torch.from_numpy(off.view(np.int64)).cuda()
        ln = torch.empty((n, 4), dtype=torch.int64, device="cuda")
        nn = torch.empty((n - 1, 4), dtype=torch.int64, device="cuda")
        ctx = cfg.context(0)
        N.check(N.lib.cpb_merkle_poseidon_build_ragged_dev(ctx, ctx, v.data_ptr(), o.data_ptr(), n, ln.data_ptr(), nn.data_ptr(),
                                                           stream.cuda_stream))
    stream.synchronize()
    return ln.cpu().numpy().view(np.uint64), nn.cpu().numpy().view(np.uint64)


def test_ragged_tree_against_python_oracle():
    import torch
    _, ocfg = oracle_config("bn254_r2")
    cfg = product_config("bn254_r2")
    rnd = random.Random(11)
    n = 1 << 10
    vals, off, parts = _batch(ocfg.p, [rnd.randrange(9) for _ in range(n)], 70)
    ints = [cref.mont_to_ints(x, ocfg.p) if x.shape[0] else [] for x in parts]
    comp = lambda a, b: OP.two_to_one_compress(ocfg, a, b)                  # noqa: E731
    otree = OM.MerkleTree.new(ints, lambda x: OP.crh_evaluate(ocfg, x), comp, comp)
    t = MerkleTree.new(cfg, cfg, parts)
    assert cref.mont_to_ints(t.leaf_nodes, ocfg.p) == otree.leaf_nodes
    assert cref.mont_to_ints(t.non_leaf_nodes, ocfg.p) == otree.non_leaf_nodes
    ln, nn = _build_dev(cfg, vals, off, torch.cuda.Stream())
    assert np.array_equal(ln, t.leaf_nodes) and np.array_equal(nn, t.non_leaf_nodes)


def test_ragged_tree_2_20_against_c_oracle():
    import torch
    _, ocfg = oracle_config("bn254_r2")
    cfg = product_config("bn254_r2")
    n = 1 << 20
    lens = np.random.default_rng(3).integers(0, 9, n)
    vals, off, parts = _batch(ocfg.p, lens, 80)
    O = cref.Poseidon(ocfg)
    level = _oracle_crh_flat(O, vals, off)
    want_leaf, nodes = level, []
    while level.shape[0] > 1:
        level = O.compress_batch(level.reshape(-1, 2, 4), threads=os.cpu_count() or 8)
        nodes.insert(0, level)
    want_nodes = np.concatenate(nodes)                                        # heap order: root level first
    ln, nn = _build_host(cfg, vals, off)
    assert np.array_equal(ln, want_leaf) and np.array_equal(nn, want_nodes)
    ln, nn = _build_dev(cfg, vals, off, torch.cuda.Stream())
    assert np.array_equal(ln, want_leaf) and np.array_equal(nn, want_nodes)


def _build_host(cfg, vals, off):
    from crypto_primitives_b200.merkle_tree import PoseidonFieldConfig
    return PoseidonFieldConfig().build_ragged(cfg, cfg, vals, off, 0)


def test_ragged_tree_python_api():
    _, ocfg = oracle_config("jubjub_merkle_fixture")
    cfg = product_config("jubjub_merkle_fixture")
    p, r = ocfg.p, ocfg.rate
    rnd = random.Random(21)
    n = 64
    _, _, parts = _batch(p, [rnd.randrange(3 * r + 2) for _ in range(n)], 90)
    leaves = [x.copy() for x in parts]
    tree = MerkleTree.new(cfg, cfg, leaves)
    root = tree.root()
    proofs = [tree.generate_proof(i) for i in range(n)]
    assert all(proofs[i].verify(cfg, cfg, root, leaves[i]) for i in range(n))
    assert tree.verify_proofs_batch(proofs, leaves).all()
    assert tree.verify_proofs_batch(tree.generate_proofs_batch(range(n)), leaves).all()
    assert cp.merkle_tree.verify_paths_batch(cfg, cfg, root, leaves, proofs).all()
    assert tree.generate_multi_proof(range(n)).verify(cfg, cfg, root, leaves)

    # one more zero element: the oracle's answer, and the path verifies exactly when the zero stays inside the last block
    zero = np.zeros((1, 4), dtype=np.uint64)
    for i in range(n):
        L = leaves[i].shape[0]
        ext = np.concatenate([leaves[i], zero])
        inside = L % r != 0 or L == 0
        want = OP.crh_evaluate(ocfg, cref.mont_to_ints(ext, p))
        assert cref.mont_to_ints(CRH.evaluate(cfg, ext), p) == [want]
        assert proofs[i].verify(cfg, cfg, root, ext) == inside, (i, L)
    ext_leaves = [np.concatenate([x, zero]) for x in leaves]
    ok = tree.verify_proofs_batch(proofs, ext_leaves)
    assert ok.tolist() == [x.shape[0] % r != 0 or x.shape[0] == 0 for x in leaves]

    # updates with new leaves of new lengths agree with the oracle tree of the updated leaves
    idx = [3, 17, 40, 63]
    _, _, new = _batch(p, [0, 3 * r + 3, 1, 2 * r], 91)
    for k, i in enumerate(idx):
        leaves[i] = new[k]
    ints = [cref.mont_to_ints(x, p) if x.shape[0] else [] for x in leaves]
    comp = lambda a, b: OP.two_to_one_compress(ocfg, a, b)                  # noqa: E731
    otree = OM.MerkleTree.new(ints, lambda x: OP.crh_evaluate(ocfg, x), comp, comp)
    t2 = MerkleTree.new(cfg, cfg, [x.copy() for x in parts])
    assert t2.check_update_batch(idx, new, root) is False                    # wrong root: untouched
    assert np.array_equal(t2.root(), root)
    t2.update_batch(idx[:2], new[:2])
    assert t2.check_update_batch(idx[2:], new[2:], cfg.field.elements([otree.root()])[0])
    assert cref.mont_to_ints(t2.non_leaf_nodes, p) == otree.non_leaf_nodes
    assert cref.mont_to_ints(t2.leaf_nodes, p) == otree.leaf_nodes


def test_ragged_errors():
    import torch
    cfg = product_config("bls_default_r2")
    vals = cref.synth_field_mont(5, 12, OF.BLS12_381_FR).reshape(-1, 4)
    with pytest.raises(ValueError):
        CRH.evaluate_ragged(cfg, vals, [0, 4, 2, 6])                        # decreasing offsets: CPB_BAD_LENGTH
    with pytest.raises(ValueError):
        cp.absorb_squeeze_ragged(cfg, vals, [0, 4, 2, 6], 2)
    from crypto_primitives_b200.merkle_tree import PoseidonFieldConfig
    with pytest.raises(ValueError):
        PoseidonFieldConfig().build_ragged(cfg, cfg, vals, [0, 4, 2, 6, 7], 0)
    with pytest.raises(ValueError):
        MerkleTree.new(cfg, cfg, [vals[:1], vals[:2], vals[:3]])             # three leaves: not a power of two
    assert CRH.evaluate_ragged(cfg, vals, [5]).shape == (0, 4)
    assert cp.absorb_squeeze_ragged(cfg, vals, [2], 3).shape == (0, 3, 4)
    v = torch.from_numpy(vals.view(np.int64)).cuda()
    assert CRH.evaluate_ragged_dev(cfg, v, torch.tensor([3], dtype=torch.int64, device="cuda")).shape == (0, 4)
    # the _dev form reads a decreasing pair as an empty input and nothing outside [offsets[0], offsets[n])
    _, ocfg = oracle_config("bls_default_r2")
    O = cref.Poseidon(ocfg)
    for off, parts in (([2, 5, 3, 9, 11], [vals[2:5], vals[0:0], vals[3:9], vals[9:11]]),
                       ([2, 5, 1, 9, 11], [vals[2:5], vals[0:0], vals[2:9], vals[9:11]])):      # 1 < offsets[0]: clamped
        out = CRH.evaluate_ragged_dev(cfg, v, torch.tensor(off, dtype=torch.int64, device="cuda"))
        assert np.array_equal(out.cpu().numpy().view(np.uint64), _oracle_crh(O, parts))


def test_cpp_ragged_root_matches_python():
    out_dir = os.path.join(ROOT, "tests", "host", "_build")
    os.makedirs(out_dir, exist_ok=True)
    exe = os.path.join(out_dir, "test_ragged")
    lib_dir = os.path.join(ROOT, "crypto_primitives_b200")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "test_ragged.cpp"),
                           "-L", lib_dir, "-l:libcpb200.so", f"-Wl,-rpath,{lib_dir}", "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "cpp ragged ok" in r.stdout
    line = [l for l in r.stdout.splitlines() if l.startswith("ragged root")][0]
    words = [int(w, 16) for w in line.split("=")[1].split()][::-1]
    f = cp.BLS12_381_FR
    cfg = cp.get_default_poseidon_parameters(f, 2, False)
    leaves = [f.elements([31 * i + 7 * k + 1 + (k << 64) for k in range(i % 9)]) for i in range(16)]
    tree = MerkleTree.new(cfg, cfg, leaves)
    assert tree.root().tolist() == words
