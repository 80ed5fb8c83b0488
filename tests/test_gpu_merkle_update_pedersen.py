"""Merkle update / check_update on the GPU for byte trees with Pedersen inner nodes (cpb_merkle_pedersen_update*, include/cpb200.h):
host and _dev forms against the C oracle on Jubjub trees with 8-, 12- and 18-bit table contexts, ed-on-BLS12-377 against a device
rebuild, the check_update rule, the _dev bounds rule, leaf and digest forms, CUDA-graph capture, a 2^20-leaf tree, the Python and
torch mirrors and the C++ mirror."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from helpers import ROOT
import crypto_primitives_b200 as cp
from crypto_primitives_b200 import _native as N
from crypto_primitives_b200.crh.pedersen import CRH, Parameters, Window
from crypto_primitives_b200.merkle_tree import MerkleTree, PedersenByteConfig
from oracle import cref, fields as OF, pedersen as OPD

pytestmark = pytest.mark.gpu

_cache = {}


def _p(a):
    return a.ctypes.data_as(N.u64p)


def _torch():
    import torch
    return torch


def setup(chunk_bits=8):
    """Jubjub, window 4 x 256 (R/merkle_tree/tests/mod.rs:12-17): (oracle C context, product parameters at `chunk_bits`)."""
    if chunk_bits not in _cache:
        ow = OPD.Window(4, 256)
        oprm = OPD.setup(ow, 5)
        g = cp.BLS12_381_FR.elements([c for w in oprm.generators for pt in w for c in pt]).reshape(256, 4, 2, 4)
        _cache[chunk_bits] = (cref.Pedersen(oprm, ow), Parameters(cp.curves.JUBJUB, Window(4, 256), g, chunk_bits=chunk_bits))
    return _cache[chunk_bits]


def to_dev(a):
    torch = _torch()
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.int64) if a.dtype == np.uint64 else a).cuda()


def to_np(t):
    return t.cpu().numpy().view(np.uint64)


def sequential(leaves, idx, new):
    out = leaves.copy()
    for j, i in enumerate(idx):
        if i < out.shape[0]:
            out[i] = new[j]
    return out


def update_host(prm, ln, nn, idx, new, asserted=None):
    ok = C.c_int(-1)
    ix = np.ascontiguousarray(idx, dtype=np.uint64)
    a = None if asserted is None else np.ascontiguousarray(asserted, dtype=np.uint64)
    lv = np.ascontiguousarray(new, dtype=np.uint8)
    N.check(N.lib.cpb_merkle_pedersen_update(prm.context(0), prm.context(0), _p(ln), _p(nn), ln.shape[0], _p(ix), lv.ctypes.data_as(N.u8p),
                                             lv.shape[1], ix.size, None if a is None else _p(a), C.byref(ok)))
    return ok.value


def update_dev(prm, ln, nn, idx, new, asserted=None):
    """The leaf form on device tensors through CudaPedersenBackend.update."""
    torch = _torch()
    from crypto_primitives_b200.distributed import CudaPedersenBackend
    be = CudaPedersenBackend(prm, prm, 0)
    ix = to_dev(np.asarray(idx, dtype=np.uint64))
    applied = be.update(ln, nn, ix, to_dev(np.ascontiguousarray(new, dtype=np.uint8)), None if asserted is None else to_dev(asserted))
    torch.cuda.synchronize()
    return int(applied.item())


@pytest.mark.parametrize("leaf_len", [32, 128])
@pytest.mark.parametrize("n", [2, 4, 1 << 10, 1 << 12])
def test_random_updates_match_oracle(n, leaf_len):
    oc, prm8 = setup(8)
    ctxs = [prm8, setup(0)[1], setup(12)[1]]                          # 8-bit (shared-memory tables), default (18-bit), 12-bit
    leaves = np.ascontiguousarray(cref.synth_bytes(40 + n + leaf_len, n * leaf_len).reshape(n, leaf_len))
    t0 = MerkleTree.new(prm8, prm8, leaves, config=PedersenByteConfig())
    rng = np.random.default_rng(n + leaf_len)
    for k in sorted({1, 2, 17, n // 2, n}):
        idx = rng.integers(0, n, size=k).astype(np.uint64)
        if k >= 2:
            idx[-1] = idx[0]                                              # a repeated index: the last occurrence wins
        new = np.ascontiguousarray(cref.synth_bytes(int(rng.integers(1 << 30)), k * leaf_len).reshape(k, leaf_len))
        exp_leaf, exp_nodes = cref.pedersen_merkle(oc, oc, sequential(leaves, idx, new), threads=8)
        for prm in ctxs:
            ln, nn = t0.leaf_nodes.copy(), t0.non_leaf_nodes.copy()
            assert update_host(prm, ln, nn, idx, new) == 1
            assert np.array_equal(ln, exp_leaf) and np.array_equal(nn, exp_nodes), ("host", k, prm.chunk_bits)
            dl, dn = to_dev(t0.leaf_nodes), to_dev(t0.non_leaf_nodes)
            assert update_dev(prm, dl, dn, idx, new) == 1
            assert np.array_equal(to_np(dl), exp_leaf), ("dev", k, prm.chunk_bits)
            assert np.array_equal(to_np(dn), exp_nodes), ("dev", k, prm.chunk_bits)


def test_ed_on_bls12_377_against_rebuild():
    curve = cp.curves.ED_ON_BLS12_377
    prm = CRH.setup(OF.SplitMix64(42), Window(4, 256), curve)
    cfg = PedersenByteConfig()
    n, L = 1 << 10, 64
    leaves = np.ascontiguousarray(cref.synth_bytes(377, n * L).reshape(n, L))
    t0 = MerkleTree.new(prm, prm, leaves, config=cfg)
    rng = np.random.default_rng(377)
    for k in (1, 17, n):
        idx = rng.integers(0, n, size=k).astype(np.uint64)
        if k >= 2:
            idx[-1] = idx[0]
        new = np.ascontiguousarray(cref.synth_bytes(400 + k, k * L).reshape(k, L))
        ref = MerkleTree.new(prm, prm, sequential(leaves, idx, new), config=cfg)
        ln, nn = t0.leaf_nodes.copy(), t0.non_leaf_nodes.copy()
        assert update_host(prm, ln, nn, idx, new) == 1
        assert np.array_equal(ln, ref.leaf_nodes) and np.array_equal(nn, ref.non_leaf_nodes), k
        dl, dn = to_dev(t0.leaf_nodes), to_dev(t0.non_leaf_nodes)
        assert update_dev(prm, dl, dn, idx, new) == 1
        assert np.array_equal(to_np(dl).reshape(ref.leaf_nodes.shape), ref.leaf_nodes)
        assert np.array_equal(to_np(dn).reshape(ref.non_leaf_nodes.shape), ref.non_leaf_nodes)


def test_check_update_rule():
    oc, prm = setup(8)
    n, L = 1 << 10, 32
    leaves = np.ascontiguousarray(cref.synth_bytes(7, n * L).reshape(n, L))
    t0 = MerkleTree.new(prm, prm, leaves, config=PedersenByteConfig())
    idx = np.array([5, 900, 5, 1023, 0], dtype=np.uint64)
    new = np.ascontiguousarray(cref.synth_bytes(8, 5 * L).reshape(5, L))
    exp_leaf, exp_nodes = cref.pedersen_merkle(oc, oc, sequential(leaves, idx, new), threads=8)
    wrong = exp_nodes[0].copy()
    wrong[1, 3] ^= np.uint64(1)                                           # only y differs: all 16 words are compared
    for fn, mk, back in ((update_host, lambda a: a.copy(), lambda a: a), (update_dev, to_dev, lambda t: to_np(t))):
        ln, nn = mk(t0.leaf_nodes), mk(t0.non_leaf_nodes)
        assert fn(prm, ln, nn, idx, new, asserted=wrong) == 0
        assert np.array_equal(back(ln).reshape(t0.leaf_nodes.shape), t0.leaf_nodes)          # bit for bit untouched
        assert np.array_equal(back(nn).reshape(t0.non_leaf_nodes.shape), t0.non_leaf_nodes)
        assert fn(prm, ln, nn, idx, new, asserted=exp_nodes[0]) == 1
        assert np.array_equal(back(ln).reshape(exp_leaf.shape), exp_leaf) and np.array_equal(back(nn).reshape(exp_nodes.shape), exp_nodes)
        empty = np.zeros((0, L), dtype=np.uint8)
        assert fn(prm, ln, nn, np.zeros(0, dtype=np.uint64), empty, asserted=exp_nodes[0]) == 1      # k = 0, current root
        assert fn(prm, ln, nn, np.zeros(0, dtype=np.uint64), empty, asserted=wrong) == 0
    # the Python mirror keeps its contract: distinct indexes, False on a wrong root
    tree = MerkleTree.new(prm, prm, leaves, config=PedersenByteConfig())
    assert tree.check_update_batch([3, 4], new[:2], wrong) is False
    assert np.array_equal(tree.non_leaf_nodes, t0.non_leaf_nodes) and np.array_equal(tree.leaf_nodes, t0.leaf_nodes)
    with pytest.raises(AssertionError):
        tree.update_batch([3, 3], new[:2])
    with pytest.raises(ValueError):
        tree.update_batch([3], np.zeros((1, 129), dtype=np.uint8))       # over the 1024-bit window


def test_dev_bounds_guard_regions():
    torch = _torch()
    oc, prm = setup(8)
    n, G, L = 256, 16, 32
    leaves = np.ascontiguousarray(cref.synth_bytes(11, n * L).reshape(n, L))
    t0 = MerkleTree.new(prm, prm, leaves, config=PedersenByteConfig())
    sentinel = np.full((G, 2, 4), 0x5A5A5A5A5A5A5A5A, dtype=np.uint64)
    buf = to_dev(np.concatenate([sentinel, t0.leaf_nodes, sentinel, t0.non_leaf_nodes, sentinel]))
    ln, nn = buf[G:G + n], buf[2 * G + n:2 * G + 2 * n - 1]
    idx = np.array([n, 3, n + 1, 1 << 40, n - 1, (1 << 64) - 1], dtype=np.uint64)
    new = np.ascontiguousarray(cref.synth_bytes(12, idx.size * L).reshape(idx.size, L))
    assert update_dev(prm, ln, nn, idx, new) == 1
    exp_leaf, exp_nodes = cref.pedersen_merkle(oc, oc, sequential(leaves, idx, new), threads=8)
    got = to_np(buf).reshape(-1, 2, 4)
    for g in (got[:G], got[G + n:2 * G + n], got[2 * G + 2 * n - 1:]):
        assert np.array_equal(g, sentinel)
    assert np.array_equal(got[G:G + n], exp_leaf) and np.array_equal(got[2 * G + n:2 * G + 2 * n - 1], exp_nodes)
    torch.cuda.synchronize()


def test_leaf_form_with_stride_equals_digest_form():
    torch = _torch()
    oc, prm = setup(0)
    n, L, S = 1 << 10, 32, 48
    leaves = np.ascontiguousarray(cref.synth_bytes(13, n * L).reshape(n, L))
    t0 = MerkleTree.new(prm, prm, leaves, config=PedersenByteConfig())
    idx = np.array([9, 1000, 9, 0, 511, 512], dtype=np.uint64)
    k = idx.size
    wide = np.ascontiguousarray(cref.synth_bytes(14, k * S).reshape(k, S))
    rows = wide[:, :L]                                                    # leaf_stride 48 > leaf_len 32
    dig = CRH.evaluate_batch(prm, np.ascontiguousarray(rows))
    s = torch.cuda.current_stream().cuda_stream
    ctx = prm.context(0)
    a = torch.zeros(3, dtype=torch.uint8, device="cuda")
    dl1, dn1 = to_dev(t0.leaf_nodes), to_dev(t0.non_leaf_nodes)
    tw, ti = to_dev(wide), to_dev(idx)
    N.check(N.lib.cpb_merkle_pedersen_update_dev(ctx, ctx, dl1.data_ptr(), dn1.data_ptr(), n, ti.data_ptr(), tw.data_ptr(), L, S, k, None,
                                                 a[0:1].data_ptr(), s))
    dl2, dn2 = to_dev(t0.leaf_nodes), to_dev(t0.non_leaf_nodes)
    td = to_dev(dig)
    N.check(N.lib.cpb_merkle_pedersen_update_digests_dev(ctx, dl2.data_ptr(), dn2.data_ptr(), n, ti.data_ptr(), td.data_ptr(), k, None,
                                                         a[1:2].data_ptr(), s))
    hl, hn = t0.leaf_nodes.copy(), t0.non_leaf_nodes.copy()
    ok = C.c_int(-1)
    N.check(N.lib.cpb_merkle_pedersen_update_digests(ctx, _p(hl), _p(hn), n, _p(idx), _p(np.ascontiguousarray(dig)), k, None, C.byref(ok)))
    torch.cuda.synchronize()
    assert a[:2].tolist() == [1, 1] and ok.value == 1
    assert torch.equal(dl1, dl2) and torch.equal(dn1, dn2)
    assert np.array_equal(to_np(dl1).reshape(hl.shape), hl) and np.array_equal(to_np(dn1).reshape(hn.shape), hn)
    exp_leaf, exp_nodes = cref.pedersen_merkle(oc, oc, sequential(leaves, idx, np.ascontiguousarray(rows)), threads=8)
    assert np.array_equal(hl, exp_leaf) and np.array_equal(hn, exp_nodes)


def test_dev_update_is_graph_capturable():
    """No host synchronisation in the _dev form: one update captured in a CUDA graph and replayed equals the eager update."""
    torch = _torch()
    from crypto_primitives_b200.distributed import CudaPedersenBackend
    oc, prm = setup(0)
    n, L = 1 << 12, 128
    leaves = np.ascontiguousarray(cref.synth_bytes(21, n * L).reshape(n, L))
    be = CudaPedersenBackend(prm, prm, 0)
    tl, tn = be.build_local(to_dev(leaves))
    l0, n0 = tl.clone(), tn.clone()
    idx = torch.tensor([4, 4000, 17, 4], dtype=torch.int64, device="cuda")
    new = to_dev(np.ascontiguousarray(cref.synth_bytes(22, 4 * L).reshape(4, L)))
    el, en = l0.clone(), n0.clone()
    be.update(el, en, idx, new)                                           # eager (also warms the kernels up)
    gl, gn = l0.clone(), n0.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            applied = be.update(gl, gn, idx, new)
    torch.cuda.synchronize()
    assert torch.equal(gl, l0)                                            # capture ran nothing
    graph.replay()
    torch.cuda.synchronize()
    assert int(applied.item()) == 1
    assert torch.equal(gl, el) and torch.equal(gn, en)
    exp_leaf, exp_nodes = cref.pedersen_merkle(oc, oc, sequential(leaves, idx.cpu().numpy(), new.cpu().numpy()), threads=8)
    assert np.array_equal(to_np(gn).reshape(exp_nodes.shape), exp_nodes) and np.array_equal(to_np(gl).reshape(exp_leaf.shape), exp_leaf)


def test_large_tree_update_equals_rebuild():
    """2^20 leaves of 128 bytes, k = 2^16 random indexes with the _dev form in place = a device rebuild of the modified leaves."""
    torch = _torch()
    from crypto_primitives_b200.distributed import CudaPedersenBackend
    _, prm = setup(0)
    n, L, k = 1 << 20, 128, 1 << 16
    g = torch.Generator(device="cuda").manual_seed(3)
    leaves = torch.randint(0, 256, (n, L), dtype=torch.uint8, device="cuda", generator=g)
    be = CudaPedersenBackend(prm, prm, 0)
    ln, nn = be.build_local(leaves)
    ln, nn = ln.clone(), nn.clone()
    idx = torch.randint(0, n, (k,), device="cuda", generator=g)
    new = torch.randint(0, 256, (k, L), dtype=torch.uint8, device="cuda", generator=g)
    applied = be.update(ln, nn, idx, new)
    uniq, inv = torch.unique(idx, return_inverse=True)                    # a repeated index takes its last new leaf
    last = torch.full((uniq.shape[0],), -1, dtype=torch.int64, device="cuda").scatter_reduce(0, inv, torch.arange(k, device="cuda"),
                                                                                             reduce="amax")
    leaves[uniq] = new[last]
    rl, rn = CudaPedersenBackend(prm, prm, 0).build_local(leaves)
    torch.cuda.synchronize()
    assert int(applied.item()) == 1
    assert torch.equal(ln, rl) and torch.equal(nn, rn)


class _LevelLoopConfig(PedersenByteConfig):
    """The same Config under another type: MerkleTree takes the generic level loop for it."""


def test_python_mirror_equals_level_loop():
    _, prm = setup(8)
    n, L = 512, 32
    leaves = np.ascontiguousarray(cref.synth_bytes(31, n * L).reshape(n, L))
    fast = MerkleTree.new(prm, prm, leaves, config=PedersenByteConfig())
    slow = MerkleTree.new(prm, prm, leaves, config=_LevelLoopConfig())
    assert fast._updates_on_device() and not slow._updates_on_device()
    idx = [0, 1, 77, 300, 511]
    new = np.ascontiguousarray(cref.synth_bytes(32, len(idx) * L).reshape(len(idx), L))
    fast.update_batch(idx, new)
    slow.update_batch(idx, new)
    assert np.array_equal(fast.leaf_nodes, slow.leaf_nodes) and np.array_equal(fast.non_leaf_nodes, slow.non_leaf_nodes)
    fast.update(5, new[0])
    slow.update(5, new[0])
    assert np.array_equal(fast.non_leaf_nodes, slow.non_leaf_nodes)
    probe = MerkleTree.new(prm, prm, leaves, config=_LevelLoopConfig())
    probe.leaf_nodes, probe.non_leaf_nodes = slow.leaf_nodes.copy(), slow.non_leaf_nodes.copy()
    probe.update_batch([9, 10], new[1:3])
    good = probe.root()
    assert fast.check_update_batch([9, 10], new[1:3], good) is True
    assert slow.check_update_batch([9, 10], new[1:3], good) is True
    assert np.array_equal(fast.non_leaf_nodes, slow.non_leaf_nodes) and np.array_equal(fast.leaf_nodes, slow.leaf_nodes)
    bad = good.copy()
    bad[0, 0] ^= np.uint64(1)
    assert fast.check_update(3, new[4], bad) is False and slow.check_update(3, new[4], bad) is False
    assert np.array_equal(fast.non_leaf_nodes, slow.non_leaf_nodes)


def test_cpp_update_mirror(tmp_path):
    _, prm = setup(8)
    gens = tmp_path / "gens.bin"
    gens.write_bytes(np.ascontiguousarray(prm.generators, dtype=np.uint64).tobytes())
    out_dir = os.path.join(ROOT, "tests", "host", "_build")
    os.makedirs(out_dir, exist_ok=True)
    exe = os.path.join(out_dir, "test_update_pedersen")
    lib_dir = os.path.join(ROOT, "crypto_primitives_b200")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "test_update_pedersen.cpp"), "-L", lib_dir, "-l:libcpb200.so",
                           f"-Wl,-rpath,{lib_dir}", "-o", exe])
    r = subprocess.run([exe, str(gens)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "cpp pedersen update ok" in r.stdout
