"""Pedersen-node Merkle update without a GPU: the CPB_HD pieces of csrc/cpb_merkle_update_pedersen.cu run on the CPU through a host
shim -- the TwoToOneCRH row of a node against the Python oracle's serialisation, and which scratch slot or tree node each child of a
candidate slot is read from against a model of the tree, the narrow-level warp kernel's lane split and shuffle reduction against the
oracle's TwoToOneCRH -- and the argument rules of the four cpb_merkle_pedersen_update* entry
points of include/cpb200.h."""
import ctypes as C

import numpy as np
import pytest

from helpers import build_host_shim
from crypto_primitives_b200 import _native as N
from oracle import cref, fields as OF, jubjub as jj, pedersen as OPD

u64p = C.POINTER(C.c_uint64)
u32p = C.POINTER(C.c_uint32)


@pytest.fixture(scope="module")
def shim():
    lib = build_host_shim("merkle_update_pedersen_shim")
    lib.host_ped_node_row.argtypes = [C.c_int, u32p, u32p, u32p]
    lib.host_ped_child_src.restype = C.c_int
    lib.host_ped_child_src.argtypes = [u64p, C.c_uint64, C.c_uint64, C.c_int, C.c_int, C.c_uint64, u64p]
    lib.host_ped_warp_hash.argtypes = [u32p, C.c_int, u32p, C.POINTER(C.c_uint8), C.c_long, C.c_int, C.c_int, u32p, u32p]
    return lib


def _p(a):
    return a.ctypes.data_as(u64p)


def _p32(a):
    return a.ctypes.data_as(u32p)


def _mont_point(P, p):
    return cref.ints_to_mont([P[0], P[1]], p).reshape(2, 4)


def test_node_row_is_the_oracle_serialisation(shim):
    """te_node_row: canonical x_l || y_l || x_r || y_r, the bytes TwoToOneCRH::compress hashes (R/crh/pedersen/mod.rs:187-197)."""
    rng = OF.SplitMix64(31)
    pts = [OPD.synthetic_base(rng) for _ in range(6)] + [(0, 1), (0, OF.BLS12_381_FR - 1)]
    w = OPD.Window(4, 256)
    prm = OPD.setup(w, 3)
    for a, b in zip(pts, pts[::-1]):
        row = np.zeros(32, dtype=np.uint32)
        la, rb = _mont_point(a, OF.BLS12_381_FR), _mont_point(b, OF.BLS12_381_FR)
        shim.host_ped_node_row(0, _p32(la.view(np.uint32)), _p32(rb.view(np.uint32)), _p32(row))
        assert row.tobytes() == jj.serialize_uncompressed(a) + jj.serialize_uncompressed(b)
    # the row, cut to the window's two-to-one length, is the oracle's TwoToOneCRH input: same hash
    a, b = pts[0], pts[1]
    shim.host_ped_node_row(0, _p32(_mont_point(a, OF.BLS12_381_FR).view(np.uint32)), _p32(_mont_point(b, OF.BLS12_381_FR).view(np.uint32)),
                           _p32(row))
    half = (w.window_size * w.num_windows) // 2
    assert OPD.crh_evaluate(prm, w, row.tobytes()[:min(128, (half + half) // 8)]) == OPD.two_to_one_compress(prm, w, a, b)


def test_node_row_ed_on_bls12_377(shim):
    p = OF.BLS12_377_FR
    vals = [1, 2, p - 1, 12345678901234567890, (1 << 250) + 7, 0, 3, p - 2]
    for four in (vals[:4], vals[4:]):                                     # one row: left (x, y), right (x, y)
        m = cref.ints_to_mont(four, p).reshape(2, 2, 4)
        row = np.zeros(32, dtype=np.uint32)
        shim.host_ped_node_row(1, _p32(np.ascontiguousarray(m[0]).view(np.uint32)), _p32(np.ascontiguousarray(m[1]).view(np.uint32)),
                               _p32(row))
        assert row.tobytes() == b"".join(v.to_bytes(32, "little") for v in four)


def _jubjub_d2():
    p = OF.BLS12_381_FR
    d = (-10240 * pow(10241, p - 2, p)) % p
    return cref.ints_to_mont([2 * d % p], p).reshape(4).view(np.uint32)


@pytest.mark.parametrize("cb", [8, 12, 18, 21])
@pytest.mark.parametrize("ws,nw", [(4, 256), (4, 200), (5, 33)])
def test_warp_lane_split_and_reduction(shim, cb, ws, nw):
    """k_ped_upd_top's node hash on the CPU: lookup c at bits [c cb, (c + 1) cb) of the row (zero beyond the two-to-one length,
    across byte boundaries), lane c % 32, then the five-round shuffle reduction -- equal to the oracle's TwoToOneCRH."""
    w = OPD.Window(ws, nw)
    prm = OPD.setup(w, 7)
    p = OF.BLS12_381_FR
    gens = [pt for win in prm.generators for pt in win]
    half = (ws * nw) // 2
    length = min(128, (half + half) // 8)                                 # two_to_one_len
    settable = ((ws * nw) // 8) * 8
    n_chunks = (settable + cb - 1) // cb
    gxy = cref.ints_to_mont([c for pt in gens for c in pt], p).reshape(-1).view(np.uint32)
    rng = OF.SplitMix64(cb * 1000 + ws * nw)
    a, b = OPD.synthetic_base(rng), OPD.synthetic_base(rng)
    row = np.frombuffer(jj.serialize_uncompressed(a) + jj.serialize_uncompressed(b), dtype=np.uint8).copy()
    values = np.zeros(n_chunks, dtype=np.uint32)
    out = np.zeros(16, dtype=np.uint32)
    shim.host_ped_warp_hash(_p32(gxy), len(gens), _p32(_jubjub_d2()), row.ctypes.data_as(C.POINTER(C.c_uint8)), length, cb, n_chunks,
                            _p32(values), _p32(out))
    msg = int.from_bytes(row.tobytes()[:length], "little")
    assert [int(v) for v in values] == [(msg >> (c * cb)) & ((1 << cb) - 1) for c in range(n_chunks)]
    got = cref.mont_to_ints(out.view(np.uint64).reshape(2, 4), p)
    assert tuple(got) == tuple(OPD.two_to_one_compress(prm, w, a, b))


def model_child_src(U, k, h, l, node, b):
    """Where child b of touched node `node` (level l) is read: the scratch slot when the child is touched, else the tree."""
    c = 2 * node + b
    s = h - l - 1
    under = [i for i, u in enumerate(U) if u >> s == c]
    widths = [min(k, 1 << j) for j in range(h + 1)]
    off = [sum(widths[:j]) for j in range(h + 2)]
    if under:
        slot = c if (1 << (l + 1)) <= k else under[0]
        return 0, off[l + 1] + slot
    if l + 1 == h:
        return 1, c
    return 2, (1 << (l + 1)) - 1 + c


@pytest.mark.parametrize("n", [2, 4, 64, 1024])
def test_candidate_children(shim, n):
    h = n.bit_length() - 1
    rng = np.random.default_rng(n)
    cases = [[0], [n - 1], [0, 1], list(range(n)), sorted(set(int(x) for x in rng.integers(0, n, size=17))),
             sorted(set(int(x) for x in rng.integers(0, max(n // 8, 1), size=9)))]
    for U in cases:
        for k in sorted({len(U), len(U) + 3, 2 * len(U) + 1}):            # k counts the pairs given (repeats included)
            u = np.array(U, dtype=np.uint64)
            for l in range(h):
                width = min(k, 1 << l)
                touched = sorted({x >> (h - l) for x in U})
                seen = set()
                for cand in range(width):
                    src = np.zeros(4, dtype=np.uint64)
                    t = shim.host_ped_child_src(_p(u), u.size, k, h, l, cand, _p(src))
                    if not t:
                        continue
                    node = cand if (1 << l) <= k else U[cand] >> (h - l)
                    seen.add(node)
                    for b in (0, 1):
                        assert tuple(int(x) for x in src[2 * b:2 * b + 2]) == model_child_src(U, k, h, l, node, b), (U, k, l, cand, b)
                assert sorted(seen) == touched, (U, k, l)                  # every touched node has exactly one candidate


# ---------------------------------------------------------------------------------------------------- ABI argument rules
def _pts(n):
    return np.zeros((max(n, 1), 2, 4), dtype=np.uint64)


def test_update_entry_points_validate_before_touching_a_device():
    ln, nn, idx, dg = _pts(8), _pts(7), np.array([1, 2], dtype=np.uint64), _pts(2)
    leaves = np.zeros((2, 32), dtype=np.uint8)
    lb = leaves.ctypes.data_as(N.u8p)
    ok = C.c_int(7)
    H, HL = N.lib.cpb_merkle_pedersen_update_digests, N.lib.cpb_merkle_pedersen_update
    D, DL = N.lib.cpb_merkle_pedersen_update_digests_dev, N.lib.cpb_merkle_pedersen_update_dev
    # null contexts, otherwise valid
    assert H(None, _p(ln), _p(nn), 8, _p(idx), _p(dg), 2, None, C.byref(ok)) == N.CPB_NULL_POINTER
    assert HL(None, None, _p(ln), _p(nn), 8, _p(idx), lb, 32, 2, None, C.byref(ok)) == N.CPB_NULL_POINTER
    assert D(None, ln.ctypes.data, nn.ctypes.data, 8, idx.ctypes.data, dg.ctypes.data, 2, None, None, None) == N.CPB_NULL_POINTER
    assert DL(None, None, ln.ctypes.data, nn.ctypes.data, 8, idx.ctypes.data, leaves.ctypes.data, 32, 32, 2, None, None,
              None) == N.CPB_NULL_POINTER
    # n not a power of two > 1
    for n in (0, 1, 3, 6):
        assert H(None, _p(ln), _p(nn), n, _p(idx), _p(dg), 2, None, None) == N.CPB_NOT_POW2
        assert D(None, ln.ctypes.data, nn.ctypes.data, n, idx.ctypes.data, dg.ctypes.data, 2, None, None, None) == N.CPB_NOT_POW2
    # k >= 2^32, checked before any array is read
    assert H(None, _p(ln), _p(nn), 8, _p(idx), _p(dg), 1 << 32, None, None) == N.CPB_BAD_LENGTH
    assert D(None, ln.ctypes.data, nn.ctypes.data, 8, idx.ctypes.data, dg.ctypes.data, 1 << 32, None, None, None) == N.CPB_BAD_LENGTH
    assert DL(None, None, ln.ctypes.data, nn.ctypes.data, 8, idx.ctypes.data, leaves.ctypes.data, 32, 32, 1 << 32, None, None,
              None) == N.CPB_NULL_POINTER                                 # a null leaf context is reported first
    # host forms: an index >= n is rejected before any copy
    bad = np.array([1, 8], dtype=np.uint64)
    assert H(None, _p(ln), _p(nn), 8, _p(bad), _p(dg), 2, None, C.byref(ok)) == N.CPB_BAD_PARAMS
    # null arrays
    assert H(None, None, _p(nn), 8, _p(idx), _p(dg), 2, None, None) == N.CPB_NULL_POINTER
    assert H(None, _p(ln), _p(nn), 8, None, _p(dg), 2, None, None) == N.CPB_NULL_POINTER
    assert H(None, _p(ln), _p(nn), 8, _p(idx), None, 2, None, None) == N.CPB_NULL_POINTER
    assert D(None, ln.ctypes.data, None, 8, idx.ctypes.data, dg.ctypes.data, 2, None, None, None) == N.CPB_NULL_POINTER
    assert N.lib.cpb_abi_version() == 5


# A leaf longer than the window (leaf_len * 8 > WINDOW_SIZE * NUM_WINDOWS -> CPB_BAD_LENGTH) is checked against the leaf context,
# which cannot be created without a device; tests/test_gpu_merkle_update_pedersen.py covers it through the C-ABI.


@pytest.mark.skipif(N.lib.cpb_device_count() > 0, reason="an H100 is present")
def test_update_has_no_cpu_fallback():
    import crypto_primitives_b200 as cp
    from crypto_primitives_b200.crh.pedersen import Parameters, Window
    from crypto_primitives_b200.merkle_tree import MerkleTree, PedersenByteConfig
    w = OPD.Window(4, 8)
    oprm = OPD.setup(w, 3)
    g = cp.BLS12_381_FR.elements([c for ws in oprm.generators for pt in ws for c in pt]).reshape(8, 4, 2, 4)
    prm = Parameters(cp.curves.JUBJUB, Window(4, 8), g)
    tree = MerkleTree(PedersenByteConfig(), np.zeros((4, 2, 4), dtype=np.uint64), np.zeros((3, 2, 4), dtype=np.uint64), prm, prm, 0)
    with pytest.raises(N.CpbError) as e:
        tree.update_batch([1], np.zeros((1, 4), dtype=np.uint8))
    assert e.value.status in (N.CPB_NO_DEVICE, N.CPB_CUDA_ERROR)
