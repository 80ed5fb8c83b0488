"""Ragged Poseidon batches without a GPU: why the kernels must not pad (oracle), the ordering helpers of the device code
(csrc/poseidon.cuh: ragged_span / ragged_key / ragged_scan / ragged_ranges) through a host shim, the per-item device code run on
the CPU against the oracle at every width, the Python packing helpers, and the null-context rule of every new C-ABI symbol."""
import ctypes as C
import random

import numpy as np
import pytest

from helpers import build_host_shim, oracle_config
from oracle import cref, fields as OF, poseidon as OP
from test_poseidon_lane1_basis import random_config
from test_poseidon_scaled_lane0 import FID, _arrays, _P

u32p = C.POINTER(C.c_uint32)
FIELD_CONFIGS = ["bls_default_r2", "bn254_r2", "jubjub_merkle_fixture", "bls377_random"]     # one per field


@pytest.fixture(scope="module")
def shim():
    lib = build_host_shim("ragged_shim", defines=["CPB_POS_SPLIT=1"])
    lib.host_ragged_span.restype = C.c_long
    lib.host_ragged_span.argtypes = [C.c_void_p, C.c_long, C.c_long, C.POINTER(C.c_uint64)]
    lib.host_ragged_key.argtypes = [C.c_long, C.c_int]
    lib.host_ragged_order.argtypes = [C.c_void_p, C.c_long, C.c_int, C.c_int, u32p, u32p, u32p]
    return lib


# ---------------------------------------------------------------------------------------------------- the oracle: no padding
@pytest.mark.parametrize("which", FIELD_CONFIGS)
def test_zero_padding_is_exact_only_inside_the_last_block(which):
    """Absorbing zeros that stay inside the last rate block leaves the CRH unchanged; one more zero starts a new block, costs a
    permutation and changes it.  So a ragged batch cannot be padded to its longest input: every input is hashed at its length."""
    _, cfg = oracle_config(which)
    r, p = cfg.rate, cfg.p
    rnd = random.Random(FID[oracle_config(which)[0]])
    for L in range(0, 2 * r + 1):
        x = [rnd.randrange(p) for _ in range(L)]
        h = OP.crh_evaluate(cfg, x)
        blocks = max(1, -(-L // r))
        assert OP.crh_evaluate(cfg, x + [0] * (blocks * r - L)) == h, L
        assert OP.crh_evaluate(cfg, x + [0] * (blocks * r - L + 1)) != h, L


# ---------------------------------------------------------------------------------------------------- ordering helpers
def _order(shim, offsets, rate, single=True):
    off = np.ascontiguousarray(offsets, dtype=np.uint64)
    n = off.shape[0] - 1
    nb = shim.host_ragged_buckets()
    order = np.zeros(max(n, 1), dtype=np.uint32)
    starts = np.zeros(nb + 1, dtype=np.uint32)
    rng = np.zeros(4, dtype=np.uint32)
    shim.host_ragged_order(off.ctypes.data, n, rate, int(single), order.ctypes.data_as(u32p), starts.ctypes.data_as(u32p),
                           rng.ctypes.data_as(u32p))
    return order[:n], starts, rng


def _span(shim, off, i):
    lo = C.c_uint64()
    ln = shim.host_ragged_span(np.ascontiguousarray(off, dtype=np.uint64).ctypes.data, i, len(off) - 1, C.byref(lo))
    return lo.value, ln


def _expected_len(off, i):
    a, b = int(off[0]), int(off[-1])
    lo, hi = max(int(off[i]), a), min(int(off[i + 1]), b)
    return max(hi - lo, 0)


ORDER_CASES = {
    "n0": [7],
    "n1": [3, 8],
    "all_equal": [5 + 2 * i for i in range(40)],
    "all_distinct": list(np.cumsum([11] + list(range(0, 30)))),
    "above_cap": list(np.cumsum([0, 1, 200, 130, 127, 128, 129, 2, 500, 126])),
    "decreasing_pair": [10, 12, 9, 15, 15, 20],
}


@pytest.mark.parametrize("case", list(ORDER_CASES))
@pytest.mark.parametrize("rate", [1, 2, 4])
def test_order_is_a_permutation_sorted_by_bucket(shim, case, rate):
    off = np.array(ORDER_CASES[case], dtype=np.uint64)
    n = len(off) - 1
    nb = shim.host_ragged_buckets()
    order, starts, rng = _order(shim, off, rate)
    lens = [_expected_len(off, i) for i in range(n)]
    keys = [min(max(1, -(-L // rate)), nb) - 1 for L in lens]
    assert [shim.host_ragged_key(L, rate) for L in lens] == keys
    assert sorted(order.tolist()) == list(range(n))                          # a permutation
    sk = [keys[i] for i in order]
    assert sk == sorted(sk)                                                  # buckets come out sorted
    for b in range(nb + 1):
        assert starts[b] == sum(1 for k in keys if k < b), b                 # bucket b is order[starts[b] .. starts[b+1])
    assert rng.tolist() == [0, starts[1], starts[1], n]
    _, _, rng0 = _order(shim, off, rate, single=False)
    assert rng0.tolist() == [0, 0, 0, n]
    if case == "above_cap" and rate == 1:
        assert keys.count(nb - 1) == 7                                       # 64 blocks or more share the last bucket


def test_span_reads_nothing_outside_the_window(shim):
    """A decreasing pair is an empty input; offsets outside [offsets[0], offsets[n]) are clamped to it."""
    off = [10, 12, 9, 15, 30, 4, 20]
    n = len(off) - 1
    assert _span(shim, off, 0) == (10, 2)
    assert _span(shim, off, 1)[1] == 0 and _span(shim, off, 1)[0] == 10      # 12 -> 9
    assert _span(shim, off, 2) == (10, 5)                                    # 9 < offsets[0]: starts at 10
    assert _span(shim, off, 3) == (15, 5)                                    # 30 > offsets[n] = 20: ends at 20
    assert _span(shim, off, 4)[1] == 0                                       # 30 -> 4
    assert _span(shim, off, 5) == (10, 10)
    for i in range(n):
        lo, ln = _span(shim, off, i)
        assert 10 <= lo and lo + ln <= 20


# ---------------------------------------------------------------------------------------------------- per-item device code, every width
def _ragged_case(p, rate, seed, front=5):
    """Lengths 0 .. 3*rate+1, shuffled, behind `front` junk elements (offsets[0] = front)."""
    rnd = random.Random(seed)
    lens = list(range(3 * rate + 2)) * 2
    rnd.shuffle(lens)
    ints = [[rnd.randrange(p) for _ in range(L)] for L in lens]
    ints[0] = [p - 1] * len(ints[0])
    flat = [rnd.randrange(p) for _ in range(front)] + [x for row in ints for x in row]
    offsets = np.array(np.cumsum([front] + lens), dtype=np.uint64)
    return ints, cref.ints_to_mont(flat, p).reshape(-1, 4), offsets


def _run(shim, fname, cfg, values, vbase, offsets, n_out):
    arkm, mdsm = _arrays(cfg)
    n = len(offsets) - 1
    out = np.zeros((n, n_out, 4), dtype=np.uint64)
    rc = shim.host_ragged_sponge_any_width(FID[fname], cfg.rate, cfg.capacity, cfg.full_rounds, cfg.partial_rounds,
                                           C.c_ulonglong(cfg.alpha), _P(arkm), _P(mdsm), _P(np.ascontiguousarray(values)),
                                           C.c_uint64(vbase), _P(offsets), C.c_long(n), C.c_long(n_out), _P(out))
    assert rc == 0
    return out


def _oracle_sponge(cfg, x, n_out):
    s = OP.PoseidonSponge(cfg)
    s.absorb(x)
    return s.squeeze_native_field_elements(n_out)


@pytest.mark.parametrize("t", range(2, 10))
def test_ragged_device_code_every_width(shim, t):
    for fname, alpha in (("bls12_381_fr", 5), ("bn254_fr", 5), ("jubjub_fr", 5), ("bls12_377_fr", 11)):
        p = OF.MODULI[fname]
        cfg = random_config(p, t, 8, 21, alpha, 100 * t + FID[fname])
        ints, values, offsets = _ragged_case(p, cfg.rate, t + 10 * FID[fname])
        want = [OP.crh_evaluate(cfg, x) for x in ints]
        got = _run(shim, fname, cfg, values, 0, offsets, 1)
        assert cref.mont_to_ints(got.reshape(-1, 4), p) == want, fname
        got = _run(shim, fname, cfg, values[5:], 5, offsets, 1)              # values start at offsets[0]
        assert cref.mont_to_ints(got.reshape(-1, 4), p) == want, fname


@pytest.mark.parametrize("which", ["bn254_r2", "bls_sponge_fixture"])
def test_ragged_device_code_squeezes(shim, which):
    fname, cfg = oracle_config(which)
    p, r = cfg.p, cfg.rate
    ints, values, offsets = _ragged_case(p, r, 3)
    for n_out in (1, r, r + 1, 3 * r):
        got = _run(shim, fname, cfg, values, 0, offsets, n_out)
        for i, x in enumerate(ints):
            assert cref.mont_to_ints(got[i], p) == _oracle_sponge(cfg, x, n_out), (n_out, i)


# ---------------------------------------------------------------------------------------------------- Python packing
def test_pack_and_is_ragged():
    from crypto_primitives_b200 import ragged as R
    a, b = np.arange(8, dtype=np.uint64).reshape(2, 4), np.arange(12, dtype=np.uint64).reshape(3, 4)
    assert R.is_ragged([a, b]) and R.is_ragged((b, a, np.zeros((0, 4), dtype=np.uint64)))
    assert not R.is_ragged([a, a]) and not R.is_ragged(np.stack([a, a])) and not R.is_ragged([a])
    vals, off = R.pack([a, np.zeros((0, 4), dtype=np.uint64), b])
    assert off.tolist() == [0, 2, 2, 5] and off.dtype == np.uint64
    assert np.array_equal(vals, np.concatenate([a, b]))
    with pytest.raises(ValueError):
        R.as_arrays(vals, [0, 2, 6])                                         # reaches past the values


# ---------------------------------------------------------------------------------------------------- C-ABI: null contexts
def test_every_ragged_symbol_rejects_a_null_context():
    from crypto_primitives_b200 import _native as N
    L = N.lib
    off = np.zeros(3, dtype=np.uint64)
    vals = np.zeros((1, 4), dtype=np.uint64)
    out = np.zeros((4, 4), dtype=np.uint64)
    ok = np.zeros(2, dtype=np.uint8)
    u8 = ok.ctypes.data_as(N.u8p)
    assert L.cpb_poseidon_crh_ragged_batch(None, _P(vals), _P(off), _P(out), 2) == N.CPB_NULL_POINTER
    assert L.cpb_poseidon_crh_ragged_batch_dev(None, None, None, None, 2, None) == N.CPB_NULL_POINTER
    assert L.cpb_poseidon_sponge_ragged_batch(None, _P(vals), _P(off), _P(out), 1, 2) == N.CPB_NULL_POINTER
    assert L.cpb_poseidon_sponge_ragged_batch_dev(None, None, None, None, 1, 2, None) == N.CPB_NULL_POINTER
    assert L.cpb_merkle_poseidon_build_ragged(None, None, _P(vals), _P(off), 2, _P(out), _P(out)) == N.CPB_NULL_POINTER
    assert L.cpb_merkle_poseidon_build_ragged_dev(None, None, None, None, 2, None, None, None) == N.CPB_NULL_POINTER
    assert L.cpb_merkle_poseidon_verify_ragged_batch(None, None, _P(vals), _P(vals), _P(off), _P(vals), None, 0, _P(off), u8, 2) == N.CPB_NULL_POINTER
    assert L.cpb_merkle_poseidon_verify_ragged_batch_dev(None, None, None, None, None, None, None, 0, None, None, 2, None) == N.CPB_NULL_POINTER
