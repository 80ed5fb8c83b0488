"""CPU checks of signatures and encryption over ed-on-BLS12-377: the device arithmetic of its scalar field
(Ed_On_Bls12_377_Fr in csrc/fp.cuh) at crafted full-width operands, the curve operations of csrc/te_ops.cuh over BLS12-377 Fr
(both through the host shim tests/host/signature_ed377_shim.cpp) against the oracle tests/signature_ed377_oracle.py, the oracle
on the reference's scenarios, and the C-ABI's argument rules for the new field and curve without a device."""
import ctypes as C
import functools
import random

import numpy as np
import pytest

from helpers import build_host_shim
from crypto_primitives_b200 import _native as N
import crypto_primitives_b200 as cp
from oracle import jubjub as J
from oracle import wire
import signature_ed377_oracle as E
from test_fp_host import _crafted_factor_pairs, _crafted_square_roots, _pattern_value

Q, R = E.Q, E.R
RINV = pow(1 << 256, -1, R)
u8p, u64p, u32p = C.POINTER(C.c_uint8), C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)


@pytest.fixture(scope="module")
def shim():
    lib = build_host_shim("signature_ed377_shim")
    lib.host_fr_op.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_long]
    lib.host_fr_consts.argtypes = [u32p, u32p, u32p, u32p, C.POINTER(C.c_int)]
    lib.host_compress.argtypes = [u64p, u8p]
    lib.host_from_random_bytes.argtypes = [u8p, u64p]
    lib.host_from_random_bytes.restype = C.c_int
    lib.host_dbl.argtypes = [u64p, u64p]
    lib.host_add.argtypes = [u64p, u64p, u64p]
    lib.host_neg.argtypes = [u64p, u64p]
    lib.host_mul_words.argtypes = [u64p, u64p, C.c_int, u64p]
    lib.host_mul_bitrev_bytes.argtypes = [u64p, u8p, C.c_uint64, u64p]
    return lib


def _w32(x):
    return [(x >> (32 * i)) & 0xFFFFFFFF for i in range(8)]


def _val(a):
    return sum(int(v) << (32 * i) for i, v in enumerate(a))


def _limbs(v: int):
    return np.array([(v >> (64 * i)) & (2**64 - 1) for i in range(4)], dtype=np.uint64)


def _pt(P):
    return np.concatenate([_limbs((P[0] << 256) % Q), _limbs((P[1] << 256) % Q)])


def _unpt(a):
    rinv = pow(1 << 256, -1, Q)
    v = [sum(int(a[4 * k + i]) << (64 * i) for i in range(4)) * rinv % Q for k in range(2)]
    return (v[0], v[1])


def _p64(a):
    return a.ctypes.data_as(u64p)


def _buf(data: bytes):
    a = np.frombuffer(bytes(data) + b"\0", dtype=np.uint8).copy()
    return a, a.ctypes.data_as(u8p)


def random_point(rng):
    while True:
        P = E.point_from_y(rng.randrange(Q))
        if P is not None:
            return P


@functools.lru_cache(None)
def torsion4():
    """The 4 points of order dividing 4: the identity, (0, -1) and (+-sqrt(-1), 0) -- the cofactor part of the group."""
    i = E.sqrt(Q - 1)
    pts = [E.IDENTITY, (0, Q - 1), (i, 0), (Q - i, 0)]
    assert all(E.is_on_curve(P) and E.mul(4, P) == E.IDENTITY for P in pts)
    assert E.double((i, 0)) == (0, Q - 1)
    return pts


# ---- the scalar-field tag ---------------------------------------------------------------------------------------------------
def test_scalar_field_constants_recomputed(shim):
    p, one, r2, ninv, bits = (C.c_uint32 * 8)(), (C.c_uint32 * 8)(), (C.c_uint32 * 8)(), C.c_uint32(), C.c_int()
    shim.host_fr_consts(p, one, r2, C.byref(ninv), C.byref(bits))
    assert _val(p) == R == cp.curves.ED_ON_BLS12_377.scalar_modulus
    assert _val(one) == (1 << 256) % R
    assert _val(r2) == (1 << 512) % R
    assert ninv.value == (-pow(R, -1, 1 << 32)) % (1 << 32)
    assert bits.value == R.bit_length() == 251
    assert R & 0xFFFFFFFF != 1 and (R >> 32) & 0xFFFFFFFF != 0xFFFFFFFF        # P0_ONE, P1_ALLONES false: the generic rows
    assert all(R & 0xFFFFFFFF != (1 << 32) - (1 << k) + 1 for k in range(1, 32))  # P0_POW = 0


def _run(shim, which, A, B):
    a = np.array([_w32(x) for x in A], dtype=np.uint32)
    b = np.array([_w32(x) for x in B], dtype=np.uint32)
    r = np.zeros_like(a)
    shim.host_fr_op(which, a.ctypes.data, b.ctypes.data, r.ctypes.data, len(A))
    return [_val(x) for x in r]


def test_scalar_field_ops_random_and_edge(shim):
    rnd = random.Random(377)
    edge = [0, 1, 2, R - 1, R - 2, (1 << 255) % R, (1 << 256) % R, R >> 1, (0xDEADBEEF << 32) % R, (7 << 224) % R,
            (R - 1) & ~0xFFFFFFFF, 1 << 250, (1 << 251) - 1 - R]
    A = [x for x in edge for _ in edge] + [rnd.randrange(R) for _ in range(600)]
    B = [y for _ in edge for y in edge] + [rnd.randrange(R) for _ in range(600)]
    assert _run(shim, 0, A, B) == [x * y * RINV % R for x, y in zip(A, B)]
    assert _run(shim, 1, A, B) == [(x + y) % R for x, y in zip(A, B)]
    assert _run(shim, 2, A, B) == [(x - y) % R for x, y in zip(A, B)]
    assert _run(shim, 3, A, A) == [x * x * RINV % R for x in A]
    assert _run(shim, 5, A, A) == [x * RINV % R for x in A]
    r2 = pow(1 << 256, 2, R)
    assert _run(shim, 4, A[:60], A[:60]) == [pow(x, -1, R) * r2 % R if x else 0 for x in A[:60]]


def test_scalar_field_adversarial_carry_patterns(shim):
    """Squares and products whose 512-bit results have all-ones / zero limb runs, limb-pattern operands and near-modulus
    operands (DESIGN §2.1: random operands reach a carry out of an all-ones limb with probability about 2^-32)."""
    rnd = random.Random(1377)
    A = _crafted_square_roots(rnd, R, 6000)
    assert _run(shim, 3, A, A) == [x * x * RINV % R for x in A]
    assert _run(shim, 0, A, A) == [x * x * RINV % R for x in A]
    pairs = _crafted_factor_pairs(rnd, R, 6000)
    A, B = [x for x, _ in pairs], [y for _, y in pairs]
    assert _run(shim, 0, A, B) == [x * y * RINV % R for x, y in pairs]
    assert _run(shim, 0, B, A) == [x * y * RINV % R for x, y in pairs]
    P = []
    while len(P) < 8000:
        v = _pattern_value(rnd, 8, 0.85)
        if rnd.random() < 0.5:
            v = (v & ((1 << 224) - 1)) | (rnd.choice((R >> 224, (R >> 224) - 1, 0, 1)) << 224)
        if v < R:
            P.append(v)
    A, B = P[:4000], P[4000:]
    assert _run(shim, 0, A, B) == [x * y * RINV % R for x, y in zip(A, B)]
    assert _run(shim, 3, P, P) == [x * x * RINV % R for x in P]
    assert _run(shim, 1, A, B) == [(x + y) % R for x, y in zip(A, B)]
    assert _run(shim, 2, A, B) == [(x - y) % R for x, y in zip(A, B)]
    near = [R - 1 - rnd.getrandbits(rnd.choice((1, 8, 32, 64))) for _ in range(2000)]
    assert _run(shim, 0, near, near[::-1]) == [x * y * RINV % R for x, y in zip(near, near[::-1])]
    assert _run(shim, 3, near, near) == [x * x * RINV % R for x in near]


# ---- the curve: complete law, compression, from_random_bytes ---------------------------------------------------------------
def test_the_law_is_complete():
    """a = -1 is a square and d = 3021 a non-square in Fq: the affine law has no exceptional points, and te_dbl's
    denominators d x^2 y^2 +- 1 never vanish."""
    assert pow(Q - 1, (Q - 1) // 2, Q) == 1
    assert pow(E.D, (Q - 1) // 2, Q) == Q - 1
    assert cp.curves.ED_ON_BLS12_377.d == E.D and cp.curves.ED_ON_BLS12_377.q == Q
    rng = random.Random(3)
    G = E.mul(E.COFACTOR, random_point(rng))
    assert E.mul(R, G) == E.IDENTITY and G != E.IDENTITY


def test_compression(shim):
    rng = random.Random(4)
    pts = torsion4() + [random_point(rng) for _ in range(40)]
    pts += [E.neg(P) for P in pts]
    for P in pts:
        o = np.zeros(32, dtype=np.uint8)
        shim.host_compress(_p64(_pt(P)), o.ctypes.data_as(u8p))
        assert o.tobytes() == E.compress(P) == wire.te_point(P, Q, compress=True), P


def test_from_random_bytes_at_251_bits(shim):
    rng = random.Random(5)
    cases = [R - 1, R, R + 1, 0, 1, (1 << 251) - 1, (1 << 256) - 1, R | (1 << 251), (R - 1) | (0x1F << 251), (R - 1) | (1 << 255),
             R | (0x1F << 251), 1 << 251, 1 << 250, (1 << 250) | 1]
    cases += [rng.getrandbits(256) for _ in range(400)]
    valid = 0
    for v in cases:
        d = v.to_bytes(32, "little")
        b, bp = _buf(d)
        mont = np.zeros(4, dtype=np.uint64)
        ok = shim.host_from_random_bytes(bp, _p64(mont))
        exp = E.from_random_bytes(d)
        assert bool(ok) == (exp is not None), hex(v)
        if ok:
            valid += 1
            assert sum(int(mont[i]) << (64 * i) for i in range(4)) == (exp << 256) % R
    # bits 251..255 are cleared, not reduced: they never decide validity
    assert E.from_random_bytes(((R - 1) | (0x1F << 251)).to_bytes(32, "little")) == R - 1
    assert E.from_random_bytes((R | (0x1F << 251)).to_bytes(32, "little")) is None
    assert E.from_random_bytes(((1 << 256) - 1).to_bytes(32, "little")) is None
    assert 0.45 < valid / len(cases) < 0.7                                        # r / 2^251 = 0.583


# ---- group operations -----------------------------------------------------------------------------------------------------
def _bases():
    rng = random.Random(6)
    return [random_point(rng) for _ in range(6)] + [E.mul(4, random_point(rng))] + torsion4()


def test_doubling_and_addition_agree_with_the_complete_law(shim):
    bases = _bases()
    o = np.zeros(8, dtype=np.uint64)
    for P in bases:
        shim.host_dbl(_p64(_pt(P)), _p64(o))
        assert _unpt(o) == E.double(P), P
        shim.host_neg(_p64(_pt(P)), _p64(o))
        assert _unpt(o) == E.neg(P)
        for P2 in bases:
            shim.host_add(_p64(_pt(P)), _p64(_pt(P2)), _p64(o))
            assert _unpt(o) == E.add(P, P2), (P, P2)


SCALARS = [0, 1, 2, 3, 7, 8, 9, 15, 16, 17, R - 1, R - 2, R, R + 1, (1 << 251) - 1, (1 << 252) - 1, int("88" * 32, 16) >> 4,
           int("88" * 32, 16) >> 8, int("8" * 63, 16), int("01" * 32, 16) >> 8, 1 << 250, (1 << 128) + 1, 0x7777777777777777,
           int("87" * 32, 16) >> 8]


def test_variable_base_multiplication(shim):
    """te_mul_var at 63 nibbles (the kernels' count for scalars below 2^251): 0, 1, r - 1, all-8 nibbles (every Booth digit
    at -8 with carries), alternating extremes and random scalars, on full-order, prime-order and 4-torsion bases."""
    rng = random.Random(7)
    scalars = SCALARS + [rng.randrange(R) for _ in range(8)] + [rng.getrandbits(252) for _ in range(4)]
    for P in _bases():
        base = _pt(P)
        for k in scalars:
            assert k < 1 << 252
            o = np.zeros(8, dtype=np.uint64)
            shim.host_mul_words(_p64(base), _p64(_limbs(k)), 63, _p64(o))
            assert _unpt(o) == E.mul(k, P), (P, hex(k))
        for k in ((1 << 256) - 1, int("88" * 32, 16)):                           # 64 nibbles
            o = np.zeros(8, dtype=np.uint64)
            shim.host_mul_words(_p64(base), _p64(_limbs(k)), 64, _p64(o))
            assert _unpt(o) == E.mul(k, P), (P, hex(k))


def test_multiplication_by_randomness_bytes(shim):
    rng = random.Random(8)
    G = random_point(rng)
    for P in [G] + torsion4()[1:]:
        for ln in (0, 1, 2, 31, 32, 33, 100):
            for data in (bytes(rng.randrange(256) for _ in range(ln)), b"\xff" * ln, b"\x01" * ln, b"\x80" * ln):
                b, bp = _buf(data)
                o = np.zeros(8, dtype=np.uint64)
                shim.host_mul_bitrev_bytes(_p64(_pt(P)), bp, ln, _p64(o))
                assert _unpt(o) == E.mul(E.randomizer_int(data), P), (ln, data[:4])
                assert _unpt(o) == E.randomize_public_key(P, E.IDENTITY, data)


def test_fast_oracle_products_match_the_affine_oracle():
    rng = random.Random(9)
    G = E.mul(E.COFACTOR, random_point(rng))
    fb = E.FixedBase(G)
    for k in SCALARS[:16] + [rng.randrange(R) for _ in range(5)]:
        assert fb.mul(k) == E.mul(k, G) == E.mul_ext(k, G)
    for P in torsion4():
        assert E.mul_ext(5, P) == E.mul(5, P)
    assert E.randomizer_int(b"\x01\x80") == 0x80 | (0x01 << 8)


# ---- the reference's scenarios on the oracle (R/signature/mod.rs:52-105, R/encryption/elgamal/mod.rs:102-128) ----------
def _setup(rng):
    return E.mul(E.COFACTOR, random_point(rng)), bytes(rng.randrange(256) for _ in range(32))


def _sign(G, salt, sk, msg, rng):
    while True:
        sig = E.sign(G, salt, sk, msg, rng.randrange(R))
        if sig is not None:
            return sig


def test_oracle_sign_and_verify():
    rng = random.Random(10)
    for msg in (b"Hi, I am a Schnorr signature!", b"\x00" * 4 + b"hello", bytes([100]) * 128):
        G, salt = _setup(rng)
        sk = rng.randrange(R)
        pk = E.keygen(G, sk)
        sig = _sign(G, salt, sk, msg, rng)
        assert E.verify(G, salt, pk, msg, sig)


def test_oracle_failed_verification():
    rng = random.Random(11)
    G, salt = _setup(rng)
    sk = rng.randrange(R)
    pk = E.keygen(G, sk)
    sig = _sign(G, salt, sk, b"Bad message", rng)
    assert not E.verify(G, salt, pk, b"Hi, I am a Schnorr signature!", sig)


def test_oracle_randomize_and_verify():
    rng = random.Random(12)
    G, salt = _setup(rng)
    msg = b"Hi, I am a Schnorr signature!"
    sk = rng.randrange(R)
    pk = E.keygen(G, sk)
    sig = _sign(G, salt, sk, msg, rng)
    assert E.verify(G, salt, pk, msg, sig)
    for randomness in (bytes(32), b"\x01" * 32, bytes(rng.randrange(256) for _ in range(32))):
        assert E.verify(G, salt, E.randomize_public_key(G, pk, randomness), msg, E.randomize_signature(sig, randomness))


def test_oracle_elgamal_round_trip():
    rng = random.Random(13)
    G = E.mul(E.COFACTOR, random_point(rng))
    sk = rng.randrange(R)
    pk = E.keygen(G, sk)
    for msg in (E.mul(E.COFACTOR, random_point(rng)), random_point(rng)):
        ct = E.elgamal_encrypt(G, pk, msg, rng.randrange(R))
        assert E.elgamal_decrypt(sk, ct) == msg


def test_oracle_rejection_rate():
    """About 1 - r / 2^251 = 41.7 % of nonces give no challenge (Jubjub: 1 - r / 2^252 = 9.4 %)."""
    assert abs((1 - R / 2**251) - 0.4166) < 1e-3
    rng = random.Random(14)
    rej = sum(E.from_random_bytes(E.blake2s256(rng.getrandbits(64).to_bytes(8, "little"))) is None for _ in range(20000))
    assert 0.39 < rej / 20000 < 0.44


# ---- ABI rules without a device ----------------------------------------------------------------------------------------------
def test_field_id_4_in_the_field_level_calls():
    out = (C.c_uint64 * 4)()
    assert N.lib.cpb_field_modulus(4, out) == N.CPB_OK
    assert sum(int(out[i]) << (64 * i) for i in range(4)) == R == cp.ED_ON_BLS12_377_FR.modulus
    assert cp.ED_ON_BLS12_377_FR.modulus_bit_size == 251
    assert N.lib.cpb_field_modulus(5, out) == N.CPB_BAD_PARAMS
    assert N.lib.cpb_field_serialized_size(4) == 32 and N.lib.cpb_field_serialized_size(5) == 0
    vals = [0, 1, R - 1, 12345, R >> 1]
    mont = cp.ED_ON_BLS12_377_FR.elements(vals)
    ser = np.zeros(32 * len(vals), dtype=np.uint8)
    assert N.lib.cpb_field_serialize(4, _p64(mont), len(vals), ser.ctypes.data_as(u8p)) == N.CPB_OK
    assert ser.tobytes() == b"".join(v.to_bytes(32, "little") for v in vals)
    back = np.zeros_like(mont)
    assert N.lib.cpb_field_deserialize(4, ser.ctypes.data_as(u8p), len(vals), _p64(back)) == N.CPB_OK
    assert np.array_equal(back, mont)
    bad = np.frombuffer(R.to_bytes(32, "little"), dtype=np.uint8).copy()        # r itself is not reduced
    assert N.lib.cpb_field_deserialize(4, bad.ctypes.data_as(u8p), 1, _p64(back)) == N.CPB_BAD_PARAMS
    # Montgomery conversion: id 4 is known (n == 0 needs no device); an unknown id stays CPB_BAD_PARAMS
    for f in (N.lib.cpb_field_to_montgomery, N.lib.cpb_field_from_montgomery):
        assert f(4, 0, None, None, 0) == N.CPB_OK
        assert f(5, 0, None, None, 0) == N.CPB_BAD_PARAMS
    for f in (N.lib.cpb_field_to_montgomery_dev, N.lib.cpb_field_from_montgomery_dev):
        assert f(4, 0, None, None, 0, None) == N.CPB_OK
        assert f(5, 0, None, None, 0, None) == N.CPB_BAD_PARAMS


def test_field_id_4_is_not_a_hash_field():
    """Every entry point that takes the field of a Poseidon config, context or digest answers for id 4 as for an unknown id."""
    for fid in (4, 5):
        ark = np.zeros(4 * 3 * 40, dtype=np.uint64)
        mds = np.zeros(4 * 9, dtype=np.uint64)
        assert N.lib.cpb_poseidon_find_ark_and_mds(fid, 251, 2, 8, 31, 0, _p64(ark), _p64(mds)) == N.CPB_BAD_PARAMS
        a, f, p, s = C.c_uint64(), C.c_int(), C.c_int(), C.c_int()
        assert N.lib.cpb_poseidon_default_entry(fid, 2, 0, C.byref(a), C.byref(f), C.byref(p), C.byref(s)) == N.CPB_BAD_PARAMS
        out = N.vp()
        assert N.lib.cpb_poseidon_ctx_create(fid, 2, 1, 8, 31, 17, _p64(ark), _p64(mds), 0, C.byref(out)) == N.CPB_BAD_PARAMS
        w = C.c_size_t()
        assert N.lib.cpb_poseidon_config_serialize(fid, 2, 1, 8, 31, 17, _p64(ark), _p64(mds), None, 0, C.byref(w)) == N.CPB_BAD_PARAMS
        buf = np.zeros(64, dtype=np.uint8)
        assert N.lib.cpb_poseidon_config_deserialize(fid, buf.ctypes.data_as(u8p), 64, None, None, None, None, None, None, 0, None,
                                                     0) == N.CPB_BAD_PARAMS
        d = np.zeros(8, dtype=np.uint64)
        assert N.lib.cpb_path_serialize(0, fid, 0, 0, _p64(d), _p64(d), 1, 0, None, 0, C.byref(w)) == N.CPB_BAD_PARAMS
        assert N.lib.cpb_path_serialize(0, 0, 0, fid, _p64(d), _p64(d), 1, 0, None, 0, C.byref(w)) == N.CPB_BAD_PARAMS
        plen, idx = C.c_size_t(), C.c_uint64()
        assert N.lib.cpb_path_deserialize(0, fid, 0, 0, 0, buf.ctypes.data_as(u8p), 64, _p64(d), _p64(d), 1, C.byref(plen),
                                          C.byref(idx)) == N.CPB_BAD_PARAMS
        z = np.zeros(1, dtype=np.uint64)
        assert N.lib.cpb_multipath_serialize(0, fid, 0, 0, 1, _p64(d), _p64(z), _p64(z), _p64(d), _p64(z), None, 0,
                                             C.byref(w)) == N.CPB_BAD_PARAMS
        n1, n2 = C.c_size_t(), C.c_size_t()
        assert N.lib.cpb_multipath_deserialize(0, 0, 0, fid, 0, buf.ctypes.data_as(u8p), 64, C.byref(n1), C.byref(n2), None, None, None,
                                               None, None, 0, 0) == N.CPB_BAD_PARAMS
    assert 4 not in [f.id for f in cp.FIELDS.values()]


def _jubjub_generator():
    rng = random.Random(14)
    while True:
        P = J.point_from_y(rng.randrange(J.Q))
        if P is not None:
            return J.mul(8, P)


def _jpt(P):
    return np.concatenate([_limbs((P[0] << 256) % J.Q), _limbs((P[1] << 256) % J.Q)])


def test_ed377_context_argument_rules():
    """cpb_te_base_ctx_create_ex takes both curves and checks the generator on the curve it names."""
    X = N.lib.cpb_te_base_ctx_create_ex
    out = N.vp()
    rng = random.Random(15)
    G = E.mul(E.COFACTOR, random_point(rng))
    g = _pt(G)
    assert X(1, _p64(g), 0, None) == N.CPB_NULL_POINTER
    assert X(1, None, 0, C.byref(out)) == N.CPB_NULL_POINTER
    assert X(2, _p64(g), 0, C.byref(out)) == N.CPB_UNSUPPORTED
    assert X(-1, _p64(g), 0, C.byref(out)) == N.CPB_UNSUPPORTED
    off = g.copy()
    off[4] ^= np.uint64(1)                                                                     # y changed: off the curve
    assert X(1, _p64(off), 0, C.byref(out)) == N.CPB_BAD_PARAMS
    unreduced = g.copy()
    unreduced[3] = np.uint64(2**64 - 1)
    assert X(1, _p64(unreduced), 0, C.byref(out)) == N.CPB_BAD_PARAMS
    at_q = g.copy()
    at_q[:4] = _limbs(Q)
    assert X(1, _p64(at_q), 0, C.byref(out)) == N.CPB_BAD_PARAMS
    jg = _jpt(_jubjub_generator())                                                             # a Jubjub point is not on this curve
    assert X(1, _p64(jg), 0, C.byref(out)) == N.CPB_BAD_PARAMS
    assert X(0, _p64(g), 0, C.byref(out)) == N.CPB_BAD_PARAMS                                # and the converse
    if N.lib.cpb_device_count() == 0:
        assert X(1, _p64(g), 0, C.byref(out)) == N.CPB_NO_DEVICE
        assert X(0, _p64(jg), 0, C.byref(out)) == N.CPB_NO_DEVICE
        for P in torsion4():                                                                   # any curve point is a generator
            assert X(1, _p64(_pt(P)), 0, C.byref(out)) == N.CPB_NO_DEVICE


def test_the_jubjub_form_keeps_its_contract():
    """cpb_te_base_ctx_create stays the Jubjub form: every other curve id, ed-on-BLS12-377 included and with a valid generator, is
    CPB_UNSUPPORTED before the generator is read; for Jubjub it answers as the _ex form."""
    out = N.vp()
    g = _pt(E.mul(E.COFACTOR, random_point(random.Random(16))))
    jg = _jpt(_jubjub_generator())
    for curve in (1, 2, 7, -1):
        assert N.lib.cpb_te_base_ctx_create(curve, _p64(g), 0, C.byref(out)) == N.CPB_UNSUPPORTED
        assert N.lib.cpb_te_base_ctx_create(curve, None, 0, C.byref(out)) == N.CPB_UNSUPPORTED
    assert N.lib.cpb_te_base_ctx_create(1, _p64(g), 0, None) == N.CPB_NULL_POINTER
    for gen in (g, None):
        p = None if gen is None else _p64(gen)
        assert N.lib.cpb_te_base_ctx_create(0, p, 0, C.byref(out)) == N.lib.cpb_te_base_ctx_create_ex(0, p, 0, C.byref(out))
    if N.lib.cpb_device_count() == 0:
        assert N.lib.cpb_te_base_ctx_create(0, _p64(jg), 0, C.byref(out)) == N.CPB_NO_DEVICE


def test_python_mirror_uses_the_curve_scalar_field():
    assert cp.curves.JUBJUB.scalar_field is cp.JUBJUB_FR
    assert cp.curves.ED_ON_BLS12_377.scalar_field is cp.ED_ON_BLS12_377_FR
    for c in cp.curves.CURVES.values():
        assert c.scalar_field.modulus == c.scalar_modulus
