"""CPU checks of the Schnorr / ElGamal / Blake2s device code (csrc/blake2s.cuh, csrc/te_ops.cuh, run through the host shim
tests/host/signature_shim.cpp) against the oracle, the oracle itself on the reference's scenarios, and the argument rules of
the C-ABI entry points (include/cpb200.h) without a device."""
import ctypes as C
import functools
import hashlib
import random

import numpy as np
import pytest

from helpers import build_host_shim
from crypto_primitives_b200 import _native as N
from oracle import jubjub as J
from oracle import wire
import signature_oracle as O

Q, R = J.Q, J.ORDER


@pytest.fixture(scope="module")
def shim():
    lib = build_host_shim("signature_shim")
    u8, u64 = C.POINTER(C.c_uint8), C.POINTER(C.c_uint64)
    lib.host_blake2s.argtypes = [u8, C.c_uint64, u8]
    lib.host_blake2s_concat.argtypes = [u8, C.c_uint64, u8, C.c_uint64, u8]
    lib.host_schnorr_digest.argtypes = [u8, u64, u8, C.c_uint64, u8]
    lib.host_compress.argtypes = [u64, u8]
    lib.host_from_random_bytes.argtypes = [u8, u64]
    lib.host_from_random_bytes.restype = C.c_int
    lib.host_dbl.argtypes = [u64, u64]
    lib.host_add.argtypes = [u64, u64, u64]
    lib.host_neg.argtypes = [u64, u64]
    lib.host_mul_words.argtypes = [u64, u64, C.c_int, u64]
    lib.host_mul_bitrev_bytes.argtypes = [u64, u8, C.c_uint64, u64]
    return lib


def _buf(data: bytes):
    a = np.frombuffer(bytes(data) + b"\0", dtype=np.uint8).copy()
    return a, a.ctypes.data_as(C.POINTER(C.c_uint8))


def _out(n):
    a = np.zeros(n, dtype=np.uint8)
    return a, a.ctypes.data_as(C.POINTER(C.c_uint8))


def _limbs(v: int, n: int = 4):
    return np.array([(v >> (64 * i)) & (2**64 - 1) for i in range(n)], dtype=np.uint64)


def _pt(P):
    """affine point (ints) -> Montgomery limbs x || y"""
    return np.concatenate([_limbs((P[0] << 256) % Q), _limbs((P[1] << 256) % Q)])


def _unpt(a):
    rinv = pow(1 << 256, -1, Q)
    v = [sum(int(a[4 * k + i]) << (64 * i) for i in range(4)) * rinv % Q for k in range(2)]
    return (v[0], v[1])


def _p64(a):
    return a.ctypes.data_as(C.POINTER(C.c_uint64))


@functools.lru_cache(None)
def torsion8():
    """The 8 points of order dividing 8 (the identity, (0, -1), the two of order 4 with y = 0 and four of order 8): the
    multiples of r*P for a point P whose r-multiple has order 8 (the torsion part of Jubjub's group is cyclic)."""
    rng = random.Random(99)
    while True:
        T = J.mul(R, random_point(rng))
        if J.mul(4, T) != J.IDENTITY:
            break
    pts = {J.mul(k, T) for k in range(8)}
    assert len(pts) == 8 and all(J.is_on_curve(P) and J.mul(8, P) == J.IDENTITY for P in pts)
    assert (0, Q - 1) in pts and sum(1 for P in pts if P[1] == 0) == 2
    return sorted(pts)


def random_point(rng):
    while True:
        P = J.point_from_y(rng.randrange(Q))
        if P is not None:
            return P


# ---- Blake2s ---------------------------------------------------------------------------------------------------------------
def test_hashlib_blake2s_rfc7693_vector():
    assert hashlib.blake2s(b"abc", digest_size=32).hexdigest() == "508c5e8c327c14e2e1a72ba34eeb452f37458b209ed63a294d999b4c86675982"


def test_blake2s_every_length(shim):
    rng = random.Random(1)
    data = bytes(rng.randrange(256) for _ in range(300))
    for ln in range(0, 301):
        b, bp = _buf(data[:ln])
        o, op = _out(32)
        shim.host_blake2s(bp, ln, op)
        assert o.tobytes() == hashlib.blake2s(data[:ln], digest_size=32).digest(), ln


def test_blake2s_concatenated_sources(shim):
    """The commitment's input || randomness and a ragged batch: every split point of a message."""
    rng = random.Random(2)
    for ln in (0, 1, 31, 32, 33, 63, 64, 65, 128, 129, 200):
        data = bytes(rng.randrange(256) for _ in range(ln))
        r = bytes(rng.randrange(256) for _ in range(32))
        a, ap = _buf(data)
        b, bp = _buf(r)
        o, op = _out(32)
        shim.host_blake2s_concat(ap, ln, bp, 32, op)
        assert o.tobytes() == O.blake2s_commit(data, r)
    # a ragged batch: inputs back to back, each hashed from its own offset
    lens = [rng.randrange(0, 140) for _ in range(40)]
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    vals = bytes(rng.randrange(256) for _ in range(int(offs[-1])))
    vb, _ = _buf(vals)
    for i in range(len(lens)):
        r = bytes([i]) * 32
        b, bp = _buf(r)
        o, op = _out(32)
        shim.host_blake2s_concat(vb[int(offs[i]):].ctypes.data_as(C.POINTER(C.c_uint8)), lens[i], bp, 32, op)
        assert o.tobytes() == O.blake2s_commit(vals[int(offs[i]):int(offs[i + 1])], r)


def test_schnorr_hash_input_layout(shim):
    rng = random.Random(3)
    salt = bytes(rng.randrange(256) for _ in range(32))
    for ln in (0, 1, 7, 8, 55, 56, 57, 64, 120, 200, 300):
        P = random_point(rng)
        msg = bytes(rng.randrange(256) for _ in range(ln))
        m, mp = _buf(msg)
        s, sp = _buf(salt)
        pt = _pt(P)
        o, op = _out(32)
        shim.host_schnorr_digest(sp, _p64(pt), mp, ln, op)
        assert o.tobytes() == O.blake2s256(O.hash_input(salt, P, msg)), ln


# ---- compression, from_random_bytes ------------------------------------------------------------------------------------
def test_compression(shim):
    rng = random.Random(4)
    pts = [J.IDENTITY, (0, Q - 1)] + torsion8() + [random_point(rng) for _ in range(40)]
    pts += [J.neg(P) for P in pts]
    for P in pts:
        o, op = _out(32)
        pt = _pt(P)
        shim.host_compress(_p64(pt), op)
        assert o.tobytes() == wire.te_point(P, Q, compress=True), P


def test_from_random_bytes(shim):
    rng = random.Random(5)
    cases = [R - 1, R, (1 << 252) - 1, 0, 1, R + 1, (1 << 256) - 1, R | (1 << 252), (R - 1) | (0xF << 252), 1 << 255]
    cases += [rng.getrandbits(256) for _ in range(300)]
    for v in cases:
        d = v.to_bytes(32, "little")
        b, bp = _buf(d)
        mont = np.zeros(4, dtype=np.uint64)
        ok = shim.host_from_random_bytes(bp, _p64(mont))
        exp = O.from_random_bytes(d)
        assert bool(ok) == (exp is not None), hex(v)
        if ok:
            assert sum(int(mont[i]) << (64 * i) for i in range(4)) == (exp << 256) % R
    # masking, not reduction: bits >= 252 never make a value valid or invalid on their own
    assert O.from_random_bytes(((1 << 256) - 1).to_bytes(32, "little")) is None
    assert O.from_random_bytes(((1 << 256) - 1 - (1 << 251)).to_bytes(32, "little")) == (1 << 251) - 1
    assert O.from_random_bytes((R - 1 + (0xF << 252)).to_bytes(32, "little")) == R - 1


# ---- group operations ---------------------------------------------------------------------------------------------------
def _bases():
    rng = random.Random(6)
    return [random_point(rng) for _ in range(6)] + torsion8()


def test_doubling_and_addition_agree_with_the_complete_law(shim):
    bases = _bases()
    for P in bases:
        o = np.zeros(8, dtype=np.uint64)
        shim.host_dbl(_p64(_pt(P)), _p64(o))
        assert _unpt(o) == J.double(P), P
        shim.host_neg(_p64(_pt(P)), _p64(o))
        assert _unpt(o) == J.neg(P)
        for Q2 in bases:
            shim.host_add(_p64(_pt(P)), _p64(_pt(Q2)), _p64(o))
            assert _unpt(o) == J.add(P, Q2), (P, Q2)


SCALARS = [0, 1, 2, 3, 7, 8, 9, 15, 16, 17, R - 1, R - 2, (1 << 252) - 1, (1 << 256) - 1, int("88" * 32, 16), int("01" * 32, 16),
           1 << 251, (1 << 128) + 1, 0x7777777777777777, int("87" * 32, 16)]


def test_variable_base_multiplication(shim):
    rng = random.Random(7)
    scalars = SCALARS + [rng.getrandbits(256) for _ in range(4)] + [rng.randrange(R) for _ in range(4)]
    for P in _bases():
        base = _pt(P)
        for k in scalars:
            o = np.zeros(8, dtype=np.uint64)
            nib = 64 if k >> 252 else 63
            shim.host_mul_words(_p64(base), _p64(_limbs(k)), nib, _p64(o))
            assert _unpt(o) == J.mul(k, P), (P, hex(k))


def test_multiplication_by_randomness_bytes(shim):
    rng = random.Random(8)
    G = random_point(rng)
    for P in [G] + torsion8()[:3]:
        for ln in (0, 1, 2, 31, 32, 33, 100):
            for data in (bytes(rng.randrange(256) for _ in range(ln)), b"\xff" * ln, b"\x01" * ln, b"\x80" * ln):
                b, bp = _buf(data)
                o = np.zeros(8, dtype=np.uint64)
                shim.host_mul_bitrev_bytes(_p64(_pt(P)), bp, ln, _p64(o))
                assert _unpt(o) == J.mul(O.randomizer_int(data), P), (ln, data[:4])
                assert _unpt(o) == J.add(O.randomize_public_key(P, J.IDENTITY, data), J.IDENTITY)


def test_fast_oracle_products_match_the_affine_oracle():
    rng = random.Random(9)
    G = random_point(rng)
    fb = O.FixedBase(G)
    for k in SCALARS[:14] + [rng.randrange(R) for _ in range(5)]:
        k &= (1 << 256) - 1
        assert fb.mul(k) == J.mul(k, G) == O.mul_ext(k, G)
    for P in torsion8():
        assert O.mul_ext(5, P) == J.mul(5, P)


# ---- the reference's scenarios on the oracle (R/signature/mod.rs:52-105, R/encryption/elgamal/mod.rs:102-128) ----------
def _setup(rng):
    G = J.mul(J.COFACTOR, random_point(rng))
    salt = bytes(rng.randrange(256) for _ in range(32))
    return G, salt


def _sign(G, salt, sk, msg, rng):
    while True:
        sig = O.sign(G, salt, sk, msg, rng.randrange(R))
        if sig is not None:
            return sig


def test_oracle_sign_and_verify():
    rng = random.Random(10)
    for msg in (b"Hi, I am a Schnorr signature!", b"\x00" * 4 + b"hello"):
        G, salt = _setup(rng)
        sk = rng.randrange(R)
        pk = O.keygen(G, sk)
        sig = _sign(G, salt, sk, msg, rng)
        assert O.verify(G, salt, pk, msg, sig)


def test_oracle_failed_verification():
    rng = random.Random(11)
    G, salt = _setup(rng)
    sk = rng.randrange(R)
    pk = O.keygen(G, sk)
    sig = _sign(G, salt, sk, b"Bad message", rng)
    assert not O.verify(G, salt, pk, b"Hi, I am a Schnorr signature!", sig)


def test_oracle_randomize_and_verify():
    rng = random.Random(12)
    G, salt = _setup(rng)
    msg = b"Hi, I am a Schnorr signature!"
    sk = rng.randrange(R)
    pk = O.keygen(G, sk)
    sig = _sign(G, salt, sk, msg, rng)
    assert O.verify(G, salt, pk, msg, sig)
    for randomness in (bytes(32), b"\x01" * 32, bytes(rng.randrange(256) for _ in range(32))):
        rpk = O.randomize_public_key(G, pk, randomness)
        rsig = O.randomize_signature(sig, randomness)
        assert O.verify(G, salt, rpk, msg, rsig)


def test_oracle_elgamal_round_trip():
    rng = random.Random(13)
    G = J.mul(J.COFACTOR, random_point(rng))
    sk = rng.randrange(R)
    pk = O.keygen(G, sk)
    msg = J.mul(J.COFACTOR, random_point(rng))
    ct = O.elgamal_encrypt(G, pk, msg, rng.randrange(R))
    assert O.elgamal_decrypt(sk, ct) == msg


# ---- ABI rules without a device --------------------------------------------------------------------------------------------
def test_abi_rules_without_a_device():
    out = N.vp()
    rng = random.Random(14)
    G = J.mul(8, random_point(rng))
    g = _pt(G)
    assert N.lib.cpb_te_base_ctx_create(0, _p64(g), 0, None) == N.CPB_NULL_POINTER
    assert N.lib.cpb_te_base_ctx_create(1, _p64(g), 0, C.byref(out)) == N.CPB_UNSUPPORTED     # ed-on-BLS12-377
    assert N.lib.cpb_te_base_ctx_create(7, _p64(g), 0, C.byref(out)) == N.CPB_UNSUPPORTED
    assert N.lib.cpb_te_base_ctx_create(0, None, 0, C.byref(out)) == N.CPB_NULL_POINTER
    off = g.copy()
    off[4] ^= np.uint64(1)                                                                     # y changed: off the curve
    assert N.lib.cpb_te_base_ctx_create(0, _p64(off), 0, C.byref(out)) == N.CPB_BAD_PARAMS
    unreduced = g.copy()
    unreduced[3] = np.uint64(2**64 - 1)
    assert N.lib.cpb_te_base_ctx_create(0, _p64(unreduced), 0, C.byref(out)) == N.CPB_BAD_PARAMS
    if N.lib.cpb_device_count() == 0:
        assert N.lib.cpb_te_base_ctx_create(0, _p64(g), 0, C.byref(out)) == N.CPB_NO_DEVICE
        for P in torsion8():                                                                   # any curve point is a generator
            assert N.lib.cpb_te_base_ctx_create(0, _p64(_pt(P)), 0, C.byref(out)) == N.CPB_NO_DEVICE

    salt = (C.c_uint8 * 32)()
    sc = np.zeros(4 * 4, dtype=np.uint64)
    sig = np.zeros(8 * 4, dtype=np.uint64)
    flags = np.zeros(4, dtype=np.uint8)
    msgs = np.zeros(16, dtype=np.uint8)
    u8 = lambda a: a.ctypes.data_as(N.u8p)                                                     # noqa: E731
    dec = np.array([0, 4, 2, 6, 8], dtype=np.uint64)
    inc = np.array([0, 4, 4, 6, 8], dtype=np.uint64)
    S, V = N.lib.cpb_schnorr_sign_batch, N.lib.cpb_schnorr_verify_batch
    # decreasing offsets (host forms) -> CPB_BAD_LENGTH before the context is looked at
    assert S(None, salt, _p64(sc), _p64(sc), u8(msgs), _p64(dec), _p64(sig), u8(flags), 4) == N.CPB_BAD_LENGTH
    assert V(None, salt, _p64(sig), u8(msgs), _p64(dec), _p64(sig), u8(flags), 4) == N.CPB_BAD_LENGTH
    assert N.lib.cpb_blake2s_commit_batch(0, u8(msgs), _p64(dec), u8(msgs), u8(msgs), 4) == N.CPB_BAD_LENGTH
    # n >= 2^32
    big = 1 << 32
    assert S(None, salt, _p64(sc), _p64(sc), u8(msgs), _p64(inc), _p64(sig), u8(flags), big) == N.CPB_BAD_LENGTH
    assert V(None, salt, _p64(sig), u8(msgs), _p64(inc), _p64(sig), u8(flags), big) == N.CPB_BAD_LENGTH
    assert N.lib.cpb_te_base_mul_batch(None, _p64(sc), _p64(sig), big) == N.CPB_BAD_LENGTH
    assert N.lib.cpb_elgamal_encrypt_batch(None, _p64(sig), _p64(sig), _p64(sc), _p64(sig), big) == N.CPB_BAD_LENGTH
    assert N.lib.cpb_elgamal_decrypt_batch(None, _p64(sc), _p64(sig), _p64(sig), big) == N.CPB_BAD_LENGTH
    assert N.lib.cpb_schnorr_randomize_public_key_batch(None, _p64(sig), u8(msgs), 4, 4, _p64(sig), big) == N.CPB_BAD_LENGTH
    assert N.lib.cpb_schnorr_randomize_signature_batch(None, _p64(sig), u8(msgs), 4, 4, _p64(sig), big) == N.CPB_BAD_LENGTH
    assert N.lib.cpb_blake2s_commit_batch(0, u8(msgs), _p64(inc), u8(msgs), u8(msgs), big) == N.CPB_BAD_LENGTH
    assert N.lib.cpb_schnorr_verify_batch_dev(None, salt, None, None, None, None, None, big, None) == N.CPB_BAD_LENGTH
    assert N.lib.cpb_blake2s_commit_batch_dev(0, None, None, None, None, big, None) == N.CPB_BAD_LENGTH
    # n == 0: nothing to do
    assert S(None, salt, None, None, None, None, None, None, 0) == N.CPB_OK
    assert N.lib.cpb_blake2s_commit_batch_dev(0, None, None, None, None, 0, None) == N.CPB_OK
    # null context, otherwise valid
    assert S(None, salt, _p64(sc), _p64(sc), u8(msgs), _p64(inc), _p64(sig), u8(flags), 4) == N.CPB_NULL_POINTER
    assert V(None, salt, _p64(sig), u8(msgs), _p64(inc), _p64(sig), u8(flags), 4) == N.CPB_NULL_POINTER
    assert N.lib.cpb_te_base_mul_batch(None, _p64(sc), _p64(sig), 4) == N.CPB_NULL_POINTER
    assert N.lib.cpb_elgamal_decrypt_batch_dev(None, sc.ctypes.data, sig.ctypes.data, sig.ctypes.data, 1, None) == N.CPB_NULL_POINTER
    assert S(None, None, _p64(sc), _p64(sc), u8(msgs), _p64(inc), _p64(sig), u8(flags), 4) == N.CPB_NULL_POINTER    # null salt
    # no context needed: the commitment fails on the device
    if N.lib.cpb_device_count() == 0:
        assert N.lib.cpb_blake2s_commit_batch(0, u8(msgs), _p64(inc), u8(msgs), u8(msgs), 4) == N.CPB_NO_DEVICE
