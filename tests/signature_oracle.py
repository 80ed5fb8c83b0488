"""Oracle for Schnorr signatures, ElGamal encryption and the Blake2s commitment (test infrastructure only).

A restatement of R/signature/schnorr/mod.rs, R/encryption/elgamal/mod.rs and R/commitment/blake2s/mod.rs over the affine
Jubjub oracle (oracle/jubjub.py), with the hash input built from oracle/wire.py.  Blake2s256 is Python's hashlib.blake2s
(digest_size 32), an implementation of RFC 7693 independent of the library's.  The *dep* conventions (ark-ff 0.4
`from_random_bytes`, ark-serialize 0.4 encodings) are restated each in one function.

`mul` below is the affine oracle's double-and-add; `mul_ext` and `FixedBase` compute the same points faster (extended
coordinates, one inversion at the end) for the large GPU comparisons, and are checked against `mul` in the CPU tests.
"""
from __future__ import annotations

import hashlib

from oracle import jubjub as J
from oracle import wire

Q = J.Q
R = J.ORDER
R_BITS = R.bit_length()          # MODULUS_BIT_SIZE = 252


# ---- dep: ark-ff 0.4 / ark-serialize 0.4 conventions ------------------------------------------------------------------
def from_random_bytes(digest: bytes):
    """Fp::from_random_bytes with empty flags: LE integer, bits >= MODULUS_BIT_SIZE cleared, None when >= r."""
    v = int.from_bytes(digest[:32], "little") & ((1 << R_BITS) - 1)
    return v if v < R else None


def hash_input(salt: bytes, point, message: bytes) -> bytes:
    """salt.serialize_compressed ([u8; 32], no length) || point.serialize_compressed || message.serialize_compressed (u64 length
    + bytes); schnorr/mod.rs:96-99, 131-134."""
    return bytes(salt) + wire.te_point(point, Q, compress=True) + wire.u64(len(message)) + bytes(message)


def bytes_to_bits(data: bytes):
    """schnorr/mod.rs:185-194: each byte MSB first."""
    return [((b >> (8 - i - 1)) & 1) == 1 for b in data for i in range(8)]


def blake2s256(data: bytes) -> bytes:
    return hashlib.blake2s(bytes(data), digest_size=32).digest()


# ---- Schnorr -------------------------------------------------------------------------------------------------------------
def keygen(generator, sk: int):
    return J.mul(sk, generator)


def sign(generator, salt: bytes, sk: int, message: bytes, k: int, mul=J.mul):
    """One iteration of the loop of mod.rs:87-104 with nonce k; None when the challenge is not a field element."""
    prover_commitment = mul(k, generator)
    e = from_random_bytes(blake2s256(hash_input(salt, prover_commitment, message)))
    if e is None:
        return None
    return ((k - e * sk) % R, e)


def verify(generator, salt: bytes, pk, message: bytes, signature, mul=J.mul) -> bool:
    """mod.rs:117-148."""
    s, e = signature
    claimed = J.add(mul(s, generator), mul(e, pk))
    e2 = from_random_bytes(blake2s256(hash_input(salt, claimed, message)))
    if e2 is None:
        return False
    return e == e2


def randomize_public_key(generator, pk, randomness: bytes):
    """mod.rs:150-174: double-and-add over the reversed bits, leading zeros skipped, then + pk."""
    encoded = J.IDENTITY
    bits = list(reversed(bytes_to_bits(randomness)))
    while bits and not bits[0]:
        bits.pop(0)
    for bit in bits:
        encoded = J.double(encoded)
        if bit:
            encoded = J.add(encoded, generator)
    return J.add(encoded, pk)


def randomizer_int(randomness: bytes) -> int:
    """The integer the bits of bytes_to_bits stand for, little-endian: sum_b bitrev8(byte_b) 2^(8b)."""
    return sum(1 << i for i, b in enumerate(bytes_to_bits(randomness)) if b)


def randomize_signature(signature, randomness: bytes):
    """mod.rs:176-198."""
    s, e = signature
    base, multiplier = 1, 0
    for bit in bytes_to_bits(randomness):
        if bit:
            multiplier = (multiplier + base) % R
        base = base * 2 % R
    return ((s - e * multiplier) % R, e)


# ---- ElGamal -------------------------------------------------------------------------------------------------------------
def elgamal_encrypt(generator, pk, message, r: int, mul=J.mul):
    """elgamal/mod.rs:69-84."""
    s = mul(r, pk)
    c1 = mul(r, generator)
    return (c1, J.add(message, s))


def elgamal_decrypt(sk: int, ciphertext, mul=J.mul):
    """elgamal/mod.rs:86-101."""
    c1, c2 = ciphertext
    s = mul(sk, c1)
    return J.add(c2, J.neg(s))


# ---- Blake2s commitment ----------------------------------------------------------------------------------------------
def blake2s_commit(data: bytes, r: bytes) -> bytes:
    """R/commitment/blake2s/mod.rs:21-32."""
    assert len(r) == 32
    return blake2s256(bytes(data) + bytes(r))


# ---- faster equivalents of J.mul for bulk comparisons ---------------------------------------------------------------------
_D2 = 2 * J.D % Q


def _ext(P):
    return (P[0], P[1], 1, P[0] * P[1] % Q)


def _ext_add(P, R_):
    X1, Y1, Z1, T1 = P
    X2, Y2, Z2, T2 = R_
    a = (Y1 - X1) * (Y2 - X2) % Q
    b = (Y1 + X1) * (Y2 + X2) % Q
    c = T1 * _D2 % Q * T2 % Q
    d = 2 * Z1 * Z2 % Q
    e, f, g, h = b - a, d - c, d + c, b + a
    return (e * f % Q, g * h % Q, f * g % Q, e * h % Q)


def _affine(P):
    zi = pow(P[2], -1, Q)
    return (P[0] * zi % Q, P[1] * zi % Q)


def mul_ext(k: int, P):
    acc, base = (0, 1, 1, 0), _ext(P)
    while k:
        if k & 1:
            acc = _ext_add(acc, base)
        base = _ext_add(base, base)
        k >>= 1
    return _affine(acc)


class FixedBase:
    """k*G from 32 tables of v * 256^j * G (v < 256): 32 additions per product."""

    def __init__(self, G, nbytes: int = 32):
        self.tables = []
        base = _ext(G)
        for _ in range(nbytes):
            row, acc = [(0, 1, 1, 0)], (0, 1, 1, 0)
            for _v in range(1, 256):
                acc = _ext_add(acc, base)
                row.append(acc)
            self.tables.append(row)
            base = _ext_add(acc, base)                    # 256 * base
        self.nbytes = nbytes

    def mul(self, k: int, P=None):
        acc = (0, 1, 1, 0)
        for j in range(self.nbytes):
            v = (k >> (8 * j)) & 0xFF
            if v:
                acc = _ext_add(acc, self.tables[j][v])
        assert k >> (8 * self.nbytes) == 0
        return _affine(acc)
