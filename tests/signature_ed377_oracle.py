"""Oracle for Schnorr signatures and ElGamal encryption over ed-on-BLS12-377 (test infrastructure only).

The curve of the reference's signature benchmark, `Schnorr<ark_ed_on_bls12_377::EdwardsProjective, Blake2s256>`
(R/benches/signature.rs:5-10), restated from its definition: the twisted Edwards curve a x^2 + y^2 = 1 + d x^2 y^2 over
q = the BLS12-377 scalar field, a = -1, d = 3021, whose group has order 4 r with r prime.  The group law is the affine
addition law; a = -1 is a square and d a non-square in Fq, so that law is complete (checked in the tests).  The schemes are
R/signature/schnorr/mod.rs and R/encryption/elgamal/mod.rs over this group, with the same *dep* conventions as
tests/signature_oracle.py (ark-ff 0.4 `from_random_bytes`, ark-serialize 0.4 compression), here at MODULUS_BIT_SIZE = 251.

`mul` is the affine double-and-add; `mul_ext` and `FixedBase` compute the same points in extended coordinates with one
inversion at the end, for the large GPU comparisons, and are checked against `mul` in the CPU tests.
"""
from __future__ import annotations

import hashlib

Q = 0x12AB655E9A2CA55660B44D1E5C37B00159AA76FED00000010A11800000000001      # BLS12-377 Fr
R = 0x04AAD957A68B2955982D1347970DEC005293A3AFC43C8AFEB95AEE9AC33FD9FF      # prime-order subgroup
R_BITS = R.bit_length()          # MODULUS_BIT_SIZE = 251
A = Q - 1
D = 3021
COFACTOR = 4
IDENTITY = (0, 1)


# ---- affine group law ------------------------------------------------------------------------------------------------------
def is_on_curve(P) -> bool:
    x, y = P
    return (A * x * x + y * y - 1 - D * x * x % Q * y * y) % Q == 0


def add(P, P2):
    x1, y1 = P
    x2, y2 = P2
    k = D * x1 % Q * x2 % Q * y1 % Q * y2 % Q
    x3 = (x1 * y2 + y1 * x2) * pow((1 + k) % Q, -1, Q) % Q
    y3 = (y1 * y2 - A * x1 * x2) * pow((1 - k) % Q, -1, Q) % Q
    return (x3, y3)


def double(P):
    return add(P, P)


def neg(P):
    return ((-P[0]) % Q, P[1])


def mul(k: int, P):
    acc, base = IDENTITY, P
    while k:
        if k & 1:
            acc = add(acc, base)
        base = double(base)
        k >>= 1
    return acc


def sqrt(n: int):
    """Tonelli-Shanks in Fq; None for a non-residue."""
    n %= Q
    if n == 0:
        return 0
    if pow(n, (Q - 1) // 2, Q) != 1:
        return None
    s, t = 0, Q - 1
    while t % 2 == 0:
        s, t = s + 1, t // 2
    z = 2
    while pow(z, (Q - 1) // 2, Q) == 1:
        z += 1
    m, c, tt, r = s, pow(z, t, Q), pow(n, t, Q), pow(n, (t + 1) // 2, Q)
    while tt != 1:
        i, x = 0, tt
        while x != 1:
            x, i = x * x % Q, i + 1
        b = pow(c, 1 << (m - i - 1), Q)
        m, c = i, b * b % Q
        tt, r = tt * c % Q, r * b % Q
    return r


def point_from_y(y: int):
    """x^2 = (1 - y^2) / (a - d y^2); the root with even canonical x, or None."""
    y %= Q
    den = (A - D * y * y) % Q
    if den == 0:
        return None
    x = sqrt((1 - y * y) * pow(den, -1, Q) % Q)
    if x is None:
        return None
    return (Q - x if x & 1 else x, y)


def compress(P) -> bytes:
    """ark-serialize 0.4 compressed TE point: 32-byte LE canonical y, bit 7 of the last byte set when x > -x."""
    out = bytearray(P[1].to_bytes(32, "little"))
    if P[0] > (-P[0]) % Q:
        out[31] |= 0x80
    return bytes(out)


# ---- Schnorr (R/signature/schnorr/mod.rs) -----------------------------------------------------------------------------------
def from_random_bytes(digest: bytes):
    """Fp::from_random_bytes with empty flags: LE integer, bits >= MODULUS_BIT_SIZE cleared, None when >= r."""
    v = int.from_bytes(digest[:32], "little") & ((1 << R_BITS) - 1)
    return v if v < R else None


def blake2s256(data: bytes) -> bytes:
    return hashlib.blake2s(bytes(data), digest_size=32).digest()


def hash_input(salt: bytes, point, message: bytes) -> bytes:
    """salt || compress(point) || u64_le(len) || message (mod.rs:96-99, 131-134)."""
    return bytes(salt) + compress(point) + len(message).to_bytes(8, "little") + bytes(message)


def keygen(generator, sk: int, mul=mul):
    return mul(sk, generator)


def sign(generator, salt: bytes, sk: int, message: bytes, k: int, mul=mul):
    """One iteration of the signing loop (mod.rs:87-104) with nonce k; None when the challenge is not a field element."""
    e = from_random_bytes(blake2s256(hash_input(salt, mul(k, generator), message)))
    if e is None:
        return None
    return ((k - e * sk) % R, e)


def verify(generator, salt: bytes, pk, message: bytes, signature, mul=mul) -> bool:
    """mod.rs:117-148."""
    s, e = signature
    e2 = from_random_bytes(blake2s256(hash_input(salt, add(mul(s, generator), mul(e, pk)), message)))
    return e2 is not None and e == e2


def randomizer_int(randomness: bytes) -> int:
    """The integer of bytes_to_bits (mod.rs:185-194, each byte MSB first) read as little-endian bits."""
    return sum(int(f"{b:08b}"[::-1], 2) << (8 * i) for i, b in enumerate(randomness))


def randomize_public_key(generator, pk, randomness: bytes, mul=mul):
    """mod.rs:150-174: pk + m*G for the exact (unreduced) integer m."""
    return add(mul(randomizer_int(randomness), generator), pk)


def randomize_signature(signature, randomness: bytes):
    """mod.rs:176-198: (s - e*m, e) in Fr."""
    s, e = signature
    return ((s - e * randomizer_int(randomness)) % R, e)


# ---- ElGamal (R/encryption/elgamal/mod.rs) ----------------------------------------------------------------------------------
def elgamal_encrypt(generator, pk, message, r: int, mul=mul):
    """mod.rs:69-84: (r*G, m + r*pk)."""
    return (mul(r, generator), add(message, mul(r, pk)))


def elgamal_decrypt(sk: int, ciphertext, mul=mul):
    """mod.rs:86-101: c2 - sk*c1."""
    c1, c2 = ciphertext
    return add(c2, neg(mul(sk, c1)))


# ---- faster equivalents of `mul` for bulk comparisons -----------------------------------------------------------------------
_D2 = 2 * D % Q
_ID_EXT = (0, 1, 1, 0)


def _ext(P):
    return (P[0], P[1], 1, P[0] * P[1] % Q)


def _ext_add(P, P2):
    """Extended coordinates, a = -1 (the unified formula; complete here)."""
    X1, Y1, Z1, T1 = P
    X2, Y2, Z2, T2 = P2
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
    acc, base = _ID_EXT, _ext(P)
    while k:
        if k & 1:
            acc = _ext_add(acc, base)
        base = _ext_add(base, base)
        k >>= 1
    return _affine(acc)


class FixedBase:
    """k*G from tables of v * 256^j * G (v < 256, j < nbytes): one addition per non-zero byte of k."""

    def __init__(self, G, nbytes: int = 32):
        self.tables = []
        base = _ext(G)
        for _ in range(nbytes):
            row, acc = [_ID_EXT], _ID_EXT
            for _v in range(1, 256):
                acc = _ext_add(acc, base)
                row.append(acc)
            self.tables.append(row)
            base = _ext_add(acc, base)                    # 256 * base
        self.nbytes = nbytes

    def mul(self, k: int, P=None):
        assert k >> (8 * self.nbytes) == 0
        acc = _ID_EXT
        for j in range(self.nbytes):
            v = (k >> (8 * j)) & 0xFF
            if v:
                acc = _ext_add(acc, self.tables[j][v])
        return _affine(acc)
