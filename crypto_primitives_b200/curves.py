"""Twisted-Edwards curves known to the CUDA library (ids of `cpb_curve`) and the small amount of
host-side group arithmetic that parameter *setup* needs (random base points and their doublings,
R/crh/pedersen/mod.rs:38-56).  Hashing itself never runs here -- it is done by the GPU kernels."""
from __future__ import annotations

from dataclasses import dataclass

from .fields import BLS12_377_FR, BLS12_381_FR, ED_ON_BLS12_377_FR, JUBJUB_FR, Field


@dataclass(frozen=True)
class TECurve:
    id: int
    name: str
    base_field: Field
    scalar_modulus: int
    cofactor: int
    d_num: int
    d_den: int          # d = -(d_num/d_den) when d_den != 1 else d_num ; a = -1
    scalar_field: Field     # the field of scalar_modulus: secret keys, nonces and signatures are its elements

    @property
    def q(self) -> int:
        return self.base_field.modulus

    @property
    def d(self) -> int:
        q = self.q
        return (-(self.d_num * pow(self.d_den, -1, q))) % q if self.d_den != 1 else self.d_num % q

    @property
    def scalar_modulus_bit_size(self) -> int:
        return self.scalar_modulus.bit_length()

    def is_on_curve(self, P) -> bool:
        q, x, y = self.q, P[0], P[1]
        return (-x * x + y * y - 1 - self.d * x * x % q * y * y) % q == 0

    def add(self, P, R):
        q, d = self.q, self.d
        x1, y1 = P
        x2, y2 = R
        k = d * x1 % q * x2 % q * y1 % q * y2 % q
        x3 = (x1 * y2 + y1 * x2) % q * pow((1 + k) % q, -1, q) % q
        y3 = (y1 * y2 + x1 * x2) % q * pow((1 - k) % q, -1, q) % q
        return (x3, y3)

    def double(self, P):
        return self.add(P, P)

    def mul(self, k: int, P):
        acc, base = (0, 1), P
        while k:
            if k & 1:
                acc = self.add(acc, base)
            base = self.double(base)
            k >>= 1
        return acc

    def _sqrt(self, n: int):
        q = self.q
        n %= q
        if n == 0:
            return 0
        if pow(n, (q - 1) // 2, q) != 1:
            return None
        s, t = 0, q - 1
        while t % 2 == 0:
            s, t = s + 1, t // 2
        z = 2
        while pow(z, (q - 1) // 2, q) == 1:
            z += 1
        m, c, tt, r = s, pow(z, t, q), pow(n, t, q), pow(n, (t + 1) // 2, q)
        while tt != 1:
            i, x = 0, tt
            while x != 1:
                x, i = x * x % q, i + 1
            b = pow(c, 1 << (m - i - 1), q)
            m, c = i, b * b % q
            tt, r = tt * c % q, r * b % q
        return r

    def random_point(self, rng):
        """A point of the prime-order subgroup drawn from `rng` (any object with .field(q) -> int):
        the analogue of `C::rand(rng)`.  y is drawn until x exists; even x; times the cofactor."""
        q, d = self.q, self.d
        while True:
            y = rng.field(q)
            den = (-1 - d * y * y) % q
            if den == 0:
                continue
            x = self._sqrt((1 - y * y) % q * pow(den, -1, q) % q)
            if x is None:
                continue
            if x & 1:
                x = q - x
            P = self.mul(self.cofactor, (x, y))
            if P != (0, 1):
                return P


JUBJUB = TECurve(0, "jubjub", BLS12_381_FR, 0x0E7DB4EA6533AFA906673B0101343B00A6682093CCC81082D0970E5ED6F72CB7,
                 8, 10240, 10241, JUBJUB_FR)
ED_ON_BLS12_377 = TECurve(1, "ed_on_bls12_377", BLS12_377_FR,
                          0x04AAD957A68B2955982D1347970DEC005293A3AFC43C8AFEB95AEE9AC33FD9FF, 4, 3021, 1,
                          ED_ON_BLS12_377_FR)
CURVES = {c.name: c for c in (JUBJUB, ED_ON_BLS12_377)}
