"""Prime fields known to the CUDA library (ids of `cpb_field`, include/cpb200.h) and the
Montgomery interchange layout: an element is 4 x uint64 little-endian limbs, R = 2^256, fully
reduced -- the memory image of ark-ff's Fp<MontBackend<_,4>,4>.  Arrays are numpy uint64 (..., 4).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import _native as N

MASK64 = (1 << 64) - 1


@dataclass(frozen=True)
class Field:
    id: int
    name: str

    @property
    def modulus(self) -> int:
        out = (C.c_uint64 * 4)()
        N.check(N.lib.cpb_field_modulus(self.id, out))
        return sum(int(out[i]) << (64 * i) for i in range(4))

    @property
    def modulus_bit_size(self) -> int:
        return self.modulus.bit_length()

    # -- small-scale conversions (Python ints; used for parameters and tests)
    def to_mont_int(self, x: int) -> int:
        return ((x % self.modulus) << 256) % self.modulus

    def from_mont_int(self, x: int) -> int:
        p = self.modulus
        return x * pow(1 << 256, -1, p) % p

    def elements(self, values) -> np.ndarray:
        """Python ints -> (n, 4) Montgomery limbs."""
        p = self.modulus
        out = np.empty((len(values), 4), dtype=np.uint64)
        for i, v in enumerate(values):
            m = ((int(v) % p) << 256) % p
            out[i] = [(m >> (64 * k)) & MASK64 for k in range(4)]
        return out

    def to_ints(self, arr) -> list[int]:
        p = self.modulus
        rinv = pow(1 << 256, -1, p)
        a = np.asarray(arr, dtype=np.uint64).reshape(-1, 4)
        return [sum(int(a[i, k]) << (64 * k) for k in range(4)) * rinv % p for i in range(a.shape[0])]

    # -- bulk conversions on the GPU (canonical LE limbs <-> Montgomery limbs)
    def to_montgomery(self, canonical: np.ndarray, device: int = 0) -> np.ndarray:
        a = np.ascontiguousarray(canonical, dtype=np.uint64)
        out = np.empty_like(a)
        N.check(N.lib.cpb_field_to_montgomery(self.id, device, a.ctypes.data_as(N.u64p), out.ctypes.data_as(N.u64p), a.size // 4))
        return out

    def from_montgomery(self, mont: np.ndarray, device: int = 0) -> np.ndarray:
        a = np.ascontiguousarray(mont, dtype=np.uint64)
        out = np.empty_like(a)
        N.check(N.lib.cpb_field_from_montgomery(self.id, device, a.ctypes.data_as(N.u64p), out.ctypes.data_as(N.u64p), a.size // 4))
        return out


BLS12_381_FR = Field(0, "bls12_381_fr")
BN254_FR = Field(1, "bn254_fr")
JUBJUB_FR = Field(2, "jubjub_fr")
BLS12_377_FR = Field(3, "bls12_377_fr")
FIELDS = {f.name: f for f in (BLS12_381_FR, BN254_FR, JUBJUB_FR, BLS12_377_FR)}     # the hash fields (Poseidon, Merkle)
# The scalar field of ed-on-BLS12-377: the field-level calls above and the signature layer only, so not in FIELDS.
ED_ON_BLS12_377_FR = Field(4, "ed_on_bls12_377_fr")
