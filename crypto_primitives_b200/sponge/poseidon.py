"""PoseidonConfig and parameter generation -- host mirror of R/sponge/poseidon/mod.rs:26-45,189-217
and R/sponge/poseidon/traits.rs:59-146 (R = /root/reference/crypto-primitives/src).  The Grain LFSR
and Cauchy-matrix arithmetic run in the library's host code (csrc/poseidon_host.hpp); permutations
run only on the GPU (see crh/poseidon.py).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field as _f

import numpy as np

from .. import _native as N
from ..fields import Field


@dataclass(eq=False)
class PoseidonConfig:
    """Same members as the reference struct (mod.rs:26-45); `ark` is (full+partial, t, 4) and `mds`
    (t, t, 4) uint64 Montgomery limbs; `field` replaces the Rust type parameter."""
    field: Field
    full_rounds: int
    partial_rounds: int
    alpha: int
    mds: np.ndarray
    ark: np.ndarray
    rate: int
    capacity: int
    _ctx: dict = _f(default_factory=dict, repr=False)

    def __post_init__(self):
        t = self.rate + self.capacity
        self.ark = np.ascontiguousarray(self.ark, dtype=np.uint64)
        self.mds = np.ascontiguousarray(self.mds, dtype=np.uint64)
        # PoseidonConfig::new asserts, mod.rs:198-206
        assert self.ark.shape == (self.full_rounds + self.partial_rounds, t, 4), "ark shape"
        assert self.mds.shape == (t, t, 4), "mds shape"

    @classmethod
    def new(cls, field, full_rounds, partial_rounds, alpha, mds, ark, rate, capacity):
        """Argument order of PoseidonConfig::new (mod.rs:189-197)."""
        return cls(field, full_rounds, partial_rounds, alpha, mds, ark, rate, capacity)

    @classmethod
    def from_ints(cls, field: Field, full_rounds, partial_rounds, alpha, mds, ark, rate, capacity):
        t = rate + capacity
        a = field.elements([x for row in ark for x in row]).reshape(full_rounds + partial_rounds, t, 4)
        m = field.elements([x for row in mds for x in row]).reshape(t, t, 4)
        return cls(field, full_rounds, partial_rounds, alpha, m, a, rate, capacity)

    # -- device context (created on first use, one per device)
    def context(self, device: int = 0):
        h = self._ctx.get(device)
        if h is None:
            out = N.vp()
            N.check(N.lib.cpb_poseidon_ctx_create(
                self.field.id, self.rate, self.capacity, self.full_rounds, self.partial_rounds, self.alpha,
                self.ark.ctypes.data_as(N.u64p), self.mds.ctypes.data_as(N.u64p), device, C.byref(out)))
            h = _Ctx(out.value)
            self._ctx[device] = h
        return h.handle


class _Ctx:
    def __init__(self, handle):
        self.handle = handle

    def __del__(self):
        try:
            if self.handle:
                N.lib.cpb_poseidon_ctx_destroy(self.handle)
                self.handle = None
        except Exception:
            pass


def find_poseidon_ark_and_mds(field: Field, prime_bits: int, rate: int, full_rounds: int, partial_rounds: int,
                              skip_matrices: int):
    """traits.rs:105-146 -> (ark (R, t, 4), mds (t, t, 4)) Montgomery limbs."""
    t = rate + 1
    ark = np.empty((full_rounds + partial_rounds, t, 4), dtype=np.uint64)
    mds = np.empty((t, t, 4), dtype=np.uint64)
    N.check(N.lib.cpb_poseidon_find_ark_and_mds(field.id, prime_bits, rate, full_rounds, partial_rounds, skip_matrices,
                                                ark.ctypes.data_as(N.u64p), mds.ctypes.data_as(N.u64p)))
    return ark, mds


def get_default_poseidon_parameters(field: Field, rate: int, optimized_for_weights: bool):
    """PoseidonDefaultConfigField::get_default_poseidon_parameters (traits.rs:59-103).  The entry tables are per field
    (`PoseidonDefaultConfig`); the reference implements them for its BLS12-381 Fr test field only
    (R/sponge/test.rs:13-32).  As in the reference, a rate without an entry yields None; so does a field without a table
    (there the reference would not compile) -- derive parameters for other fields explicitly with
    find_poseidon_ark_and_mds and a round count / alpha chosen for that field."""
    alpha = C.c_uint64()
    rf, rp, skip = C.c_int(), C.c_int(), C.c_int()
    st = N.lib.cpb_poseidon_default_entry(field.id, rate, int(bool(optimized_for_weights)), C.byref(alpha), C.byref(rf), C.byref(rp), C.byref(skip))
    if st != N.CPB_OK:
        return None
    ark, mds = find_poseidon_ark_and_mds(field, field.modulus_bit_size, rate, rf.value, rp.value, skip.value)
    return PoseidonConfig(field, rf.value, rp.value, alpha.value, mds, ark, rate, 1)


FULL = "Full"        # FieldElementSize::Full; an int is FieldElementSize::Truncated(bits) (R/sponge/mod.rs:24-36)


class PoseidonSponge:
    """Duplex sponge over the GPU permutation -- host mirror of PoseidonSponge<F> (R/sponge/poseidon/mod.rs:47-63):
    CryptographicSponge::{new, absorb, squeeze_bytes, squeeze_bits, squeeze_field_elements} (mod.rs:220-321) and
    FieldBasedCryptographicSponge::squeeze_native_field_elements (mod.rs:323-345), with the same mode bookkeeping
    (absorb_internal / squeeze_internal, mod.rs:124-186), `fork` (R/sponge/mod.rs:145-153), the sized squeezes
    (R/sponge/mod.rs:57-96,170-187) and SpongeExt::{from_state, into_state} (mod.rs:347-370).  `absorb` takes native
    field elements as (k, 4) Montgomery limbs or any value sponge/absorb.py can encode (R/sponge/absorb.rs).  Every
    permutation is one GPU call of batch size 1: correct but slow -- a single transcript is sequential by nature; for
    many independent sponges use `absorb_squeeze_batch`."""

    def __init__(self, parameters: PoseidonConfig, device: int = 0):
        self.parameters = parameters
        self.device = device
        t = parameters.rate + parameters.capacity
        self.state = np.zeros((t, 4), dtype=np.uint64)
        self.mode = ("Absorbing", 0)            # DuplexSpongeMode::{Absorbing{next_absorb_index}, Squeezing{next_squeeze_index}}

    @classmethod
    def new(cls, parameters: PoseidonConfig, device: int = 0):
        return cls(parameters, device)

    # -- internals
    def _permute(self):
        out = np.empty_like(self.state)
        N.check(N.lib.cpb_poseidon_permute_batch(self.parameters.context(self.device), self.state.ctypes.data_as(N.u64p),
                                                 out.ctypes.data_as(N.u64p), 1))
        self.state = out

    def _add(self, lane: int, elem: np.ndarray):
        f = self.parameters.field
        a, b = f.to_ints(self.state[lane])[0], f.to_ints(elem)[0]
        self.state[lane] = f.elements([(a + b) % f.modulus])[0]

    def _absorb_internal(self, rate_start: int, elems: np.ndarray):           # mod.rs:124-153
        c = self.parameters
        rem = elems
        while True:
            if rate_start + len(rem) <= c.rate:
                for i, e in enumerate(rem):
                    self._add(c.capacity + i + rate_start, e)
                self.mode = ("Absorbing", rate_start + len(rem))
                return
            k = c.rate - rate_start
            for i, e in enumerate(rem[:k]):
                self._add(c.capacity + i + rate_start, e)
            self._permute()
            rem = rem[k:]
            rate_start = 0

    def _squeeze_internal(self, rate_start: int, n_out: int) -> np.ndarray:  # mod.rs:156-186
        c = self.parameters
        out = []
        rem = n_out
        while True:
            if rate_start + rem <= c.rate:
                out.extend(self.state[c.capacity + rate_start: c.capacity + rate_start + rem])
                self.mode = ("Squeezing", rate_start + rem)
                return np.array(out, dtype=np.uint64).reshape(-1, 4)
            k = c.rate - rate_start
            out.extend(self.state[c.capacity + rate_start: c.capacity + rate_start + k])
            rem -= k
            if rem != 0:
                self._permute()
            rate_start = 0

    # -- public surface
    def clone(self) -> "PoseidonSponge":
        c = PoseidonSponge(self.parameters, self.device)
        c.state, c.mode = self.state.copy(), self.mode
        return c

    @classmethod
    def from_state(cls, state, parameters: PoseidonConfig, device: int = 0):   # mod.rs:357-362
        s = cls(parameters, device)
        s.state, s.mode = np.array(state[0], dtype=np.uint64).reshape(-1, 4), state[1]
        return s

    def into_state(self):                                                       # mod.rs:364-369
        return (self.state, self.mode)

    def fork(self, domain: bytes) -> "PoseidonSponge":
        """R/sponge/mod.rs:145-153: clone, then absorb usize(len(domain)) bytes || domain as one byte string."""
        new = self.clone()
        new.absorb(len(domain).to_bytes(8, "little") + bytes(domain))
        return new

    def absorb(self, elems):
        """elems: (k, 4) Montgomery limbs (or a single (4,) element), or any absorbable of sponge/absorb.py."""
        if isinstance(elems, np.ndarray):
            e = np.asarray(elems, dtype=np.uint64).reshape(-1, 4)
        else:
            from .absorb import to_sponge_field_elements
            e = to_sponge_field_elements(elems, self.parameters.field)
        if e.shape[0] == 0:
            return
        kind, idx = self.mode
        if kind == "Absorbing":
            if idx == self.parameters.rate:
                self._permute()
                idx = 0
            self._absorb_internal(idx, e)
        else:
            self._absorb_internal(0, e)

    def squeeze_native_field_elements(self, num_elements: int) -> np.ndarray:
        kind, idx = self.mode
        if kind == "Absorbing":
            self._permute()
            return self._squeeze_internal(0, num_elements)
        if idx == self.parameters.rate:
            self._permute()
            idx = 0
        return self._squeeze_internal(idx, num_elements)

    def squeeze_field_elements(self, num_elements: int, field: Field | None = None) -> np.ndarray:
        """mod.rs:309-320: the native fast path, else `num_elements` Full-size elements of `field`."""
        if field is None or field.id == self.parameters.field.id:
            return self.squeeze_native_field_elements(num_elements)
        return self.squeeze_field_elements_with_sizes([FULL] * num_elements, field)

    def squeeze_native_field_elements_with_sizes(self, sizes) -> np.ndarray:
        """R/sponge/mod.rs:170-187.  sizes: FULL or an int bit count (FieldElementSize::Truncated)."""
        return self.squeeze_field_elements_with_sizes(sizes, None)

    def squeeze_field_elements_with_sizes(self, sizes, field: Field | None = None) -> np.ndarray:
        """mod.rs:291-307 over R/sponge/mod.rs:57-96: (len(sizes), 4) Montgomery limbs of `field` (default: native)."""
        native = self.parameters.field
        field = native if field is None else field
        sizes = list(sizes)
        # native field: an empty `sizes` is "all Full" and still goes through squeeze_native_field_elements(0), which
        # permutes from Absorbing mode and switches to Squeezing{0} (mod.rs:291-307, R/sponge/mod.rs:164-179, mod.rs:323-345);
        # only the non-native default implementation returns early (R/sponge/mod.rs:61-63)
        if field.modulus == native.modulus and all(s == FULL for s in sizes):
            return self.squeeze_native_field_elements(len(sizes)).reshape(-1, 4)
        if not sizes:
            return np.zeros((0, 4), dtype=np.uint64)
        widths = []
        for s in sizes:
            if s == FULL:
                widths.append(field.modulus_bit_size - 1)
            elif s > field.modulus_bit_size:
                raise ValueError("num_bits is greater than the capacity of the field.")   # R/sponge/mod.rs:39-42
            else:
                widths.append(int(s))
        bits = self.squeeze_bits(sum(widths))
        vals, pos = [], 0
        for w in widths:
            vals.append(sum(1 << i for i, b in enumerate(bits[pos:pos + w]) if b))
            pos += w
        return field.elements(vals)

    def squeeze_bytes(self, num_bytes: int) -> bytes:
        """mod.rs:259-274."""
        f = self.parameters.field
        usable = (f.modulus_bit_size - 1) // 8
        n = (num_bytes + usable - 1) // usable
        out = b"".join(v.to_bytes(32, "little")[:usable] for v in f.to_ints(self.squeeze_native_field_elements(n)))
        return out[:num_bytes]

    def squeeze_bits(self, num_bits: int) -> list:
        """mod.rs:276-291."""
        f = self.parameters.field
        usable = f.modulus_bit_size - 1
        n = (num_bits + usable - 1) // usable
        bits = []
        for v in f.to_ints(self.squeeze_native_field_elements(n)):
            bits.extend(bool((v >> i) & 1) for i in range(usable))
        return bits[:num_bits]


def absorb_squeeze_batch(parameters: PoseidonConfig, inputs, num_squeeze: int, device: int = 0) -> np.ndarray:
    """n independent sponges in one kernel launch: new -> absorb(inputs[i]) -> squeeze_native_field_elements(num_squeeze).
    inputs (n, len, 4) -> (n, num_squeeze, 4).  A list of (L_i, 4) arrays whose lengths differ goes through absorb_squeeze_ragged."""
    from .. import ragged as R
    if R.is_ragged(inputs):
        return absorb_squeeze_ragged(parameters, *R.pack(inputs), num_squeeze, device)
    inp = np.ascontiguousarray(inputs, dtype=np.uint64)
    assert inp.ndim == 3 and inp.shape[2] == 4
    n, ln = inp.shape[0], inp.shape[1]
    out = np.empty((n, num_squeeze, 4), dtype=np.uint64)
    N.check(N.lib.cpb_poseidon_sponge_batch(parameters.context(device), inp.ctypes.data_as(N.u64p), ln, out.ctypes.data_as(N.u64p),
                                            num_squeeze, n))
    return out


def absorb_squeeze_ragged(parameters: PoseidonConfig, values, offsets, num_squeeze: int, device: int = 0) -> np.ndarray:
    """absorb_squeeze_batch over inputs of different lengths: sponge i absorbs values[offsets[i] .. offsets[i+1]).
    -> (n, num_squeeze, 4) with n = len(offsets) - 1; offsets that decrease raise ValueError."""
    from .. import ragged as R
    vals, off = R.as_arrays(values, offsets)
    n = off.shape[0] - 1
    out = np.empty((n, num_squeeze, 4), dtype=np.uint64)
    if n and num_squeeze:
        R.check(N.lib.cpb_poseidon_sponge_ragged_batch(parameters.context(device), vals.ctypes.data_as(N.u64p), off.ctypes.data_as(N.u64p),
                                                       out.ctypes.data_as(N.u64p), num_squeeze, n))
    return out
