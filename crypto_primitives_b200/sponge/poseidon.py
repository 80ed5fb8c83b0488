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


def _c_mode(mode) -> "N.SpongeMode":
    kind, idx = mode
    if kind not in ("Absorbing", "Squeezing"):
        raise ValueError(f"unknown sponge mode {kind!r}")
    return N.SpongeMode(int(kind == "Squeezing"), int(idx))


def _py_mode(m) -> tuple:
    return ("Squeezing" if m.squeezing else "Absorbing", int(m.index))


class PoseidonSponge:
    """Duplex sponge over the GPU permutation -- host mirror of PoseidonSponge<F> (R/sponge/poseidon/mod.rs:47-63):
    CryptographicSponge::{new, absorb, squeeze_bytes, squeeze_bits, squeeze_field_elements} (mod.rs:220-321) and
    FieldBasedCryptographicSponge::squeeze_native_field_elements (mod.rs:323-345), `fork` (R/sponge/mod.rs:145-153), the sized
    squeezes (R/sponge/mod.rs:57-96,170-187) and SpongeExt::{from_state, into_state} (mod.rs:347-370).  `absorb` takes native
    field elements as (k, 4) Montgomery limbs or any value sponge/absorb.py can encode (R/sponge/absorb.rs).  It is the n = 1 case
    of the batched duplex (cpb_poseidon_duplex_*, host form): one library call per absorb or squeeze, which runs every permutation
    that call needs and the reference's mode bookkeeping (absorb_internal / squeeze_internal, mod.rs:124-186) on the GPU.  For many
    sponges running the same script use PoseidonSpongeBatch."""

    def __init__(self, parameters: PoseidonConfig, device: int = 0):
        self.parameters = parameters
        self.device = device
        t = parameters.rate + parameters.capacity
        self.state = np.zeros((t, 4), dtype=np.uint64)
        self.mode = ("Absorbing", 0)            # DuplexSpongeMode::{Absorbing{next_absorb_index}, Squeezing{next_squeeze_index}}

    @classmethod
    def new(cls, parameters: PoseidonConfig, device: int = 0):
        return cls(parameters, device)

    # -- internals: one duplex call of batch size 1 on the host-form C-ABI
    def _call(self, fn, *args):
        st = np.ascontiguousarray(self.state, dtype=np.uint64).copy()
        m = _c_mode(self.mode)
        N.check(fn(self.parameters.context(self.device), st.ctypes.data_as(N.u64p), C.byref(m), *args, 1))
        self.state, self.mode = st, _py_mode(m)

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
        if isinstance(elems, (bytes, bytearray)):                              # the [u8] rule, encoded on the device
            b = np.frombuffer(bytes(elems), dtype=np.uint8)
            self._call(N.lib.cpb_poseidon_duplex_absorb_bytes, b.ctypes.data_as(N.u8p) if len(b) else None, len(b), 0)
            return
        if isinstance(elems, np.ndarray):
            e = np.ascontiguousarray(elems, dtype=np.uint64).reshape(-1, 4)
        else:
            from .absorb import to_sponge_field_elements
            e = np.ascontiguousarray(to_sponge_field_elements(elems, self.parameters.field))
        self._call(N.lib.cpb_poseidon_duplex_absorb, e.ctypes.data_as(N.u64p), e.shape[0])

    def squeeze_native_field_elements(self, num_elements: int) -> np.ndarray:
        out = np.zeros((max(num_elements, 1), 4), dtype=np.uint64)
        self._call(N.lib.cpb_poseidon_duplex_squeeze, out.ctypes.data_as(N.u64p), num_elements, 0)
        return out[:num_elements]

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


class PoseidonSpongeBatch:
    """n independent PoseidonSponge over one PoseidonConfig that run the same script: the states are a torch CUDA int64 tensor
    (n, t, 4) of Montgomery limbs on `device`, and the batch has one DuplexSpongeMode.  Every absorb or squeeze is one call of the
    _dev C-ABI (cpb_poseidon_duplex_*) on the current torch stream, which runs every permutation of the call for all n sponges in
    one kernel launch.  Results are torch tensors on the device; sponge(i) continues item i as an independent PoseidonSponge."""

    def __init__(self, parameters: PoseidonConfig, n: int, device=None):
        import torch
        self.parameters = parameters
        self.n = int(n)
        self.device = _cuda_device(device)
        t = parameters.rate + parameters.capacity
        self.states = torch.zeros((self.n, t, 4), dtype=torch.int64, device=self.device)
        self._mode = N.SpongeMode(0, 0)

    # -- state
    @property
    def mode(self) -> tuple:
        return _py_mode(self._mode)

    @classmethod
    def from_states(cls, states, mode, parameters: PoseidonConfig, device=None) -> "PoseidonSpongeBatch":
        """SpongeExt::from_state for the batch: states (n, t, 4) Montgomery limbs (torch or numpy), mode ("Absorbing"|"Squeezing", index)."""
        st = _as_i64(states, _cuda_device(device))
        b = cls(parameters, st.shape[0], st.device)
        t = parameters.rate + parameters.capacity
        if tuple(st.shape[1:]) != (t, 4):
            raise ValueError(f"states must be (n, {t}, 4)")
        b.states = st.contiguous().clone()
        b._mode = _c_mode(mode)
        return b

    def into_states(self):
        return self.states, self.mode

    def clone(self) -> "PoseidonSpongeBatch":
        c = PoseidonSpongeBatch.__new__(PoseidonSpongeBatch)
        c.parameters, c.n, c.device = self.parameters, self.n, self.device
        c.states = self.states.clone()
        c._mode = N.SpongeMode(self._mode.squeezing, self._mode.index)
        return c

    def sponge(self, i: int) -> PoseidonSponge:
        """Item i as an independent PoseidonSponge (host state)."""
        st = self.states[i].cpu().numpy().view(np.uint64)
        return PoseidonSponge.from_state((st, self.mode), self.parameters, self.device.index)

    # -- internals
    def _stream(self):
        import torch
        return torch.cuda.current_stream(self.device).cuda_stream

    def _ctx(self):
        return self.parameters.context(self.device.index)

    # -- absorb
    def absorb(self, x):
        """x: (n, k, 4) native elements (torch or numpy limbs); (n, L) uint8 byte strings, one per sponge; one `bytes` value for every
        sponge; or a sequence of n absorbables (sponge/absorb.py), one per sponge, that encode to the same number of elements."""
        import torch
        if isinstance(x, (bytes, bytearray)):
            b = torch.tensor(list(x), dtype=torch.uint8, device=self.device)
            N.check(N.lib.cpb_poseidon_duplex_absorb_bytes_dev(self._ctx(), self.states.data_ptr(), C.byref(self._mode),
                                                               b.data_ptr() if len(x) else None, len(x), 0, self.n, self._stream()))
            return
        if isinstance(x, (np.ndarray, torch.Tensor)) and x.dtype in (np.uint8, torch.uint8):
            b = torch.as_tensor(x).to(self.device).contiguous()
            if b.ndim != 2 or b.shape[0] != self.n:
                raise ValueError(f"byte strings must be (n={self.n}, L) uint8")
            L = b.shape[1]
            N.check(N.lib.cpb_poseidon_duplex_absorb_bytes_dev(self._ctx(), self.states.data_ptr(), C.byref(self._mode),
                                                               b.data_ptr() if L else None, L, L, self.n, self._stream()))
            return
        if isinstance(x, (np.ndarray, torch.Tensor)):
            e = _as_i64(x, self.device)
        else:
            from .absorb import to_sponge_field_elements
            items = list(x)
            if len(items) != self.n:
                raise ValueError(f"expected {self.n} absorbables, one per sponge (got {len(items)})")
            enc = [to_sponge_field_elements(v, self.parameters.field) for v in items]
            if len({a.shape[0] for a in enc}) > 1:
                raise ValueError("the items encode to different numbers of field elements; a batch absorbs one length "
                                 "(RaggedPoseidonSpongeBatch absorbs each at its own)")
            e = _as_i64(np.stack(enc) if enc else np.zeros((0, 0, 4), dtype=np.uint64), self.device)
        e = e.reshape(self.n, -1, 4).contiguous()
        k = e.shape[1]
        N.check(N.lib.cpb_poseidon_duplex_absorb_dev(self._ctx(), self.states.data_ptr(), C.byref(self._mode),
                                                     e.data_ptr() if k else None, k, self.n, self._stream()))

    def fork(self, domain) -> "PoseidonSpongeBatch":
        """R/sponge/mod.rs:145-153 for every sponge: clone, then absorb the byte string usize(len(domain)) || domain.  domain: one
        `bytes` value for every sponge or (n, L) uint8, one per sponge."""
        import torch
        new = self.clone()
        if isinstance(domain, (bytes, bytearray)):
            new.absorb(len(domain).to_bytes(8, "little") + bytes(domain))
            return new
        d = torch.as_tensor(domain).to(self.device, torch.uint8)
        if d.ndim != 2 or d.shape[0] != self.n:
            raise ValueError(f"domains must be (n={self.n}, L) uint8")
        prefix = torch.tensor(list(d.shape[1].to_bytes(8, "little")), dtype=torch.uint8, device=self.device).expand(self.n, 8)
        new.absorb(torch.cat([prefix, d], dim=1))
        return new

    # -- squeeze
    def _squeeze(self, m: int, canonical: bool):
        import torch
        out = torch.empty((self.n, m, 4), dtype=torch.int64, device=self.device)
        N.check(N.lib.cpb_poseidon_duplex_squeeze_dev(self._ctx(), self.states.data_ptr(), C.byref(self._mode),
                                                      out.data_ptr() if out.numel() else None, m, int(canonical), self.n,
                                                      self._stream()))
        return out

    def squeeze_native_field_elements(self, num_elements: int):
        """(n, num_elements, 4) Montgomery limbs (torch int64 on the device)."""
        return self._squeeze(num_elements, False)

    def squeeze_canonical(self, num_elements: int):
        """squeeze_native_field_elements as canonical integers: (n, num_elements, 4) little-endian limbs."""
        return self._squeeze(num_elements, True)

    def squeeze_bytes(self, num_bytes: int):
        """mod.rs:259-274: (n, num_bytes) uint8."""
        usable = (self.parameters.field.modulus_bit_size - 1) // 8
        m = (num_bytes + usable - 1) // usable
        c = self.squeeze_canonical(m).view(__import__("torch").uint8).reshape(self.n, m, 32)
        return c[:, :, :usable].reshape(self.n, m * usable)[:, :num_bytes]

    def squeeze_bits(self, num_bits: int):
        """mod.rs:276-291: (n, num_bits) bool."""
        import torch
        usable = self.parameters.field.modulus_bit_size - 1
        m = (num_bits + usable - 1) // usable
        c = self.squeeze_canonical(m).view(torch.uint8).reshape(self.n, m, 32)
        bits = (c[..., None] >> torch.arange(8, device=self.device, dtype=torch.uint8)) & 1
        return bits.reshape(self.n, m, 256)[:, :, :usable].reshape(self.n, m * usable)[:, :num_bits].bool()

    def squeeze_field_elements(self, num_elements: int, field: Field | None = None):
        """mod.rs:309-320: (n, num_elements, 4) Montgomery limbs of `field` (default: native)."""
        if field is None or field.id == self.parameters.field.id:
            return self.squeeze_native_field_elements(num_elements)
        return self.squeeze_field_elements_with_sizes([FULL] * num_elements, field)

    def squeeze_native_field_elements_with_sizes(self, sizes):
        return self.squeeze_field_elements_with_sizes(sizes, None)

    def squeeze_field_elements_with_sizes(self, sizes, field: Field | None = None):
        """mod.rs:291-307 over R/sponge/mod.rs:57-96 (PoseidonSponge.squeeze_field_elements_with_sizes for every sponge):
        (n, len(sizes), 4) Montgomery limbs of `field`, converted on the device."""
        import torch
        native = self.parameters.field
        field = native if field is None else field
        sizes = list(sizes)
        if field.modulus == native.modulus and all(s == FULL for s in sizes):
            return self.squeeze_native_field_elements(len(sizes))
        if not sizes:
            return torch.zeros((self.n, 0, 4), dtype=torch.int64, device=self.device)
        widths = []
        for s in sizes:
            if s == FULL:
                widths.append(field.modulus_bit_size - 1)
            elif s > field.modulus_bit_size:
                raise ValueError("num_bits is greater than the capacity of the field.")   # R/sponge/mod.rs:39-42
            else:
                widths.append(int(s))
        bits = self.squeeze_bits(sum(widths))
        S = len(sizes)
        padded = torch.zeros((self.n, S, 256), dtype=torch.int64, device=self.device)
        pos = 0
        for j, w in enumerate(widths):
            padded[:, j, :w] = bits[:, pos:pos + w]
            pos += w
        shifts = torch.arange(64, device=self.device, dtype=torch.int64)
        limbs = (padded.view(self.n, S, 4, 64) << shifts).sum(-1).contiguous()       # disjoint bits: the sum is the OR
        N.check(N.lib.cpb_field_to_montgomery_dev(field.id, self.device.index, limbs.data_ptr(), limbs.data_ptr(), self.n * S,
                                                  self._stream()))
        return limbs


class RaggedPoseidonSpongeBatch:
    """n independent PoseidonSponge over one PoseidonConfig, each with its own DuplexSpongeMode, so that every call can absorb or
    squeeze a different number of elements per sponge (transcripts whose messages, labels or challenge counts differ).  States are a
    torch CUDA int64 tensor (n, t, 4) of Montgomery limbs, modes an int64 tensor (n, 2) of [squeezing, index] rows (the
    cpb_sponge_mode layout), both on `device`.  Every call is one _dev call of the C-ABI (cpb_poseidon_duplex_*_ragged) on the current
    torch stream: the device sorts the sponges by their permutation count and runs every permutation of the call in one launch.
    Ragged data is (values, offsets): sponge i's part is values[offsets[i] .. offsets[i+1])."""

    def __init__(self, parameters: PoseidonConfig, n: int, device=None):
        import torch
        self.parameters = parameters
        self.n = int(n)
        self.device = _cuda_device(device)
        t = parameters.rate + parameters.capacity
        self.states = torch.zeros((self.n, t, 4), dtype=torch.int64, device=self.device)
        self.modes = torch.zeros((self.n, 2), dtype=torch.int64, device=self.device)

    # -- state
    @classmethod
    def from_batch(cls, batch: PoseidonSpongeBatch) -> "RaggedPoseidonSpongeBatch":
        """A copy of a PoseidonSpongeBatch: its states, and its one mode in every row."""
        b = cls(batch.parameters, batch.n, batch.device)
        b.states = batch.states.clone()
        b.modes[:, 0] = int(batch._mode.squeezing)
        b.modes[:, 1] = int(batch._mode.index)
        return b

    @classmethod
    def from_states(cls, states, modes, parameters: PoseidonConfig, device=None) -> "RaggedPoseidonSpongeBatch":
        """states (n, t, 4) Montgomery limbs and modes (n, 2) [squeezing, index] rows, torch or numpy."""
        dev = _cuda_device(device)
        st = _as_i64(states, dev)
        md = _as_i64(modes, dev)
        t = parameters.rate + parameters.capacity
        if st.ndim != 3 or tuple(st.shape[1:]) != (t, 4):
            raise ValueError(f"states must be (n, {t}, 4)")
        if tuple(md.shape) != (st.shape[0], 2):
            raise ValueError(f"modes must be (n={st.shape[0]}, 2)")
        b = cls(parameters, st.shape[0], st.device)
        b.states = st.clone()
        b.modes = md.clone()
        return b

    def into_states(self):
        return self.states, self.modes

    def clone(self) -> "RaggedPoseidonSpongeBatch":
        c = RaggedPoseidonSpongeBatch.__new__(RaggedPoseidonSpongeBatch)
        c.parameters, c.n, c.device = self.parameters, self.n, self.device
        c.states, c.modes = self.states.clone(), self.modes.clone()
        return c

    def sponge(self, i: int) -> PoseidonSponge:
        """Item i as an independent PoseidonSponge (host state) in its own mode."""
        st = self.states[i].cpu().numpy().view(np.uint64)
        sq, idx = (int(v) for v in self.modes[i].cpu())
        return PoseidonSponge.from_state((st, _py_mode(N.SpongeMode(sq & 0xFFFFFFFF, idx))), self.parameters, self.device.index)

    # -- internals
    def _call(self, fn, data, offsets, *args):
        import torch
        N.check(fn(self.parameters.context(self.device.index), self.states.data_ptr(), self.modes.data_ptr(),
                   data.data_ptr() if data.numel() else None, offsets.data_ptr(), *args, self.n,
                   torch.cuda.current_stream(self.device).cuda_stream))

    def _offsets(self, offsets):
        import torch
        if isinstance(offsets, np.ndarray):
            offsets = torch.from_numpy(np.ascontiguousarray(offsets, dtype=np.uint64).view(np.int64))
        off = torch.as_tensor(offsets, dtype=torch.int64).to(self.device).reshape(-1).contiguous()
        if off.shape[0] != self.n + 1:
            raise ValueError(f"offsets needs n + 1 = {self.n + 1} entries (got {off.shape[0]})")
        return off

    def _pack(self, parts, dtype):
        """Per-item parts -> (values, offsets) on the device."""
        import torch
        if len(parts) != self.n:
            raise ValueError(f"expected {self.n} items, one per sponge (got {len(parts)})")
        off = np.zeros(self.n + 1, dtype=np.int64)
        np.cumsum([len(x) for x in parts], out=off[1:])
        vals = np.concatenate(parts) if parts else np.zeros((0,), dtype=dtype)
        return torch.from_numpy(np.ascontiguousarray(vals).view(np.int64 if dtype == np.uint64 else np.uint8)).to(self.device), \
            torch.from_numpy(off).to(self.device)

    # -- absorb
    def absorb(self, x):
        """x: a (values (S, 4), offsets (n + 1)) tuple of Montgomery limbs, torch or numpy; or a list of n items, one per sponge, each a
        (L_i, 4) limb array or any absorbable of sponge/absorb.py, encoded at its own length."""
        import torch
        if isinstance(x, tuple):
            values, offsets = x
            v = _as_i64(values, self.device).reshape(-1, 4)
            off = self._offsets(offsets)
        else:
            from .absorb import to_sponge_field_elements
            parts = []
            for item in x:
                if isinstance(item, torch.Tensor):
                    item = item.cpu().numpy()
                if isinstance(item, np.ndarray) and item.dtype in (np.uint64, np.int64) and item.ndim == 2 and item.shape[1] == 4:
                    parts.append(np.ascontiguousarray(item).view(np.uint64))
                else:
                    parts.append(to_sponge_field_elements(item, self.parameters.field))
            v, off = self._pack([p.reshape(-1, 4) for p in parts], np.uint64)
            v = v.reshape(-1, 4)
        self._call(N.lib.cpb_poseidon_duplex_absorb_ragged_dev, v, off)

    def absorb_bytes(self, x):
        """x: a list of n `bytes`, one [u8] value per sponge, or a (uint8 values, offsets (n + 1)) tuple."""
        import torch
        if isinstance(x, tuple):
            values, offsets = x
            b = torch.as_tensor(values).to(self.device, torch.uint8).reshape(-1).contiguous()
            off = self._offsets(offsets)
        else:
            b, off = self._pack([np.frombuffer(bytes(s), dtype=np.uint8) for s in x], np.uint8)
        self._call(N.lib.cpb_poseidon_duplex_absorb_bytes_ragged_dev, b, off)

    def fork(self, domains) -> "RaggedPoseidonSpongeBatch":
        """R/sponge/mod.rs:145-153 for every sponge with its own domain: clone, then sponge i absorbs the byte string
        usize(len(domains[i])) || domains[i]."""
        new = self.clone()
        new.absorb_bytes([len(d).to_bytes(8, "little") + bytes(d) for d in domains])
        return new

    # -- squeeze
    def _squeeze(self, counts, canonical: bool):
        import torch
        if isinstance(counts, int):
            if counts < 0:
                raise ValueError("counts must not be negative")
            off = torch.arange(self.n + 1, dtype=torch.int64, device=self.device) * counts
            total = self.n * counts
        else:
            c = torch.as_tensor(counts, dtype=torch.int64).to(self.device).reshape(-1)
            if c.shape[0] != self.n:
                raise ValueError(f"expected {self.n} counts (got {c.shape[0]})")
            if self.n and int(c.min()) < 0:
                raise ValueError("counts must not be negative")
            off = torch.zeros(self.n + 1, dtype=torch.int64, device=self.device)
            torch.cumsum(c, 0, out=off[1:])
            total = int(off[-1]) if self.n else 0
        out = torch.empty((total, 4), dtype=torch.int64, device=self.device)
        self._call(N.lib.cpb_poseidon_duplex_squeeze_ragged_dev, out, off, int(canonical))
        return out, off

    def squeeze_native_field_elements(self, counts):
        """Sponge i squeezes counts[i] (or counts, an int, for all) native elements: (values (S, 4) Montgomery limbs, offsets (n + 1)),
        torch int64 on the device; sponge i's are values[offsets[i] .. offsets[i+1])."""
        return self._squeeze(counts, False)

    def squeeze_canonical(self, counts):
        """squeeze_native_field_elements as canonical integers (little-endian limbs)."""
        return self._squeeze(counts, True)


def _cuda_device(device):
    import torch
    if device is None:
        return torch.device("cuda", torch.cuda.current_device())
    if isinstance(device, int):
        return torch.device("cuda", device)
    d = torch.device(device)
    if d.type != "cuda":
        raise ValueError("PoseidonSpongeBatch keeps its states on a CUDA device")
    return torch.device("cuda", torch.cuda.current_device() if d.index is None else d.index)


def _as_i64(x, device):
    """Montgomery limbs (numpy uint64/int64 or torch int64) -> contiguous torch int64 on `device`."""
    import torch
    if isinstance(x, np.ndarray):
        x = torch.from_numpy(np.ascontiguousarray(x, dtype=np.uint64).view(np.int64))
    if x.dtype != torch.int64:
        raise TypeError("field elements are int64 (or uint64) limbs")
    return x.to(device).contiguous()


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
