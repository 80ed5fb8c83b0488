"""signature::schnorr::{Parameters, Schnorr} -- host mirror of R/signature/schnorr/mod.rs over the CUDA library, for
Schnorr<EdwardsProjective, Blake2s256> over Jubjub, the instantiation of the reference's tests (R/signature/mod.rs:52-105), and
over ed-on-BLS12-377, the curve of the reference's signature benchmark (R/benches/signature.rs:5-10); `Parameters.curve` picks it.

Scalars (secret keys, nonces, s and e) are elements of the curve's scalar field as Montgomery limbs, numpy uint64 (..., 4)
(`parameters.curve.scalar_field.elements` converts Python ints); points are affine Montgomery limbs (..., 2, 4); a signature is (prover_response, verifier_challenge),
(..., 2, 4).  The single-item functions keep the trait signatures; the `*_batch` forms are the GPU path.  The `*_dev` forms take
torch CUDA tensors (int64 views of the same layouts) and run asynchronously on the current torch stream.
Signing is not constant time: secret scalars select table entries by value, as the reference's `mul` does.
"""
from __future__ import annotations

import ctypes as C
import weakref
from dataclasses import dataclass, field as _f

import numpy as np

from .. import _native as N
from ..curves import JUBJUB, TECurve


def _u8(a):
    return a.ctypes.data_as(N.u8p)


def _u64(a):
    return a.ctypes.data_as(N.u64p)


class _Ctx:
    def __init__(self, handle):
        self.handle = handle

    def __del__(self):
        try:
            if self.handle:
                N.lib.cpb_te_base_ctx_destroy(self.handle)
                self.handle = None
        except Exception:
            pass


# One device context (about 0.4 GB of fixed-base tables) per (curve, generator, device), shared by every Parameters object with
# that generator -- Schnorr parameters that differ only in the salt, and ElGamal parameters over the same generator.  Held
# weakly: the tables are freed when the last Parameters object using them goes.
_CONTEXTS: "weakref.WeakValueDictionary" = weakref.WeakValueDictionary()


@dataclass(eq=False)
class BaseParameters:
    """A generator (2, 4) and its device tables (cpb_te_base_ctx), shared by Schnorr and ElGamal."""
    generator: np.ndarray
    curve: TECurve = JUBJUB
    _ctx: dict = _f(default_factory=dict, repr=False)

    def __post_init__(self):
        self.generator = np.ascontiguousarray(np.asarray(self.generator, dtype=np.uint64).reshape(2, 4))

    def context(self, device: int = 0):
        h = self._ctx.get(device)
        if h is None:
            key = (self.curve.id, self.generator.tobytes(), device)
            h = _CONTEXTS.get(key)
            if h is None:
                out = N.vp()
                N.check(N.lib.cpb_te_base_ctx_create_ex(self.curve.id, _u64(self.generator), device, C.byref(out)))
                h = _Ctx(out.value)
                _CONTEXTS[key] = h
            self._ctx[device] = h
        return h.handle


@dataclass(eq=False)
class Parameters(BaseParameters):
    """schnorr::Parameters{generator, salt} (mod.rs:24-29)."""
    salt: bytes = bytes(32)

    def __post_init__(self):
        super().__post_init__()
        assert len(self.salt) == 32, "salt is [u8; 32]"
        self.salt = bytes(self.salt)

    def salt_arg(self):
        return (C.c_uint8 * 32).from_buffer_copy(self.salt)


def pack_messages(messages):
    """A list of byte strings -> (values uint8, offsets uint64[n+1]): message i = values[offsets[i]:offsets[i+1]]."""
    msgs = [bytes(m) for m in messages]
    offsets = np.zeros(len(msgs) + 1, dtype=np.uint64)
    offsets[1:] = np.cumsum([len(m) for m in msgs], dtype=np.uint64) if msgs else []
    values = np.frombuffer(b"".join(msgs) + b"\0", dtype=np.uint8)     # never empty, so the pointer is valid
    return values, offsets


def _scalars(a, n=None) -> np.ndarray:
    s = np.ascontiguousarray(np.asarray(a, dtype=np.uint64).reshape(-1, 4))
    assert n is None or s.shape[0] == n
    return s


def _points(a, n=None) -> np.ndarray:
    p = np.ascontiguousarray(np.asarray(a, dtype=np.uint64).reshape(-1, 2, 4))
    assert n is None or p.shape[0] == n
    return p


def _randomness(randomness):
    """A list of equal-length byte strings, or a (n, len) uint8 array -> (array, len)."""
    if isinstance(randomness, np.ndarray):
        r = np.ascontiguousarray(randomness, dtype=np.uint8)
    else:
        rows = [bytes(x) for x in randomness]
        assert len({len(x) for x in rows}) <= 1, "one randomness length per batch"
        ln = len(rows[0]) if rows else 0
        r = np.frombuffer(b"".join(rows), dtype=np.uint8).reshape(len(rows), ln).copy()
    assert r.ndim == 2
    return np.ascontiguousarray(np.concatenate([r.reshape(-1), np.zeros(1, dtype=np.uint8)])), r.shape[1]


def base_mul_batch(parameters: BaseParameters, scalars, device: int = 0) -> np.ndarray:
    """scalars (n, 4) Fr Montgomery -> (n, 2, 4) affine scalar * generator."""
    s = _scalars(scalars)
    out = np.empty((s.shape[0], 2, 4), dtype=np.uint64)
    N.check(N.lib.cpb_te_base_mul_batch(parameters.context(device), _u64(s), _u64(out), s.shape[0]))
    return out


def _torch_stream():
    import torch
    return torch.cuda.current_stream().cuda_stream


class Schnorr:
    """SignatureScheme for Schnorr<C, Blake2s256> (mod.rs:40-183), C = Jubjub or ed-on-BLS12-377."""

    @staticmethod
    def setup(rng, curve: TECurve = JUBJUB) -> Parameters:
        """mod.rs:48-63: a 32-byte salt, then a random generator (`rng`: .bytes(n) and .field(q), e.g. oracle SplitMix64)."""
        salt = rng.bytes(32)
        G = curve.random_point(rng)
        return Parameters(curve.base_field.elements(list(G)).reshape(2, 4), curve, salt=salt)

    @staticmethod
    def keygen(parameters: Parameters, rng, device: int = 0):
        """mod.rs:65-78 -> (public_key (2, 4), secret_key (4,))."""
        sk = parameters.curve.scalar_field.elements([rng.field(parameters.curve.scalar_modulus)])
        return Schnorr.keygen_batch(parameters, sk, device)[0], sk[0]

    @staticmethod
    def keygen_batch(parameters: Parameters, secret_keys, device: int = 0) -> np.ndarray:
        return base_mul_batch(parameters, secret_keys, device)

    @staticmethod
    def sign(parameters: Parameters, sk, message, rng, device: int = 0) -> np.ndarray:
        """mod.rs:80-115 -> signature (2, 4)."""
        return Schnorr.sign_batch(parameters, _scalars(sk), [message], rng, device)[0]

    @staticmethod
    def sign_batch(parameters: Parameters, secret_keys, messages, rng, device: int = 0) -> np.ndarray:
        """The reference's loop, per batch: nonces are drawn from `rng` and redrawn for the items whose challenge was not a
        field element until every item is signed."""
        sks = _scalars(secret_keys)
        n = sks.shape[0]
        msgs = [bytes(m) for m in messages]
        assert len(msgs) == n
        sigs = np.zeros((n, 2, 4), dtype=np.uint64)
        todo = np.arange(n)
        r = parameters.curve.scalar_modulus
        while todo.size:
            nonces = parameters.curve.scalar_field.elements([rng.field(r) for _ in range(todo.size)])
            s, ok = Schnorr.sign_with_nonces_batch(parameters, sks[todo], nonces, [msgs[i] for i in todo], device)
            sigs[todo[ok]] = s[ok]
            todo = todo[~ok]
        return sigs

    @staticmethod
    def sign_with_nonces_batch(parameters: Parameters, secret_keys, nonces, messages, device: int = 0):
        """One iteration of the signing loop per item with the given nonce -> (signatures (n, 2, 4), signed (n,) bool).
        signed[i] is False when the challenge of nonce i is not a field element; that signature is zero."""
        sks = _scalars(secret_keys)
        n = sks.shape[0]
        k = _scalars(nonces, n)
        values, offsets = pack_messages(messages)
        assert offsets.size == n + 1
        sigs = np.empty((n, 2, 4), dtype=np.uint64)
        ok = np.empty(n, dtype=np.uint8)
        N.check(N.lib.cpb_schnorr_sign_batch(parameters.context(device), parameters.salt_arg(), _u64(sks), _u64(k), _u8(values),
                                             _u64(offsets), _u64(sigs), _u8(ok), n))
        return sigs, ok.astype(bool)

    @staticmethod
    def verify(parameters: Parameters, pk, message, signature, device: int = 0) -> bool:
        """mod.rs:117-148."""
        return bool(Schnorr.verify_batch(parameters, _points(pk), [message], np.asarray(signature).reshape(1, 2, 4), device)[0])

    @staticmethod
    def verify_batch(parameters: Parameters, public_keys, messages, signatures, device: int = 0) -> np.ndarray:
        pks = _points(public_keys)
        n = pks.shape[0]
        sigs = _points(signatures, n)
        values, offsets = pack_messages(messages)
        assert offsets.size == n + 1
        ok = np.empty(n, dtype=np.uint8)
        N.check(N.lib.cpb_schnorr_verify_batch(parameters.context(device), parameters.salt_arg(), _u64(pks), _u8(values), _u64(offsets),
                                               _u64(sigs), _u8(ok), n))
        return ok.astype(bool)

    @staticmethod
    def randomize_public_key(parameters: Parameters, public_key, randomness, device: int = 0) -> np.ndarray:
        """mod.rs:150-174."""
        return Schnorr.randomize_public_key_batch(parameters, _points(public_key), [bytes(randomness)], device)[0]

    @staticmethod
    def randomize_public_key_batch(parameters: Parameters, public_keys, randomness, device: int = 0) -> np.ndarray:
        """randomness: n byte strings of one length, or (n, len) uint8."""
        pks = _points(public_keys)
        n = pks.shape[0]
        rnd, ln = _randomness(randomness)
        out = np.empty((n, 2, 4), dtype=np.uint64)
        N.check(N.lib.cpb_schnorr_randomize_public_key_batch(parameters.context(device), _u64(pks), _u8(rnd), ln, ln, _u64(out), n))
        return out

    @staticmethod
    def randomize_signature(parameters: Parameters, signature, randomness, device: int = 0) -> np.ndarray:
        """mod.rs:176-198."""
        return Schnorr.randomize_signature_batch(parameters, np.asarray(signature).reshape(1, 2, 4), [bytes(randomness)], device)[0]

    @staticmethod
    def randomize_signature_batch(parameters: Parameters, signatures, randomness, device: int = 0) -> np.ndarray:
        sigs = _points(signatures)
        n = sigs.shape[0]
        rnd, ln = _randomness(randomness)
        out = np.empty((n, 2, 4), dtype=np.uint64)
        N.check(N.lib.cpb_schnorr_randomize_signature_batch(parameters.context(device), _u64(sigs), _u8(rnd), ln, ln, _u64(out), n))
        return out

    # ---- torch CUDA tensors (device-pointer forms, asynchronous on the current stream)
    @staticmethod
    def keygen_dev(parameters: Parameters, secret_keys, out=None):
        """secret_keys: (n, 4) int64 CUDA tensor -> (n, 2, 4)."""
        import torch
        n = secret_keys.shape[0]
        out = torch.empty((n, 2, 4), dtype=torch.int64, device=secret_keys.device) if out is None else out
        N.check(N.lib.cpb_te_base_mul_batch_dev(parameters.context(secret_keys.device.index), secret_keys.data_ptr(), out.data_ptr(), n,
                                                _torch_stream()))
        return out

    @staticmethod
    def sign_with_nonces_dev(parameters: Parameters, secret_keys, nonces, values, offsets, sigs_out=None, signed_out=None):
        """values: uint8 CUDA tensor of the messages back to back, offsets: (n + 1) int64 -> (sigs (n, 2, 4), signed (n,) uint8)."""
        import torch
        n = secret_keys.shape[0]
        dev = secret_keys.device
        sigs_out = torch.empty((n, 2, 4), dtype=torch.int64, device=dev) if sigs_out is None else sigs_out
        signed_out = torch.empty(n, dtype=torch.uint8, device=dev) if signed_out is None else signed_out
        N.check(N.lib.cpb_schnorr_sign_batch_dev(parameters.context(dev.index), parameters.salt_arg(), secret_keys.data_ptr(), nonces.data_ptr(),
                                                 values.data_ptr(), offsets.data_ptr(), sigs_out.data_ptr(), signed_out.data_ptr(), n,
                                                 _torch_stream()))
        return sigs_out, signed_out

    @staticmethod
    def verify_dev(parameters: Parameters, public_keys, values, offsets, signatures, ok_out=None):
        import torch
        n = public_keys.shape[0]
        ok_out = torch.empty(n, dtype=torch.uint8, device=public_keys.device) if ok_out is None else ok_out
        N.check(N.lib.cpb_schnorr_verify_batch_dev(parameters.context(public_keys.device.index), parameters.salt_arg(), public_keys.data_ptr(),
                                                   values.data_ptr(), offsets.data_ptr(), signatures.data_ptr(), ok_out.data_ptr(), n,
                                                   _torch_stream()))
        return ok_out

    @staticmethod
    def randomize_public_key_dev(parameters: Parameters, public_keys, randomness, out=None):
        """randomness: (n, len) uint8 CUDA tensor."""
        import torch
        n, ln = public_keys.shape[0], randomness.shape[1]
        out = torch.empty((n, 2, 4), dtype=torch.int64, device=public_keys.device) if out is None else out
        N.check(N.lib.cpb_schnorr_randomize_public_key_batch_dev(parameters.context(public_keys.device.index), public_keys.data_ptr(),
                                                                 randomness.data_ptr(), ln, randomness.stride(0), out.data_ptr(), n,
                                                                 _torch_stream()))
        return out

    @staticmethod
    def randomize_signature_dev(parameters: Parameters, signatures, randomness, out=None):
        import torch
        n, ln = signatures.shape[0], randomness.shape[1]
        out = torch.empty((n, 2, 4), dtype=torch.int64, device=signatures.device) if out is None else out
        N.check(N.lib.cpb_schnorr_randomize_signature_batch_dev(parameters.context(signatures.device.index), signatures.data_ptr(),
                                                                randomness.data_ptr(), ln, randomness.stride(0), out.data_ptr(), n,
                                                                _torch_stream()))
        return out
