"""encryption::elgamal::{Parameters, ElGamal} -- host mirror of R/encryption/elgamal/mod.rs over the CUDA library, for
ElGamal<EdwardsProjective (Jubjub)> (the reference's test curve, mod.rs:102-128).

Layouts as in signature/schnorr.py: scalars (..., 4) Fr Montgomery limbs, points (..., 2, 4) affine Montgomery limbs, a
ciphertext (c1, c2) is (..., 2, 2, 4).  The `*_dev` forms take torch CUDA int64 tensors on the current stream."""
from __future__ import annotations

import numpy as np

from .. import _native as N
from ..curves import JUBJUB, TECurve
from ..fields import JUBJUB_FR
from ..signature.schnorr import BaseParameters, _points, _scalars, _torch_stream, _u64, base_mul_batch


class Parameters(BaseParameters):
    """elgamal::Parameters{generator} (mod.rs:14-16)."""


class ElGamal:
    """AsymmetricEncryptionScheme for ElGamal<C> (mod.rs:34-101)."""

    @staticmethod
    def setup(rng, curve: TECurve = JUBJUB) -> Parameters:
        """mod.rs:47-53 (`rng`: .field(q))."""
        G = curve.random_point(rng)
        return Parameters(curve.base_field.elements(list(G)).reshape(2, 4), curve)

    @staticmethod
    def keygen(parameters: Parameters, rng, device: int = 0):
        """mod.rs:55-67 -> (public_key (2, 4), secret_key (4,))."""
        sk = JUBJUB_FR.elements([rng.field(parameters.curve.scalar_modulus)])
        return base_mul_batch(parameters, sk, device)[0], sk[0]

    @staticmethod
    def keygen_batch(parameters: Parameters, secret_keys, device: int = 0) -> np.ndarray:
        return base_mul_batch(parameters, secret_keys, device)

    @staticmethod
    def encrypt(parameters: Parameters, pk, message, r, device: int = 0) -> np.ndarray:
        """mod.rs:69-84 -> (c1, c2) (2, 2, 4)."""
        return ElGamal.encrypt_batch(parameters, _points(pk), _points(message), _scalars(r), device)[0]

    @staticmethod
    def encrypt_batch(parameters: Parameters, public_keys, messages, randomness, device: int = 0) -> np.ndarray:
        pks = _points(public_keys)
        n = pks.shape[0]
        ms = _points(messages, n)
        rs = _scalars(randomness, n)
        out = np.empty((n, 2, 2, 4), dtype=np.uint64)
        N.check(N.lib.cpb_elgamal_encrypt_batch(parameters.context(device), _u64(pks), _u64(ms), _u64(rs), _u64(out), n))
        return out

    @staticmethod
    def decrypt(parameters: Parameters, sk, ciphertext, device: int = 0) -> np.ndarray:
        """mod.rs:86-101."""
        return ElGamal.decrypt_batch(parameters, _scalars(sk), np.asarray(ciphertext).reshape(1, 2, 2, 4), device)[0]

    @staticmethod
    def decrypt_batch(parameters: Parameters, secret_keys, ciphertexts, device: int = 0) -> np.ndarray:
        sks = _scalars(secret_keys)
        n = sks.shape[0]
        cts = np.ascontiguousarray(np.asarray(ciphertexts, dtype=np.uint64).reshape(n, 2, 2, 4))
        out = np.empty((n, 2, 4), dtype=np.uint64)
        N.check(N.lib.cpb_elgamal_decrypt_batch(parameters.context(device), _u64(sks), _u64(cts), _u64(out), n))
        return out

    @staticmethod
    def encrypt_dev(parameters: Parameters, public_keys, messages, randomness, out=None):
        import torch
        n = public_keys.shape[0]
        out = torch.empty((n, 2, 2, 4), dtype=torch.int64, device=public_keys.device) if out is None else out
        N.check(N.lib.cpb_elgamal_encrypt_batch_dev(parameters.context(public_keys.device.index), public_keys.data_ptr(), messages.data_ptr(),
                                                    randomness.data_ptr(), out.data_ptr(), n, _torch_stream()))
        return out

    @staticmethod
    def decrypt_dev(parameters: Parameters, secret_keys, ciphertexts, out=None):
        import torch
        n = secret_keys.shape[0]
        out = torch.empty((n, 2, 4), dtype=torch.int64, device=secret_keys.device) if out is None else out
        N.check(N.lib.cpb_elgamal_decrypt_batch_dev(parameters.context(secret_keys.device.index), secret_keys.data_ptr(), ciphertexts.data_ptr(),
                                                    out.data_ptr(), n, _torch_stream()))
        return out
