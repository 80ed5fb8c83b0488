"""commitment::blake2s::Commitment -- host mirror of R/commitment/blake2s/mod.rs over the CUDA library:
commit(input, r) = Blake2s256(input || r), r of 32 bytes, hashed on the GPU one input per thread."""
from __future__ import annotations

import numpy as np

from .. import _native as N
from ..signature.schnorr import _torch_stream, _u8, _u64, pack_messages


class Commitment:
    """CommitmentScheme{Parameters=(), Randomness=[u8; 32], Output=[u8; 32]} (mod.rs:11-33)."""

    @staticmethod
    def setup(rng=None):
        return None

    @staticmethod
    def commit(parameters, input, r, device: int = 0) -> bytes:
        return Commitment.commit_batch(parameters, [input], [r], device)[0].tobytes()

    @staticmethod
    def commit_batch(parameters, inputs, randomness, device: int = 0) -> np.ndarray:
        """inputs: n byte strings of any lengths; randomness: n x 32 bytes (list or (n, 32) uint8) -> (n, 32) uint8."""
        values, offsets = pack_messages(inputs)
        n = offsets.size - 1
        rnd = np.ascontiguousarray(np.frombuffer(b"".join(bytes(r) for r in randomness), dtype=np.uint8)
                                   if not isinstance(randomness, np.ndarray) else randomness, dtype=np.uint8).reshape(-1)
        assert rnd.size == 32 * n, "randomness is [u8; 32] per input"
        out = np.empty((n, 32), dtype=np.uint8)
        N.check(N.lib.cpb_blake2s_commit_batch(device, _u8(values), _u64(offsets), _u8(rnd), _u8(out), n))
        return out

    @staticmethod
    def commit_dev(values, offsets, randomness, out=None):
        """torch CUDA tensors: values uint8, offsets (n + 1) int64, randomness (n, 32) uint8 -> (n, 32) uint8."""
        import torch
        n = offsets.shape[0] - 1
        out = torch.empty((n, 32), dtype=torch.uint8, device=values.device) if out is None else out
        N.check(N.lib.cpb_blake2s_commit_batch_dev(values.device.index, values.data_ptr(), offsets.data_ptr(), randomness.data_ptr(),
                                                   out.data_ptr(), n, _torch_stream()))
        return out
