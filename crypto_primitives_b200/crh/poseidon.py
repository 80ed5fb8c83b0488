"""crh::poseidon::{CRH, TwoToOneCRH} -- host mirror of R/crh/poseidon/mod.rs:15-80 over the CUDA
library.  Inputs/outputs are Montgomery limb arrays (numpy uint64 (..., 4)); `*_dev` variants take
torch CUDA tensors (int64 (..., 4)) and launch on the current torch stream."""
from __future__ import annotations

import numpy as np

from .. import _native as N
from .. import ragged as R
from ..sponge.poseidon import PoseidonConfig


def _p(a: np.ndarray):
    return a.ctypes.data_as(N.u64p)


def _stream_ptr():
    import torch
    return torch.cuda.current_stream().cuda_stream


class CRH:
    """CRHScheme{Input=[F], Output=F, Parameters=PoseidonConfig<F>} (mod.rs:19-41)."""

    @staticmethod
    def setup(rng=None):
        # mod.rs:24-28: unimplemented!() -- parameters must be supplied by the caller
        raise NotImplementedError("automatic generation of parameters are not implemented yet")

    @staticmethod
    def evaluate(parameters: PoseidonConfig, input, device: int = 0) -> np.ndarray:
        inp = np.ascontiguousarray(input, dtype=np.uint64).reshape(-1, 4)
        return CRH.evaluate_batch(parameters, inp.reshape(1, inp.shape[0], 4), device)[0]

    @staticmethod
    def evaluate_batch(parameters: PoseidonConfig, inputs, device: int = 0) -> np.ndarray:
        """inputs (n, len, 4) -> (n, 4).  A list of (L_i, 4) arrays whose lengths differ is hashed as a ragged batch, each input at
        its own length (evaluate_ragged)."""
        if R.is_ragged(inputs):
            return CRH.evaluate_ragged(parameters, *R.pack(inputs), device)
        inp = np.ascontiguousarray(inputs, dtype=np.uint64)
        assert inp.ndim == 3 and inp.shape[2] == 4
        n, ln = inp.shape[0], inp.shape[1]
        out = np.empty((n, 4), dtype=np.uint64)
        N.check(N.lib.cpb_poseidon_crh_batch(parameters.context(device), _p(inp), ln, _p(out), n))
        return out

    @staticmethod
    def evaluate_batch_dev(parameters: PoseidonConfig, inputs, out=None):
        import torch
        assert inputs.is_cuda and inputs.is_contiguous() and inputs.dtype == torch.int64 and inputs.shape[-1] == 4
        n, ln = inputs.shape[0], inputs.shape[1]
        if out is None:
            out = torch.empty((n, 4), dtype=torch.int64, device=inputs.device)
        N.check(N.lib.cpb_poseidon_crh_batch_dev(parameters.context(inputs.device.index), inputs.data_ptr(), ln,
                                                 out.data_ptr(), n, _stream_ptr()))
        return out

    @staticmethod
    def evaluate_ragged(parameters: PoseidonConfig, values, offsets, device: int = 0) -> np.ndarray:
        """n = len(offsets) - 1 inputs of different lengths: input i = values[offsets[i] .. offsets[i+1]) -> (n, 4).
        Offsets that decrease raise ValueError."""
        vals, off = R.as_arrays(values, offsets)
        n = off.shape[0] - 1
        out = np.empty((n, 4), dtype=np.uint64)
        if n:
            R.check(N.lib.cpb_poseidon_crh_ragged_batch(parameters.context(device), _p(vals), _p(off), _p(out), n))
        return out

    @staticmethod
    def evaluate_ragged_dev(parameters: PoseidonConfig, values, offsets, out=None):
        """evaluate_ragged on torch CUDA tensors (values int64 (m, 4), offsets int64 (n + 1,)), on the current stream.  The
        offsets are not checked: they must not decrease (a decreasing pair hashes as an empty input)."""
        import torch
        assert values.is_cuda and values.is_contiguous() and values.dtype == torch.int64 and values.shape[-1] == 4
        assert offsets.is_cuda and offsets.is_contiguous() and offsets.dtype == torch.int64 and offsets.dim() == 1
        assert offsets.device == values.device
        n = offsets.numel() - 1
        if out is None:
            out = torch.empty((n, 4), dtype=torch.int64, device=values.device)
        R.check(N.lib.cpb_poseidon_crh_ragged_batch_dev(parameters.context(values.device.index), values.data_ptr(), offsets.data_ptr(),
                                                        out.data_ptr(), n, _stream_ptr()))
        return out


class TwoToOneCRH:
    """TwoToOneCRHScheme{Input=F, Output=F} (mod.rs:47-80); evaluate is an alias of compress (:58-64)."""

    @staticmethod
    def setup(rng=None):
        raise NotImplementedError("automatic generation of parameters are not implemented yet")

    @staticmethod
    def compress(parameters: PoseidonConfig, left_input, right_input, device: int = 0) -> np.ndarray:
        pair = np.stack([np.asarray(left_input, dtype=np.uint64).reshape(4),
                         np.asarray(right_input, dtype=np.uint64).reshape(4)])[None]
        return TwoToOneCRH.compress_batch(parameters, pair, device)[0]

    evaluate = compress

    @staticmethod
    def compress_batch(parameters: PoseidonConfig, pairs, device: int = 0) -> np.ndarray:
        """pairs (n, 2, 4) -> (n, 4)."""
        pr = np.ascontiguousarray(pairs, dtype=np.uint64)
        assert pr.ndim == 3 and pr.shape[1:] == (2, 4)
        out = np.empty((pr.shape[0], 4), dtype=np.uint64)
        N.check(N.lib.cpb_poseidon_compress_batch(parameters.context(device), _p(pr), _p(out), pr.shape[0]))
        return out

    evaluate_batch = compress_batch

    @staticmethod
    def compress_batch_dev(parameters: PoseidonConfig, pairs, out=None):
        import torch
        assert pairs.is_cuda and pairs.is_contiguous() and pairs.dtype == torch.int64
        n = pairs.numel() // 8
        if out is None:
            out = torch.empty((n, 4), dtype=torch.int64, device=pairs.device)
        N.check(N.lib.cpb_poseidon_compress_batch_dev(parameters.context(pairs.device.index), pairs.data_ptr(),
                                                      out.data_ptr(), n, _stream_ptr()))
        return out


def permute_batch(parameters: PoseidonConfig, states, device: int = 0) -> np.ndarray:
    """n bare permutations (PoseidonSponge::permute, R/sponge/poseidon/mod.rs:98-121): (n, t, 4) -> (n, t, 4)."""
    st = np.ascontiguousarray(states, dtype=np.uint64)
    t = parameters.rate + parameters.capacity
    assert st.ndim == 3 and st.shape[1:] == (t, 4)
    out = np.empty_like(st)
    N.check(N.lib.cpb_poseidon_permute_batch(parameters.context(device), _p(st), _p(out), st.shape[0]))
    return out
