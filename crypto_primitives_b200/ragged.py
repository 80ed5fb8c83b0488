"""Ragged batches: n inputs of different lengths as one flat `values` array and n + 1 `offsets` (include/cpb200.h, "Poseidon
over inputs of different lengths").  Input i is values[offsets[i] .. offsets[i+1]); offsets[0] need not be 0."""
from __future__ import annotations

import numpy as np

from . import _native as N


def is_ragged(inputs) -> bool:
    """True for a list or tuple of inputs whose lengths differ -- what no (n, len, 4) array can hold.  Arrays and equal-length
    sequences are not ragged and keep taking the uniform calls."""
    if isinstance(inputs, np.ndarray) or not isinstance(inputs, (list, tuple)) or len(inputs) < 2:
        return False
    try:
        n0 = len(inputs[0])
        return any(len(x) != n0 for x in inputs)
    except TypeError:
        return False


def pack(inputs):
    """A sequence of (L_i, 4) Montgomery limb arrays -> (values (sum L_i, 4), offsets (n + 1,)), both uint64."""
    parts = [np.asarray(x, dtype=np.uint64).reshape(-1, 4) for x in inputs]
    offsets = np.zeros(len(parts) + 1, dtype=np.uint64)
    np.cumsum([p.shape[0] for p in parts], out=offsets[1:])
    values = np.concatenate(parts) if parts else np.zeros((0, 4), dtype=np.uint64)
    return np.ascontiguousarray(values, dtype=np.uint64), offsets


def as_arrays(values, offsets):
    """Contiguous uint64 views of a caller's (values, offsets) pair, with the bounds a host call relies on checked: offsets[n]
    must lie inside `values` (whether offsets decrease is the library's check, CPB_BAD_LENGTH)."""
    vals = np.ascontiguousarray(values, dtype=np.uint64).reshape(-1, 4)
    off = np.ascontiguousarray(offsets, dtype=np.uint64).reshape(-1)
    if off.shape[0] < 1:
        raise ValueError("offsets needs n + 1 entries")
    if off.shape[0] > 1 and int(off.max()) > vals.shape[0]:
        raise ValueError(f"offsets reach element {int(off.max())} of {vals.shape[0]} values")
    return vals, off


def check(status: int):
    """N.check, with CPB_BAD_LENGTH (offsets that decrease) raised as ValueError like every other malformed input."""
    try:
        N.check(status)
    except N.CpbError as e:
        if e.status == N.CPB_BAD_LENGTH:
            raise ValueError(str(e)) from e
        raise
