"""Ragged duplex calls without a GPU: the per-sponge step of csrc/poseidon_duplex.cuh (duplex_ragged_step / duplex_ragged_key, which
the kernel, the ordering and the host all run) against the instrumented oracle sponge, an emulated ragged call (the ordering, then
the kernel's per-sponge body pos_duplex_ragged with the real permutation) against independent oracle sponges in any order, invalid
per-sponge modes, the argument rules of the cpb_poseidon_duplex_*_ragged entry points that need no device, and the cpb_sponge_mode
layout."""
import ctypes as C
import random

import numpy as np
import pytest

from helpers import build_host_shim
import crypto_primitives_b200 as cp
from crypto_primitives_b200 import _native as N
from crypto_primitives_b200.sponge import absorb as A
from oracle import poseidon as OP
from test_poseidon_duplex_host import P61, Traced, replay

lp = C.POINTER(C.c_long)
KABSORB, KBYTES, KSQUEEZE, KCANON = range(4)
BUCKETS = 64


@pytest.fixture(scope="module")
def shim():
    lib = build_host_shim("poseidon_duplex_ragged_shim")
    lib.host_duplex_ragged_step.argtypes = [C.c_int, N.u64p, N.u64p, C.c_long, C.c_long, C.c_uint64, C.c_long, lp]
    lib.host_duplex_ragged_run.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_ulonglong, N.u64p, N.u64p, N.u64p, N.u64p,
                                           C.c_long, C.c_int, C.c_void_p, N.u64p, C.c_uint64, C.c_int, C.POINTER(C.c_uint)]
    return lib


def clamp(off, i):
    """ragged_span: (lo, len) of item i, clamped to [off[0], off[n])."""
    a, b = off[0], off[-1]
    lo, hi = max(off[i], a), min(off[i + 1], b)
    return (lo, hi - lo) if hi > lo else (a, 0)


def step(shim, kind, modes, off, i, vbase, rate):
    out = (C.c_long * 12)()
    m = np.ascontiguousarray(modes, dtype=np.uint64)
    o = np.ascontiguousarray(off, dtype=np.uint64)
    shim.host_duplex_ragged_step(kind, m.ctypes.data_as(N.u64p), o.ctypes.data_as(N.u64p), i, len(off) - 1, vbase, rate, out)
    return list(out)


def mode_words(kind, idx, pad=0):
    return [int(kind == "S") | (pad << 32), idx]


@pytest.mark.parametrize("rate", range(1, 9))
@pytest.mark.parametrize("cap", [1, 2])
def test_step_matches_the_oracle(shim, rate, cap):
    """Permute-first, start lane, boundaries, new mode and the ordering key of one sponge's step, from its own mode and a span of
    `count` elements placed among other sponges' spans, against the oracle sponge with its permutation instrumented."""
    t = rate + cap
    cfg = OP.PoseidonConfig(P61, 0, 0, 5, [], [[0] * t for _ in range(t)], rate, cap)
    rnd = random.Random(rate * 10 + cap)
    for kind in ("A", "S"):
        for idx in range(rate + 1):
            for count in range(3 * rate + 2):
                for squeeze in (False, True):
                    o = Traced(cfg, (kind, idx), squeeze)
                    if squeeze:
                        outs = o.squeeze_native_field_elements(count)
                    else:
                        o.absorb(list(range(1, count + 1)))
                        outs = []
                    a = rnd.randrange(0, 50)
                    b = a + rnd.randrange(0, 5)
                    off = [a, b, b + count, b + count + rnd.randrange(0, 5)]
                    modes = [mode_words("A", 0), mode_words(kind, idx, pad=rnd.choice([0, 0xDEADBEEF])), mode_words("S", rate)]
                    s = step(shim, KSQUEEZE if squeeze else KABSORB, modes, off, 1, a, rate)
                    valid, noop, first, start, boundaries, cnt, sq2, idx2, perms, key, ln, doff = s
                    case = (kind, idx, count, squeeze)
                    assert valid == 1 and cnt == ln == count and doff == (b - a if count else 0), case
                    assert replay([noop, first, start, boundaries], cap, rate, count, squeeze) == (o.perms, o.snaps, o.state, outs), case
                    assert ("S" if sq2 else "A", idx2) == o.mode, case
                    assert perms == o.perms and key == min(o.perms, BUCKETS - 1), case


def test_spans_are_clamped_and_byte_spans_count_their_encoding(shim):
    """Random offsets with decreasing pairs and values outside [offsets[0], offsets[n]): every step sees ragged_span's clamped span.
    Byte spans count ceil((len + 8) / 31) elements, the empty string included.  Keys clamp at the last bucket."""
    rnd = random.Random(7)
    for trial in range(300):
        n = rnd.randrange(1, 9)
        off = [rnd.randrange(0, 200) for _ in range(n + 1)]
        if trial % 3 == 0:
            off = sorted(off)
        rate = rnd.randrange(1, 9)
        modes = [mode_words(rnd.choice("AS"), rnd.randrange(rate + 1)) for _ in range(n)]
        for i in range(n):
            lo, ln = clamp(off, i)
            for kind in range(4):
                s = step(shim, kind, modes, off, i, off[0], rate)
                assert s[10] == ln and s[11] == lo - off[0], (off, i, kind)
                assert s[5] == (-(-(ln + 8) // 31) if kind == KBYTES else ln), (off, i, kind)
    big = [0, 1000]
    s = step(shim, KABSORB, [mode_words("A", 0)], big, 0, 0, 1)
    assert s[8] == 999 and s[9] == BUCKETS - 1                                 # the last block is not permuted


def test_invalid_modes_are_reported_and_left_alone(shim):
    for rate in (1, 2, 5):
        for sq, idx in ((2, 0), (-1, 0), (0, rate + 1), (1, rate + 1), (0, 1 << 63)):
            modes = [[sq & 0xFFFFFFFFFFFFFFFF, idx]]
            for kind in range(4):
                s = step(shim, kind, modes, [3, 7], 0, 3, rate)
                assert s[0] == 0 and s[8] == 0 and s[9] == 0, (sq, idx, kind)
        # only the low 4 bytes of the first word are the flag: padding does not make a mode invalid
        s = step(shim, KSQUEEZE, [[(0xFFFFFFFF << 32) | 1, rate]], [0, 2], 0, 0, rate)
        assert s[0] == 1 and s[2] == 1 and s[6:8] == [1, 2 - rate * ((2 - 1) // rate)]           # Squeezing{rate}: permute, 2 lanes


def _call(shim, field, ocfg, am, mm, states, modes, kind, data, off, vbase, order_kind):
    n = states.shape[0]
    order = (C.c_uint * max(n, 1))()
    rc = shim.host_duplex_ragged_run(field.id, ocfg.rate, ocfg.capacity, ocfg.full_rounds, ocfg.partial_rounds, ocfg.alpha,
                                     am.ctypes.data_as(N.u64p), mm.ctypes.data_as(N.u64p), states.ctypes.data_as(N.u64p),
                                     modes.ctypes.data_as(N.u64p), n, kind, data.ctypes.data,
                                     np.ascontiguousarray(off, dtype=np.uint64).ctypes.data_as(N.u64p), vbase, order_kind, order)
    assert rc >= 0
    return list(order)[:n]


@pytest.mark.parametrize("field", list(cp.FIELDS.values()), ids=lambda f: f.name)
@pytest.mark.parametrize("t", [2, 3, 4, 5])
def test_emulated_ragged_call_matches_independent_oracle_sponges(shim, field, t):
    """A seeded script of ragged absorbs, byte absorbs and squeezes (both output forms) over n = 6 sponges, each span 0 .. 3*rate+2 and
    some pairs decreasing, run in input order, in the counting-sort order and reversed: the three agree bit for bit, the sorted order's
    keys do not decrease, and every output, state and mode equals n independent oracle sponges."""
    p = field.modulus
    rnd = random.Random(100 * field.id + t)
    rate, n = t - 1, 6
    ark = [[rnd.randrange(p) for _ in range(t)] for _ in range(8 + 3)]
    mds = [[rnd.randrange(1, p) for _ in range(t)] for _ in range(t)]
    if t % 2:
        mds[0][0] = 0                                                       # the dense schedule
    ocfg = OP.PoseidonConfig(p, 8, 3, 5, ark, mds, rate, 1)
    oracles = [OP.PoseidonSponge(ocfg) for _ in range(n)]
    am, mm = field.elements([x for r in ark for x in r]), field.elements([x for r in mds for x in r])
    states = np.zeros((n, t, 4), dtype=np.uint64)
    modes = np.zeros((n, 2), dtype=np.uint64)
    kinds = [KABSORB, KBYTES, KSQUEEZE, KCANON]
    for stp in range(12):
        kind = kinds[stp] if stp < 4 else rnd.choice(kinds)
        lens = [rnd.randrange(0, 3 * rate + 3) if kind != KBYTES else rnd.randrange(0, 80) for _ in range(n)]
        base = rnd.randrange(0, 4)
        off = [base]
        for ln in lens:
            off.append(off[-1] + ln)
        if stp % 3 == 1:                                                    # below the window: sponge 0 empty, sponge 1 clamped
            off[1] = 0
        if stp % 3 == 2 and kind < KSQUEEZE:                                # a decreasing pair: sponge 2's span is empty
            off[3] = off[2] - 1 if off[2] > off[0] else off[2]
        if stp % 3 == 2 and kind >= KSQUEEZE:                               # above the window: sponge n-1 empty (outputs must not
            off[n - 1] = off[n] + 3                                         # overlap, so only at the window's edges)
        spans = [clamp(off, i) for i in range(n)]
        total = off[-1]
        if kind == KABSORB:
            vals = [rnd.randrange(p) for _ in range(total)]
            data = field.elements(vals) if total else np.zeros((1, 4), dtype=np.uint64)
        elif kind == KBYTES:
            raw = bytes(rnd.randrange(256) for _ in range(total))
            data = np.frombuffer(raw + b"\0", dtype=np.uint8).copy()
        else:
            data = np.zeros((max(total, 1), 4), dtype=np.uint64)
        results = []
        for order_kind in (0, 1, 2):
            s, m = states.copy(), modes.copy()
            d = data.copy()
            order = _call(shim, field, ocfg, am, mm, s, m, kind, d, off, 0, order_kind)
            if order_kind == 1:
                keys = [step(shim, kind, modes, off, i, 0, rate)[9] for i in order]
                assert keys == sorted(keys) and sorted(order) == list(range(n))
            results.append((s, m, d))
        for s, m, d in results[1:]:
            assert np.array_equal(s, results[0][0]) and np.array_equal(m, results[0][1]) and np.array_equal(d, results[0][2]), stp
        states, modes, d = results[0]
        for i, o in enumerate(oracles):
            lo, ln = spans[i]
            if kind == KABSORB:
                o.absorb(vals[lo:lo + ln])
            elif kind == KBYTES:
                o.absorb(A._ints(raw[lo:lo + ln], field))
            else:
                want = o.squeeze_native_field_elements(ln)
                got = field.to_ints(d[lo:lo + ln]) if kind == KSQUEEZE else [int.from_bytes(r.tobytes(), "little") for r in d[lo:lo + ln]]
                assert got == want, (stp, i)
            assert field.to_ints(states[i]) == o.state, (stp, i)
            assert ("S" if modes[i, 0] else "A", int(modes[i, 1])) == o.mode, (stp, i)


def test_invalid_mode_items_are_untouched_and_their_output_zeroed(shim):
    field = cp.BN254_FR
    p, t, rate, n = field.modulus, 3, 2, 5
    rnd = random.Random(3)
    ark = [[rnd.randrange(p) for _ in range(t)] for _ in range(11)]
    mds = [[rnd.randrange(1, p) for _ in range(t)] for _ in range(t)]
    ocfg = OP.PoseidonConfig(p, 8, 3, 5, ark, mds, rate, 1)
    am, mm = field.elements([x for r in ark for x in r]), field.elements([x for r in mds for x in r])
    states = np.stack([field.elements([rnd.randrange(p) for _ in range(t)]) for _ in range(n)])
    modes = np.array([[0, 1], [2, 0], [0xFFFFFFFF00000001, 1], [0, rate + 1], [1, 2]], dtype=np.uint64)
    s, m = states.copy(), modes.copy()
    off = [0, 2, 5, 7, 8, 10]
    out = np.full((10, 4), 0x55, dtype=np.uint64)
    _call(shim, field, ocfg, am, mm, s, m, KSQUEEZE, out, off, 0, 1)
    for i in (1, 3):                                                         # invalid: untouched, output zeroed
        assert np.array_equal(s[i], states[i]) and np.array_equal(m[i], modes[i])
        assert not out[off[i]:off[i + 1]].any()
    for i in (0, 2, 4):                                                      # valid: squeezed, the mode's padding written as zero
        o = OP.PoseidonSponge(ocfg)
        o.state = field.to_ints(states[i])
        o.mode = ("S" if int(modes[i, 0]) & 0xFFFFFFFF else "A", int(modes[i, 1]))
        assert field.to_ints(out[off[i]:off[i + 1]]) == o.squeeze_native_field_elements(off[i + 1] - off[i]), i
        assert field.to_ints(s[i]) == o.state and [int(x) for x in m[i]] == [1, o.mode[1]], i
    # an absorb leaves the invalid items alone too
    s2, m2 = s.copy(), m.copy()
    vals = field.elements(list(range(1, 11)))
    _call(shim, field, ocfg, am, mm, s2, m2, KABSORB, vals, off, 0, 0)
    for i in (1, 3):
        assert np.array_equal(s2[i], states[i]) and np.array_equal(m2[i], modes[i])


# ---------------------------------------------------------------------------------------------------- ABI argument rules
def test_sponge_mode_layout():
    assert C.sizeof(N.SpongeMode) == 16 and N.SpongeMode.squeezing.offset == 0 and N.SpongeMode.index.offset == 8


def _ragged_entry_points():
    """(name, host form?, kind, call(ctx, states, modes, data, offsets, n))."""
    L = N.lib
    return [
        ("absorb", True, KABSORB, lambda c, s, m, d, o, n: L.cpb_poseidon_duplex_absorb_ragged(c, s, m, d, o, n)),
        ("absorb_dev", False, KABSORB, lambda c, s, m, d, o, n: L.cpb_poseidon_duplex_absorb_ragged_dev(c, s, m, d, o, n, None)),
        ("absorb_bytes", True, KBYTES, lambda c, s, m, d, o, n: L.cpb_poseidon_duplex_absorb_bytes_ragged(c, s, m, C.cast(d, N.u8p) if d else None, o, n)),
        ("absorb_bytes_dev", False, KBYTES, lambda c, s, m, d, o, n: L.cpb_poseidon_duplex_absorb_bytes_ragged_dev(c, s, m, d, o, n, None)),
        ("squeeze", True, KSQUEEZE, lambda c, s, m, d, o, n: L.cpb_poseidon_duplex_squeeze_ragged(c, s, m, d, o, 0, n)),
        ("squeeze_dev", False, KSQUEEZE, lambda c, s, m, d, o, n: L.cpb_poseidon_duplex_squeeze_ragged_dev(c, s, m, d, o, 1, n, None)),
    ]


@pytest.mark.parametrize("name,host,kind,call", _ragged_entry_points(), ids=[e[0] for e in _ragged_entry_points()])
def test_ragged_entry_points_validate_in_the_header_order(name, host, kind, call):
    n = 3
    states = np.zeros((n, 3, 4), dtype=np.uint64)
    buf = np.zeros(64, dtype=np.uint64)
    off = np.array([2, 4, 4, 7], dtype=np.uint64)
    modes = (N.SpongeMode * n)(N.SpongeMode(0, 0), N.SpongeMode(1, 2), N.SpongeMode(0, 1))
    st, bp, op = states.ctypes.data_as(N.u64p), buf.ctypes.data_as(N.u64p), off.ctypes.data_as(N.u64p)
    mp = C.cast(modes, N.modep)
    # n >= 2^32 first, then n == 0: a no-op even with every pointer null
    assert call(None, None, None, None, None, 1 << 32) == N.CPB_BAD_LENGTH
    assert call(None, None, None, None, None, 0) == N.CPB_OK
    # then states, modes, offsets
    assert call(None, None, mp, bp, op, n) == N.CPB_NULL_POINTER
    assert call(None, st, None, bp, op, n) == N.CPB_NULL_POINTER
    assert call(None, st, mp, bp, None, n) == N.CPB_NULL_POINTER
    dec = np.array([2, 5, 4, 7], dtype=np.uint64)
    bad = (N.SpongeMode * n)(N.SpongeMode(0, 0), N.SpongeMode(2, 0), N.SpongeMode(0, 0))
    if host:
        # host forms: decreasing offsets, then a null data buffer with a span that is not empty, then a bad squeezing flag -- all
        # before the context (a null one here), so without a device
        assert call(None, st, mp, bp, dec.ctypes.data_as(N.u64p), n) == N.CPB_BAD_LENGTH
        assert call(None, st, mp, None, op, n) == N.CPB_NULL_POINTER
        assert b"data" in N.lib.cpb_last_error()
        assert call(None, st, C.cast(bad, N.modep), bp, op, n) == N.CPB_BAD_PARAMS
        assert b"squeezing" in N.lib.cpb_last_error()
        # all spans empty: a null data buffer is fine and the context comes next
        empty = np.array([4, 4, 4, 4], dtype=np.uint64)
        assert call(None, st, mp, None, empty.ctypes.data_as(N.u64p), n) == N.CPB_NULL_POINTER
        assert b"null context" in N.lib.cpb_last_error()
    else:
        # _dev forms check nothing in device memory: offsets and modes go straight to the context check
        assert call(None, st, mp, bp, dec.ctypes.data_as(N.u64p), n) == N.CPB_NULL_POINTER
        assert call(None, st, C.cast(bad, N.modep), bp, op, n) == N.CPB_NULL_POINTER
        assert b"null context" in N.lib.cpb_last_error()
    assert call(None, st, mp, bp, op, n) == N.CPB_NULL_POINTER
    assert b"null context" in N.lib.cpb_last_error()
    # a refused call leaves the modes and states as they were
    assert [(m.squeezing, m.index) for m in modes] == [(0, 0), (1, 2), (0, 1)] and not states.any()

