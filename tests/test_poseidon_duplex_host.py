"""Batched duplex sponges without a GPU: the mode plan of csrc/poseidon_duplex.cuh (duplex_plan, which both the host and the kernel
run) against oracle/poseidon.py::PoseidonSponge with its permutation instrumented, the kernel's per-sponge body pos_duplex itself
(CPU build, real permutation) against independent oracle sponges, the [u8] chunk encoding against sponge/absorb.py, and the argument
rules of the cpb_poseidon_duplex_* entry points that need no device."""
import ctypes as C
import random

import numpy as np
import pytest

from helpers import build_host_shim
import crypto_primitives_b200 as cp
from crypto_primitives_b200 import _native as N
from crypto_primitives_b200.sponge import absorb as A
from oracle import poseidon as OP

lp = C.POINTER(C.c_long)
u32p = C.POINTER(C.c_uint32)


@pytest.fixture(scope="module")
def shim():
    lib = build_host_shim("poseidon_duplex_shim")
    lib.host_duplex_plan.argtypes = [C.c_int, C.c_int, C.c_long, C.c_long, C.c_long, lp]
    lib.host_duplex_mode_valid.argtypes = [C.c_int, C.c_ulonglong, C.c_long]
    lib.host_duplex_byte_elems.argtypes = [C.c_long]
    lib.host_duplex_byte_elems.restype = C.c_long
    lib.host_duplex_byte_chunk.argtypes = [C.c_char_p, C.c_long, C.c_long, C.c_int, C.c_int, u32p]
    lib.host_duplex_run.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_ulonglong, N.u64p, N.u64p, N.u64p, C.c_long, C.c_int,
                                    C.c_long, N.u64p, C.c_char_p, C.c_long, C.c_long, N.u64p, C.POINTER(C.c_int), lp]
    return lib


P61 = (1 << 61) - 1


class Traced(OP.PoseidonSponge):
    """The oracle sponge with a permutation that records what it sees: an absorb's state is snapshotted and cleared, so each
    segment shows which lanes took which elements; a squeeze reads marker values 1000 * (permutations so far) + lane."""

    def __init__(self, cfg, mode, squeeze):
        super().__init__(cfg)
        self.mode = mode
        self.squeeze = squeeze
        self.perms, self.snaps = 0, []
        self._fill()

    def _fill(self):
        t = len(self.state)
        self.state = [1000 * self.perms + i for i in range(t)] if self.squeeze else [0] * t

    def _permute(self):
        self.snaps.append(list(self.state))
        self.perms += 1
        self._fill()


def plan(shim, squeeze, mode, rate, count):
    out = (C.c_long * 6)()
    shim.host_duplex_plan(int(squeeze), int(mode[0] == "S"), mode[1], rate, count, out)
    return list(out)


def replay(p, cap, rate, count, squeeze):
    """The block / lane walk the plan prescribes, on the same instrumented state as Traced (the plan's meaning; the kernel's own loop
    is run in test_pos_duplex_matches_independent_oracle_sponges)."""
    noop, first, start, boundaries = p[:4]
    t = rate + cap
    tr = Traced(OP.PoseidonConfig(P61, 0, 0, 5, [], [[0] * t for _ in range(t)], rate, cap), ("A", 0), squeeze)
    outs = []
    if not noop:
        done = 0
        for b in range(boundaries + 1):
            if b > 0 or first:
                tr._permute()
            lo = start if b == 0 else 0
            hi = min(rate, lo + count - done)
            for lane in range(lo, hi):
                e = done + lane - lo
                if squeeze:
                    outs.append(tr.state[cap + lane])
                else:
                    tr.state[cap + lane] += e + 1
            done += hi - lo
    return tr.perms, tr.snaps, tr.state, outs


@pytest.mark.parametrize("rate", range(1, 9))
@pytest.mark.parametrize("cap", [1, 2])
def test_plan_matches_the_oracle(shim, rate, cap):
    t = rate + cap
    cfg = OP.PoseidonConfig(P61, 0, 0, 5, [], [[0] * t for _ in range(t)], rate, cap)
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
                    p = plan(shim, squeeze, (kind, idx), rate, count)
                    perms, snaps, state, routs = replay(p, cap, rate, count, squeeze)
                    case = (kind, idx, count, squeeze)
                    assert (perms, snaps, state, routs) == (o.perms, o.snaps, o.state, outs), case
                    assert ("S" if p[4] else "A", p[5]) == o.mode, case
                    assert 0 <= p[2] < rate, case


def test_mode_validity(shim):
    for rate in range(1, 9):
        for idx in range(rate + 3):
            for sq in (-1, 0, 1, 2):
                assert shim.host_duplex_mode_valid(sq, idx, rate) == int(sq in (0, 1) and idx <= rate)
    assert shim.host_duplex_mode_valid(0, (1 << 64) - 1, 8) == 0


@pytest.mark.parametrize("field", list(cp.FIELDS.values()), ids=lambda f: f.name)
def test_byte_chunks_match_absorb_encoding(shim, field):
    rng = np.random.default_rng(field.id)
    for L in range(101):
        s = bytes(rng.integers(0, 256, size=L, dtype=np.uint8))
        want = A._ints(s, field)
        n = shim.host_duplex_byte_elems(L)
        assert n == len(want) == -(-(L + 8) // 31), L
        mont = field.elements(want)
        for j in range(n):
            out = np.zeros(8, dtype=np.uint32)
            shim.host_duplex_byte_chunk(s, L, j, 0, field.id, out.ctypes.data_as(u32p))
            assert int.from_bytes(out.tobytes(), "little") == want[j], (L, j)
            shim.host_duplex_byte_chunk(s, L, j, 1, field.id, out.ctypes.data_as(u32p))
            assert np.array_equal(out.view(np.uint64), mont[j]), (L, j)


@pytest.mark.parametrize("field", list(cp.FIELDS.values()), ids=lambda f: f.name)
@pytest.mark.parametrize("t", [2, 3, 4, 5])
def test_pos_duplex_matches_independent_oracle_sponges(shim, field, t):
    """The kernel's per-sponge body (pos_duplex with pos_permute, on the product's schedule, sparse or dense) over a seeded script of
    every call kind, for n = 3 sponges, against three oracle sponges: every output, the states and the mode."""
    p = field.modulus
    rnd = random.Random(100 * field.id + t)
    rate, n = t - 1, 3
    ark = [[rnd.randrange(p) for _ in range(t)] for _ in range(8 + 3)]
    mds = [[rnd.randrange(1, p) for _ in range(t)] for _ in range(t)]
    if t % 2:
        mds[0][0] = 0                                                       # the dense schedule
    ocfg = OP.PoseidonConfig(p, 8, 3, 5, ark, mds, rate, 1)
    oracles = [OP.PoseidonSponge(ocfg) for _ in range(n)]
    am, mm = field.elements([x for r in ark for x in r]), field.elements([x for r in mds for x in r])
    states = np.zeros((n, t, 4), dtype=np.uint64)
    sq, idx = C.c_int(0), C.c_long(0)

    def call(kind, count=0, inp=None, data=None, length=0, stride=0, out=None):
        rc = shim.host_duplex_run(field.id, rate, 1, 8, 3, 5, am.ctypes.data_as(N.u64p), mm.ctypes.data_as(N.u64p),
                                  states.ctypes.data_as(N.u64p), n, kind, count, None if inp is None else inp.ctypes.data_as(N.u64p),
                                  data, length, stride, None if out is None else out.ctypes.data_as(N.u64p), C.byref(sq), C.byref(idx))
        assert rc == int(t % 2 == 0)

    kinds = ["absorb", "bytes", "bcast", "squeeze", "canonical"]
    for step in range(14):
        op = kinds[step] if step < len(kinds) else rnd.choice(kinds)
        if op == "absorb":
            k = rnd.randrange(0, 3 * rate + 2)
            vals = [[rnd.randrange(p) for _ in range(k)] for _ in range(n)]
            x = np.ascontiguousarray(np.stack([field.elements(v) for v in vals]) if k else np.zeros((n, 0, 4), dtype=np.uint64))
            call(0, k, inp=x if k else None)
            for o, v in zip(oracles, vals):
                o.absorb(v)
        elif op in ("bytes", "bcast"):
            L = rnd.randrange(0, 70)
            strings = [bytes(rnd.randrange(256) for _ in range(L)) for _ in range(n)]
            if op == "bcast":
                strings = [strings[0]] * n
            call(1, data=b"".join(strings) if op == "bytes" else strings[0], length=L, stride=L if op == "bytes" else 0)
            for o, b in zip(oracles, strings):
                o.absorb(A._ints(b, field))
        else:
            m = rnd.randrange(0, 2 * rate + 2)
            out = np.zeros((n, max(m, 1), 4), dtype=np.uint64)
            call(2 if op == "squeeze" else 3, m, out=out)
            for i, o in enumerate(oracles):
                want = o.squeeze_native_field_elements(m)
                got = field.to_ints(out[i, :m]) if op == "squeeze" else [int.from_bytes(r.tobytes(), "little") for r in out[i, :m]]
                assert got == want, (op, step, i)
        for i, o in enumerate(oracles):
            assert field.to_ints(states[i]) == o.state, (op, step, i)
            assert ("S" if sq.value else "A", idx.value) == o.mode, (op, step)


# ---------------------------------------------------------------------------------------------------- ABI argument rules
def _entry_points():
    """(name, call(ctx, states, mode, buf, size, n)) for the six entry points; `size` is k, len or m."""
    L = N.lib
    return [
        ("absorb", lambda c, s, m, b, k, n: L.cpb_poseidon_duplex_absorb(c, s, m, b, k, n)),
        ("absorb_dev", lambda c, s, m, b, k, n: L.cpb_poseidon_duplex_absorb_dev(c, s, m, b, k, n, None)),
        ("absorb_bytes", lambda c, s, m, b, k, n: L.cpb_poseidon_duplex_absorb_bytes(c, s, m, C.cast(b, N.u8p) if b else None, k, k, n)),
        ("absorb_bytes_dev", lambda c, s, m, b, k, n: L.cpb_poseidon_duplex_absorb_bytes_dev(c, s, m, b, k, k, n, None)),
        ("squeeze", lambda c, s, m, b, k, n: L.cpb_poseidon_duplex_squeeze(c, s, m, b, k, 0, n)),
        ("squeeze_dev", lambda c, s, m, b, k, n: L.cpb_poseidon_duplex_squeeze_dev(c, s, m, b, k, 1, n, None)),
    ]


@pytest.mark.parametrize("name,call", _entry_points(), ids=[e[0] for e in _entry_points()])
def test_duplex_entry_points_validate_before_touching_a_device(name, call):
    states = np.zeros((2, 3, 4), dtype=np.uint64)
    buf = np.zeros(64, dtype=np.uint64)
    st, bp = states.ctypes.data_as(N.u64p), buf.ctypes.data_as(N.u64p)
    # the mode first: null, then squeezing outside {0, 1}, with null context and buffers
    assert call(None, None, None, None, 1, 2) == N.CPB_NULL_POINTER
    for sq in (-1, 2, 7):
        m = N.SpongeMode(sq, 0)
        assert call(None, None, C.byref(m), None, 1, 2) == N.CPB_BAD_PARAMS
        assert (m.squeezing, m.index) == (sq, 0)
    m = N.SpongeMode(1, 1)
    # then the sizes
    assert call(None, st, C.byref(m), bp, 1, 1 << 62) == N.CPB_BAD_LENGTH
    assert call(None, st, C.byref(m), bp, 1 << 62, 2) == N.CPB_BAD_LENGTH
    # then the buffers the call needs (n > 0)
    assert call(None, None, C.byref(m), bp, 1, 2) == N.CPB_NULL_POINTER
    assert call(None, st, C.byref(m), None, 1, 2) == N.CPB_NULL_POINTER
    # then the context, also when n == 0 (advancing the mode needs the rate)
    assert call(None, st, C.byref(m), bp, 1, 2) == N.CPB_NULL_POINTER
    assert call(None, None, C.byref(m), None, 0, 0) == N.CPB_NULL_POINTER
    assert b"null context" in N.lib.cpb_last_error()
    # a buffer that is not read or written (k, len or m == 0) may be null, as in the other calls
    assert call(None, st, C.byref(m), None, 0, 2) == N.CPB_NULL_POINTER
    assert b"null context" in N.lib.cpb_last_error()
    assert (m.squeezing, m.index) == (1, 1), "a refused call leaves the mode as it was"
    # a mode index past the rate is refused once the context is known (test_mode_validity); without one the context comes first
    m = N.SpongeMode(0, 99)
    assert call(None, st, C.byref(m), bp, 1, 2) == N.CPB_NULL_POINTER
