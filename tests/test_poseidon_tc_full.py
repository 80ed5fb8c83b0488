"""The full rounds' dense rows on the tensor cores (csrc/poseidon_tc.cuh: tc_full_round; the row tables of poseidon_host.hpp:
tc_full_tables).  The row tables of the bench schedule and of a random-constant BN254 Fr t = 3 alpha = 5 sparse schedule against
Python integers, a CPU emulation of one warp's full round (staging, ldmatrix, IMMA, the C buffer, tc_finish, the conditional
subtraction) against the field algebra on extreme operands -- every matrix, the entry row and the last round's rows -- and the
bounds of a row as exact rationals."""
import ctypes as C
import random
from fractions import Fraction as Fr

import numpy as np
import pytest

from helpers import OF, build_host_shim, oracle_config
from test_poseidon_lane1_basis import random_config, regions
from test_poseidon_scaled_lane0 import FID, _arrays, _P, schedule
from test_poseidon_tc import emulate_output, k8, ptx_b

u32p = C.POINTER(C.c_uint32)
R = 1 << 256
ROW_WORDS, ROWS = 768, 10
# a row's product is below p * (1 + EXTRA): V = sum_{j,i} byte_i(s_j) * K8_i(c_j) < 3 * 32 * 255 * p, divided by 2^32
EXTRA = Fr(3 * 32 * 255, 1 << 32)


@pytest.fixture(scope="module")
def lib():
    return build_host_shim("poseidon_tc_full_shim")


@pytest.fixture(scope="module")
def tc_lib():
    return build_host_shim("poseidon_tc_shim")


def configs():
    return {"bench": oracle_config("bn254_r2")[1], "random": random_config(OF.BN254_FR, 3, 8, 57, 5, seed=2024)}


@pytest.fixture(scope="module", params=["bench", "random"])
def cfg(request):
    return configs()[request.param]


def full_tables(lib, cfg):
    ark, mds = _arrays(cfg)
    args = (cfg.rate, cfg.capacity, cfg.full_rounds, cfg.partial_rounds, C.c_ulonglong(cfg.alpha), _P(ark), _P(mds))
    n = lib.host_tc_full_tables(*args, None, C.c_long(0))
    assert n == ROWS * ROW_WORDS
    out = np.zeros(n, dtype=np.uint32)
    assert lib.host_tc_full_tables(*args, out.ctypes.data_as(u32p), C.c_long(n)) == n
    return out.reshape(ROWS, ROW_WORDS)


def row_words(lib):
    words = (C.c_int * ROW_WORDS)()
    lib.host_tc_row_words(words)
    return list(words)


def row_constants(cfg):
    """The ten rows the split form's full rounds read, as field integers: rows 0..2 of M, Mpre, Mpost, then the entry row."""
    o, v = schedule(FID["bn254_fr"], cfg)
    assert o["sparse"] == 1
    reg = regions(o, v, 3, cfg.full_rounds, cfg.partial_rounds)
    rows = [reg[m][3 * i:3 * i + 3] for m in ("M", "Mpre", "Mpost") for i in range(3)]
    return rows + [reg["entry_row"]]


def test_row_word_map(lib):
    words = row_words(lib)
    assert sorted(words) == list(range(ROW_WORDS))             # every (n-tile, k-chunk, lane, register) a distinct word
    it = iter(words)
    for _nt in range(4):
        for _kc in range(3):
            for _lane in range(32):
                w0, w1 = next(it), next(it)
                assert w1 == w0 + 1 and w0 % 2 == 0           # lane's b0, b1 pair: one 8-byte load


def test_full_index(lib):
    for rf in (8, 6, 9):
        half = rf // 2
        want = [1 if fr == half - 1 else 2 if fr == half else 0 for fr in range(rf)]
        assert [lib.host_pos_full_index(rf, fr) for fr in range(rf)] == want


def test_row_tables_are_the_schedule_rows(lib, cfg):
    p = cfg.p
    tabs, words = full_tables(lib, cfg), row_words(lib)
    for row, consts in enumerate(row_constants(cfg)):
        it = iter(words)
        for nt in range(4):
            for kc in range(3):
                kk = k8(consts[kc], p)
                for lane in range(32):
                    for r in range(2):
                        w = int(tabs[row][next(it)])
                        for q in range(4):
                            krow, ncol = ptx_b(lane, r, q)
                            assert (w >> (8 * q)) & 0xFF == (kk[krow] >> (8 * (8 * nt + ncol))) & 0xFF, (row, nt, kc, lane, r, q)


def as_round_words(tab, words):
    """A row table laid out as constants 0..2 of a partial round's table (the layout emulate_output reads), through the product's
    own map."""
    out = [0] * 1024
    it = iter(words)
    for nt in range(4):
        for kc in range(3):
            for lane in range(32):
                for r in range(2):
                    out[((nt * 4 + kc) * 32 + lane) * 2 + r] = int(tab[next(it)])
    return out


def full_round(tc_lib, tabs4, m, entry, need, ops, p):
    """tc_full_round for 32 lanes: row i from table 3 m + i (row 1 from the entry table when entry), one conditional subtraction
    of p, zero for a row whose need bit is clear.  Returns [lane][row] and the unreduced products."""
    res = [[0] * 3 for _ in range(32)]
    raw = [[None] * 3 for _ in range(32)]
    for i in range(3):
        if not (need >> i) & 1:
            continue
        tab = tabs4[9] if entry and i == 1 else tabs4[3 * m + i]
        out = emulate_output(tc_lib, ops, tab, [0, 1, 2])
        for lane in range(32):
            raw[lane][i] = out[lane]
            res[lane][i] = out[lane] - p if out[lane] >= p else out[lane]     # fp_final_sub
    return res, raw


def test_warp_full_round_against_the_field(lib, tc_lib, cfg):
    p = cfg.p
    tabs, words = full_tables(lib, cfg), row_words(lib)
    tabs4 = [as_round_words(tabs[row], words) for row in range(ROWS)]
    rows = row_constants(cfg)
    rinv = pow(R, -1, p)
    rnd = random.Random(5)
    lazy = p * 124 // 100                                      # the lazy S-box outputs are below 1.24 p
    extremes = [R - 1, p - 1, 0, p, lazy, lazy - 1, 1, int("ff" * 32, 16) >> 2, 2 * p - 1]
    # (matrix, entry, need): every matrix with all rows, the entry round (Mpre with the entry row), and the last round's rows for
    # one and for two squeezed outputs (capacity 1)
    cases = [(0, False, 0b111), (1, True, 0b111), (2, False, 0b111), (0, False, 0b010), (0, False, 0b110)]
    for trial, (m, entry, need) in enumerate(cases):
        ops = []
        for lane in range(32):
            if lane < 27:
                ops.append([extremes[(lane + j * 3 + trial) % len(extremes)] for j in range(3)])
            else:
                ops.append([rnd.randrange(lazy) for _ in range(3)])
        res, raw = full_round(tc_lib, tabs4, m, entry, need, ops, p)
        for lane in range(32):
            for i in range(3):
                if not (need >> i) & 1:
                    assert res[lane][i] == 0
                    continue
                consts = rows[9] if entry and i == 1 else rows[3 * m + i]
                mont = [c * R % p for c in consts]
                want = sum(c * s for c, s in zip(mont, ops[lane])) * rinv % p
                assert raw[lane][i] < p * (1 + EXTRA), (trial, lane, i)
                assert res[lane][i] == want, (trial, lane, i)


def test_full_row_bounds_bn254():
    p = OF.BN254_FR
    col = 3 * 32 * 255 * 255                                   # column sum of three k-chunks
    assert col < 1 << 23 and col + 256 * col < 1 << 31         # s32 accumulators; a packed pair; E's chain cannot carry out
    Vmax = 3 * 32 * 255 * (p - 1)                              # any operand below 2^256: bytes <= 255, K8_i <= p - 1
    assert Vmax < 96 * 255 * p
    m = (1 << 32) - 1
    assert Vmax + m * p < 1 << 288                             # tc_finish's accumulators
    res = Fr(Vmax + m * p, 1 << 32)
    assert res < p * (1 + Fr(765, 1 << 27)) and p * (1 + Fr(765, 1 << 27)) < 2 * p   # one subtraction of p makes it canonical
    assert 2 * p < R                                           # the subtraction's operand fits 256 bits
    assert Fr(124, 100) * p < R                                # the lazy S-box outputs enter the stage as they are
