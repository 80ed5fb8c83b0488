"""The S-box's Montgomery reduction on the tensor cores (csrc/poseidon_tc.cuh: tc_redc; poseidon.cuh: pos_sbox5_tc).  The 512-bit
products fp_sqr_wide and fp_mul_wide against Python integers, the R^-1 table against Python integers, a CPU emulation of one warp's
reduction (staging, ldmatrix, IMMA, the C buffer, tc_finish) against a*b/R mod p on random and extreme operands, and the bounds
of the lazy BN254 Fr chain with the reduction's extra term as exact rationals."""
import ctypes as C
import random
from fractions import Fraction as Fr

import pytest

from helpers import build_host_shim, oracle_config
from test_poseidon_tc import emulate_output, ptx_b

R = 1 << 256
RINV_WORDS = 256
# tc_redc's result is below T_hi + p * (1 + EXTRA): V = sum_i byte_i(T_lo) * K8_i < 32 * 255 * p, divided by 2^32
EXTRA = Fr(32 * 255, 1 << 32)


@pytest.fixture(scope="module")
def lib():
    return build_host_shim("poseidon_tc_redc_shim")


@pytest.fixture(scope="module")
def tc_lib():
    return build_host_shim("poseidon_tc_shim")


@pytest.fixture(scope="module")
def p():
    return oracle_config("bn254_r2")[1].p


def limbs(x, n):
    return (C.c_uint32 * n)(*[(x >> (32 * i)) & 0xFFFFFFFF for i in range(n)])


def wide(lib, a, b, sq):
    out = (C.c_uint32 * 16)()
    lib.host_mul_wide(limbs(a, 8), limbs(b, 8), 1 if sq else 0, out)
    return sum(int(w) << (32 * i) for i, w in enumerate(out))


def test_wide_products(lib, p):
    rnd = random.Random(7)
    ones = R - 1
    cases = [ones, 0, 1, 2 * p - 1, p - 1, p, int("ffffffff00000000" * 4, 16), int("00000000ffffffff" * 4, 16)]
    cases += [rnd.randrange(R) for _ in range(200)] + [rnd.randrange(2 * p) for _ in range(200)]
    for a in cases:
        assert wide(lib, a, a, True) == a * a
        b = rnd.choice(cases)
        assert wide(lib, a, b, False) == a * b
        assert wide(lib, a, a, False) == a * a


def rinv_table(lib):
    out = (C.c_uint32 * RINV_WORDS)()
    assert lib.host_tc_rinv_table(out) == RINV_WORDS
    words = (C.c_int * RINV_WORDS)()
    lib.host_tc_rinv_words(words)
    return list(out), list(words)


def test_rinv_table_is_the_constant(lib, p):
    tab, words = rinv_table(lib)
    assert sorted(words) == list(range(RINV_WORDS))                  # every (n-tile, lane, register) a distinct word
    k8 = [(1 << (8 * i + 32)) * pow(R, -1, p) % p for i in range(32)]   # K8_i(1) = 2^(8i) * 2^32 / R mod p
    it = iter(words)
    for nt in range(4):
        for lane in range(32):
            for r in range(2):
                w = tab[next(it)]
                for q in range(4):
                    krow, ncol = ptx_b(lane, r, q)
                    assert (w >> (8 * q)) & 0xFF == (k8[krow] >> (8 * (8 * nt + ncol))) & 0xFF, (nt, lane, r, q)


def as_round_words(tab, words):
    """The R^-1 table laid out as constant 0 of a round table (the layout emulate_output reads), through the product's own map."""
    out = [0] * 1024
    it = iter(words)
    for nt in range(4):
        for lane in range(32):
            for r in range(2):
                out[((nt * 4 + 0) * 32 + lane) * 2 + r] = tab[next(it)]
    return out


def reduce_warp(tc_lib, tab4, Ts):
    """tc_redc for 32 lanes: stage T_lo, the NT = 1 product over the R^-1 table, tc_finish with y = T_hi."""
    return emulate_output(tc_lib, [[T % R] for T in Ts], tab4, [0], y=[T >> 256 for T in Ts])


def test_warp_reduction_against_the_field(lib, tc_lib, p):
    tab, words = rinv_table(lib)
    tab4 = as_round_words(tab, words)
    rinv = pow(R, -1, p)
    rnd = random.Random(11)
    hi_max = (2 * p - 1) ** 2 >> 256
    ops = [2 * p - 1, p - 1, p, 0, 1, 2 * p - 2, int("ffffffff" * 7, 16)]
    for trial in range(4):
        Ts = []
        for lane in range(32):
            kind = (lane + trial) % 8
            if kind == 0:
                Ts.append(rnd.randrange(hi_max + 1) * R)                 # T_lo = 0
            elif kind == 1:
                Ts.append(rnd.randrange(hi_max + 1) * R + R - 1)         # T_lo = 2^256 - 1
            elif kind == 2:
                Ts.append(hi_max * R + R - 1)                            # the largest T of operands below 2p, all-ones low half
            elif kind == 3:
                a = ops[(lane + trial) % len(ops)]
                Ts.append(wide(lib, a, a, True))
            elif kind == 4:
                a, b = ops[lane % len(ops)], ops[(lane + trial + 1) % len(ops)]
                Ts.append(wide(lib, a, b, False))
            elif kind == 5:
                a = rnd.randrange(2 * p)
                Ts.append(wide(lib, a, a, True))
            else:
                Ts.append(wide(lib, rnd.randrange(2 * p), rnd.randrange(2 * p), False))
        res = reduce_warp(tc_lib, tab4, Ts)
        for lane, (T, r) in enumerate(zip(Ts, res)):
            assert r % p == T * rinv % p, (trial, lane)
            assert r < (T >> 256) + p * (1 + EXTRA), (trial, lane)


def test_redc_bounds_bn254(p):
    """Every link of the lazy chain of pos_permute_split with the S-box reduced by tc_redc (result < T/R + p (1 + EXTRA))."""
    q = Fr(p, R)                                               # p / R
    red = lambda a, b: a * b * q + 1 + EXTRA                   # noqa: E731  bound / p of the reduced product of a p and b p
    # tc_finish: V + m*p < 2^288 and y + (V >> 32) < 2^256 for y = T_hi of operands below 2p (the widest S-box input)
    y_max = (2 * p - 1) ** 2 >> 256
    V = 32 * 255 * (p - 1) + y_max * (1 << 32)
    assert V + ((1 << 32) - 1) * p < 1 << 288
    assert y_max + (32 * 255 * (p - 1) >> 32) + 1 < R
    # partial rounds: x < 2p
    x2 = red(2, 2)
    x4 = red(x2, x2)
    x5 = red(x4, 2)
    assert x2 < Fr(176, 100) and x4 < Fr(159, 100) and x5 < Fr(160, 100)
    # full rounds: canonical x
    f2 = red(1, 1)
    f4 = red(f2, f2)
    f5 = red(f4, 1)
    assert f5 < Fr(124, 100)
    # every S-box input and output is below 2^256 (the dense rows' digit tables take any operand below 2^256) and the wide products
    # of x < 2p fit 512 bits
    assert 2 * x5 * p < R and 2 * p < R
    # fp_add_lazy: d = y + a' with y = x^5 < 1.60p and a' below p (1 + 3 * 255 * 2^-27) (the round's tensor-core output).  It
    # returns d canonical, and the next S-box input d + c (c < p) is below 2p again.
    assert x5 + 1 + Fr(3 * 255, 1 << 27) < 3
