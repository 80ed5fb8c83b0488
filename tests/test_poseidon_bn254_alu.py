"""Fewer non-multiply instructions in the Poseidon hash kernel (csrc/fp.cuh, csrc/poseidon.cuh, DESIGN §4.1 and §4.2): the
squaring's reduction without an overflow word, the second reduction row of fp_dot_tab without one, the partial-round lanes kept
in a wider range (lane 1 below p * (1 + t * 2^-29) on BN254, lanes >= 2 below 2p), and the compile-time alpha = 5 path.  The bounds
as exact rationals, the primitives on the narrow-limb toy fields, and the alpha = 5 device code on the CPU against the oracle."""
import ctypes as C
import os
import random
import subprocess
from fractions import Fraction as Fr
from math import isqrt

import numpy as np
import pytest

from helpers import ROOT, build_host_shim, synth_elems
from oracle import cref, fields as OF
from test_poseidon_lane1_basis import random_config
from test_poseidon_scaled_lane0 import FID, _arrays, _P

FIELDS = ["bls12_381_fr", "bn254_fr", "jubjub_fr", "bls12_377_fr"]
R = 1 << 256
W = 32


def top_limb_bound(p):
    """p < (p[7] + 1) * 2^224: the top-limb form the constexpr predicates of fp.cuh decide on."""
    return ((p >> 224) + 1) << 224


# ---------------------------------------------------------------------------------------------------- bounds, exact rationals
@pytest.mark.parametrize("fname", FIELDS)
def test_squaring_window_needs_no_overflow_word(fname):
    """fp_sqr: limb i + 7 of T = a^2 enters at row i, limb 15 after the last row.  After row i the window holds
    (T mod 2^(32(i+8)) + M*p) / 2^(32i) with M < 2^(32(i+1)), for ANY a < 2^256."""
    p = OF.MODULI[fname]
    assert p < R - (1 << 224)                                               # the static_assert of fp_sqr
    for i in range(8):
        window = ((1 << (32 * (i + 8))) - 1 + ((1 << (32 * (i + 1))) - 1) * p) // (1 << (32 * i))
        assert window < 1 << 288
    # the result, (T + M*p) / R, is below 2p for a < p and for the lazy operands (a^2 < R*p): limb 7 takes T's limb 15 uncarried
    assert Fr((p - 1) ** 2 + (R - 1) * p, R) < 2 * p < R
    if fname == "bn254_fr":
        assert (2 * p) ** 2 < R * p                                         # lane 0 below 2p is a lazy operand


def row2_needs_x(p, terms, unit, w=W):
    """detail::tab_row2_needs_x<F, T, U> of csrc/fp.cuh"""
    top = (p >> (7 * w)) + 1
    return top * (1 + unit) + ((top * (8 * terms + 1) + (1 << w) - 1) >> w) > 1 << w


@pytest.mark.parametrize("fname", FIELDS)
def test_dot_tab_second_row_bound(fname):
    """Where tab_row2_needs_x is false, the second reduction row stays below 2^288 and the result below 2^256."""
    p = OF.MODULI[fname]
    for terms in range(1, 10):
        for unit in (0, 1, 2):
            v_max = 8 * terms * (2**32 - 1) * (p - 1) + (unit * p - 1 if unit else 0) * 2**64
            after_row2 = (v_max + (2**32 - 1) * p) // 2**32 + (2**32 - 1) * p
            if not row2_needs_x(p, terms, unit):
                assert after_row2 < 1 << 288
                assert after_row2 // 2**32 < R
                assert top_limb_bound(p) * (8 * terms + 1 + (1 + unit) * 2**32) <= 1 << 320
    bn, bls = OF.MODULI["bn254_fr"], OF.MODULI["bls12_381_fr"]
    assert not row2_needs_x(bn, 3, 0) and not row2_needs_x(bn, 1, 2)        # both BN254 t = 3 partial-round products
    assert not row2_needs_x(bls, 3, 0) and not row2_needs_x(bls, 1, 1) and row2_needs_x(bls, 1, 2)


def tab_result_bound(p, terms, unit):
    """fp_dot_tab's value before its conditional subtractions, over p: (V + M*p) / (2^64 p) with y < unit * p."""
    v_max = 8 * terms * (2**32 - 1) * (p - 1) + (unit * p - 1 if unit else 0) * 2**64
    return Fr(v_max + (2**64 - 1) * p, 2**64 * p)


@pytest.mark.parametrize("fname", FIELDS)
def test_wide_lane_invariants(fname):
    """Lanes >= 2 in [0, 2p): the column update takes s_j < 2p as its unit addend (U = 2) and one pass by 2p returns it below 2p.
    Every lane is an operand of fp_dot_tab (any value below 2^256), and one pass by p makes it canonical at the loop's exit."""
    p = OF.MODULI[fname]
    b = tab_result_bound(p, 1, 2)
    assert b < 3 + Fr(1, 2**29) <= 4                                          # one pass by 2p (tab_reduce_passes<1, 2> == 1) ...
    assert b - 2 < 2                                                          # ... leaves it below 2p
    assert 2 * p < R                                                          # an fp_dot_tab operand
    assert 2 * p - 1 - p < p                                                  # the exit's fp_final_sub


def sbox5_bounds(x_over_p, rho):
    """Lazy products of x^5 = (x^2)^2 * x with Montgomery factor rho = p/R: (a*b + M*p)/R < p*(a*b*rho + 1) (in units of p)."""
    x2 = x_over_p * x_over_p * rho + 1
    x4 = x2 * x2 * rho + 1
    x5 = x4 * x_over_p * rho + 1
    return x2, x4, x5


def test_bn254_lane1_invariant():
    """Lane 1 (BN254, LZ): a' = the dot's result with its one conditional subtraction skipped, below p * (1 + t * 2^-29); its
    only addition d = xi + a' stays below 3p, which fp_add_lazy's two passes (2p, then p) make canonical, so x = d + c < 2p as
    before.  xi = x^5 for x < 2p, the lazy S-box chain."""
    p = OF.MODULI["bn254_fr"]
    rho = Fr(p, R)
    _, _, xi = sbox5_bounds(Fr(2), rho)
    assert xi < Fr(16, 10)
    for t in (2, 3):                                                          # LZ holds for t <= 3 on BN254 (no dot overflow word)
        a = tab_result_bound(p, t, 0)
        assert a < 1 + Fr(t, 2**29) < 2                                      # tab_reduce_passes<t, 0> == 0: no pass at all
        assert xi + a < 3                                                     # fp_add_lazy's precondition
        assert 3 * p < R
    # the lazy S-box operands: both squarings take a^2 < R*p, the product's full operand x^4 needs x^4 + p < 2^256
    x2, x4, _ = sbox5_bounds(Fr(2), rho)
    assert (2 * p) ** 2 < R * p and (x2 * p) ** 2 < R * p and x4 * p + p < R


def test_toy_widths_keep_the_wide_lane_bounds():
    """The narrow-limb model (w = 8) has the same pass counts: U = 2 below 4p, U = 0 below 2p."""
    for terms in (1, 2, 3, 4, 9):
        assert Fr(8 * terms * 2**8, 2**16) + 1 + 2 <= 4
        assert Fr(8 * terms * 2**8, 2**16) + 1 <= 2


# ---------------------------------------------------------------------------------------------------- toy fields
@pytest.fixture(scope="module")
def toy():
    from test_fp_toy import W as TW, write_header
    out_dir = os.path.join(ROOT, "tests", "host", "_build")
    os.makedirs(out_dir, exist_ok=True)
    mods = write_header(os.path.join(out_dir, "toy_fields.h"))
    so = os.path.join(out_dir, "alu_toy_shim.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", f"-DCPB_LIMB_BITS={TW}", "-I", out_dir, "-x", "c++",
                           os.path.join(ROOT, "tests", "host", "alu_toy_shim.cpp"), "-o", so])
    lib = C.CDLL(so)
    assert lib.toy_field_count() == len(mods)
    return lib, mods


TOY_CASES = ["sqr", "tab3_U0_lazy", "tab1_U2_lazy", "tab4_U2_lazy", "tab9_U0_lazy", "tab1_U2", "tab2_U2"]


@pytest.mark.parametrize("idx", range(9))
def test_xless_and_wide_range_primitives_on_narrow_limbs(toy, idx):
    """fp_sqr without the overflow word for operands up to sqrt(R*p) (lazy) and p (canonical); fp_dot_tab with a unit addend
    below 2p and with the pass by p skipped, all-ones limb patterns included."""
    lib, mods = toy
    name, p, _ = mods[idx]
    out = (C.c_long * 7)()
    lib.toy_check_alu(idx, C.c_ulonglong(4242 + idx), C.c_long(60000), out)
    assert {n: int(v) for n, v in zip(TOY_CASES, out) if v} == {}, (name, hex(p))


# ---------------------------------------------------------------------------------------------------- device code, alpha = 5
@pytest.mark.parametrize("t", range(2, 10))
@pytest.mark.parametrize("fname", FIELDS)
def test_alpha5_path_device_code_matches_oracle(fname, t):
    """pos_hash_single<F, T, A5 = true> (the kernel launch_crh_ft picks for alpha = 5) on the digit tables, odd RF (4 full rounds
    before the partial ones, 5 after), sparse and dense schedules.  Inputs include p - 1; the first partial round's constants
    are p - 1 - i."""
    lib = build_host_shim("poseidon_alpha5_shim")
    p = OF.MODULI[fname]
    cfg = random_config(p, t, 9, 13, 5, 5000 * t + FID[fname])
    arkm, mdsm = _arrays(cfg)
    rate = t - 1
    for sparse in (1, 0):
        n = 10
        inp = synth_elems(11 * t, (n, rate), p)
        inp[0, :] = cref.ints_to_mont([p - 1] * rate, p)
        out = np.zeros((n, 4), dtype=np.uint64)
        rc = lib.host_poseidon_crh_alpha5(FID[fname], rate, 1, 9, 13, _P(arkm), _P(mdsm), sparse, _P(np.ascontiguousarray(inp)),
                                          C.c_long(rate), C.c_long(n), _P(out))
        assert rc == sparse, (fname, t, sparse)
        assert np.array_equal(out, cref.Poseidon(cfg).crh_batch(inp)), (fname, t, sparse)


def test_bn254_lazy_sbox_on_operands_near_2p():
    """The partial-round S-box of BN254 (lazy products) on x just below 2p, on x whose square has all-ones upper limbs, and on
    random x < 2p: congruent to x^5 (Montgomery) and below 1.6p."""
    lib = build_host_shim("poseidon_alpha5_shim")
    p = OF.MODULI["bn254_fr"]
    rnd = random.Random(254)
    xs = [2 * p - 1 - i for i in range(64)] + [p, p - 1, 0, 1]
    while len(xs) < 400:                                                     # x^2 with all-ones limbs 8..15
        x = rnd.randrange(1, 2 * p)
        if ((x * x) >> 256) & 0xFFFFFFFF == 0xFFFFFFFF or rnd.random() < 0.5:
            xs.append(x)
    for k in range(160, 2 * p.bit_length()):                                 # the largest x with x^2 < 2^k, inside [0, 2p)
        x = isqrt((1 << k) - 1)
        if x < 2 * p:
            xs.append(x)
    xa = np.array([[(x >> (32 * i)) & 0xFFFFFFFF for i in range(8)] for x in xs], dtype=np.uint32)
    out = np.zeros_like(xa)
    lib.host_bn254_sbox5_lazy(xa.ctypes.data_as(C.POINTER(C.c_uint32)), C.c_long(len(xs)), out.ctypes.data_as(C.POINTER(C.c_uint32)))
    rinv = pow(R, -1, p)
    for x, row in zip(xs, out):
        got = sum(int(w) << (32 * i) for i, w in enumerate(row))
        assert got % p == pow(x, 5, p) * pow(rinv, 4, p) % p, hex(x)
        assert Fr(got, p) < Fr(16, 10), hex(x)
