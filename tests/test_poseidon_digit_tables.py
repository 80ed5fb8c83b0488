"""Products by schedule constants through pre-reduced digit tables (csrc/fp.cuh: fp_dot_tab; csrc/poseidon_host.hpp: the tables of
derive_schedule; csrc/poseidon.cuh: pos_permute_split; DESIGN §4.1).  The primitive on narrow-limb toy fields (every carry path,
operands up to 2^64 - 1 at 8-bit limbs) and at full width against Python integers, the table region of every named config against
the same algebra in Python integers, the CPU model of the device code on the tables at every field and width (sparse and dense,
odd RF, one-permutation and sponge forms) against the oracle, and the result bounds with exact rationals."""
import ctypes as C
import os
import random
import subprocess
from fractions import Fraction as Fr

import numpy as np
import pytest

from helpers import ALL_CONFIGS, ROOT, build_host_shim, oracle_config, synth_elems
from oracle import cref, fields as OF
from test_poseidon_lane1_basis import random_config, regions
from test_poseidon_scaled_lane0 import FID, _arrays, _P, needs_x, schedule

u32p = C.POINTER(C.c_uint32)
FIELDS = ["bls12_381_fr", "bn254_fr", "jubjub_fr", "bls12_377_fr"]


# ---------------------------------------------------------------------------------------------------- toy fields
@pytest.fixture(scope="module")
def toy():
    from test_fp_toy import W, write_header
    out_dir = os.path.join(ROOT, "tests", "host", "_build")
    os.makedirs(out_dir, exist_ok=True)
    mods = write_header(os.path.join(out_dir, "toy_fields.h"))
    so = os.path.join(out_dir, "dot_tab_toy_shim.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", f"-DCPB_LIMB_BITS={W}", "-I", out_dir, "-x", "c++",
                           os.path.join(ROOT, "tests", "host", "dot_tab_toy_shim.cpp"), "-o", so])
    lib = C.CDLL(so)
    assert lib.toy_field_count() == len(mods)
    return lib, mods


TOY_CASES = [f"{t}terms_U{u}" for u in (0, 1) for t in (1, 2, 3, 4, 9)]


@pytest.mark.parametrize("idx", range(9))
def test_dot_tab_on_narrow_limbs(toy, idx):
    lib, mods = toy
    name, p, _ = mods[idx]
    out = (C.c_long * 10)()
    lib.toy_check_dot_tab(idx, C.c_ulonglong(9876 + idx), C.c_long(60000), out)
    assert {n: int(v) for n, v in zip(TOY_CASES, out) if v} == {}, (name, hex(p))


# ---------------------------------------------------------------------------------------------------- full width
R = 1 << 256


def _limbs(xs):
    return np.array([[(x >> (32 * i)) & 0xFFFFFFFF for i in range(8)] for x in xs], dtype=np.uint32)


@pytest.mark.parametrize("fname", FIELDS)
def test_dot_tab_full_width_against_integers(fname):
    lib = build_host_shim("poseidon_tables_shim")
    p = OF.MODULI[fname]
    rinv = pow(R, -1, p)
    rnd = random.Random(FID[fname])
    edge_a = [R - 1, p - 1, p, 2 * p - 1, 0, 1, int("ffffffff" * 8, 16) - (1 << 128), int("ffffffff00000000" * 4, 16)]
    edge_c = [p - 1, 0, 1, p - 2]
    for nt in (1, 2, 3):
        for unit in (0, 1):
            n = 400
            a = [[rnd.choice(edge_a) if rnd.random() < 0.4 else rnd.randrange(R) for _ in range(nt)] for _ in range(n)]
            c = [[rnd.choice(edge_c) if rnd.random() < 0.3 else rnd.randrange(p) for _ in range(nt)] for _ in range(n)]
            y = [(rnd.choice([p - 1, 0, p - 2]) if rnd.random() < 0.3 else rnd.randrange(p)) if unit else 0 for _ in range(n)]
            aa = _limbs([x for row in a for x in row])
            cc = np.array([[(x >> (64 * i)) & (2**64 - 1) for i in range(4)] for row in c for x in row], dtype=np.uint64)
            yy, r = _limbs(y), np.zeros((n, 8), dtype=np.uint32)
            assert lib.host_dot_tab(FID[fname], nt, unit, aa.ctypes.data_as(u32p), _P(cc), yy.ctypes.data_as(u32p), C.c_long(n),
                                    r.ctypes.data_as(u32p)) == 0
            got = [sum(int(w) << (32 * i) for i, w in enumerate(row)) for row in r]
            want = [(sum(x * k for x, k in zip(a[i], c[i])) * rinv + y[i]) % p for i in range(n)]
            assert got == want, (fname, nt, unit)


# ---------------------------------------------------------------------------------------------------- the table region
def digit_rows(c, p):
    """K_0(c) .. K_7(c) of a plain constant c, each as its 32-bit limbs in the stored order 1, 3, 5, 7, 0, 2, 4, 6."""
    out = []
    for i in range(8):
        k = c * (1 << (32 * i + 64)) % p
        limbs = [(k >> (32 * m)) & 0xFFFFFFFF for m in range(8)]
        out.append([limbs[m] for m in (1, 3, 5, 7, 0, 2, 4, 6)])
    return out


@pytest.mark.parametrize("which", ALL_CONFIGS)
def test_digit_tables_are_the_schedule_constants_pre_reduced(which):
    fname, cfg = oracle_config(which)
    p, t, rf, rp = cfg.p, cfg.rate + cfg.capacity, cfg.full_rounds, cfg.partial_rounds
    o, v = schedule(FID[fname], cfg)
    assert o["sparse"] == 1
    g = regions(o, v, t, rf, rp)
    consts = g["M"] + g["Mpre"] + g["Mpost"] + [x for row in g["lp"] for x in row] + g["entry_row"]
    lib = build_host_shim("poseidon_tables_shim")
    ark, mds = _arrays(cfg)
    args = (FID[fname], cfg.rate, cfg.capacity, rf, rp, C.c_ulonglong(cfg.alpha), _P(ark), _P(mds))
    n = lib.host_poseidon_digit_tables(*args, None, C.c_long(0))
    assert n == 8 * len(consts) == 8 * (3 * t * t + rp * (2 * t - 2) + t)
    tabs = np.zeros((n, 4), dtype=np.uint64)
    assert lib.host_poseidon_digit_tables(*args, _P(tabs), C.c_long(n)) == n
    got = tabs.view(np.uint32).reshape(len(consts), 8, 8).tolist()
    assert got == [digit_rows(c, p) for c in consts]


# ---------------------------------------------------------------------------------------------------- device code, every width
@pytest.mark.parametrize("t", range(2, 10))
@pytest.mark.parametrize("fname,alpha", [("bls12_381_fr", 5), ("bn254_fr", 5), ("jubjub_fr", 5), ("bls12_377_fr", 11),
                                         ("bls12_381_fr", 17)])
def test_table_path_device_code_matches_oracle(fname, alpha, t):
    """pos_permute_split on the digit tables (BN254 with alpha = 5 runs its lazy lanes at t <= 3), the one-permutation and the
    sponge form, odd RF (4 full rounds before the partial ones, 5 after); the dense schedule of the same config for contrast.
    Inputs include p - 1; the first partial round's constants are p - 1 - i."""
    lib = build_host_shim("poseidon_tables_shim")
    p = OF.MODULI[fname]
    cfg = random_config(p, t, 9, 13, alpha, 1000 * t + alpha + FID[fname])
    arkm, mdsm = _arrays(cfg)
    rate = t - 1
    for sparse in (1, 0):
        for length, sponge in ((rate, 0), (2 * rate + 1, 1)):
            n = 10
            inp = synth_elems(7 * t + length, (n, length), p)
            inp[0, :] = cref.ints_to_mont([p - 1] * length, p)
            out = np.zeros((n, 4), dtype=np.uint64)
            rc = lib.host_poseidon_crh_tables(FID[fname], rate, 1, 9, 13, C.c_ulonglong(alpha), _P(arkm), _P(mdsm), sparse,
                                              _P(np.ascontiguousarray(inp)), C.c_long(length), C.c_long(n), sponge, _P(out))
            assert rc == sparse, (fname, t, sparse)
            assert np.array_equal(out, cref.Poseidon(cfg).crh_batch(inp)), (fname, t, sparse, sponge)


# ---------------------------------------------------------------------------------------------------- bounds, exact rationals
BOUND_FIELDS = {f: OF.MODULI[f] for f in FIELDS}


def tab_reduce_passes(terms, unit, w=32):
    """detail::tab_reduce_passes<T, U> of csrc/fp.cuh"""
    k = 0
    while ((1 + unit) << (w - 3)) + terms > 1 << (k + 1 + w - 3):
        k += 1
    return k


@pytest.mark.parametrize("fname", FIELDS)
def test_dot_tab_bounds(fname):
    """V = sum_j sum_i a_j[i] * K_i(c_j) + y * 2^64 for a_j < 2^256, K_i < p, y < p; two rows add M*p with M < 2^64."""
    p = BOUND_FIELDS[fname]
    for terms in range(1, 10):
        for unit in (0, 1):
            v_max = 8 * terms * (2**32 - 1) * (p - 1) + unit * (p - 1) * 2**64
            assert v_max + (2**64 - 1) * p < 2**320                      # 10 limbs: E, O and the overflow word
            if not unit and not needs_x(p, 8 * terms):                   # no overflow word: the first row stays below 2^288
                assert v_max + (2**32 - 1) * p < 2**288
            bound = Fr(v_max + (2**64 - 1) * p, 2**64 * p)               # result / p after the two rows
            assert bound < 1 + unit + Fr(terms, 2**29)
            k = tab_reduce_passes(terms, unit)
            assert k == unit and bound <= 2 ** (k + 1)                  # reduce9<F, K> leaves a canonical value
            assert 2 ** (k + 1) * p < 2**288                            # its 9-limb comparisons hold 2^(K+1) p


def test_consumers_take_the_lazy_lanes_bn254():
    """BN254 alpha = 5 (LAZY5): the lanes fp_dot_tab reads below 2^256 whatever their lazy bound, and the column's unit addend s_j
    canonical.  y = x^5 < 1.6p (tests/test_poseidon_lane1_basis.py), full-round S-box outputs < 1.24p."""
    p = OF.MODULI["bn254_fr"]
    assert Fr(16, 10) * p < R and Fr(124, 100) * p < R
    assert tab_reduce_passes(1, 1) == 1 and tab_reduce_passes(3, 0) == 0    # column: canonical s_j'; dot rows: canonical


def test_toy_widths_keep_the_same_passes():
    """The toy-field model (8-bit limbs: 2^w = 2^8) needs the same number of conditional subtractions as 32-bit limbs."""
    for terms in (1, 2, 3, 4, 9):
        for unit in (0, 1):
            assert Fr(8 * terms * 2**8, 2**16) + 1 + unit <= 2 ** (tab_reduce_passes(terms, unit, 8) + 1)
            assert tab_reduce_passes(terms, unit, 8) == tab_reduce_passes(terms, unit)
