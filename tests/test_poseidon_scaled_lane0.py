"""Sparse partial rounds with lane 0 carried scaled (csrc/poseidon_host.hpp: derive_schedule; DESIGN §4.2): every sparse row's
lane-0 coefficient is one, the kernels form the row with fp_dot_unit (csrc/fp.cuh), and the first second-half full round takes
the scale out again through Mpost.  The schedule's layout, the dense fallback when M[0][0] = 0, the row primitive on narrow-limb
toy fields against 128-bit integers, and the lazy bounds of the new row with exact rationals.  The CPU model of the device code
on the new schedule against the oracle (both loop forms, the team kernel, crafted S-box operands) is tests/test_poseidon_host.py."""
import ctypes as C
import os
import random
import subprocess
from fractions import Fraction as Fr

import numpy as np
import pytest

from helpers import ALL_CONFIGS, ROOT, build_host_shim, oracle_config, synth_elems
from oracle import cref, fields as OF, poseidon as OP

u64p = C.POINTER(C.c_uint64)
FID = {"bls12_381_fr": 0, "bn254_fr": 1, "jubjub_fr": 2, "bls12_377_fr": 3}


def _P(a):
    return a.ctypes.data_as(u64p)


def _arrays(cfg):
    p = cfg.p
    return (cref.ints_to_mont([x for r in cfg.ark for x in r], p), cref.ints_to_mont([x for r in cfg.mds for x in r], p))


def schedule(fid, cfg, allow_sparse=1):
    """(offsets dict, constants as field integers) of the product's schedule for cfg."""
    lib = build_host_shim("poseidon_schedule_shim")
    ark, mds = _arrays(cfg)
    offs = (C.c_int * 12)()
    args = (fid, cfg.rate, cfg.capacity, cfg.full_rounds, cfg.partial_rounds, C.c_ulonglong(cfg.alpha), _P(ark), _P(mds), allow_sparse, offs)
    n = lib.host_poseidon_schedule(*args, None, C.c_long(0))
    assert n > 0
    consts = np.zeros((n, 4), dtype=np.uint64)
    assert lib.host_poseidon_schedule(*args, _P(consts), C.c_long(n)) == n
    names = ["t", "sparse", "off_c", "off_m", "off_mpre", "off_cp0", "off_pc", "off_sp", "off_arkp", "off_mod", "off_sc0", "n_elems"]
    o = dict(zip(names, offs))
    vals = cref.mont_to_ints(consts[:o["off_mod"]], cfg.p) + [0] + cref.mont_to_ints(consts[o["off_mod"] + 1:], cfg.p)
    return o, vals


@pytest.mark.parametrize("which", ALL_CONFIGS)
def test_sparse_rows_have_unit_lane0_coefficient(which):
    fname, cfg = oracle_config(which)
    p, t, rp = cfg.p, cfg.rate + cfg.capacity, cfg.partial_rounds
    o, v = schedule(FID[fname], cfg)
    assert o["sparse"] == 1
    assert [v[o["off_sp"] + k * (2 * t - 1)] for k in range(rp)] == [1] * rp
    assert v[o["off_m"]:o["off_m"] + t * t] == [x for r in cfg.mds for x in r]
    # Mpost (right after Mpre) = M * diag(lam^alpha, 1, ..., 1) with lam != 0
    mpost = v[o["off_mpre"] + t * t:o["off_mpre"] + 2 * t * t]
    M = cfg.mds
    scale = mpost[0] * pow(M[0][0], -1, p) % p
    assert scale != 0
    for i in range(t):
        assert mpost[i * t] == M[i][0] * scale % p
        assert mpost[i * t + 1:(i + 1) * t] == M[i][1:]
    assert o["off_cp0"] == o["off_mpre"] + 2 * t * t


def test_dense_schedule_stores_m_in_both_extra_matrix_slots():
    _, cfg = oracle_config("bn254_r2")
    t = cfg.rate + cfg.capacity
    o, v = schedule(1, cfg, allow_sparse=0)
    M = [x for r in cfg.mds for x in r]
    assert o["sparse"] == 0
    assert v[o["off_mpre"]:o["off_mpre"] + t * t] == M and v[o["off_mpre"] + t * t:o["off_mpre"] + 2 * t * t] == M


@pytest.fixture(scope="module", params=["merged", "split"])
def shim(request):
    split = request.param == "split"
    return build_host_shim("poseidon_host_shim", defines=[f"CPB_POS_SPLIT={int(split)}"], tag="_" + request.param)


def test_zero_m00_falls_back_to_dense_and_matches_oracle(shim):
    """lam_{k+1} = m00 * lam_k^alpha divides by m00: a matrix with M[0][0] = 0 must take the dense schedule, in the
    one-hash-per-thread code (both loop forms) and in the team-kernel model."""
    rnd = random.Random(5)
    for p, fid in ((OF.BLS12_381_FR, 0), (OF.BN254_FR, 1)):
        rate, rf, rp, alpha = 2, 8, 9, 5
        t = rate + 1
        ark = [[rnd.randrange(p) for _ in range(t)] for _ in range(rf + rp)]
        mds = [[rnd.randrange(1, p) for _ in range(t)] for _ in range(t)]
        mds[0][0] = 0
        cfg = OP.PoseidonConfig(p, rf, rp, alpha, ark, mds, rate, 1)
        arkm, mdsm = _arrays(cfg)
        inp = synth_elems(17, (16, rate), p)
        exp = cref.Poseidon(cfg).crh_batch(inp)
        out = np.zeros((16, 4), dtype=np.uint64)
        rc = shim.host_poseidon_crh(fid, rate, 1, rf, rp, C.c_ulonglong(alpha), _P(arkm), _P(mdsm), 1, _P(np.ascontiguousarray(inp)),
                                    C.c_long(rate), C.c_long(16), _P(out))
        assert rc == 0 and np.array_equal(out, exp)
        exp2 = cref.Poseidon(cfg).compress_batch(inp)
        rc = shim.host_poseidon_team_compress(fid, rf, rp, C.c_ulonglong(alpha), _P(arkm), _P(mdsm), 1, _P(np.ascontiguousarray(inp)),
                                              C.c_long(16), _P(out))
        assert rc == 0 and np.array_equal(out, exp2)
        mds[0][0] = 1                                      # any nonzero m00 keeps the sparse schedule
        cfg = OP.PoseidonConfig(p, rf, rp, alpha, ark, mds, rate, 1)
        arkm, mdsm = _arrays(cfg)
        rc = shim.host_poseidon_crh(fid, rate, 1, rf, rp, C.c_ulonglong(alpha), _P(arkm), _P(mdsm), 1, _P(np.ascontiguousarray(inp)),
                                    C.c_long(rate), C.c_long(16), _P(out))
        assert rc == 1 and np.array_equal(out, cref.Poseidon(cfg).crh_batch(inp))


# ---------------------------------------------------------------------------------------------------- fp_dot_unit, toy fields
@pytest.fixture(scope="module")
def toy():
    from test_fp_toy import W, write_header
    out_dir = os.path.join(ROOT, "tests", "host", "_build")
    os.makedirs(out_dir, exist_ok=True)
    mods = write_header(os.path.join(out_dir, "toy_fields.h"))
    so = os.path.join(out_dir, "dot_unit_toy_shim.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", f"-DCPB_LIMB_BITS={W}", "-I", out_dir, "-x", "c++",
                           os.path.join(ROOT, "tests", "host", "dot_unit_toy_shim.cpp"), "-o", so])
    lib = C.CDLL(so)
    assert lib.toy_field_count() == len(mods)
    return lib, mods


CASES = [f"{n}terms_unit<{xi}p" for xi in (1, 2) for n in (1, 2, 3, 4, 8)]


@pytest.mark.parametrize("idx", range(9))
def test_dot_unit_on_narrow_limbs(toy, idx):
    lib, mods = toy
    name, p, _ = mods[idx]
    out = (C.c_long * 10)()
    lib.toy_check_dot_unit(idx, C.c_ulonglong(4321 + idx), C.c_long(100000), out)
    assert {n: int(v) for n, v in zip(CASES, out) if v} == {}, (name, hex(p))


# ---------------------------------------------------------------------------------------------------- bounds, exact rationals
R = 1 << 256
BN254 = 0x30644e72e131a029b85045b68181585d2833e84879b9709143e1f593f0000001
BLS381 = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001


def reduce_passes(p, terms, unit):
    """detail::dot_reduce_passes<F, terms, unit> of csrc/fp.cuh (decided on the top 32-bit limb)"""
    top, k = p >> 224, 0
    while terms * (top + 1) > ((2 << k) - 1 - unit) * (1 << 32):
        k += 1
    return k


def needs_x(p, terms):
    """detail::dot_needs_x<F, terms>"""
    return (terms + 1) * ((p >> 224) + 1) > (1 << 32)


def test_unit_row_chain_bn254_lazy():
    rho = Fr(BN254, R)
    mont = lambda a, b: a * b * rho + 1                     # noqa: E731  (bound in units of p of an unreduced Montgomery product)
    x = Fr(2)                                               # x = L + c, L canonical (the row's result), c canonical
    assert x * rho < 1
    y = mont(mont(mont(x, x), mont(x, x)), x)               # xi = x^5 without conditional subtractions
    assert y < Fr(16, 10) and y < 2                         # within the declared unit bound XI = 2
    assert y + 1 < 1 / rho                                  # column products v_j * xi: full operand xi + p < R
    for t in (2, 3):
        assert t * rho <= 1 and not needs_x(BN254, t - 1)   # the (t-1)-term rows need no overflow word
        value = y + (t - 1) * rho + 1                       # xi + (sum_j s_j*w_j + M*p)/R, s_j and w_j canonical
        k = reduce_passes(BN254, t - 1, 2)
        assert k == 1 and value <= 2 ** (k + 1) and 2 + (t - 1) * rho + 1 <= 2 ** (k + 1)
        assert 2 ** (k + 1) * rho < 1                       # reduce9's input fits 256 bits: the ninth limb is zero


def test_unit_row_chain_bls12_381():
    rho = Fr(BLS381, R)
    value = 1 + 2 * rho + 1                                 # canonical xi + two canonical products, t = 3
    k = reduce_passes(BLS381, 2, 1)
    assert k == 1 and value <= 2 ** (k + 1)
    assert needs_x(BLS381, 2)                               # the rows keep their overflow word


def test_reduce_passes_never_undercount():
    """the top-limb rule against the exact bound xi + p*(n*p/R + 1) < 2^(K+1)*p for every field and shape the kernels use"""
    for p in (BLS381, BN254, OF.JUBJUB_FR, OF.BLS12_377_FR):
        for n in range(1, 9):
            for unit in (1, 2):
                k = reduce_passes(p, n, unit)
                assert unit + n * Fr(p, R) + 1 <= 2 ** (k + 1)
