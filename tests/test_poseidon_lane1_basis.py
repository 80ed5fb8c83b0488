"""Sparse partial rounds with lane 1 carried as a = w_hat . s (csrc/poseidon_host.hpp: derive_schedule; csrc/poseidon.cuh:
pos_permute_split; DESIGN §4.2).  The split loop's region of the schedule against the same algebra redone in Python integers, a
Python model of the split loop on the product's schedule against the oracle permutation, the dense fallback when a row's
w_hat[1] is zero, the CPU model of the device code at every width, fp_add_lazy against Python integers, and the lazy bounds of
the new round with exact rationals."""
import ctypes as C
import random
from fractions import Fraction as Fr

import numpy as np
import pytest

from helpers import ALL_CONFIGS, build_host_shim, oracle_config, synth_elems
from oracle import cref, fields as OF, poseidon as OP
from test_poseidon_scaled_lane0 import BN254, FID, R, _arrays, _P, needs_x, reduce_passes, schedule


def regions(o, v, t, rf, rp):
    """The schedule's regions as lists of field integers (offsets as derive_schedule lays them out)."""
    q = 2 * t - 2
    lp = v[o["off_sc0"] + 1:o["n_elems"]]
    return {
        "C": v[o["off_c"]:o["off_c"] + rf * t], "M": v[o["off_m"]:o["off_m"] + t * t],
        "Mpre": v[o["off_mpre"]:o["off_mpre"] + t * t], "Mpost": v[o["off_mpre"] + t * t:o["off_mpre"] + 2 * t * t],
        "Cp0": v[o["off_cp0"]:o["off_cp0"] + t], "pc": v[o["off_pc"]:o["off_pc"] + rp],
        "sp": [v[o["off_sp"] + k * (2 * t - 1):o["off_sp"] + (k + 1) * (2 * t - 1)] for k in range(rp)],
        "lp": [lp[k * q:(k + 1) * q] for k in range(rp)], "entry_row": lp[rp * q:rp * q + t], "entry_c": lp[rp * q + t:],
    }


def random_config(p, t, rf, rp, alpha, seed):
    rnd = random.Random(seed)
    ark = [[rnd.randrange(p) for _ in range(t)] for _ in range(rf + rp)]
    ark[rf // 2] = [p - 1 - i for i in range(t)]                            # the largest constants, in the first partial round
    mds = [[rnd.randrange(1, p) for _ in range(t)] for _ in range(t)]
    return OP.PoseidonConfig(p, rf, rp, alpha, ark, mds, t - 1, 1)


# ---------------------------------------------------------------------------------------------------- the schedule's new region
@pytest.mark.parametrize("which", ALL_CONFIGS)
def test_lane1_region_is_the_basis_change_of_the_sparse_rows(which):
    fname, cfg = oracle_config(which)
    p, t, rf, rp = cfg.p, cfg.rate + cfg.capacity, cfg.full_rounds, cfg.partial_rounds
    o, v = schedule(FID[fname], cfg)
    assert o["sparse"] == 1
    assert o["n_elems"] == o["off_sc0"] + 1 + rp * (2 * t - 2) + t + 1
    g = regions(o, v, t, rf, rp)
    inv = lambda x: pow(x, -1, p)                                             # noqa: E731
    w = [row[:t] for row in g["sp"]] + [[1, 1] + [0] * (t - 2)]            # w_hat_k[1..t-1] at index 1..; w_hat_rp = e_1
    vs = [row[t:] for row in g["sp"]]                                        # v_k[1..t-1] at index 0..
    for k in range(rp):
        wk, wn = w[k], w[k + 1]
        assert wk[1] != 0
        alpha = wn[1] * inv(wk[1]) % p
        beta = [(wn[j] - alpha * wk[j]) % p for j in range(2, t)]
        gamma = sum(wn[j] * vs[k][j - 1] for j in range(1, t)) % p
        assert g["lp"][k] == [gamma, alpha] + beta + vs[k][1:], k
    Mpre, Cp0 = g["Mpre"], g["Cp0"]
    assert g["entry_row"] == [sum(w[0][j] * Mpre[j * t + i] for j in range(1, t)) % p for i in range(t)]
    assert g["entry_c"] == [sum(w[0][j] * Cp0[j] for j in range(1, t)) % p]


def split_model(g, cfg, state):
    """pos_permute_split in Python integers on the product's schedule (no PermuteHint)."""
    p, t, rf, rp, al = cfg.p, cfg.rate + cfg.capacity, cfg.full_rounds, cfg.partial_rounds, cfg.alpha
    half = rf // 2
    s = list(state)

    def full(fr, mat, entry):
        nonlocal s
        s = [pow((s[i] + g["C"][fr * t + i]) % p, al, p) for i in range(t)]
        rows = [mat[i * t:(i + 1) * t] for i in range(t)]
        if entry:
            rows[1] = g["entry_row"]
        s = [sum(r[j] * s[j] for j in range(t)) % p for r in rows]

    for fr in range(half):
        full(fr, g["Mpre"] if fr == half - 1 else g["M"], fr == half - 1)
    s = [(s[i] + (g["entry_c"][0] if i == 1 else g["Cp0"][i])) % p for i in range(t)]
    for k in range(rp):
        c = g["lp"][k]
        y = pow(s[0], al, p)
        a = (c[0] * y + sum(c[j] * s[j] for j in range(1, t))) % p
        d = (y + s[1]) % p
        for j in range(2, t):
            s[j] = (s[j] + c[t + j - 2] * y) % p
        s[0] = (d + g["pc"][k + 1]) % p if k + 1 < rp else d
        s[1] = a
    for fr in range(half, rf):
        full(fr, g["Mpost"] if fr == half else g["M"], False)
    return s


MODEL_CASES = [(w, None) for w in ALL_CONFIGS] + [("bls12_381_fr", t) for t in range(2, 10)] + [("bn254_fr", t) for t in (2, 3, 4)]


@pytest.mark.parametrize("which,t", MODEL_CASES)
def test_split_model_on_the_schedule_matches_oracle_permutation(which, t):
    if t is None:
        fname, cfg = oracle_config(which)
    else:
        fname = which
        p = OF.MODULI[fname]
        cfg = random_config(p, t, 8, 13, 5, 40 + t)
    o, v = schedule(FID[fname], cfg)
    assert o["sparse"] == 1
    tt = cfg.rate + cfg.capacity
    g = regions(o, v, tt, cfg.full_rounds, cfg.partial_rounds)
    rnd = random.Random(7)
    for _ in range(3):
        st = [rnd.randrange(cfg.p) for _ in range(tt)]
        assert split_model(g, cfg, st) == OP.permute(cfg, st)
    assert split_model(g, cfg, [0] * tt) == OP.permute(cfg, [0] * tt)


# ---------------------------------------------------------------------------------------------------- fallback
@pytest.fixture(scope="module", params=["merged", "split"])
def shim(request):
    split = request.param == "split"
    return build_host_shim("poseidon_host_shim", defines=[f"CPB_POS_SPLIT={int(split)}"], tag="_" + request.param)


def test_zero_w_hat1_falls_back_to_dense_and_matches_oracle(shim):
    """t = 2: w_hat_k[1] = M[0][1] / N_k[1][1], so M[0][1] = 0 leaves lane 1 no basis to change to: the schedule must be dense
    (with M[0][0] != 0 and the minors invertible, i.e. for this reason only), and the digests still the oracle's."""
    rnd = random.Random(9)
    for p, fid in ((OF.BLS12_381_FR, 0), (OF.BN254_FR, 1)):
        rate, rf, rp, alpha = 1, 8, 9, 5
        ark = [[rnd.randrange(p) for _ in range(2)] for _ in range(rf + rp)]
        for m01, sparse in ((0, 0), (rnd.randrange(1, p), 1)):
            mds = [[rnd.randrange(1, p), m01], [rnd.randrange(1, p), rnd.randrange(1, p)]]
            cfg = OP.PoseidonConfig(p, rf, rp, alpha, ark, mds, rate, 1)
            assert schedule(fid, cfg)[0]["sparse"] == sparse
            arkm, mdsm = _arrays(cfg)
            inp = synth_elems(19, (16, rate), p)
            out = np.zeros((16, 4), dtype=np.uint64)
            rc = shim.host_poseidon_crh(fid, rate, 1, rf, rp, C.c_ulonglong(alpha), _P(arkm), _P(mdsm), 1, _P(np.ascontiguousarray(inp)),
                                        C.c_long(rate), C.c_long(16), _P(out))
            assert rc == sparse and np.array_equal(out, cref.Poseidon(cfg).crh_batch(inp)), (hex(p), m01)


# ---------------------------------------------------------------------------------------------------- device code, every width
@pytest.mark.parametrize("t", range(2, 10))
def test_split_loop_device_code_every_width(t):
    """The device's split loop compiled for the CPU (PTX emulated) at every instantiated width and field, sparse schedule,
    against the oracle: BN254 with alpha = 5 runs lazy at t <= 3; inputs include p - 1, round constants p - 1 - i."""
    shim = build_host_shim("poseidon_widths_shim", defines=["CPB_POS_SPLIT=1"])
    for fname, alpha in (("bls12_381_fr", 5), ("bn254_fr", 5), ("jubjub_fr", 5), ("bls12_377_fr", 11)):
        p = OF.MODULI[fname]
        cfg = random_config(p, t, 8, 21, alpha, 100 * t + FID[fname])
        arkm, mdsm = _arrays(cfg)
        rate, n = t - 1, 24
        inp = synth_elems(t, (n, rate), p)
        inp[0, :] = cref.ints_to_mont([p - 1] * rate, p)
        out = np.zeros((n, 4), dtype=np.uint64)
        rc = shim.host_poseidon_crh_any_width(FID[fname], rate, 1, 8, 21, C.c_ulonglong(alpha), _P(arkm), _P(mdsm),
                                              _P(np.ascontiguousarray(inp)), C.c_long(rate), C.c_long(n), _P(out))
        assert rc == 1 and np.array_equal(out, cref.Poseidon(cfg).crh_batch(inp)), fname


# ---------------------------------------------------------------------------------------------------- fp_add_lazy
def _limbs(xs):
    return np.array([[(x >> (32 * i)) & 0xFFFFFFFF for i in range(8)] for x in xs], dtype=np.uint32)


def test_add_lazy_bn254_against_integers():
    lib = build_host_shim("add_lazy_shim")
    p = BN254
    rnd = random.Random(13)
    edge = [(2 * p - 1, p - 1), (2 * p - 1, 0), (p, p - 1), (p - 1, 1), (0, 0), (2 * p - 2, 2), (p - 1, p - 1), (0, p - 1)]
    pairs = edge + [(rnd.randrange(2 * p), rnd.randrange(p)) for _ in range(20000)]
    pairs += [(2 * p - 1 - rnd.randrange(1 << 40), p - 1 - rnd.randrange(1 << 40)) for _ in range(2000)]
    a, b = _limbs([x for x, _ in pairs]), _limbs([y for _, y in pairs])
    r = np.zeros_like(a)
    u32p = C.POINTER(C.c_uint32)
    lib.host_add_lazy_bn254(a.ctypes.data_as(u32p), b.ctypes.data_as(u32p), r.ctypes.data_as(u32p), C.c_long(len(pairs)))
    got = [sum(int(w) << (32 * i) for i, w in enumerate(row)) for row in r]
    assert got == [(x + y) % p for x, y in pairs]


# ---------------------------------------------------------------------------------------------------- bounds, exact rationals
def test_lane1_round_chain_bn254_lazy():
    """One lazy partial round (F::LAZY5, alpha = 5, t <= 3), in units of p: x = d + c < 2p on entry, and again on exit."""
    rho = Fr(BN254, R)
    mont = lambda a, b: a * b * rho + 1                     # noqa: E731  (bound of an unreduced Montgomery product)
    x = Fr(2)
    assert x * x * rho < 1                                  # lazy squaring: x^2 < R*p
    y = mont(mont(mont(x, x), mont(x, x)), x)               # xi = x^5, no conditional subtractions
    assert y < Fr(16, 10)
    assert y + 1 < 1 / rho                                  # column products v_j * xi: full operand xi + p < R
    for t in (2, 3):
        # a' = fp_dot<F, t, EX = 1>: xi is the one unreduced term, every other lane canonical
        assert y + (t - 1) < t + 1
        assert not needs_x(BN254, t + 1)                    # (t + 2) * p < R: no overflow word
        value = (y + (t - 1)) * rho + 1                     # (sum_j a_j*b_j + M*p)/R, b_j canonical
        k = reduce_passes(BN254, t + 1, 0)                  # dot_reduce_passes<F, t + 1>
        assert k == 0 and value <= 2 ** (k + 1) and 2 ** (k + 1) * rho < 1
    d = y + 1                                               # d = xi + a, a canonical: fp_add_lazy
    assert d < 3 and 3 * rho < 1                            # its 8-limb sum does not overflow; 2p then p makes it canonical
    assert 1 + 1 <= x                                       # x' = d + c with d, c canonical: the bound the round started from
