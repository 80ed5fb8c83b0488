"""The tensor-core hash kernel's staged constants and its ring of partial-round tables (csrc/poseidon_host.hpp: tc_const_image;
csrc/poseidon_tc.cuh: tc_ring_slot, tc_ring_parity, tc_ring_next).  Every constant the kernel's path of pos_permute_split reads,
taken at its offset in the compact image, is the full schedule's element -- for the bench schedule and a random-constant BN254 Fr
t = 3 alpha = 5 sparse schedule -- and round g of the ring lands in the slot, phase and refill order the kernel assumes."""
import ctypes as C

import numpy as np
import pytest

from helpers import OF, build_host_shim, oracle_config
from test_poseidon_lane1_basis import random_config
from test_poseidon_scaled_lane0 import _arrays, _P

u64p = C.POINTER(C.c_uint64)


@pytest.fixture(scope="module")
def lib():
    return build_host_shim("poseidon_tc_ring_shim")


def configs():
    return {"bench": oracle_config("bn254_r2")[1], "random": random_config(OF.BN254_FR, 3, 8, 57, 5, seed=2024)}


@pytest.fixture(scope="module", params=["bench", "random"])
def cfg(request):
    return configs()[request.param]


def full_schedule(cfg):
    """(offsets, raw Montgomery limbs (n, 4)) of the product's schedule for cfg."""
    lib = build_host_shim("poseidon_schedule_shim")
    ark, mds = _arrays(cfg)
    offs = (C.c_int * 12)()
    args = (1, cfg.rate, cfg.capacity, cfg.full_rounds, cfg.partial_rounds, C.c_ulonglong(cfg.alpha), _P(ark), _P(mds), 1, offs)
    n = lib.host_poseidon_schedule(*args, None, C.c_long(0))
    consts = np.zeros((n, 4), dtype=np.uint64)
    assert lib.host_poseidon_schedule(*args, _P(consts), C.c_long(n)) == n
    names = ["t", "sparse", "off_c", "off_m", "off_mpre", "off_cp0", "off_pc", "off_sp", "off_arkp", "off_mod", "off_sc0", "n_elems"]
    return dict(zip(names, offs)), consts


def const_image(lib, cfg):
    ark, mds = _arrays(cfg)
    offs = (C.c_int * 6)()
    args = (cfg.rate, cfg.capacity, cfg.full_rounds, cfg.partial_rounds, C.c_ulonglong(cfg.alpha), _P(ark), _P(mds), offs)
    n = lib.host_tc_const_image(*args, None, C.c_long(0))
    assert n > 0
    img = np.zeros((n, 4), dtype=np.uint64)
    assert lib.host_tc_const_image(*args, img.ctypes.data_as(u64p), C.c_long(n)) == n
    return dict(zip(["off_c", "off_cp0", "off_pc", "off_mod", "off_sc0", "n_elems"], offs)), img


def test_image_holds_every_constant_the_tc_path_reads(lib, cfg):
    o, full = full_schedule(cfg)
    io, img = const_image(lib, cfg)
    t, rf, rp = 3, cfg.full_rounds, cfg.partial_rounds
    assert o["sparse"] == 1 and io["n_elems"] == img.shape[0]
    # full-round constants, rf x t
    assert np.array_equal(img[io["off_c"]:io["off_c"] + rf * t], full[o["off_c"]:o["off_c"] + rf * t])
    # S(c0), the modulus, and the lane-0 constants read after partial rounds 0 .. rp-2 (entries 1 .. rp-1)
    assert np.array_equal(img[io["off_sc0"]], full[o["off_sc0"]])
    assert np.array_equal(img[io["off_mod"]], full[o["off_mod"]])
    assert np.array_equal(img[io["off_pc"] + 1:io["off_pc"] + rp], full[o["off_pc"] + 1:o["off_pc"] + rp])
    # Cp0: lanes 0 and 2 as the schedule has them, lane 1 the entry constant in the w_hat_0 basis (after the lp rounds' rows and
    # the Mpre row 1 at off_sc0 + 1)
    lp_entry = o["off_sc0"] + 1 + rp * (2 * t - 2)
    assert np.array_equal(img[io["off_cp0"] + 0], full[o["off_cp0"] + 0])
    assert np.array_equal(img[io["off_cp0"] + 1], full[lp_entry + t])
    assert np.array_equal(img[io["off_cp0"] + 2], full[o["off_cp0"] + 2])
    # small enough that the kernel's CTA keeps room for its warp buffers, the R^-1 table and the ring at 6 CTAs per SM
    assert io["n_elems"] * 32 <= 3 * 1024


@pytest.mark.parametrize("rp", [57, 2, 3])
def test_ring_round_map(lib, rp):
    n = 4 * rp + 7
    out = (C.c_int * (3 * n))()
    S = lib.host_tc_ring_map(n, rp, out)
    assert S == 2
    rows = [tuple(out[3 * g:3 * g + 3]) for g in range(n)]
    for g, (slot, parity, nxt) in enumerate(rows):
        assert slot == g % S
        assert parity == (g // S) & 1                 # the phase of the slot's barrier that round g waits for
        assert nxt == (g % rp + S) % rp               # the table the refill after round g brings: round g + S's
    # consecutive uses of a slot alternate parity, so a wait never mistakes the previous phase for its own
    for g in range(n - S):
        assert rows[g][0] == rows[g + S][0] and rows[g][1] != rows[g + S][1]
