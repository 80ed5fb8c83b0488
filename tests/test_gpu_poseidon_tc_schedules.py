"""The tensor-core BN254 Fr hash kernel (k_poseidon_crh_tc) on every kind of schedule the C-ABI sends it, not only the
benchmark's RF = 8, RP = 57.  cpb_poseidon_ctx_create routes every BN254 Fr, t = 3, alpha = 5 configuration whose factorisation
is sparse to that kernel, for any RF >= 2 and RP >= 1, and the kernel's control flow forks on both:

  * RF: the entry round (Mpre and the entry row) is full round RF/2 - 1, so at RF in {2, 3} it is also the first round, where
    lane 0's S-box is the schedule constant S(c0) (first_j and entry in one round of pos_permute_split); odd RF puts one more
    round after the partial rounds than before them.
  * RP: the CTA's ring of partial-round tables (TcRing) takes slot g mod 2 and parity (g / 2) mod 2 of g = batch * RP + k, so
    an odd RP alternates the slot a round starts in from batch to batch, RP = 1 refills a slot with its own round
    (tc_ring_next(0, 1) = 0), and the CTA's last round g_end - 1 decides which copies are never issued.
  * Past the grid cap (SMs x occupancy x 64 CTAs of 128 hashes) CTAs loop over batches and differ in g_end.

Each configuration asserts cpb_poseidon_ctx_is_sparse, so none silently reaches the integer kernel instead, and the digests are
compared bit for bit with the C oracle at every one-permutation (len, n_out) shape and at batch sizes that end in partial warps
and partly idle CTAs.  A defect in any of the forks above -- a wrong ring slot or parity after a batch boundary, a refill of
the wrong round, the entry row applied in the wrong round, S(c0) and the entry round mixed up -- gives wrong digests here.  The
short-RF schedules also run through the other kernels of the family (the tree-top team kernel, the alpha = 5 integer kernel,
the Merkle build and the ragged kernels), and RF in {2, 3} runs through every kernel of one width of each other field."""
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest

from helpers import ROOT, synth_elems
from crypto_primitives_b200 import _native as N
from crypto_primitives_b200 import ragged as RG
from crypto_primitives_b200.crh.poseidon import CRH, TwoToOneCRH
from crypto_primitives_b200.merkle_tree import MerkleTree
from crypto_primitives_b200.sponge.poseidon import absorb_squeeze_batch
from oracle import cref, fields as OF, poseidon as OP
import test_gpu_poseidon_instances as instances
from test_gpu_poseidon_instances import THREADS, inputs, oracle_ragged, oracle_sponge, product, random_config
from test_poseidon_scaled_lane0 import FID, schedule

P = OF.BN254_FR


# ------------------------------------------------------------------------------------------------------------- configurations
def _edge_ark(rf, rp, seed):
    """Random constants with whole rows of 0 and p - 1 and rows that mix them (the first and last full rounds, the entry round,
    the first and last partial rounds)."""
    cfg = random_config(P, 3, 5, 1, rf, rp, seed=seed)
    ark = [list(r) for r in cfg.ark]
    half = rf // 2
    ark[0] = [0, P - 1, 0]
    ark[half - 1] = [P - 1, P - 1, P - 1]
    ark[half] = [0, 0, 0]
    ark[half + rp - 1] = [P - 1, 0, P - 1]
    ark[-1] = [0, 0, P - 1]
    return OP.PoseidonConfig(P, rf, rp, 5, ark, cfg.mds, 2, 1)


SMALL_MDS = [[2, 1, 1], [1, 2, 1], [1, 1, 3]]


def _config(name):
    kind, rest = name.split(":")
    vals = dict(kv.split("=") for kv in rest.split(","))
    rf, rp, cap = int(vals["rf"]), int(vals["rp"]), int(vals.get("cap", 1))
    seed = 254000 + 1000 * rf + rp + 100 * cap
    if kind == "random":
        return random_config(P, 3, 5, cap, rf, rp, seed=seed)
    if kind == "grain":                                        # the Grain LFSR constants of traits.rs, as the benchmark's
        ark, mds = OP.find_poseidon_ark_and_mds(P, 254, 2, rf, rp, 0)
        return OP.PoseidonConfig(P, rf, rp, 5, ark, mds, 2, 1)
    if kind == "small_mds":
        cfg = random_config(P, 3, 5, 1, rf, rp, seed=seed)
        return OP.PoseidonConfig(P, rf, rp, 5, cfg.ark, SMALL_MDS, 2, 1)
    if kind == "edge_ark":
        return _edge_ark(rf, rp, seed)
    raise KeyError(name)


CONFIGS = ([f"random:rf={rf},rp=57" for rf in (2, 3, 4, 5, 6, 7, 10)]
           + [f"random:rf=8,rp={rp}" for rp in (1, 2, 3, 4, 5, 8, 31, 32, 33, 56, 58, 64, 65, 128)]
           + [f"random:rf={rf},rp={rp},cap=2" for rf, rp in ((2, 1), (3, 2), (8, 57))]
           + ["grain:rf=8,rp=56", "grain:rf=8,rp=60", "small_mds:rf=8,rp=57", "edge_ark:rf=8,rp=57", "edge_ark:rf=3,rp=5"])
NS = (1, 31, 32, 33, 97, 127, 128, 129, 4097)
_cache = {}


def config(name):
    if name not in _cache:
        ocfg = _config(name)
        _cache[name] = (ocfg, product("bn254_fr", ocfg))
    return _cache[name]


def shapes(ocfg):
    """Every one-permutation (absorbed elements, squeezed elements) pair: len <= rate, 1 <= n_out <= rate."""
    return [(L, k) for L in range(ocfg.rate + 1) for k in range(1, ocfg.rate + 1)]


def _seed(name, n, L):
    return 40000 + 7919 * CONFIGS.index(name) + 10 * n + L


# ------------------------------------------------------------------------------------------------------------- CPU: the matrix is sparse
@pytest.mark.parametrize("name", CONFIGS + ["random:rf=2,rp=2", "random:rf=3,rp=3", "random:rf=8,rp=4"])
def test_every_configuration_has_a_sparse_schedule(name):
    """The host schedule of every configuration here is the sparse one, so the device runs it on the tensor-core kernel (the
    GPU tests assert the same through the context)."""
    ocfg = _config(name)
    o, _ = schedule(FID["bn254_fr"], ocfg)
    assert o["sparse"] == 1 and o["t"] == 3


# ------------------------------------------------------------------------------------------------------------- GPU: every shape
@pytest.mark.gpu
@pytest.mark.parametrize("name", CONFIGS)
def test_tc_kernel_schedule_every_shape(name):
    ocfg, cfg = config(name)
    assert N.lib.cpb_poseidon_ctx_is_sparse(cfg.context(0)) == 1, "the configuration does not reach the tensor-core kernel"
    O = cref.Poseidon(ocfg)
    for n in NS:
        for L in range(ocfg.rate + 1):
            x = inputs(P, n, L, _seed(name, n, L))
            if L:
                assert np.array_equal(CRH.evaluate_batch(cfg, x), O.crh_batch(x, threads=THREADS)), ("crh", n, L)
            for L_, k in shapes(ocfg):
                if L_ == L:
                    assert np.array_equal(absorb_squeeze_batch(cfg, x, k), oracle_sponge(O, ocfg, x, k)), (n, L, k)


# ------------------------------------------------------------------------------------------------------------- GPU: past the grid cap
BIG = [(2, 1), (2, 2), (3, 3), (8, 4)]
BIG_N = (1 << 23) + 37
_BIG_CHILD = """
import sys
import numpy as np
sys.path.insert(0, {root!r}); sys.path.insert(0, {tests!r})
from test_gpu_poseidon_tc_schedules import big_case
from crypto_primitives_b200.crh.poseidon import CRH
for rf, rp in {big!r}:
    _, cfg, x = big_case(rf, rp)
    np.save({out!r} + "_%d_%d.npy" % (rf, rp), CRH.evaluate_batch(cfg, x))
"""


def big_case(rf, rp):
    name = f"random:rf={rf},rp={rp}"
    ocfg, cfg = config(name)
    return ocfg, cfg, inputs(P, BIG_N, 2, 70000 + 100 * rf + rp)


@pytest.mark.gpu
def test_tc_kernel_past_the_grid_cap(tmp_path):
    """n = 2^23 + 37, past the grid cap of an H100 (132 SMs x 5 CTAs x 64 x 128 hashes): CTAs loop over batches, and the last
    batch leaves them with different numbers of rounds (g_end), so the ring's slots and parities run across batch boundaries.
    Every digest against the alpha = 5 integer kernel (CPB_POS_TC=0, in a child process since the switch is read once), and 4096
    random rows plus the first and last 256 against the C oracle."""
    out = str(tmp_path / "int")
    code = _BIG_CHILD.format(root=ROOT, tests=os.path.join(ROOT, "tests"), big=BIG, out=out)
    subprocess.run([sys.executable, "-c", code], env=dict(os.environ, CPB_POS_TC="0"), check=True)
    for rf, rp in BIG:
        ocfg, cfg, x = big_case(rf, rp)
        assert N.lib.cpb_poseidon_ctx_is_sparse(cfg.context(0)) == 1
        got = CRH.evaluate_batch(cfg, x)
        ref = np.load(f"{out}_{rf}_{rp}.npy")
        assert np.array_equal(got, ref), ("integer kernel", rf, rp, int(np.nonzero((got != ref).any(axis=1))[0][0]))
        idx = np.unique(np.concatenate([np.random.default_rng(rf * 100 + rp).integers(0, BIG_N, 4096), np.arange(256),
                                        np.arange(BIG_N - 256, BIG_N)]))
        assert np.array_equal(got[idx], cref.Poseidon(ocfg).crh_batch(np.ascontiguousarray(x[idx]), threads=THREADS)), ("oracle", rf, rp)
        del x, got, ref


# ------------------------------------------------------------------------------------------------------------- GPU: short RF, other kernels
SHORT = ["random:rf=2,rp=57", "random:rf=3,rp=57", "edge_ark:rf=3,rp=5"]
TWO_NS = (1, 33, 4096)


@pytest.mark.gpu
@pytest.mark.parametrize("name", SHORT)
def test_short_rf_team_merkle_and_ragged(name):
    """RF in {2, 3} through the tree-top team kernel (the two-to-one shape at n <= 4096), a 2^13-leaf Merkle build, and a ragged
    batch (one-permutation and sponge ragged kernels in one call)."""
    ocfg, cfg = config(name)
    O = cref.Poseidon(ocfg)
    for n in TWO_NS:
        pairs = inputs(P, n, 2, _seed(name, n, 7))
        assert np.array_equal(TwoToOneCRH.compress_batch(cfg, pairs), O.compress_batch(pairs, threads=THREADS)), ("two-to-one", n)
    leaves = inputs(P, 1 << 13, 2, _seed(name, 8192, 8))
    tree = MerkleTree.new(cfg, cfg, leaves)
    exp_leaf, exp_nodes = cref.poseidon_merkle(O, O, leaves, threads=THREADS)
    assert np.array_equal(tree.leaf_nodes, exp_leaf) and np.array_equal(tree.non_leaf_nodes, exp_nodes), "tree"
    rnd = random.Random(_seed(name, 0, 9))
    lens = [rnd.choice((0, 1, 2, 3, 5)) for _ in range(1000)]
    vals = synth_elems(_seed(name, 1, 9), (sum(lens) + 1, ), P)
    parts = [vals[a:a + L] for a, L in zip(np.cumsum([0] + lens[:-1]), lens)]
    assert np.array_equal(CRH.evaluate_ragged(cfg, *RG.pack(parts)), oracle_ragged(O, parts)), "ragged crh"


_AGREE_CHILD = """
import json, sys
import numpy as np
sys.path.insert(0, {root!r}); sys.path.insert(0, {tests!r})
from test_gpu_poseidon_tc_schedules import config
from crypto_primitives_b200.crh.poseidon import TwoToOneCRH
from crypto_primitives_b200.sponge.poseidon import absorb_squeeze_batch
d = np.load({inp!r})
out = {{}}
for name, L, k, n in json.loads({jobs!r}):
    x = d["x_%s_%d_%d" % (name, L, n)]
    out["%s_%d_%d_%d" % (name, L, k, n)] = absorb_squeeze_batch(config(name)[1], x, k)
    if L == 2 and k == 1:
        out["two_%s_%d" % (name, n)] = TwoToOneCRH.compress_batch(config(name)[1], x)
np.savez({out!r}, **out)
"""


@pytest.mark.gpu
def test_short_rf_kernels_agree(tmp_path):
    """The short-RF schedules in child processes (the switches are read once per process): CPB_TEAM_MAX=0 sends the two-to-one
    shape at n <= 4096 to the tensor-core kernel instead of the team kernel; with CPB_POS_TC=0 as well the alpha = 5 integer kernel
    runs everything.  Both against the C oracle."""
    ns = (33, 4096)
    jobs = [(nm, L, k, n) for nm in SHORT for n in ns for L, k in shapes(config(nm)[0])]
    xs = {f"x_{nm}_{L}_{n}": inputs(P, n, L, _seed(nm, n, L) + 3) for nm in SHORT for n in ns for L in range(3)}
    inp = str(tmp_path / "in.npz")
    np.savez(inp, **xs)
    exp = {}
    for nm, L, k, n in jobs:
        ocfg = config(nm)[0]
        exp[(nm, L, k, n)] = oracle_sponge(cref.Poseidon(ocfg), ocfg, xs[f"x_{nm}_{L}_{n}"], k)
    for tag, env in (("tc", {"CPB_TEAM_MAX": "0"}), ("int", {"CPB_TEAM_MAX": "0", "CPB_POS_TC": "0"})):
        out = str(tmp_path / f"out_{tag}.npz")
        code = _AGREE_CHILD.format(root=ROOT, tests=os.path.join(ROOT, "tests"), inp=inp, jobs=json.dumps(jobs), out=out)
        subprocess.run([sys.executable, "-c", code], env=dict(os.environ, **env), check=True)
        got = np.load(out)
        for nm, L, k, n in jobs:
            assert np.array_equal(got[f"{nm}_{L}_{k}_{n}"], exp[(nm, L, k, n)]), (tag, nm, L, k, n)
            if L == 2 and k == 1:
                assert np.array_equal(got[f"two_{nm}_{n}"], exp[(nm, L, k, n)][:, 0]), (tag, "two-to-one", nm, n)


# ------------------------------------------------------------------------------------------------------------- GPU: short RF, other fields
SHORT_RF_PAIRS = [("bls12_381_fr", 3), ("jubjub_fr", 4), ("bls12_377_fr", 5)]
SHORT_RF_VARIANTS = {"rf2": (lambda t: 5, 1, 2, None, False, 1), "rf3": (lambda t: 5, 1, 3, None, False, 1)}


@pytest.mark.parametrize("variant", list(SHORT_RF_VARIANTS))
@pytest.mark.parametrize("fname,t", SHORT_RF_PAIRS)
def test_short_rf_other_fields_are_sparse(monkeypatch, fname, t, variant):
    for name, v in SHORT_RF_VARIANTS.items():
        monkeypatch.setitem(instances.VARIANTS, name, v)
    ocfg = instances.case_config(fname, t, variant)[0]
    assert ocfg.full_rounds == int(variant[2:]) and schedule(FID[fname], ocfg)[0]["sparse"] == 1


@pytest.mark.gpu
@pytest.mark.parametrize("variant", list(SHORT_RF_VARIANTS))
@pytest.mark.parametrize("fname,t", SHORT_RF_PAIRS)
def test_short_rf_other_fields_every_kernel(monkeypatch, fname, t, variant):
    """RF in {2, 3} (random constants, RP in 1..13, sparse) as two more variants of the instance matrix of
    test_gpu_poseidon_instances.py, run through its own body: every kernel of the field's unit against the C oracle.  The entry
    round is then the first round, the one that meets S(c0), in the split loop every field shares."""
    for name, v in SHORT_RF_VARIANTS.items():
        monkeypatch.setitem(instances.VARIANTS, name, v)
    instances.test_instance_matches_oracle(fname, t, variant)
