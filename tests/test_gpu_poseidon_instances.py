"""Every compiled Poseidon kernel instance on the GPU against the C oracle, bit for bit.

The library instantiates its Poseidon kernels for four fields x state widths t = 2..9 (CPB_POS_WIDTHS), and the code inside them
forks at compile time on the field and the width (lazy bounds for BN254 Fr at t <= 4, wide lanes everywhere but BLS12-381 Fr, the
unrolled or rolled column update, x^5 or the bit loop) and at run time on the schedule (the split loop of a sparse schedule, the
merged loop of a dense one).  Here every (field, t) pair runs a generated matrix of configurations through every kernel of its
field unit -- one-permutation CRH, sponge, multi-lane squeeze, bare permutation, two-to-one (and the tree-top kernel at t = 3),
ragged CRH, Merkle build, path verification and ragged path verification -- together with the BN254 Fr t = 3, alpha = 5 family
(tensor-core and integer alpha = 5 kernels) at every one-permutation shape, and the argument paths of widths that are not built.
"""
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest

from helpers import ROOT, crafted_sbox_inputs, oracle_config, product_config, synth_elems
import crypto_primitives_b200 as cp
from crypto_primitives_b200 import _native as N
from crypto_primitives_b200 import ragged as R
from crypto_primitives_b200.crh.poseidon import CRH, TwoToOneCRH, permute_batch
from crypto_primitives_b200.merkle_tree import MerkleTree, PoseidonFieldConfig, verify_paths_batch
from crypto_primitives_b200.sponge.poseidon import absorb_squeeze_batch
from oracle import cref, fields as OF, poseidon as OP

pytestmark = pytest.mark.gpu

THREADS = os.cpu_count() or 8
FIELD_NAMES = ["bls12_381_fr", "bn254_fr", "jubjub_fr", "bls12_377_fr"]


# ------------------------------------------------------------------------------------------------------------- configurations
def random_config(p, t, alpha, cap=1, rf=8, rp=None, dense=False, seed=0):
    """Random MDS and round constants in the shape of test_poseidon_lane1_basis.random_config: RP in 1..13 unless given, the
    largest constants in the first partial round.  dense: M[0][0] = 0, or at t = 2 M[0][1] = 0 (w_hat_1 = 0), either of which
    makes the host schedule fall back to the dense form."""
    rnd = random.Random(seed)
    if rp is None:
        rp = rnd.randrange(1, 14)
    ark = [[rnd.randrange(p) for _ in range(t)] for _ in range(rf + rp)]
    if rp:
        ark[rf // 2] = [p - 1 - i for i in range(t)]
    mds = [[rnd.randrange(1, p) for _ in range(t)] for _ in range(t)]
    if dense:
        mds[0][1 if t == 2 else 0] = 0
    return OP.PoseidonConfig(p, rf, rp, alpha, ark, mds, t - cap, cap)


def product(fname, ocfg):
    return cp.PoseidonConfig.from_ints(cp.FIELDS[fname], ocfg.full_rounds, ocfg.partial_rounds, ocfg.alpha, ocfg.mds, ocfg.ark,
                                       ocfg.rate, ocfg.capacity)


# variant -> (alpha(t), capacity, RF, RP (None: random), dense tweak, the schedule the host must derive: 1 sparse / 0 dense)
VARIANTS = {
    "a5": (lambda t: 5, 1, 8, None, False, 1),
    "a17": (lambda t: 17, 1, 8, None, False, 1),               # the bit-loop S-box
    "a3": (lambda t: 3, 1, 8, None, False, 1),                 # BN254 Fr, t <= 4: the lazy path must stay off
    "dense": (lambda t: 5 if t % 2 == 0 else 17, 1, 8, None, True, 0),
    "rp0": (lambda t: 5, 1, 8, 0, False, 0),                   # no partial rounds: dense
    "cap2": (lambda t: 5, 2, 8, None, False, 1),
    "odd_rf": (lambda t: 5, 1, 7, 1, False, 1),                # floor(RF/2) full rounds before, ceil(RF/2) after
}
RP0_PAIRS = [("bls12_381_fr", 2), ("bn254_fr", 3), ("jubjub_fr", 5), ("bls12_377_fr", 8)]
ODD_RF_PAIRS = [("bls12_381_fr", 9), ("bn254_fr", 4), ("jubjub_fr", 3), ("bls12_377_fr", 6)]


def _cases():
    out = []
    for f in FIELD_NAMES:
        for t in range(2, 10):
            out += [(f, t, "a5"), (f, t, "a17")]
            if f == "bn254_fr" and t <= 4:
                out.append((f, t, "a3"))
            out.append((f, t, "dense"))
            if t >= 3:
                out.append((f, t, "cap2"))
            if (f, t) in RP0_PAIRS:
                out.append((f, t, "rp0"))
            if (f, t) in ODD_RF_PAIRS:
                out.append((f, t, "odd_rf"))
    return out


CASES = _cases()


def case_config(fname, t, variant):
    alpha, cap, rf, rp, dense, sparse = VARIANTS[variant]
    seed = 100000 * FIELD_NAMES.index(fname) + 1000 * t + list(VARIANTS).index(variant)
    ocfg = random_config(OF.MODULI[fname], t, alpha(t), cap, rf, rp, dense, seed)
    return ocfg, product(fname, ocfg), sparse, seed


# ------------------------------------------------------------------------------------------------------------- inputs, oracle
def inputs(p, n, L, seed):
    """(n, L, 4) Montgomery limbs; row 0 all p - 1, row 1 all zero."""
    x = np.ascontiguousarray(synth_elems(seed, (n, max(L, 1)), p)[:, :L])
    if L and n > 1:
        x[0] = cref.ints_to_mont([p - 1] * L, p)
        x[1] = 0
    return x


def _add_mont(a, b, p):
    """(a + b) mod p on Montgomery limbs (the Montgomery map is additive)."""
    v = (OF.from_limbs(a) + OF.from_limbs(b)) % p
    return np.array(OF.to_limbs(v), dtype=np.uint64)


def oracle_sponge(O, ocfg, x, n_out):
    """PoseidonSponge::new -> absorb(x[i]) -> squeeze_native_field_elements(n_out) for every row, each permutation on the C oracle
    (R/sponge/poseidon/mod.rs:124-186, 323-345): fill `rate` lanes and permute while more input remains, permute once to leave
    absorbing mode, then read `rate` lanes per permutation."""
    n, L = x.shape[:2]
    rate, cap = ocfg.rate, ocfg.capacity
    if n_out == 1:
        return O.crh_batch(x, threads=THREADS)[:, None]
    out = np.empty((n, n_out, 4), dtype=np.uint64)
    for i in range(n):
        s = np.zeros((rate + cap, 4), dtype=np.uint64)
        pos = 0
        while True:
            k = min(rate, L - pos)
            for j in range(k):
                s[cap + j] = _add_mont(s[cap + j], x[i, pos + j], ocfg.p)
            pos += k
            if pos == L:
                break
            s = O.permute(s)
        got = 0
        while got < n_out:
            s = O.permute(s)
            k = min(rate, n_out - got)
            out[i, got:got + k] = s[cap:cap + k]
            got += k
    return out


def oracle_ragged(O, parts):
    vals, off = R.pack(parts)
    off = off.astype(np.int64)
    lens = np.diff(off)
    out = np.empty((lens.size, 4), dtype=np.uint64)
    for L in np.unique(lens):
        idx = np.nonzero(lens == L)[0]
        out[idx] = O.crh_batch(vals[off[idx][:, None] + np.arange(L)[None, :]], threads=THREADS)
    return out


def oracle_levels(O, digests):
    """The inner nodes (heap order) over given leaf digests (R/merkle_tree/mod.rs:424-523) with the C oracle's two-to-one."""
    n = digests.shape[0]
    nodes = np.empty((n - 1, 4), dtype=np.uint64)
    start = n // 2 - 1
    nodes[start:] = O.compress_batch(np.ascontiguousarray(digests.reshape(-1, 2, 4)), threads=THREADS)
    while start > 0:
        upper, start = start, (start - 1) // 2
        nodes[start:upper] = O.compress_batch(np.ascontiguousarray(nodes[upper:2 * upper + 1].reshape(-1, 2, 4)), threads=THREADS)
    return nodes


def _other(a, b):
    assert not np.array_equal(a, b)
    return b.copy()


# ------------------------------------------------------------------------------------------------------------- the matrix
@pytest.mark.parametrize("fname,t,variant", CASES, ids=[f"{f}-t{t}-{v}" for f, t, v in CASES])
def test_instance_matches_oracle(fname, t, variant):
    ocfg, cfg, sparse, seed = case_config(fname, t, variant)
    p, rate, cap = ocfg.p, ocfg.rate, ocfg.capacity
    assert N.lib.cpb_poseidon_ctx_is_sparse(cfg.context(0)) == sparse, "the case does not reach the schedule it is meant for"
    O = cref.Poseidon(ocfg)

    # CRH, one permutation (and the sponge kernel past `rate` elements)
    for L in sorted({0, 1, rate, rate + 1, 2 * rate + 1}):
        x = inputs(p, 97, L, seed + L)
        assert np.array_equal(CRH.evaluate_batch(cfg, x), O.crh_batch(x, threads=THREADS)), ("crh", L)
    if cap == 1 and rate >= 2:
        x = crafted_sbox_inputs(ocfg, 64, seed=seed)
        if rate > 2:
            x = np.concatenate([x, synth_elems(seed + 50, (64, rate - 2), p)], axis=1)
        x = np.ascontiguousarray(x)
        assert np.array_equal(CRH.evaluate_batch(cfg, x), O.crh_batch(x, threads=THREADS)), "crafted S-box operands"

    # several lanes squeezed: one permutation for n_out <= rate, the sponge kernel past it
    x = inputs(p, 97, rate, seed + 60)
    for n_out in sorted({2, rate, rate + 1}):
        got = absorb_squeeze_batch(cfg, x, n_out)
        assert np.array_equal(got, oracle_sponge(O, ocfg, x, n_out)), ("squeeze", n_out)
        if n_out > rate:
            for i in (0, 1, 50):
                sp = OP.PoseidonSponge(ocfg)
                sp.absorb(cref.mont_to_ints(x[i], p))
                assert cref.mont_to_ints(got[i], p) == sp.squeeze_native_field_elements(n_out), ("sponge state machine", n_out, i)

    # bare permutation
    st = synth_elems(seed + 70, (65, t), p)
    st[0] = cref.ints_to_mont([p - 1] * t, p)
    assert np.array_equal(permute_batch(cfg, st), np.stack([O.permute(s) for s in st])), "permute"

    # ragged CRH: the one-permutation and the sponge ragged kernels in one call
    rnd = random.Random(seed)
    lens = [rnd.choice(sorted({0, 1, rate - 1, rate, rate + 1, 2 * rate + 1})) for _ in range(100)]
    vals = synth_elems(seed + 80, (sum(lens) + 1, ), p)
    parts = [vals[a:a + L] for a, L in zip(np.cumsum([0] + lens[:-1]), lens)]
    assert np.array_equal(CRH.evaluate_ragged(cfg, *R.pack(parts)), oracle_ragged(O, parts)), "ragged crh"

    if rate < 2:
        return
    # two-to-one; at t = 3, capacity 1 also the tree-top kernel (<= 4096 hashes) and the one-hash kernel past it
    for n in (97, 4096, 5000) if (t == 3 and cap == 1) else (97,):
        pairs = inputs(p, n, 2, seed + 90 + n)
        assert np.array_equal(TwoToOneCRH.compress_batch(cfg, pairs), O.compress_batch(pairs, threads=THREADS)), ("two-to-one", n)

    # Merkle tree (leaf hash = node hash) node for node, then every path through the one-launch verify kernel
    leaves = inputs(p, 64, rate, seed + 100)
    tree = MerkleTree.new(cfg, cfg, leaves)
    exp_leaf, exp_nodes = cref.poseidon_merkle(O, O, leaves, threads=THREADS)
    assert np.array_equal(tree.leaf_nodes, exp_leaf) and np.array_equal(tree.non_leaf_nodes, exp_nodes), "tree"
    sib, paths, idx = tree.generate_proofs_batch(np.arange(64))
    assert tree.verify_proofs_batch((sib, paths, idx), leaves).all(), "verify"
    bad_leaves = leaves.copy()
    bad_leaves[5, 0] = _other(leaves[5, 0], leaves[6, 0])
    bad_sib = sib.copy()
    bad_sib[9] = _other(sib[9], sib[10])
    bad_paths = paths.copy()
    bad_paths[20, 1] = _other(paths[20, 1], paths[20, 2])
    for (s_, p_, lv), bad in (((sib, paths, bad_leaves), 5), ((bad_sib, paths, leaves), 9), ((sib, bad_paths, leaves), 20)):
        ok = tree.verify_proofs_batch((s_, p_, idx), lv)
        assert not ok[bad] and ok[np.arange(64) != bad].all(), ("tampered verify", bad)
    proofs = [tree.generate_proof(i) for i in range(64)]
    assert verify_paths_batch(cfg, cfg, tree.root(), leaves, proofs).all(), "verify_paths_batch"
    ok = verify_paths_batch(cfg, cfg, tree.root(), bad_leaves, proofs)
    assert not ok[5] and ok[np.arange(64) != 5].all(), "verify_paths_batch, tampered leaf"
    proofs[9].leaf_sibling_hash = bad_sib[9]
    ok = verify_paths_batch(cfg, cfg, tree.root(), leaves, proofs)
    assert not ok[9] and ok[np.arange(64) != 9].all(), "verify_paths_batch, tampered sibling"

    # a tree over leaves of different lengths: the ragged leaf hash and the ragged verify kernel
    rlens = [rnd.choice((1, rate, rate + 1)) for _ in range(16)]
    rvals = synth_elems(seed + 110, (sum(rlens), ), p)
    rparts = [rvals[a:a + L] for a, L in zip(np.cumsum([0] + rlens[:-1]), rlens)]
    rtree = MerkleTree.new(cfg, cfg, rparts)
    exp_leaf = oracle_ragged(O, rparts)
    assert np.array_equal(rtree.leaf_nodes, exp_leaf) and np.array_equal(rtree.non_leaf_nodes, oracle_levels(O, exp_leaf)), "ragged tree"
    rproofs = rtree.generate_proofs_batch(np.arange(16))
    assert rtree.verify_proofs_batch(rproofs, rparts).all(), "ragged verify"
    bad = list(rparts)
    bad[3] = rparts[3].copy()
    bad[3][0] = _other(rparts[3][0], rvals[-1])
    ok = rtree.verify_proofs_batch(rproofs, bad)
    assert not ok[3] and ok[np.arange(16) != 3].all(), "ragged verify, tampered leaf"


# ------------------------------------------------------------------------------------------------------------- BN254 Fr, t = 3, alpha = 5
# The pair with kernels of its own: k_poseidon_crh_tc (tensor cores; sparse schedules, the default) and k_poseidon_crh<.., A5>
# (integer pipe; CPB_POS_TC=0, and every dense schedule, which builds no byte-digit tables and takes the merged loop).
BN_SHAPES = [(L, k) for L in (0, 1, 2) for k in (1, 2)]        # (absorbed elements, squeezed elements)
BN_NS = (1, 31, 33, 4097)
_bn_oracle = {}


def bn254_family(name):
    """-> (oracle config, product config, expected is_sparse)."""
    p = OF.BN254_FR
    if name == "bn254_r2":                                     # RP = 57, the Merkle benchmark's parameters
        return oracle_config("bn254_r2")[1], product_config("bn254_r2"), 1
    ocfg = {"rate1_cap2": lambda: random_config(p, 3, 5, cap=2, seed=254001),
            "dense": lambda: random_config(p, 3, 5, dense=True, seed=254002)}[name]()
    return ocfg, product("bn254_fr", ocfg), int(name != "dense")


def bn_inputs(name, L, n):
    return inputs(OF.BN254_FR, n, L, 9700 + 10 * L + n + 100000 * ["bn254_r2", "rate1_cap2", "dense"].index(name))


def bn_expected(name, L, k, n):
    key = (name, L, k, n)
    if key not in _bn_oracle:
        ocfg = bn254_family(name)[0]
        _bn_oracle[key] = oracle_sponge(cref.Poseidon(ocfg), ocfg, bn_inputs(name, L, n), k)
    return _bn_oracle[key]


@pytest.mark.parametrize("name", ["bn254_r2", "rate1_cap2", "dense"])
def test_bn254_t3_alpha5_every_shape(name):
    """Every (len, n_out) of one permutation the capacity allows (and, at rate 1, the sponge shapes next to them) at batch sizes
    that end in partial warps, through the default kernels: the tensor-core kernel for sparse schedules (two-row last round at
    n_out = 2; rate 1 with capacity 2), the alpha = 5 integer kernel's merged loop for the dense one."""
    ocfg, cfg, sparse = bn254_family(name)
    assert N.lib.cpb_poseidon_ctx_is_sparse(cfg.context(0)) == sparse
    for n in BN_NS:
        for L, k in BN_SHAPES:
            got = absorb_squeeze_batch(cfg, bn_inputs(name, L, n), k)
            assert np.array_equal(got, bn_expected(name, L, k, n)), (L, k, n)


_CHILD = """
import json, sys
import numpy as np
sys.path.insert(0, {root!r})
import crypto_primitives_b200 as cp
from crypto_primitives_b200.sponge.poseidon import absorb_squeeze_batch
d = np.load({inp!r})
cfgs, out = {{}}, {{}}
for name, L, k, n in json.loads({jobs!r}):
    if name not in cfgs:
        rf, rp, alpha, rate, cap = (int(v) for v in d["meta_" + name])
        cfgs[name] = cp.PoseidonConfig(cp.BN254_FR, rf, rp, alpha, d["mds_" + name], d["ark_" + name], rate, cap)
    out["%s_%d_%d_%d" % (name, L, k, n)] = absorb_squeeze_batch(cfgs[name], d["x_%s_%d_%d" % (name, L, n)], k)
np.savez({out!r}, **out)
"""


def test_bn254_t3_alpha5_kernels_agree(tmp_path):
    """The same batches in child processes (the switches are read once per process): CPB_TEAM_MAX=0 sends the two-to-one shape
    at n <= 4096 to the tensor-core kernel instead of the tree-top kernel; CPB_POS_TC=0 then runs the alpha = 5 integer kernel.
    Both equal the oracle, hence each other and the default kernels."""
    names = ["bn254_r2", "rate1_cap2", "dense"]
    jobs = [(nm, L, k, n) for nm in names for n in BN_NS for L, k in BN_SHAPES]
    arrays = {}
    for nm in names:
        ocfg, cfg, _ = bn254_family(nm)
        arrays["meta_" + nm] = np.array([cfg.full_rounds, cfg.partial_rounds, cfg.alpha, cfg.rate, cfg.capacity], dtype=np.int64)
        arrays["mds_" + nm], arrays["ark_" + nm] = cfg.mds, cfg.ark
        for n in BN_NS:
            for L in (0, 1, 2):
                arrays[f"x_{nm}_{L}_{n}"] = bn_inputs(nm, L, n)
    inp = str(tmp_path / "in.npz")
    np.savez(inp, **arrays)
    for tag, env in (("tc", {"CPB_TEAM_MAX": "0"}), ("int", {"CPB_TEAM_MAX": "0", "CPB_POS_TC": "0"})):
        out = str(tmp_path / f"out_{tag}.npz")
        code = _CHILD.format(root=ROOT, inp=inp, jobs=json.dumps(jobs), out=out)
        subprocess.run([sys.executable, "-c", code], env=dict(os.environ, **env), check=True)
        got = np.load(out)
        for nm, L, k, n in jobs:
            assert np.array_equal(got[f"{nm}_{L}_{k}_{n}"], bn_expected(nm, L, k, n)), (tag, nm, L, k, n)


# ------------------------------------------------------------------------------------------------------------- argument paths
@pytest.mark.parametrize("t", [10, 16])
def test_widths_without_kernels_are_unsupported(t):
    """rate + capacity <= 16 is a valid shape (the context and its schedule are built), but kernels exist for t = 2..9 only: every
    launch answers CPB_UNSUPPORTED and computes nothing."""
    p = OF.BLS12_381_FR
    ocfg = random_config(p, t, 5, rp=2, seed=1600 + t)
    cfg = product("bls12_381_fr", ocfg)
    assert cfg.context(0)
    x = inputs(p, 33, 2, t)
    four = MerkleTree(PoseidonFieldConfig(), np.zeros((4, 4), np.uint64), np.zeros((3, 4), np.uint64), cfg, cfg, 0)
    calls = {
        "crh": lambda: CRH.evaluate_batch(cfg, x),
        "sponge": lambda: absorb_squeeze_batch(cfg, x, 3),
        "permute": lambda: permute_batch(cfg, synth_elems(t, (5, t), p)),
        "two-to-one": lambda: TwoToOneCRH.compress_batch(cfg, x),
        "ragged": lambda: CRH.evaluate_ragged(cfg, *R.pack([x[0], x[1, :1], x[2]])),
        "tree": lambda: MerkleTree.new(cfg, cfg, x[:32]),
        "verify": lambda: four.verify_proofs_batch((x[:4, 0], np.zeros((4, 1, 4), np.uint64), np.arange(4, dtype=np.uint64)), x[:4]),
        "ragged verify": lambda: four.verify_proofs_batch((x[:4, 0], np.zeros((4, 1, 4), np.uint64), np.arange(4, dtype=np.uint64)),
                                                          [x[0], x[1, :1], x[2], x[3]]),
    }
    for what, call in calls.items():
        with pytest.raises(N.CpbError) as e:
            call()
        assert e.value.status == N.CPB_UNSUPPORTED, what
    big = random_config(p, 17, 5, rp=2, seed=1617)
    with pytest.raises(N.CpbError) as e:
        product("bls12_381_fr", big).context(0)
    assert e.value.status == N.CPB_BAD_PARAMS


def test_verify_with_leaf_and_node_widths_that_differ_is_unsupported():
    """The one-launch verify kernels are built for one width: a leaf hash of t = 4 under a t = 3 two-to-one builds (separate
    launches) but its paths answer CPB_UNSUPPORTED there, uniform and ragged; the level-synchronous verify_paths_batch takes them."""
    p = OF.JUBJUB_FR
    oleaf, onode = random_config(p, 4, 5, seed=41), random_config(p, 3, 5, seed=31)
    leaf, node = product("jubjub_fr", oleaf), product("jubjub_fr", onode)
    leaves = inputs(p, 8, 3, 7)
    tree = MerkleTree.new(leaf, node, leaves)
    exp_leaf, exp_nodes = cref.poseidon_merkle(cref.Poseidon(oleaf), cref.Poseidon(onode), leaves)
    assert np.array_equal(tree.leaf_nodes, exp_leaf) and np.array_equal(tree.non_leaf_nodes, exp_nodes)
    proofs = tree.generate_proofs_batch(np.arange(8))
    for lv in (leaves, [leaves[i, :1 + i % 3] for i in range(8)]):
        with pytest.raises(N.CpbError) as e:
            tree.verify_proofs_batch(proofs, lv)
        assert e.value.status == N.CPB_UNSUPPORTED
    assert verify_paths_batch(leaf, node, tree.root(), leaves, [tree.generate_proof(i) for i in range(8)]).all()
