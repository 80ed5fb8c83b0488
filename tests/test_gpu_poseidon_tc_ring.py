"""The tensor-core BN254 Fr hash kernel with its staged constant image and per-CTA ring of partial-round tables
(k_poseidon_crh_tc): batch sizes whose last CTA has 0 to 3 idle warps and a partly filled warp, every one-permutation (len, n_out)
shape, against the C oracle and against the integer-pipe kernel (CPB_POS_TC=0, in a child process since the switch is read once),
a sampled 2^23 batch, and a guard after the last output that must stay untouched."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from helpers import ROOT, oracle_config, product_config, synth_elems
from crypto_primitives_b200.crh.poseidon import CRH
from crypto_primitives_b200.sponge.poseidon import absorb_squeeze_batch
from oracle import cref
from test_gpu_poseidon_instances import oracle_sponge

pytestmark = pytest.mark.gpu

NS = (1, 32, 33, 95, 96, 97, 127, 128, 129)
SHAPES = [(L, k) for L in (0, 1, 2) for k in (1, 2)]          # (absorbed elements, squeezed elements)


def _inputs(n, L, seed, p):
    x = np.ascontiguousarray(synth_elems(seed, (n, max(L, 1)), p)[:, :L])
    if L and n > 1:
        x[0] = cref.ints_to_mont([p - 1] * L, p)               # largest canonical operands
        x[1] = 0
    return x


def _seed(n, L):
    return 31000 + 10 * n + L


def test_ring_kernel_every_shape_against_oracle():
    _, ocfg = oracle_config("bn254_r2")
    cfg = product_config("bn254_r2")
    O = cref.Poseidon(ocfg)
    for n in NS:
        for L, k in SHAPES:
            x = _inputs(n, L, _seed(n, L), ocfg.p)
            got = absorb_squeeze_batch(cfg, x, k)
            assert np.array_equal(got, oracle_sponge(O, ocfg, x, k)), (n, L, k)


_CHILD = """
import json, sys
import numpy as np
sys.path.insert(0, {root!r}); sys.path.insert(0, {tests!r})
from helpers import product_config
from crypto_primitives_b200.sponge.poseidon import absorb_squeeze_batch
d = np.load({inp!r})
cfg = product_config("bn254_r2")
np.savez({out!r}, **{{"%d_%d_%d" % (n, L, k): absorb_squeeze_batch(cfg, d["x_%d_%d" % (n, L)], k) for n, L, k in json.loads({jobs!r})}})
"""


def test_ring_kernel_matches_integer_kernel(tmp_path):
    _, ocfg = oracle_config("bn254_r2")
    cfg = product_config("bn254_r2")
    jobs = [(n, L, k) for n in NS for L, k in SHAPES]
    xs = {f"x_{n}_{L}": _inputs(n, L, _seed(n, L), ocfg.p) for n in NS for L in (0, 1, 2)}
    inp, out = str(tmp_path / "in.npz"), str(tmp_path / "out.npz")
    np.savez(inp, **xs)
    code = _CHILD.format(root=ROOT, tests=os.path.join(ROOT, "tests"), inp=inp, out=out, jobs=json.dumps(jobs))
    subprocess.run([sys.executable, "-c", code], env=dict(os.environ, CPB_POS_TC="0"), check=True)
    ref = np.load(out)
    for n, L, k in jobs:
        assert np.array_equal(absorb_squeeze_batch(cfg, xs[f"x_{n}_{L}"], k), ref["%d_%d_%d" % (n, L, k)]), (n, L, k)


def test_ring_kernel_at_2_23_sampled():
    _, ocfg = oracle_config("bn254_r2")
    cfg = product_config("bn254_r2")
    n = 1 << 23
    x = _inputs(n, 2, 31500, ocfg.p)
    got = CRH.evaluate_batch(cfg, x)
    idx = np.unique(np.concatenate([np.random.default_rng(23).integers(0, n, 4096), np.arange(n - 200, n), np.arange(200)]))
    assert np.array_equal(got[idx], cref.Poseidon(ocfg).crh_batch(np.ascontiguousarray(x[idx]), threads=8))


@pytest.mark.parametrize("n", [1, 33, 97, 129])
def test_ring_kernel_leaves_the_guard_after_the_outputs(n):
    import torch
    _, ocfg = oracle_config("bn254_r2")
    cfg = product_config("bn254_r2")
    x = _inputs(n, 2, _seed(n, 2), ocfg.p)
    guard = 64
    sentinel = 0x5A5A5A5A5A5A5A5A
    buf = torch.full((n + guard, 4), sentinel, dtype=torch.int64, device="cuda")
    CRH.evaluate_batch_dev(cfg, torch.from_numpy(x.view(np.int64)).cuda(), out=buf[:n])
    torch.cuda.synchronize()
    got = buf.cpu().numpy()
    assert (got[n:] == sentinel).all()
    assert np.array_equal(got[:n].view(np.uint64), cref.Poseidon(ocfg).crh_batch(x, threads=8))
