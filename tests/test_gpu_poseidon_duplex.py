"""Batched duplex sponges on the GPU (cpb_poseidon_duplex_*, sponge.poseidon.PoseidonSpongeBatch) against n independent oracle
sponges (oracle/poseidon.py::PoseidonSponge with every permutation on the C oracle), bit for bit: seeded random scripts of every
operation, the mode edge cases, agreement with absorb_squeeze_batch, the reference KATs and PoseidonSponge, host form against _dev
form, and CUDA-graph replay."""
import copy
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

from helpers import ROOT, kats
import crypto_primitives_b200 as cp
from crypto_primitives_b200 import _native as N
from crypto_primitives_b200.sponge import absorb as A
from crypto_primitives_b200.sponge.poseidon import FULL, PoseidonSponge, PoseidonSpongeBatch, absorb_squeeze_batch
from oracle import cref, fields as OF, poseidon as OP

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

FIELD_NAMES = ["bls12_381_fr", "bn254_fr", "jubjub_fr", "bls12_377_fr"]


def random_config(p, t, alpha, dense, seed):
    """Random MDS and constants, capacity 1, RP in 1..13; dense: M[0][0] = 0 (M[0][1] at t = 2) forces the dense schedule."""
    rnd = random.Random(seed)
    rp = rnd.randrange(1, 14)
    ark = [[rnd.randrange(p) for _ in range(t)] for _ in range(8 + rp)]
    mds = [[rnd.randrange(1, p) for _ in range(t)] for _ in range(t)]
    if dense:
        mds[0][1 if t == 2 else 0] = 0
    return OP.PoseidonConfig(p, 8, rp, alpha, ark, mds, t - 1, 1)


def product(fname, ocfg):
    return cp.PoseidonConfig.from_ints(cp.FIELDS[fname], ocfg.full_rounds, ocfg.partial_rounds, ocfg.alpha, ocfg.mds, ocfg.ark,
                                       ocfg.rate, ocfg.capacity)


class CSponge(OP.PoseidonSponge):
    """The oracle sponge with its permutation on the C oracle."""

    def __init__(self, cfg, O):
        super().__init__(cfg)
        self.O = O

    def _permute(self):
        p = self.cfg.p
        self.state = cref.mont_to_ints(self.O.permute(cref.ints_to_mont(self.state, p)), p)


def o_bytes(o, nb, bits):
    usable = (bits - 1) // 8
    vals = o.squeeze_native_field_elements(-(-nb // usable))
    return b"".join(v.to_bytes(32, "little")[:usable] for v in vals)[:nb]


def o_bits(o, nbits, bits):
    usable = bits - 1
    out = []
    for v in o.squeeze_native_field_elements(-(-nbits // usable)):
        out += [(v >> i) & 1 for i in range(usable)]
    return out[:nbits]


def o_sized(o, sizes, bits_native, target):
    if target.modulus == o.cfg.p and all(s == FULL for s in sizes):
        return o.squeeze_native_field_elements(len(sizes))
    widths = [target.modulus_bit_size - 1 if s == FULL else s for s in sizes]
    b = o_bits(o, sum(widths), bits_native) if sizes else []
    vals, pos = [], 0
    for w in widths:
        vals.append(sum(bit << i for i, bit in enumerate(b[pos:pos + w])) % target.modulus)
        pos += w
    return vals


def ints(field, t):
    return field.to_ints(t.cpu().numpy().view(np.uint64).reshape(-1, 4))


def check_states(batch, oracles, field):
    got = ints(field, batch.states)
    t = batch.states.shape[1]
    for i, o in enumerate(oracles):
        assert got[t * i:t * (i + 1)] == o.state, ("state", i)
        assert batch.mode == ({"A": "Absorbing", "S": "Squeezing"}[o.mode[0]], o.mode[1])


def run_script(fname, ocfg, n, seed, steps=14):
    field = cp.FIELDS[fname]
    p, bits = ocfg.p, field.modulus_bit_size
    prm = product(fname, ocfg)
    O = cref.Poseidon(ocfg)
    rnd = random.Random(seed)
    rng = np.random.default_rng(seed)
    batch = PoseidonSpongeBatch(prm, n, 0)
    oracles = [CSponge(ocfg, O) for _ in range(n)]
    rate = ocfg.rate
    ops = ["absorb", "absorb_bytes", "absorb_bcast", "squeeze", "squeeze_canonical", "squeeze_bytes", "squeeze_bits", "sized",
           "fork", "clone"]
    for step in range(steps):
        op = ops[step] if step < len(ops) else rnd.choice(ops)
        if op == "absorb":
            k = rnd.randrange(0, 3 * rate + 2)
            vals = [[rnd.randrange(p) for _ in range(k)] for _ in range(n)]
            batch.absorb(np.stack([field.elements(v) for v in vals]) if k else np.zeros((n, 0, 4), dtype=np.uint64))
            for o, v in zip(oracles, vals):
                o.absorb(v)
        elif op == "absorb_bytes":
            L = rnd.randrange(0, 80)
            b = rng.integers(0, 256, size=(n, L), dtype=np.uint8)
            batch.absorb(b)
            for o, row in zip(oracles, b):
                o.absorb(A._ints(row.tobytes(), field))
        elif op == "absorb_bcast":
            s = bytes(rng.integers(0, 256, size=rnd.randrange(0, 70), dtype=np.uint8))
            batch.absorb(s)
            for o in oracles:
                o.absorb(A._ints(s, field))
        elif op in ("squeeze", "squeeze_canonical"):
            m = rnd.randrange(0, 2 * rate + 2)
            got = batch.squeeze_native_field_elements(m) if op == "squeeze" else batch.squeeze_canonical(m)
            g = got.cpu().numpy().view(np.uint64).reshape(n, m, 4)
            for i, o in enumerate(oracles):
                want = o.squeeze_native_field_elements(m)
                have = field.to_ints(g[i]) if op == "squeeze" else [OF.from_limbs(r) for r in g[i]]
                assert have == want, (op, step, i)
        elif op == "squeeze_bytes":
            nb = rnd.randrange(0, 100)
            got = batch.squeeze_bytes(nb).cpu().numpy()
            for i, o in enumerate(oracles):
                assert got[i].tobytes() == o_bytes(o, nb, bits), (op, step, i)
        elif op == "squeeze_bits":
            nbits = rnd.randrange(0, 600)
            got = batch.squeeze_bits(nbits).cpu().numpy()
            for i, o in enumerate(oracles):
                assert [int(x) for x in got[i]] == o_bits(o, nbits, bits), (op, step, i)
        elif op == "sized":
            target = field if rnd.random() < 0.5 else cp.FIELDS[rnd.choice(FIELD_NAMES)]
            sizes = [rnd.choice([FULL, rnd.randrange(1, target.modulus_bit_size + 1)]) for _ in range(rnd.randrange(0, 4))]
            got = batch.squeeze_field_elements_with_sizes(sizes, target).cpu().numpy().view(np.uint64)
            for i, o in enumerate(oracles):
                assert target.to_ints(got[i]) == o_sized(o, sizes, bits, target), (op, step, i, sizes)
        elif op == "fork":
            if rnd.random() < 0.5:
                d = bytes(rng.integers(0, 256, size=rnd.randrange(0, 40), dtype=np.uint8))
                batch = batch.fork(d)
                doms = [d] * n
            else:
                dd = rng.integers(0, 256, size=(n, rnd.randrange(0, 40)), dtype=np.uint8)
                batch = batch.fork(torch.from_numpy(dd))
                doms = [r.tobytes() for r in dd]
            oracles = [copy.copy(o) for o in oracles]
            for o, d in zip(oracles, doms):
                o.state = list(o.state)
                o.absorb(A._ints(len(d).to_bytes(8, "little") + d, field))
        elif op == "clone":
            before = batch.states.clone()
            c = batch.clone()
            c.absorb(b"x")
            assert torch.equal(batch.states, before)
            batch = c
            for o in oracles:
                o.absorb(A._ints(b"x", field))
    torch.cuda.synchronize()
    check_states(batch, oracles, field)
    return batch, oracles


def _script_cases():
    out = []
    for f in FIELD_NAMES:
        for dense in (False, True):
            out.append((f, 3, dense, 33))
    for f in ("bls12_381_fr", "bn254_fr"):
        for t in range(2, 10):
            out.append((f, t, t % 2 == 0, 33 if t in (2, 9) else 1))
    out += [("bn254_fr", 3, False, 4097), ("bls12_381_fr", 3, True, 4097)]
    return out


@pytest.mark.parametrize("fname,t,dense,n", _script_cases())
def test_random_script_matches_independent_oracle_sponges(fname, t, dense, n):
    seed = 1000 * FIELD_NAMES.index(fname) + 10 * t + int(dense) + n
    ocfg = random_config(OF.MODULI[fname], t, 5 if t % 2 else 17, dense, seed)
    batch, _ = run_script(fname, ocfg, n, seed, steps=14 if n < 4097 else 10)
    assert N.lib.cpb_poseidon_ctx_is_sparse(batch.parameters.context(0)) == int(not dense)


EDGES = {
    "absorb_to_rate_then_absorb": [("a", "rate"), ("a", 1), ("s", 1)],
    "squeeze_rate_then_squeeze": [("a", 1), ("s", "rate"), ("s", 2)],
    "squeeze0_from_absorbing": [("a", 1), ("s", 0), ("s", 1)],
    "squeeze0_from_squeezing": [("s", 1), ("s", 0), ("s", "rate"), ("s", 0), ("a", 1)],
    "absorb_nothing": [("a", 0), ("a", 1), ("a", 0), ("s", 1), ("a", 0), ("s", 1)],
    "absorb_after_squeeze": [("a", 2), ("s", 1), ("a", 1), ("s", 1), ("a", "rate")],
    "absorb_spanning_blocks": [("a", "3rate+1"), ("s", 1), ("a", "2rate"), ("s", "2rate+1")],
}


@pytest.mark.parametrize("edge", list(EDGES))
@pytest.mark.parametrize("rate", [1, 2, 4])
def test_edge_cases(edge, rate):
    fname = "bn254_fr"
    field = cp.FIELDS[fname]
    ocfg = random_config(field.modulus, rate + 1, 5, False, rate)
    O = cref.Poseidon(ocfg)
    n = 5
    batch = PoseidonSpongeBatch(product(fname, ocfg), n, 0)
    oracles = [CSponge(ocfg, O) for _ in range(n)]
    rnd = random.Random(rate)
    for kind, k in EDGES[edge]:
        k = {"rate": rate, "3rate+1": 3 * rate + 1, "2rate": 2 * rate, "2rate+1": 2 * rate + 1}.get(k, k)
        if kind == "a":
            vals = [[rnd.randrange(field.modulus) for _ in range(k)] for _ in range(n)]
            batch.absorb(np.stack([field.elements(v) for v in vals]) if k else np.zeros((n, 0, 4), dtype=np.uint64))
            for o, v in zip(oracles, vals):
                o.absorb(v)
        else:
            got = batch.squeeze_native_field_elements(k).cpu().numpy().view(np.uint64)
            for i, o in enumerate(oracles):
                assert field.to_ints(got[i]) == o.squeeze_native_field_elements(k), (edge, i)
        check_states(batch, oracles, field)


def test_matches_absorb_squeeze_batch():
    for fname in FIELD_NAMES:
        field = cp.FIELDS[fname]
        ocfg = random_config(field.modulus, 3, 5, False, 7)
        prm = product(fname, ocfg)
        for L, m in ((2, 1), (0, 1), (5, 3), (1, 2)):
            x = np.stack([field.elements([(31 * i + j) % field.modulus for j in range(L)]) for i in range(257)]) if L else \
                np.zeros((257, 0, 4), dtype=np.uint64)
            b = PoseidonSpongeBatch(prm, 257, 0)
            b.absorb(x)
            got = b.squeeze_native_field_elements(m).cpu().numpy().view(np.uint64)
            assert np.array_equal(got, absorb_squeeze_batch(prm, x, m)), (fname, L, m)


def test_reference_kats_hold_in_every_sponge():
    K = kats()["sponge"]
    prm = cp.get_default_poseidon_parameters(cp.BLS12_381_FR, K["rate"], K["optimized_for_weights"])
    f = cp.BLS12_381_FR
    n = 300
    b = PoseidonSpongeBatch(prm, n, 0)
    b.absorb(np.broadcast_to(f.elements([int(x) for x in K["absorb"]]), (n, 3, 4)).copy())
    got = b.squeeze_native_field_elements(3).cpu().numpy().view(np.uint64)
    for i in range(n):
        assert f.to_ints(got[i]) == [int(x) for x in K["squeeze3"]], i


def test_sponge_i_continues_like_an_independent_sponge():
    ocfg = random_config(OF.BLS12_377_FR, 4, 17, False, 3)
    prm = product("bls12_377_fr", ocfg)
    f = cp.BLS12_377_FR
    n = 40
    b = PoseidonSpongeBatch(prm, n, 0)
    x = np.stack([f.elements([i, i + 1, i + 2, 5]) for i in range(n)])
    b.absorb(x)
    b.squeeze_native_field_elements(2)
    for i in (0, 17, n - 1):
        single = PoseidonSponge(prm)
        single.absorb(x[i])
        single.squeeze_native_field_elements(2)
        s = b.sponge(i)
        assert s.mode == single.mode and np.array_equal(s.state, single.state)
        s.absorb(b"tail")
        single.absorb(b"tail")
        assert np.array_equal(s.squeeze_native_field_elements(5), single.squeeze_native_field_elements(5))
    b.absorb(b"tail")
    sq = b.squeeze_native_field_elements(5).cpu().numpy().view(np.uint64)
    single = PoseidonSponge(prm)
    single.absorb(x[3])
    single.squeeze_native_field_elements(2)
    single.absorb(b"tail")
    assert np.array_equal(sq[3], single.squeeze_native_field_elements(5))


def _script_calls(ctx, states, mode, bufs, host, stream):
    """The same script through the host or the _dev form; bufs: (elems, bytes, out) host arrays or device tensors."""
    el, by, out = bufs
    n = states.shape[0]
    ptr = (lambda a, t: a.ctypes.data_as(t)) if host else (lambda a, t: a.data_ptr())
    L = N.lib
    calls = [
        lambda: (L.cpb_poseidon_duplex_absorb if host else L.cpb_poseidon_duplex_absorb_dev)(
            ctx, ptr(states, N.u64p), C.byref(mode), ptr(el, N.u64p), 5, n, *([] if host else [stream])),
        lambda: (L.cpb_poseidon_duplex_squeeze if host else L.cpb_poseidon_duplex_squeeze_dev)(
            ctx, ptr(states, N.u64p), C.byref(mode), ptr(out, N.u64p), 3, 1, n, *([] if host else [stream])),
        lambda: (L.cpb_poseidon_duplex_absorb_bytes if host else L.cpb_poseidon_duplex_absorb_bytes_dev)(
            ctx, ptr(states, N.u64p), C.byref(mode), ptr(by, N.u8p), 45, 45, n, *([] if host else [stream])),
        lambda: (L.cpb_poseidon_duplex_squeeze if host else L.cpb_poseidon_duplex_squeeze_dev)(
            ctx, ptr(states, N.u64p), C.byref(mode), ptr(out, N.u64p), 3, 0, n, *([] if host else [stream])),
    ]
    for c in calls:
        N.check(c())


def test_host_form_dev_form_and_graph_replay_agree():
    prm = cp.get_default_poseidon_parameters(cp.BLS12_381_FR, 2, False)
    ctx = prm.context(0)
    n = 1000
    rng = np.random.default_rng(5)
    el = np.stack([cp.BLS12_381_FR.elements(list(rng.integers(0, 1 << 62, size=5))) for _ in range(n)])
    by = rng.integers(0, 256, size=(n, 45), dtype=np.uint8)
    hs, hout, hm = np.zeros((n, 3, 4), dtype=np.uint64), np.zeros((n, 3, 4), dtype=np.uint64), N.SpongeMode(0, 0)
    _script_calls(ctx, hs, hm, (el, by, hout), True, None)

    dev = torch.device("cuda", 0)
    d_el, d_by = torch.from_numpy(el.view(np.int64)).to(dev), torch.from_numpy(by).to(dev)
    ds, dout, dm = torch.zeros((n, 3, 4), dtype=torch.int64, device=dev), torch.zeros((n, 3, 4), dtype=torch.int64, device=dev), N.SpongeMode(0, 0)
    stream = torch.cuda.current_stream().cuda_stream
    _script_calls(ctx, ds, dm, (d_el, d_by, dout), False, stream)
    torch.cuda.synchronize()
    assert (hm.squeezing, hm.index) == (dm.squeezing, dm.index) == (1, 1)       # squeeze(3) at rate 2 from Absorbing
    assert np.array_equal(hs, ds.cpu().numpy().view(np.uint64)) and np.array_equal(hout, dout.cpu().numpy().view(np.uint64))

    gs, gout = torch.zeros_like(ds), torch.zeros_like(dout)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    gm = N.SpongeMode(0, 0)
    with torch.cuda.stream(side):
        with torch.cuda.graph(g, stream=side):
            _script_calls(ctx, gs, gm, (d_el, d_by, gout), False, side.cuda_stream)
    torch.cuda.synchronize()
    gs.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(gs, ds) and torch.equal(gout, dout)


def test_n_zero_advances_the_mode_only():
    prm = cp.get_default_poseidon_parameters(cp.BLS12_381_FR, 3, False)
    ctx = prm.context(0)
    m = N.SpongeMode(0, 0)
    N.check(N.lib.cpb_poseidon_duplex_absorb_dev(ctx, None, C.byref(m), None, 4, 0, None))
    assert (m.squeezing, m.index) == (0, 1)
    N.check(N.lib.cpb_poseidon_duplex_squeeze_dev(ctx, None, C.byref(m), None, 0, 0, 0, None))
    assert (m.squeezing, m.index) == (1, 0)
    N.check(N.lib.cpb_poseidon_duplex_absorb_bytes(ctx, None, C.byref(m), None, 100, 0, 0))
    assert (m.squeezing, m.index) == (0, 1)          # 108 bytes = 4 elements from lane 0 at rate 3
    bad = N.SpongeMode(0, 4)
    assert N.lib.cpb_poseidon_duplex_absorb_dev(ctx, None, C.byref(bad), None, 1, 0, None) == N.CPB_BAD_PARAMS
    assert (bad.squeezing, bad.index) == (0, 4)


def test_unequal_item_encodings_are_refused():
    prm = cp.get_default_poseidon_parameters(cp.BLS12_381_FR, 2, False)
    b = PoseidonSpongeBatch(prm, 2, 0)
    with pytest.raises(ValueError):
        b.absorb([A.usize(1), "longer string than one element of thirty-one bytes"])
    b.absorb([A.usize(1), A.usize(2)])
    assert b.mode == ("Absorbing", 1)


def test_cpp_program():
    """tests/cpp/test_duplex.cpp over include/cpb200.hpp (poseidon::PoseidonSpongeBatch): it checks itself and prints the KAT squeeze."""
    out_dir = os.path.join(ROOT, "tests", "host", "_build")
    os.makedirs(out_dir, exist_ok=True)
    exe = os.path.join(out_dir, "test_duplex")
    lib_dir = os.path.join(ROOT, "crypto_primitives_b200")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "test_duplex.cpp"),
                           "-L", lib_dir, "-l:libcpb200.so", f"-Wl,-rpath,{lib_dir}", "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "duplex cpp ok" in r.stdout
    line = [l for l in r.stdout.splitlines() if l.startswith("squeeze3[0]")][0]
    assert int(line.split("=")[1].strip(), 16) == int(kats()["sponge"]["squeeze3"][0])      # R/sponge/poseidon/mod.rs:381-404
