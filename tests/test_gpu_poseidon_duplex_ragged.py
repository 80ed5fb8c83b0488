"""Ragged duplex calls on the GPU (cpb_poseidon_duplex_*_ragged, sponge.poseidon.RaggedPoseidonSpongeBatch) against n independent
oracle sponges (oracle/poseidon.py::PoseidonSponge with every permutation on the C oracle), bit for bit: seeded random scripts in every
field and width, equal spans against PoseidonSpongeBatch, the two batch types mixed, host form against _dev form, CUDA-graph replay,
the reference KAT, a large BN254 batch against grouped uniform calls, invalid per-sponge modes and the C++ program."""
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
from crypto_primitives_b200.sponge.poseidon import PoseidonSponge, PoseidonSpongeBatch, RaggedPoseidonSpongeBatch
from oracle import cref, fields as OF, poseidon as OP
from test_gpu_poseidon_duplex import FIELD_NAMES, CSponge, product, random_config

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


def clamp(off, i):
    a, b = off[0], off[-1]
    lo, hi = max(off[i], a), min(off[i + 1], b)
    return (lo, hi - lo) if hi > lo else (a, 0)


def ints(field, t):
    return field.to_ints(t.cpu().numpy().view(np.uint64).reshape(-1, 4))


def check(b, oracles, field, what):
    got = ints(field, b.states)
    modes = b.modes.cpu().numpy()
    t = b.states.shape[1]
    for i, o in enumerate(oracles):
        assert got[t * i:t * (i + 1)] == o.state, (what, "state", i)
        assert ("S" if modes[i, 0] else "A", int(modes[i, 1])) == o.mode, (what, "mode", i)


def with_decreasing_pairs(lens, base, rnd, outputs=False):
    """Offsets for spans of `lens` from `base`, with a few pairs made decreasing or pushed outside the window.  For outputs the spans
    must not overlap, so only the window's edges are moved: offsets[1] below it and offsets[n-1] above it."""
    off = [base]
    for ln in lens:
        off.append(off[-1] + ln)
    n = len(lens)
    if outputs:
        off[1], off[n - 1] = min(off[1], base - 1) if base else off[1], off[n] + 5
        return off
    for _ in range(max(1, n // 16)):
        i = rnd.randrange(1, n)
        off[i] = rnd.choice([off[i - 1] - 1 if off[i - 1] > base else off[i - 1], 0, off[-1] + 5])
    return off


def run_ragged_script(fname, ocfg, n, seed, steps=8):
    field = cp.FIELDS[fname]
    p, rate = ocfg.p, ocfg.rate
    prm = product(fname, ocfg)
    O = cref.Poseidon(ocfg)
    rnd = random.Random(seed)
    b = RaggedPoseidonSpongeBatch(prm, n, 0)
    oracles = [CSponge(ocfg, O) for _ in range(n)]
    dev = b.device
    ops = ["absorb", "absorb_bytes", "squeeze", "squeeze_canonical", "absorb_dev", "squeeze_dev", "bytes_dev"]
    for step in range(steps):
        op = ops[step] if step < len(ops) else rnd.choice(ops)
        lens = [rnd.randrange(0, 3 * rate + 3) for _ in range(n)]
        if op == "absorb":
            vals = [[rnd.randrange(p) for _ in range(ln)] for ln in lens]
            b.absorb([field.elements(v) if v else np.zeros((0, 4), dtype=np.uint64) for v in vals])
            for o, v in zip(oracles, vals):
                o.absorb(v)
        elif op == "absorb_bytes":
            strs = [bytes(rnd.randrange(256) for _ in range(rnd.randrange(0, 90))) for _ in range(n)]
            b.absorb_bytes(strs)
            for o, s in zip(oracles, strs):
                o.absorb(A._ints(s, field))
        elif op in ("squeeze", "squeeze_canonical"):
            vals, off = b.squeeze_native_field_elements(lens) if op == "squeeze" else b.squeeze_canonical(lens)
            g = vals.cpu().numpy().view(np.uint64)
            off = off.cpu().numpy()
            for i, o in enumerate(oracles):
                rows = g[off[i]:off[i + 1]]
                have = field.to_ints(rows) if op == "squeeze" else [OF.from_limbs(r) for r in rows]
                assert have == o.squeeze_native_field_elements(lens[i]), (op, step, i)
        elif op == "absorb_dev":                                                # the tuple form: offsets go to the _dev call as given
            base = rnd.randrange(0, 3)
            off = with_decreasing_pairs(lens, base, rnd)
            flat = [rnd.randrange(p) for _ in range(off[-1])]
            b.absorb((field.elements(flat) if flat else np.zeros((0, 4), dtype=np.uint64), np.array(off, dtype=np.int64)))
            for i, o in enumerate(oracles):
                lo, ln = clamp(off, i)
                o.absorb(flat[lo:lo + ln])
        elif op == "bytes_dev":
            blens = [rnd.randrange(0, 90) for _ in range(n)]
            off = with_decreasing_pairs(blens, rnd.randrange(0, 3), rnd)
            raw = bytes(rnd.randrange(256) for _ in range(off[-1]))
            b.absorb_bytes((np.frombuffer(raw, dtype=np.uint8).copy(), np.array(off, dtype=np.int64)))
            for i, o in enumerate(oracles):
                lo, ln = clamp(off, i)
                o.absorb(A._ints(raw[lo:lo + ln], field))
        else:                                                                   # squeeze_dev: a raw _dev call with decreasing pairs
            off = with_decreasing_pairs(lens, 1, rnd, outputs=True)
            out = torch.full((off[-1] + 1, 4), -1, dtype=torch.int64, device=dev)
            d_off = torch.tensor(off, dtype=torch.int64, device=dev)
            N.check(N.lib.cpb_poseidon_duplex_squeeze_ragged_dev(prm.context(0), b.states.data_ptr(), b.modes.data_ptr(), out.data_ptr(),
                                                                 d_off.data_ptr(), 0, n, torch.cuda.current_stream().cuda_stream))
            g = out.cpu().numpy().view(np.uint64)
            for i, o in enumerate(oracles):
                lo, ln = clamp(off, i)
                assert field.to_ints(g[lo:lo + ln]) == o.squeeze_native_field_elements(ln), (op, step, i)
        check(b, oracles, field, (op, step))
    return b, oracles


def _script_cases():
    out = [(f, t, 1) for f in FIELD_NAMES for t in range(2, 10)]
    return out + [("bn254_fr", 4, 2)]


@pytest.mark.parametrize("fname,t,cap", _script_cases())
def test_random_ragged_script_matches_independent_oracle_sponges(fname, t, cap):
    seed = 1000 * FIELD_NAMES.index(fname) + 10 * t + cap
    ocfg = random_config(OF.MODULI[fname], t, 5 if t % 2 else 17, t % 2 == 0, seed)
    if cap == 2:
        ocfg = OP.PoseidonConfig(ocfg.p, ocfg.full_rounds, ocfg.partial_rounds, ocfg.alpha, ocfg.ark, ocfg.mds, t - 2, 2)
    run_ragged_script(fname, ocfg, 257, seed)


def test_equal_spans_give_exactly_the_uniform_batch():
    fname = "bn254_fr"
    field = cp.FIELDS[fname]
    ocfg = random_config(field.modulus, 3, 5, False, 11)
    prm = product(fname, ocfg)
    n = 300
    rng = np.random.default_rng(4)
    u, r = PoseidonSpongeBatch(prm, n, 0), RaggedPoseidonSpongeBatch(prm, n, 0)
    for kind, k in [("a", 3), ("s", 1), ("b", 45), ("s", 0), ("a", 0), ("c", 4), ("a", 2), ("b", 0), ("s", 5)]:
        if kind == "a":
            x = np.stack([field.elements(list(rng.integers(0, 1 << 62, size=k))) for _ in range(n)]) if k else \
                np.zeros((n, 0, 4), dtype=np.uint64)
            u.absorb(x)
            r.absorb((x.reshape(-1, 4), np.arange(n + 1) * k))
        elif kind == "b":
            x = rng.integers(0, 256, size=(n, k), dtype=np.uint8)
            u.absorb(x)
            r.absorb_bytes([row.tobytes() for row in x])
        else:
            want = u.squeeze_native_field_elements(k) if kind == "s" else u.squeeze_canonical(k)
            got, off = r.squeeze_native_field_elements(k) if kind == "s" else r.squeeze_canonical(k)
            assert torch.equal(got.reshape(n, k, 4), want) and torch.equal(off.cpu(), torch.arange(n + 1) * k), (kind, k)
        assert torch.equal(u.states, r.states), (kind, k)
        assert (r.modes == torch.tensor([u._mode.squeezing, u._mode.index], device=r.device)).all(), (kind, k)


def test_the_two_batch_types_mix():
    """Uniform calls, then from_batch, then ragged calls (absorbables of different encodings too), then sponge(i) continues."""
    fname = "bls12_377_fr"
    field = cp.FIELDS[fname]
    ocfg = random_config(field.modulus, 4, 17, False, 3)
    prm = product(fname, ocfg)
    O = cref.Poseidon(ocfg)
    n = 40
    u = PoseidonSpongeBatch(prm, n, 0)
    oracles = [CSponge(ocfg, O) for _ in range(n)]
    x = np.stack([field.elements([i, i + 1, 5]) for i in range(n)])
    u.absorb(x)
    u.squeeze_native_field_elements(2)
    for i, o in enumerate(oracles):
        o.absorb([i, i + 1, 5])
        o.squeeze_native_field_elements(2)
    r = RaggedPoseidonSpongeBatch.from_batch(u)
    check(r, oracles, field, "from_batch")
    items = [A.usize(i) if i % 2 else "a string of more than thirty-one bytes, number %d" % i for i in range(n)]
    r.absorb(items)
    for o, it in zip(oracles, items):
        o.absorb(A._ints(it, field))
    r = r.fork([bytes([i]) * (i % 7) for i in range(n)])
    for i, o in enumerate(oracles):
        d = bytes([i]) * (i % 7)
        o.absorb(A._ints(len(d).to_bytes(8, "little") + d, field))
    got, off = r.squeeze_native_field_elements([i % 4 for i in range(n)])
    g = got.cpu().numpy().view(np.uint64)
    for i, o in enumerate(oracles):
        assert field.to_ints(g[off[i]:off[i + 1]]) == o.squeeze_native_field_elements(i % 4), i
    check(r, oracles, field, "ragged")
    c = r.clone()
    c.absorb_bytes([b"x"] * n)
    for i in (0, 13, n - 1):
        s = r.sponge(i)
        assert isinstance(s, PoseidonSponge) and (s.mode[0][0], s.mode[1]) == oracles[i].mode, i
        s.absorb(b"tail")
        oracles[i].absorb(A._ints(b"tail", field))
        assert field.to_ints(s.squeeze_native_field_elements(3)) == oracles[i].squeeze_native_field_elements(3), i


def _ragged_calls(ctx, states, modes, bufs, host, stream):
    """One ragged transcript through the host or the _dev form; bufs: (elems, elem offsets, bytes, byte offsets, out, out offsets)."""
    el, eo, by, bo, out, oo = bufs
    n = states.shape[0]
    L = N.lib
    if host:
        P = lambda a, t: a.ctypes.data_as(t)                                  # noqa: E731
        mp = C.cast(modes, N.modep)
        tail = []
    else:
        P = lambda a, t: a.data_ptr()                                          # noqa: E731
        mp = modes.data_ptr()
        tail = [stream]
    f = (lambda name: getattr(L, name + ("" if host else "_dev")))
    N.check(f("cpb_poseidon_duplex_absorb_ragged")(ctx, P(states, N.u64p), mp, P(el, N.u64p), P(eo, N.u64p), n, *tail))
    N.check(f("cpb_poseidon_duplex_squeeze_ragged")(ctx, P(states, N.u64p), mp, P(out, N.u64p), P(oo, N.u64p), 1, n, *tail))
    N.check(f("cpb_poseidon_duplex_absorb_bytes_ragged")(ctx, P(states, N.u64p), mp, P(by, N.u8p), P(bo, N.u64p), n, *tail))
    N.check(f("cpb_poseidon_duplex_squeeze_ragged")(ctx, P(states, N.u64p), mp, P(out, N.u64p), P(oo, N.u64p), 0, n, *tail))


def test_host_form_dev_form_and_graph_replay_agree():
    prm = cp.get_default_poseidon_parameters(cp.BLS12_381_FR, 2, False)
    ctx = prm.context(0)
    n = 1000
    rng = np.random.default_rng(5)
    el_lens, by_lens, sq_lens = rng.integers(0, 7, size=n), rng.integers(0, 130, size=n), rng.integers(0, 4, size=n)
    eo = np.concatenate([[3], 3 + np.cumsum(el_lens)]).astype(np.uint64)         # offsets[0] != 0
    bo = np.concatenate([[0], np.cumsum(by_lens)]).astype(np.uint64)
    oo = np.concatenate([[1], 1 + np.cumsum(sq_lens)]).astype(np.uint64)
    el = cp.BLS12_381_FR.elements(list(rng.integers(0, 1 << 62, size=int(eo[-1]))))
    by = rng.integers(0, 256, size=int(bo[-1]), dtype=np.uint8)
    hs, hout = np.zeros((n, 3, 4), dtype=np.uint64), np.zeros((int(oo[-1]), 4), dtype=np.uint64)
    hm = (N.SpongeMode * n)()
    _ragged_calls(ctx, hs, hm, (el, eo, by, bo, hout, oo), True, None)

    dev = torch.device("cuda", 0)
    T = lambda a: torch.from_numpy(a.view(np.int64) if a.dtype == np.uint64 else a).to(dev)   # noqa: E731
    bufs = (T(el), T(eo), T(by), T(bo))
    ds, dout, dm = torch.zeros((n, 3, 4), dtype=torch.int64, device=dev), torch.zeros((int(oo[-1]), 4), dtype=torch.int64, device=dev), \
        torch.zeros((n, 2), dtype=torch.int64, device=dev)
    stream = torch.cuda.current_stream().cuda_stream
    _ragged_calls(ctx, ds, dm, bufs + (dout, T(oo)), False, stream)
    torch.cuda.synchronize()
    assert np.array_equal(hs, ds.cpu().numpy().view(np.uint64)) and np.array_equal(hout[1:], dout.cpu().numpy().view(np.uint64)[1:])
    assert [(m.squeezing, m.index) for m in hm] == [tuple(r) for r in dm.cpu().tolist()]

    gs, gout, gm = torch.zeros_like(ds), torch.zeros_like(dout), torch.zeros_like(dm)
    d_oo = T(oo)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(g, stream=side):
            _ragged_calls(ctx, gs, gm, bufs + (gout, d_oo), False, side.cuda_stream)
    torch.cuda.synchronize()
    gs.zero_()
    gm.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(gs, ds) and torch.equal(gout, dout) and torch.equal(gm, dm)


def test_reference_kat_through_one_sponge():
    K = kats()["sponge"]
    prm = cp.get_default_poseidon_parameters(cp.BLS12_381_FR, K["rate"], K["optimized_for_weights"])
    f = cp.BLS12_381_FR
    b = RaggedPoseidonSpongeBatch(prm, 1, 0)
    b.absorb([f.elements([int(x) for x in K["absorb"]])])
    got, off = b.squeeze_native_field_elements(3)
    assert f.to_ints(got.cpu().numpy().view(np.uint64)) == [int(x) for x in K["squeeze3"]]
    assert off.tolist() == [0, 3]


def test_large_bn254_batch_matches_grouped_uniform_calls():
    """n = 2^18 transcripts of mixed shapes (message bytes, absorb count, squeeze count) through ragged calls, item by item against the
    same transcripts run through PoseidonSpongeBatch on groups of equal shape."""
    import bench
    prm = bench.poseidon_params(cp, "bn254")
    f = prm.field
    n = 1 << 18
    rng = np.random.default_rng(18)
    L_set, k_set, m_set = np.array([0, 23, 64, 128]), np.array([1, 2, 6]), np.array([1, 3])
    Li, ki, mi = L_set[rng.integers(0, 4, n)], k_set[rng.integers(0, 3, n)], m_set[rng.integers(0, 2, n)]
    dev = torch.device("cuda", 0)
    msg = torch.randint(0, 256, (n, 128), dtype=torch.uint8, generator=torch.Generator().manual_seed(1)).to(dev)
    el = torch.from_numpy(f.elements(list(range(1, 7))).view(np.int64)).to(dev)             # element j of every absorb is j + 1
    r = RaggedPoseidonSpongeBatch(prm, n, 0)
    Lt, kt, mt = (torch.from_numpy(a).to(dev) for a in (Li, ki, mi))
    mask = torch.arange(128, device=dev)[None, :] < Lt[:, None]
    boff = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    torch.cumsum(Lt, 0, out=boff[1:])
    r.absorb_bytes((msg[mask], boff))
    eoff = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    torch.cumsum(kt, 0, out=eoff[1:])
    r.absorb((el[(torch.arange(int(eoff[-1]), device=dev) - torch.repeat_interleave(eoff[:-1], kt))], eoff))
    out, ooff = r.squeeze_native_field_elements(mt)
    for L in L_set:
        for k in k_set:
            for m in m_set:
                idx = torch.nonzero((Lt == int(L)) & (kt == int(k)) & (mt == int(m))).flatten()
                if idx.numel() == 0:
                    continue
                u = PoseidonSpongeBatch(prm, idx.numel(), 0)
                u.absorb(msg[idx, :int(L)].contiguous())
                u.absorb(el[:int(k)].unsqueeze(0).expand(idx.numel(), int(k), 4).contiguous())
                want = u.squeeze_native_field_elements(int(m))
                pos = ooff[idx][:, None] + torch.arange(int(m), device=dev)[None, :]
                assert torch.equal(out[pos], want), (L, k, m)
                assert torch.equal(r.states[idx], u.states), (L, k, m)
                assert (r.modes[idx] == torch.tensor([u._mode.squeezing, u._mode.index], device=dev)).all(), (L, k, m)


def test_invalid_modes_in_a_dev_call_leave_only_those_sponges_untouched():
    prm = cp.get_default_poseidon_parameters(cp.BLS12_381_FR, 2, False)
    f = prm.field
    n = 300
    r = RaggedPoseidonSpongeBatch(prm, n, 0)
    r.absorb([f.elements([i, 2 * i]) for i in range(n)])
    bad = torch.tensor([7, 100, 250], device=r.device)
    r.modes[bad[0], 0] = 2                                                       # squeezing outside {0, 1}
    r.modes[bad[1], 1] = 3                                                       # index past the rate
    r.modes[bad[2], 0] = -1
    states0, modes0 = r.states.clone(), r.modes.clone()
    ref = RaggedPoseidonSpongeBatch.from_states(r.states, r.modes, prm)
    ref.modes[bad] = 0                                                           # the good sponges' reference run
    got, off = r.squeeze_native_field_elements(3)
    want, _ = ref.squeeze_native_field_elements(3)
    good = torch.ones(n, dtype=torch.bool, device=r.device)
    good[bad] = False
    assert torch.equal(r.states[bad], states0[bad]) and torch.equal(r.modes[bad], modes0[bad])
    assert not got.reshape(n, 3, 4)[bad].any()
    assert torch.equal(got.reshape(n, 3, 4)[good], want.reshape(n, 3, 4)[good])
    assert torch.equal(r.states[good], ref.states[good]) and torch.equal(r.modes[good], ref.modes[good])


def test_cpp_program():
    """tests/cpp/test_duplex_ragged.cpp over include/cpb200.hpp (poseidon::RaggedPoseidonSpongeBatch): it checks itself and prints
    the KAT squeeze."""
    out_dir = os.path.join(ROOT, "tests", "host", "_build")
    os.makedirs(out_dir, exist_ok=True)
    exe = os.path.join(out_dir, "test_duplex_ragged")
    lib_dir = os.path.join(ROOT, "crypto_primitives_b200")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "test_duplex_ragged.cpp"), "-L", lib_dir, "-l:libcpb200.so",
                           f"-Wl,-rpath,{lib_dir}", "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "duplex ragged cpp ok" in r.stdout
    line = [l for l in r.stdout.splitlines() if l.startswith("squeeze3[0]")][0]
    assert int(line.split("=")[1].strip(), 16) == int(kats()["sponge"]["squeeze3"][0])      # R/sponge/poseidon/mod.rs:381-404
