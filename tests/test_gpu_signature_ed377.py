"""Schnorr signatures and ElGamal encryption over ed-on-BLS12-377 on the GPU (cpb_te_base_*, cpb_schnorr_*, cpb_elgamal_* with
curve CPB_ED_ON_BLS12_377; include/cpb200.h) against the oracle tests/signature_ed377_oracle.py: the reference's scenarios through
the Python mirror, 2^16 signers bit for bit, tampering, randomisation, ElGamal, guard regions around the _dev outputs, a Jubjub
and an ed-on-BLS12-377 context used alternately, the reference benchmark's workload at 2^20 and the C++ mirror.  Every kernel
that runs te_mul_var (verify, key randomisation, encrypt, decrypt) is compared with the oracle here."""
import random

import numpy as np
import pytest

import crypto_primitives_b200 as cp
from crypto_primitives_b200 import ElGamal, Schnorr
from crypto_primitives_b200.signature.schnorr import Parameters, pack_messages
from oracle import fields as OF
import signature_ed377_oracle as E

pytestmark = pytest.mark.gpu

CURVE = cp.curves.ED_ON_BLS12_377
Fq, Fr = cp.BLS12_377_FR, cp.ED_ON_BLS12_377_FR
R = E.R


def pts_to_ints(a):
    v = Fq.to_ints(np.asarray(a).reshape(-1, 4))
    return [(v[2 * i], v[2 * i + 1]) for i in range(len(v) // 2)]


def ints_to_pts(pts):
    return Fq.elements([c for P in pts for c in P]).reshape(len(pts), 2, 4)


def sig_ints(a):
    v = Fr.to_ints(np.asarray(a).reshape(-1, 4))
    return [(v[2 * i], v[2 * i + 1]) for i in range(len(v) // 2)]


def sigs_from_ints(sigs):
    return Fr.elements([c for s in sigs for c in s]).reshape(len(sigs), 2, 4)


def random_point(rng):
    while True:
        P = E.point_from_y(rng.randrange(E.Q))
        if P is not None:
            return P


@pytest.fixture(scope="module")
def setup():
    prm = Schnorr.setup(OF.SplitMix64(2377), CURVE)
    G = pts_to_ints(prm.generator)[0]
    assert E.mul(R, G) == E.IDENTITY
    return prm, G, E.FixedBase(G)


# ---- the reference's scenarios (R/signature/mod.rs:52-105, R/encryption/elgamal/mod.rs:102-128) -------------------------
def test_reference_scenarios_through_the_mirror():
    rng = OF.SplitMix64(77)
    for msg in (b"Hi, I am a Schnorr signature!", b"\x00" * 4 + b"hello"):
        prm = Schnorr.setup(rng, CURVE)
        pk, sk = Schnorr.keygen(prm, rng)
        assert Fr.to_ints(sk)[0] < R
        sig = Schnorr.sign(prm, sk, msg, rng)
        assert Schnorr.verify(prm, pk, msg, sig)
        G = pts_to_ints(prm.generator)[0]
        assert pts_to_ints(pk)[0] == E.mul(Fr.to_ints(sk)[0], G)
        assert E.verify(G, prm.salt, pts_to_ints(pk)[0], msg, sig_ints(sig)[0])
    prm = Schnorr.setup(rng, CURVE)
    pk, sk = Schnorr.keygen(prm, rng)
    sig = Schnorr.sign(prm, sk, b"Bad message", rng)
    assert not Schnorr.verify(prm, pk, b"Hi, I am a Schnorr signature!", sig)
    msg = b"Hi, I am a Schnorr signature!"
    sig = Schnorr.sign(prm, sk, msg, rng)
    randomness = rng.bytes(32)
    rpk = Schnorr.randomize_public_key(prm, pk, randomness)
    rsig = Schnorr.randomize_signature(prm, sig, randomness)
    assert Schnorr.verify(prm, rpk, msg, rsig)
    eprm = ElGamal.setup(rng, CURVE)
    epk, esk = ElGamal.keygen(eprm, rng)
    m = ints_to_pts([E.mul(E.COFACTOR, random_point(random.Random(3)))])[0]
    r = Fr.elements([rng.field(R)])[0]
    ct = ElGamal.encrypt(eprm, epk, m, r)
    assert np.array_equal(ElGamal.decrypt(eprm, esk, ct), m)


# ---- 2^16 signers ----------------------------------------------------------------------------------------------------------
N16 = 1 << 16


@pytest.fixture(scope="module")
def signed(setup):
    prm, G, fb = setup
    rng = random.Random(16)
    sks_i = [rng.randrange(R) for _ in range(N16)]
    ks_i = [rng.randrange(R) for _ in range(N16)]
    sks_i[:3], ks_i[:3] = [0, 1, R - 1], [R - 1, 1, 0]
    msgs = [bytes(rng.randrange(256) for _ in range(rng.randrange(301))) for _ in range(N16)]
    sks, ks = Fr.elements(sks_i), Fr.elements(ks_i)
    pks = Schnorr.keygen_batch(prm, sks)
    sigs, ok = Schnorr.sign_with_nonces_batch(prm, sks, ks, msgs)
    return dict(sks_i=sks_i, ks_i=ks_i, msgs=msgs, sks=sks, ks=ks, pks=pks, sigs=sigs, ok=ok)


def test_keygen_matches_the_oracle(setup, signed):
    prm, G, fb = setup
    assert np.array_equal(signed["pks"], ints_to_pts([fb.mul(sk) for sk in signed["sks_i"]]))
    assert pts_to_ints(signed["pks"][:4]) == [E.mul(sk, G) for sk in signed["sks_i"][:4]]


def test_sign_matches_the_oracle_bit_for_bit(setup, signed):
    prm, G, fb = setup
    exp_ok = np.zeros(N16, dtype=bool)
    exp = np.zeros((N16, 2, 4), dtype=np.uint64)
    accepted = []
    for i in range(N16):
        s = E.sign(G, prm.salt, signed["sks_i"][i], signed["msgs"][i], signed["ks_i"][i], mul=fb.mul)
        if s is not None:
            exp_ok[i] = True
            accepted.append((i, s))
    idx = np.array([i for i, _ in accepted])
    exp[idx] = sigs_from_ints([s for _, s in accepted])
    assert np.array_equal(signed["ok"], exp_ok)
    assert np.array_equal(signed["sigs"], exp)                          # rejected items are (0, 0)
    rate = 1 - exp_ok.mean()
    assert 0.40 < rate < 0.435, rate                                     # 1 - r / 2^251 = 0.417


def test_verify_accepts_every_signature_and_rejects_every_tampering(setup, signed):
    prm, G, fb = setup
    idx = np.nonzero(signed["ok"])[0]
    pks, sigs = signed["pks"][idx], signed["sigs"][idx]
    msgs = [signed["msgs"][i] for i in idx]
    assert Schnorr.verify_batch(prm, pks, msgs, sigs).all()
    n_or = 48
    assert all(E.verify(G, prm.salt, pts_to_ints(pks[j])[0], msgs[j], sig_ints(sigs[j])[0], mul=E.mul_ext) for j in range(8))
    s_e = sig_ints(sigs)
    cases = {}
    nz = [j for j, m in enumerate(msgs) if len(m) > 0]
    flipped = list(msgs)
    for j in nz:
        b = bytearray(msgs[j])
        b[j % len(b)] ^= 1 << (j % 8)
        flipped[j] = bytes(b)
    cases["flip"] = (nz, pks, flipped, sigs, prm)
    cases["s+1"] = (range(len(msgs)), pks, msgs, sigs_from_ints([((s + 1) % R, e) for s, e in s_e]), prm)
    cases["e+1"] = (range(len(msgs)), pks, msgs, sigs_from_ints([(s, (e + 1) % R) for s, e in s_e]), prm)
    cases["pk"] = (range(len(msgs)), np.roll(pks, 1, axis=0), msgs, sigs, prm)
    other = Parameters(prm.generator, CURVE, salt=bytes(b ^ 0x5A for b in prm.salt))
    cases["salt"] = (range(len(msgs)), pks, msgs, sigs, other)
    cases["truncated"] = (nz, pks, [m[:-1] if m else m for m in msgs], sigs, prm)
    for name, (sel, p, m, s, pp) in cases.items():
        sel = list(sel)
        got = Schnorr.verify_batch(pp, p[sel], [m[j] for j in sel], s[sel])
        exp = [E.verify(G, pp.salt, pts_to_ints(p[j])[0], m[j], sig_ints(s[j])[0], mul=E.mul_ext) for j in sel[:n_or]]
        assert list(got[:n_or]) == exp, name
        assert not got.any(), name


@pytest.mark.parametrize("ln", [0, 1, 32, 100])
def test_randomized_keys_and_signatures(setup, signed, ln):
    prm, G, fb = setup
    rng = random.Random(ln)
    idx = np.nonzero(signed["ok"])[0][:384]
    pks, sigs = signed["pks"][idx], signed["sigs"][idx]
    msgs = [signed["msgs"][i] for i in idx]
    rnd = [bytes(rng.randrange(256) for _ in range(ln)) for _ in idx]
    if ln:
        rnd[0], rnd[1] = b"\xff" * ln, b"\x01" * ln
    rpk = Schnorr.randomize_public_key_batch(prm, pks, rnd)
    rsig = Schnorr.randomize_signature_batch(prm, sigs, rnd)
    assert pts_to_ints(rpk) == [E.add(E.mul_ext(E.randomizer_int(r), G), P) for r, P in zip(rnd, pts_to_ints(pks))]
    assert sig_ints(rsig) == [E.randomize_signature(s, r) for s, r in zip(sig_ints(sigs), rnd)]
    assert Schnorr.verify_batch(prm, rpk, msgs, rsig).all()


def test_any_generator_is_exact():
    """A generator outside the prime-order subgroup (4-torsion part kept) gives the exact integer products."""
    rng = random.Random(31)
    G = random_point(rng)
    assert E.mul(R, G) != E.IDENTITY
    prm = Parameters(ints_to_pts([G])[0], CURVE, salt=bytes(32))
    sks_i = [rng.randrange(R) for _ in range(64)] + [0, 1, R - 1]
    assert pts_to_ints(Schnorr.keygen_batch(prm, Fr.elements(sks_i))) == [E.mul_ext(k, G) for k in sks_i]
    pks = ints_to_pts([random_point(rng) for _ in range(64)])
    rnd = [bytes(rng.randrange(256) for _ in range(40)) for _ in range(64)]
    got = pts_to_ints(Schnorr.randomize_public_key_batch(prm, pks, rnd))
    assert got == [E.randomize_public_key(G, P, r, mul=E.mul_ext) for P, r in zip(pts_to_ints(pks), rnd)]
    eprm = cp.encryption_elgamal.Parameters(ints_to_pts([G])[0], CURVE)
    rs_i = [rng.randrange(R) for _ in range(64)]
    cts = ElGamal.encrypt_batch(eprm, pks, pks[::-1], Fr.elements(rs_i))
    exp = [E.elgamal_encrypt(G, P, M, r, mul=E.mul_ext) for P, M, r in zip(pts_to_ints(pks), pts_to_ints(pks[::-1]), rs_i)]
    assert np.array_equal(cts, np.stack([ints_to_pts([c1, c2]) for c1, c2 in exp]))


# ---- ElGamal ---------------------------------------------------------------------------------------------------------------
def test_elgamal(setup):
    prm, G, fb = setup
    eprm = cp.encryption_elgamal.Parameters(prm.generator, CURVE)
    rng = random.Random(44)
    n = N16
    sks_i = [rng.randrange(R) for _ in range(n)]
    sks_i[:3] = [0, 1, R - 1]
    sks = Fr.elements(sks_i)
    pks = ElGamal.keygen_batch(eprm, sks)
    ms = ElGamal.keygen_batch(eprm, Fr.elements([rng.randrange(R) for _ in range(n)]))
    rs_i = [rng.randrange(R) for _ in range(n)]
    cts = ElGamal.encrypt_batch(eprm, pks, ms, Fr.elements(rs_i))
    assert np.array_equal(ElGamal.decrypt_batch(eprm, sks, cts), ms)
    k = 512
    exp = [E.elgamal_encrypt(G, P, M, r, mul=E.mul_ext) for P, M, r in zip(pts_to_ints(pks[:k]), pts_to_ints(ms[:k]), rs_i[:k])]
    assert np.array_equal(cts[:k], np.stack([ints_to_pts([c1, c2]) for c1, c2 in exp]))
    c = [(random_point(rng), random_point(rng)) for _ in range(k)]
    ct = np.stack([ints_to_pts([c1, c2]) for c1, c2 in c])
    got = pts_to_ints(ElGamal.decrypt_batch(eprm, sks[:k], ct))
    assert got == [E.elgamal_decrypt(s, cc, mul=E.mul_ext) for s, cc in zip(sks_i[:k], c)]


# ---- _dev forms: results equal the host forms; nothing outside the outputs is written ---------------------------------------
def test_dev_forms_with_guard_regions(setup, signed):
    import torch
    prm, G, fb = setup
    dev = torch.device("cuda", 0)
    n = 1000
    GUARD = 64
    sks, pks, sigs, ks = signed["sks"][:n], signed["pks"][:n], signed["sigs"][:n], signed["ks"][:n]
    msgs = signed["msgs"][:n]
    values, offsets = pack_messages(msgs)

    def t(a, dtype=torch.int64):
        a = np.ascontiguousarray(a)
        return torch.from_numpy(a.view(np.int64) if dtype == torch.int64 else a).to(dev)

    def guarded(shape, dtype=torch.int64):
        numel = int(np.prod(shape))
        buf = torch.full((numel + 2 * GUARD,), 0x5A if dtype == torch.uint8 else 0x5A5A5A5A5A5A5A5A, dtype=dtype, device=dev)
        return buf, buf[GUARD:GUARD + numel].view(shape)

    def intact(buf):
        v = buf.cpu()
        sentinel = 0x5A if buf.dtype == torch.uint8 else 0x5A5A5A5A5A5A5A5A
        return bool((v[:GUARD] == sentinel).all() and (v[-GUARD:] == sentinel).all())

    def u64(x):
        return x.cpu().numpy().view(np.uint64)

    d_vals, d_off = t(values, torch.uint8), t(offsets)
    b1, o1 = guarded((n, 2, 4))
    Schnorr.keygen_dev(prm, t(sks), out=o1)
    b2, o2 = guarded((n, 2, 4))
    b3, o3 = guarded((n,), torch.uint8)
    Schnorr.sign_with_nonces_dev(prm, t(sks), t(ks), d_vals, d_off, sigs_out=o2, signed_out=o3)
    b4, o4 = guarded((n,), torch.uint8)
    Schnorr.verify_dev(prm, t(pks), d_vals, d_off, t(sigs), ok_out=o4)
    rnd = np.random.default_rng(1).integers(0, 256, (n, 32), dtype=np.uint8)
    b5, o5 = guarded((n, 2, 4))
    Schnorr.randomize_public_key_dev(prm, t(pks), t(rnd, torch.uint8), out=o5)
    b6, o6 = guarded((n, 2, 4))
    Schnorr.randomize_signature_dev(prm, t(sigs), t(rnd, torch.uint8), out=o6)
    eprm = cp.encryption_elgamal.Parameters(prm.generator, CURVE)
    b7, o7 = guarded((n, 2, 2, 4))
    ElGamal.encrypt_dev(eprm, t(pks), t(pks[::-1]), t(ks), out=o7)
    b8, o8 = guarded((n, 2, 4))
    ElGamal.decrypt_dev(eprm, t(sks), o7, out=o8)
    torch.cuda.synchronize()
    for b in (b1, b2, b3, b4, b5, b6, b7, b8):
        assert intact(b)
    assert np.array_equal(u64(o1), pks)
    assert np.array_equal(u64(o2), sigs) and np.array_equal(o3.cpu().numpy().astype(bool), signed["ok"][:n])
    assert o4.cpu().numpy().astype(bool).tolist() == signed["ok"][:n].tolist()          # signed items verify, (0, 0) does not
    assert np.array_equal(u64(o5), Schnorr.randomize_public_key_batch(prm, pks, rnd))
    assert np.array_equal(u64(o6), Schnorr.randomize_signature_batch(prm, sigs, rnd))
    assert np.array_equal(u64(o7), ElGamal.encrypt_batch(eprm, pks, pks[::-1], ks))
    assert np.array_equal(u64(o8), pks[::-1])


# ---- both curves in one process ----------------------------------------------------------------------------------------------
def test_jubjub_and_ed377_contexts_alternate(setup, signed):
    """Results of a Jubjub context and an ed-on-BLS12-377 context used alternately equal those of each used alone."""
    prm, G, fb = setup
    jprm = Schnorr.setup(OF.SplitMix64(2024))
    rng = random.Random(51)
    n = 2048
    msgs = signed["msgs"][:n]
    e_sks, e_ks = signed["sks"][:n], signed["ks"][:n]
    rj = cp.curves.JUBJUB.scalar_modulus
    j_sks = cp.JUBJUB_FR.elements([rng.randrange(rj) for _ in range(n)])
    j_ks = cp.JUBJUB_FR.elements([rng.randrange(rj) for _ in range(n)])
    rnd = [bytes(rng.randrange(256) for _ in range(32)) for _ in range(n)]

    def run(p, sks, ks):
        pks = Schnorr.keygen_batch(p, sks)
        sigs, ok = Schnorr.sign_with_nonces_batch(p, sks, ks, msgs)
        v = Schnorr.verify_batch(p, pks, msgs, sigs)
        rpk = Schnorr.randomize_public_key_batch(p, pks, rnd)
        return pks, sigs, ok, v, rpk

    alone_e = run(prm, e_sks, e_ks)
    alone_j = run(jprm, j_sks, j_ks)
    for _ in range(2):
        mixed_e = run(prm, e_sks, e_ks)
        mixed_j = run(jprm, j_sks, j_ks)
        for a, b in zip(alone_e + alone_j, mixed_e + mixed_j):
            assert np.array_equal(a, b)
    assert np.array_equal(alone_e[0], signed["pks"][:n]) and np.array_equal(alone_e[3], alone_e[2])
    assert np.array_equal(alone_j[3], alone_j[2])
    assert 0.05 < 1 - alone_j[2].mean() < 0.14 and 0.37 < 1 - alone_e[2].mean() < 0.47   # each curve's own rejection rate


# ---- the reference benchmark's workload (R/benches/signature.rs) -------------------------------------------------------------
def test_reference_benchmark_workload_2_20(setup):
    """Messages [100u8; 128], sign then verify at n = 2^20: every item is signed (nonces redrawn by the mirror's loop on the
    device form) and verifies; a sample is compared with the oracle."""
    import torch
    prm, G, fb = setup
    n = 1 << 20
    dev = torch.device("cuda", 0)
    g = np.random.default_rng(128)
    pyr = random.Random(128)
    base = [pyr.randrange(R) for _ in range(4096)]
    sks_i = [base[i % 4096] for i in range(n)]
    sks = np.ascontiguousarray(np.tile(Fr.elements(base), (n // 4096, 1)))
    d_sk = torch.from_numpy(sks.view(np.int64)).to(dev)
    d_vals = torch.full((128 * n,), 100, dtype=torch.uint8, device=dev)
    d_off = torch.arange(n + 1, dtype=torch.int64, device=dev) * 128
    d_pk = Schnorr.keygen_dev(prm, d_sk)
    d_sig = torch.zeros((n, 2, 4), dtype=torch.int64, device=dev)
    todo = np.arange(n)
    nonces = np.zeros((n, 4), dtype=np.uint64)
    rounds = 0
    while todo.size:
        rounds += 1
        assert rounds < 40
        k = Fr.elements([pyr.randrange(R) for _ in range(todo.size)]) if todo.size < 4096 else \
            np.ascontiguousarray(np.tile(Fr.elements([pyr.randrange(R) for _ in range(4096)]), (todo.size // 4096 + 1, 1))[:todo.size])
        sel = torch.from_numpy(todo).to(dev)
        vals_sel = torch.full((128 * todo.size,), 100, dtype=torch.uint8, device=dev)
        off_sel = torch.arange(todo.size + 1, dtype=torch.int64, device=dev) * 128
        s, ok = Schnorr.sign_with_nonces_dev(prm, d_sk[sel].contiguous(), torch.from_numpy(k.view(np.int64)).to(dev), vals_sel, off_sel)
        okb = ok.bool()
        d_sig[sel[okb]] = s[okb]
        okh = okb.cpu().numpy()
        nonces[todo[okh]] = k[okh]
        todo = todo[~okh]
    ok = Schnorr.verify_dev(prm, d_pk, d_vals, d_off, d_sig)
    torch.cuda.synchronize()
    assert bool(ok.bool().all())
    sigs = d_sig.cpu().numpy().view(np.uint64)
    msg = bytes([100]) * 128
    sample = list(range(4)) + [int(i) for i in g.integers(0, n, 60)]
    for i in sample:
        k_i = Fr.to_ints(nonces[i])[0]
        assert sig_ints(sigs[i])[0] == E.sign(G, prm.salt, sks_i[i], msg, k_i, mul=fb.mul), i
    pks = d_pk.cpu().numpy().view(np.uint64)
    assert pts_to_ints(pks[sample[:8]]) == [fb.mul(sks_i[i]) for i in sample[:8]]
    assert all(E.verify(G, prm.salt, pts_to_ints(pks[i])[0], msg, sig_ints(sigs[i])[0], mul=E.mul_ext) for i in sample[:8])


def test_cpp_signature_ed377_mirror():
    """tests/cpp/test_signature_ed377.cpp through include/cpb200.hpp."""
    import os
    import subprocess
    from helpers import ROOT
    out_dir = os.path.join(ROOT, "tests", "host", "_build")
    os.makedirs(out_dir, exist_ok=True)
    exe = os.path.join(out_dir, "test_signature_ed377")
    lib_dir = os.path.join(ROOT, "crypto_primitives_b200")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "test_signature_ed377.cpp"), "-L", lib_dir, "-l:libcpb200.so",
                           f"-Wl,-rpath,{lib_dir}", "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "cpp signature ed377 ok" in r.stdout
