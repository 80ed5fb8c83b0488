"""Schnorr signatures, ElGamal encryption and the Blake2s commitment on the GPU (cpb_te_base_*, cpb_schnorr_*, cpb_elgamal_*,
cpb_blake2s_commit_*; include/cpb200.h) against the oracle (tests/signature_oracle.py): the reference's scenarios through the Python
mirror, 2^16 signers bit for bit, tampered signatures, randomisation, ElGamal, 2^20 commitments, and guard regions around the
outputs of the _dev forms."""
import hashlib
import random

import numpy as np
import pytest

import crypto_primitives_b200 as cp
from crypto_primitives_b200 import ElGamal, Schnorr
from crypto_primitives_b200.commitment.blake2s import Commitment
from crypto_primitives_b200.signature.schnorr import Parameters, pack_messages
from oracle import fields as OF
from oracle import jubjub as J
import signature_oracle as O

pytestmark = pytest.mark.gpu

Fq, Fr = cp.BLS12_381_FR, cp.JUBJUB_FR
R = J.ORDER


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
        P = J.point_from_y(rng.randrange(J.Q))
        if P is not None:
            return P


@pytest.fixture(scope="module")
def setup():
    rng = OF.SplitMix64(2024)
    prm = Schnorr.setup(rng)
    G = pts_to_ints(prm.generator)[0]
    return prm, G, O.FixedBase(G)


# ---- the reference's scenarios (R/signature/mod.rs:52-105, R/encryption/elgamal/mod.rs:102-128, commitment) -------------
def test_reference_scenarios_through_the_mirror():
    rng = OF.SplitMix64(7)
    for msg in (b"Hi, I am a Schnorr signature!", b"\x00" * 4 + b"hello"):
        prm = Schnorr.setup(rng)
        pk, sk = Schnorr.keygen(prm, rng)
        sig = Schnorr.sign(prm, sk, msg, rng)
        assert Schnorr.verify(prm, pk, msg, sig)
        G = pts_to_ints(prm.generator)[0]
        assert O.verify(G, prm.salt, pts_to_ints(pk)[0], msg, sig_ints(sig)[0])
    # failed verification
    prm = Schnorr.setup(rng)
    pk, sk = Schnorr.keygen(prm, rng)
    sig = Schnorr.sign(prm, sk, b"Bad message", rng)
    assert not Schnorr.verify(prm, pk, b"Hi, I am a Schnorr signature!", sig)
    # randomize and verify
    msg = b"Hi, I am a Schnorr signature!"
    sig = Schnorr.sign(prm, sk, msg, rng)
    randomness = rng.bytes(32)
    rpk = Schnorr.randomize_public_key(prm, pk, randomness)
    rsig = Schnorr.randomize_signature(prm, sig, randomness)
    assert Schnorr.verify(prm, rpk, msg, rsig)
    # ElGamal round trip
    eprm = ElGamal.setup(rng)
    epk, esk = ElGamal.keygen(eprm, rng)
    m = ints_to_pts([J.mul(J.COFACTOR, random_point(random.Random(3)))])[0]
    r = Fr.elements([rng.field(R)])[0]
    ct = ElGamal.encrypt(eprm, epk, m, r)
    assert np.array_equal(ElGamal.decrypt(eprm, esk, ct), m)
    # Blake2s commitment
    assert Commitment.commit(None, b"input", bytes(range(32))) == hashlib.blake2s(b"input" + bytes(range(32)), digest_size=32).digest()


# ---- 2^16 signers ----------------------------------------------------------------------------------------------------------
N16 = 1 << 16


@pytest.fixture(scope="module")
def signed(setup):
    prm, G, fb = setup
    rng = random.Random(16)
    sks_i = [rng.randrange(R) for _ in range(N16)]
    ks_i = [rng.randrange(R) for _ in range(N16)]
    msgs = [bytes(rng.randrange(256) for _ in range(rng.randrange(301))) for _ in range(N16)]
    sks, ks = Fr.elements(sks_i), Fr.elements(ks_i)
    pks = Schnorr.keygen_batch(prm, sks)
    sigs, ok = Schnorr.sign_with_nonces_batch(prm, sks, ks, msgs)
    return dict(sks_i=sks_i, ks_i=ks_i, msgs=msgs, sks=sks, pks=pks, sigs=sigs, ok=ok)


def test_keygen_matches_the_oracle(setup, signed):
    prm, G, fb = setup
    exp = [fb.mul(sk) for sk in signed["sks_i"]]
    assert np.array_equal(signed["pks"], ints_to_pts(exp))
    assert pts_to_ints(signed["pks"][:4]) == [J.mul(sk, G) for sk in signed["sks_i"][:4]]


def test_sign_matches_the_oracle_bit_for_bit(setup, signed):
    prm, G, fb = setup
    exp_ok = np.zeros(N16, dtype=bool)
    exp = np.zeros((N16, 2, 4), dtype=np.uint64)
    accepted = []
    for i in range(N16):
        s = O.sign(G, prm.salt, signed["sks_i"][i], signed["msgs"][i], signed["ks_i"][i], mul=fb.mul)
        if s is not None:
            exp_ok[i] = True
            accepted.append((i, s))
    idx = np.array([i for i, _ in accepted])
    exp[idx] = sigs_from_ints([s for _, s in accepted])
    assert np.array_equal(signed["ok"], exp_ok)
    assert np.array_equal(signed["sigs"], exp)                          # rejected items are (0, 0)
    rate = 1 - exp_ok.mean()
    assert 0.07 < rate < 0.12, rate                                      # 1 - r / 2^252 = 0.094


def test_verify_accepts_every_signature_and_rejects_every_tampering(setup, signed):
    """Every accepted signature verifies; for each tampering every item is rejected, and the first items of each case are
    compared with the oracle's verdict (a Python oracle verification costs about 0.8 ms, so all 6 x 2^16 would take minutes)."""
    prm, G, fb = setup
    ok = signed["ok"]
    idx = np.nonzero(ok)[0]
    pks, sigs = signed["pks"][idx], signed["sigs"][idx]
    msgs = [signed["msgs"][i] for i in idx]
    assert Schnorr.verify_batch(prm, pks, msgs, sigs).all()
    n_or = 48
    assert all(O.verify(G, prm.salt, pts_to_ints(pks[j])[0], msgs[j], sig_ints(sigs[j])[0], mul=O.mul_ext) for j in range(8))

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
    other = Parameters(prm.generator, salt=bytes(b ^ 0x5A for b in prm.salt))
    cases["salt"] = (range(len(msgs)), pks, msgs, sigs, other)
    cases["truncated"] = (nz, pks, [m[:-1] if m else m for m in msgs], sigs, prm)
    for name, (sel, p, m, s, pp) in cases.items():
        sel = list(sel)
        got = Schnorr.verify_batch(pp, p[sel], [m[j] for j in sel], s[sel])
        exp = [O.verify(G, pp.salt, pts_to_ints(p[j])[0], m[j], sig_ints(s[j])[0], mul=O.mul_ext) for j in sel[:n_or]]
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
    exp_pk = [J.add(O.mul_ext(O.randomizer_int(r), G), P) for r, P in zip(rnd, pts_to_ints(pks))]
    assert pts_to_ints(rpk) == exp_pk
    assert O.randomize_public_key(G, pts_to_ints(pks[:1])[0], rnd[0]) == exp_pk[0]
    assert sig_ints(rsig) == [O.randomize_signature(s, r) for s, r in zip(sig_ints(sigs), rnd)]
    assert Schnorr.verify_batch(prm, rpk, msgs, rsig).all()


def test_any_generator_is_exact():
    """Parameters.generator is a public field: a generator outside the prime-order subgroup (cofactor part kept) gives the
    exact integer products, for keygen and for the unreduced randomize_public_key."""
    rng = random.Random(31)
    G = random_point(rng)
    assert J.mul(R, G) != J.IDENTITY
    prm = Parameters(ints_to_pts([G])[0], salt=bytes(32))
    sks_i = [rng.randrange(R) for _ in range(64)] + [0, 1, R - 1]
    assert pts_to_ints(Schnorr.keygen_batch(prm, Fr.elements(sks_i))) == [O.mul_ext(k, G) for k in sks_i]
    pks = ints_to_pts([random_point(rng) for _ in range(64)])
    rnd = [bytes(rng.randrange(256) for _ in range(40)) for _ in range(64)]
    got = pts_to_ints(Schnorr.randomize_public_key_batch(prm, pks, rnd))
    assert got == [O.randomize_public_key(G, P, r) for P, r in zip(pts_to_ints(pks), rnd)]


# ---- ElGamal ---------------------------------------------------------------------------------------------------------------
def test_elgamal(setup):
    prm, G, fb = setup
    eprm = cp.encryption_elgamal.Parameters(prm.generator)
    rng = random.Random(44)
    n = N16
    sks_i = [rng.randrange(R) for _ in range(n)]
    sks = Fr.elements(sks_i)
    pks = ElGamal.keygen_batch(eprm, sks)
    ms = ElGamal.keygen_batch(eprm, Fr.elements([rng.randrange(R) for _ in range(n)]))
    rs_i = [rng.randrange(R) for _ in range(n)]
    cts = ElGamal.encrypt_batch(eprm, pks, ms, Fr.elements(rs_i))
    assert np.array_equal(ElGamal.decrypt_batch(eprm, sks, cts), ms)
    k = 512
    exp = [O.elgamal_encrypt(G, P, M, r, mul=O.mul_ext) for P, M, r in zip(pts_to_ints(pks[:k]), pts_to_ints(ms[:k]), rs_i[:k])]
    assert np.array_equal(cts[:k], np.stack([ints_to_pts([c1, c2]) for c1, c2 in exp]))
    # decrypt of random pairs, points anywhere on the curve (cofactor part included)
    c = [(random_point(rng), random_point(rng)) for _ in range(k)]
    ct = np.stack([ints_to_pts([c1, c2]) for c1, c2 in c])
    got = pts_to_ints(ElGamal.decrypt_batch(eprm, sks[:k], ct))
    assert got == [O.elgamal_decrypt(s, cc, mul=O.mul_ext) for s, cc in zip(sks_i[:k], c)]


# ---- Blake2s commitment ----------------------------------------------------------------------------------------------------
def test_blake2s_commitment_2_20():
    n = 1 << 20
    g = np.random.default_rng(20)
    lens = g.integers(0, 301, n)
    lens[:301] = np.arange(301)
    values = g.integers(0, 256, int(lens.sum()), dtype=np.uint8)
    offsets = np.zeros(n + 1, dtype=np.uint64)
    offsets[1:] = np.cumsum(lens)
    rnd = g.integers(0, 256, (n, 32), dtype=np.uint8)
    import ctypes as C
    from crypto_primitives_b200 import _native as N
    out = np.empty((n, 32), dtype=np.uint8)
    N.check(N.lib.cpb_blake2s_commit_batch(0, values.ctypes.data_as(N.u8p), offsets.ctypes.data_as(N.u64p), rnd.ctypes.data_as(N.u8p),
                                           out.ctypes.data_as(N.u8p), n))
    vb, rb = values.tobytes(), rnd.tobytes()
    for i in range(n):
        a, b = int(offsets[i]), int(offsets[i + 1])
        assert out[i].tobytes() == hashlib.blake2s(vb[a:b] + rb[32 * i:32 * i + 32], digest_size=32).digest(), i
    # the Python mirror: list inputs
    assert np.array_equal(Commitment.commit_batch(None, [vb[:5], b""], [rb[:32], rb[32:64]]),
                          np.stack([np.frombuffer(hashlib.blake2s(x, digest_size=32).digest(), dtype=np.uint8)
                                    for x in (vb[:5] + rb[:32], rb[32:64])]))


# ---- _dev forms: results equal the host forms; nothing outside the outputs is written ---------------------------------------
def test_dev_forms_with_guard_regions(setup, signed):
    import torch
    prm, G, fb = setup
    dev = torch.device("cuda", 0)
    n = 1000
    GUARD = 64
    sks, pks, sigs = signed["sks"][:n], signed["pks"][:n], signed["sigs"][:n]
    msgs = signed["msgs"][:n]
    ks = Fr.elements([random.Random(5).randrange(R) for _ in range(n)])
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
    eprm = cp.encryption_elgamal.Parameters(prm.generator)
    b7, o7 = guarded((n, 2, 2, 4))
    ElGamal.encrypt_dev(eprm, t(pks), t(pks[::-1]), t(ks), out=o7)
    b8, o8 = guarded((n, 2, 4))
    ElGamal.decrypt_dev(eprm, t(sks), o7, out=o8)
    b9, o9 = guarded((n, 32), torch.uint8)
    Commitment.commit_dev(d_vals, d_off, t(rnd, torch.uint8), out=o9)
    torch.cuda.synchronize()
    for b in (b1, b2, b3, b4, b5, b6, b7, b8, b9):
        assert intact(b)
    assert np.array_equal(u64(o1), pks)
    hs, hok = Schnorr.sign_with_nonces_batch(prm, sks, ks, msgs)
    assert np.array_equal(u64(o2), hs) and np.array_equal(o3.cpu().numpy().astype(bool), hok)
    assert o4.cpu().numpy().astype(bool).tolist() == Schnorr.verify_batch(prm, pks, msgs, sigs).tolist()
    assert np.array_equal(u64(o5), Schnorr.randomize_public_key_batch(prm, pks, rnd))
    assert np.array_equal(u64(o6), Schnorr.randomize_signature_batch(prm, sigs, rnd))
    assert np.array_equal(u64(o7), ElGamal.encrypt_batch(eprm, pks, pks[::-1], ks))
    assert np.array_equal(u64(o8), pks[::-1])
    assert np.array_equal(o9.cpu().numpy(), Commitment.commit_batch(None, msgs, rnd))


def test_cpp_signature_mirror():
    """tests/cpp/test_signature.cpp through include/cpb200.hpp."""
    import os
    import subprocess
    from helpers import ROOT
    out_dir = os.path.join(ROOT, "tests", "host", "_build")
    os.makedirs(out_dir, exist_ok=True)
    exe = os.path.join(out_dir, "test_signature")
    lib_dir = os.path.join(ROOT, "crypto_primitives_b200")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "test_signature.cpp"),
                           "-L", lib_dir, "-l:libcpb200.so", f"-Wl,-rpath,{lib_dir}", "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "cpp signature ok" in r.stdout
