"""Throughput of the Schnorr / ElGamal / Blake2s-commitment kernels (include/cpb200.h) on one GPU: keygen, sign, verify, ElGamal
encrypt and decrypt, and the Blake2s commitment, at n = 2^20 items with messages of 32..256 bytes, through the _dev forms on
device-resident inputs.  CUDA events around each call, median of repeated calls after a warm-up; the card name and power
limit are read in the same run.  --curve picks the curve (default jubjub); ed_on_bls12_377 also times sign and verify on the
reference benchmark's message, [100u8; 128] for every item (R/benches/signature.rs).  Writes
profiles/h100_signature_perf.json for Jubjub, profiles/h100_signature_ed377_perf.json for ed-on-BLS12-377 (or --out).

    python tools/perf_signature.py [--curve jubjub|ed_on_bls12_377] [--n 1048576] [--reps 5] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import random
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import crypto_primitives_b200 as cp  # noqa: E402
from crypto_primitives_b200 import ElGamal, Schnorr  # noqa: E402
from crypto_primitives_b200.commitment.blake2s import Commitment  # noqa: E402
from crypto_primitives_b200.signature.schnorr import pack_messages  # noqa: E402
from oracle import fields as OF  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timed(fn, reps):
    fn()                                                  # warm-up: module load, pool growth
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times)), times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--curve", choices=sorted(cp.curves.CURVES), default="jubjub")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    curve = cp.curves.CURVES[args.curve]
    if args.out is None:
        args.out = os.path.join(ROOT, "profiles", "h100_signature_perf.json" if curve is cp.curves.JUBJUB else "h100_signature_ed377_perf.json")
    n = args.n
    dev = torch.device("cuda", 0)
    rng = OF.SplitMix64(1)
    prm = Schnorr.setup(rng, curve)
    eprm = cp.encryption_elgamal.Parameters(prm.generator, curve)
    g = np.random.default_rng(2)
    r = curve.scalar_modulus
    pyr = random.Random(3)
    # distinct random scalars for a slice, tiled: the kernels' work does not depend on the values beyond their bits
    base = curve.scalar_field.elements([pyr.randrange(r) for _ in range(4096)])
    sks = np.ascontiguousarray(np.tile(base, (n // 4096 + 1, 1))[:n])
    ks = np.ascontiguousarray(np.roll(sks, 1, axis=0))
    lens = g.integers(32, 257, n)
    values = g.integers(0, 256, int(lens.sum()), dtype=np.uint8)
    offsets = np.zeros(n + 1, dtype=np.uint64)
    offsets[1:] = np.cumsum(lens)

    def t(a, dtype=torch.int64):
        a = np.ascontiguousarray(a)
        return torch.from_numpy(a.view(np.int64) if dtype == torch.int64 else a).to(dev)

    d_sk, d_k = t(sks), t(ks)
    d_vals, d_off = t(values, torch.uint8), t(offsets)
    d_pk = Schnorr.keygen_dev(prm, d_sk)
    d_sig, d_ok = Schnorr.sign_with_nonces_dev(prm, d_sk, d_k, d_vals, d_off)
    d_vok = Schnorr.verify_dev(prm, d_pk, d_vals, d_off, d_sig)
    d_ct = ElGamal.encrypt_dev(eprm, d_pk, d_pk, d_k)
    d_m = ElGamal.decrypt_dev(eprm, d_sk, d_ct)
    d_rnd = t(g.integers(0, 256, (n, 32), dtype=np.uint8), torch.uint8)
    d_cm = Commitment.commit_dev(d_vals, d_off, d_rnd)
    torch.cuda.synchronize()
    signed = d_ok.cpu().numpy().astype(bool)
    checks = {"signed_fraction": float(signed.mean()),
              "every_signed_item_verifies": bool(d_vok.cpu().numpy().astype(bool)[signed].all()),
              "decrypt_returns_the_message": bool(torch.equal(d_m, d_pk))}

    ops = {
        "keygen": lambda: Schnorr.keygen_dev(prm, d_sk, out=d_pk),
        "sign": lambda: Schnorr.sign_with_nonces_dev(prm, d_sk, d_k, d_vals, d_off, sigs_out=d_sig, signed_out=d_ok),
        "verify": lambda: Schnorr.verify_dev(prm, d_pk, d_vals, d_off, d_sig, ok_out=d_vok),
        "elgamal_encrypt": lambda: ElGamal.encrypt_dev(eprm, d_pk, d_pk, d_k, out=d_ct),
        "elgamal_decrypt": lambda: ElGamal.decrypt_dev(eprm, d_sk, d_ct, out=d_m),
        "blake2s_commit": lambda: Commitment.commit_dev(d_vals, d_off, d_rnd, out=d_cm),
    }
    if curve is not cp.curves.JUBJUB:
        # the reference benchmark's message for every item: sign, then verify what was signed
        d_vals128 = t(np.full(128 * n, 100, dtype=np.uint8), torch.uint8)
        d_off128 = t(np.arange(n + 1, dtype=np.uint64) * 128)
        d_sig128, d_ok128 = Schnorr.sign_with_nonces_dev(prm, d_sk, d_k, d_vals128, d_off128)
        d_vok128 = Schnorr.verify_dev(prm, d_pk, d_vals128, d_off128, d_sig128)
        torch.cuda.synchronize()
        signed128 = d_ok128.cpu().numpy().astype(bool)
        checks["signed_fraction_128"] = float(signed128.mean())
        checks["every_signed_item_verifies_128"] = bool(d_vok128.cpu().numpy().astype(bool)[signed128].all())
        ops["sign_msg128"] = lambda: Schnorr.sign_with_nonces_dev(prm, d_sk, d_k, d_vals128, d_off128, sigs_out=d_sig128, signed_out=d_ok128)
        ops["verify_msg128"] = lambda: Schnorr.verify_dev(prm, d_pk, d_vals128, d_off128, d_sig128, ok_out=d_vok128)
    results = {}
    for name, fn in ops.items():
        med, times = timed(fn, args.reps)
        results[name] = {"median_ms": med, "items_per_s": n / (med / 1e3), "times_ms": times}
        print(f"{name:16s} {med:9.2f} ms  {n / (med / 1e3) / 1e6:8.3f} M items/s", flush=True)
    out = {"gpu": gpu_info(), "n": n, "message_bytes": "uniform 32..256", "reps": args.reps, "checks": checks, "results": results}
    if curve is not cp.curves.JUBJUB:
        out = {"curve": curve.name, **out, "msg128": "[100u8; 128] for every item (sign_msg128, verify_msg128)"}
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps({"gpu": out["gpu"], "checks": checks}))


if __name__ == "__main__":
    main()
