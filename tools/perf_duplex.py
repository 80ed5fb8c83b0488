"""Batched duplex sponges on one GPU (DESIGN §4.2): a Fiat-Shamir-shaped transcript over many sponges at once.

For the bench's BN254 Fr t = 3 config and BLS12-381 Fr default rate 2, n = 2^20 sponges (--log-n) each run one 64-byte
absorb_bytes, then 8 rounds of absorb(2) + squeeze(1).  At rate 2 the byte absorb (3 elements) and the first absorb(2) permute
once at a block boundary, every squeeze(1) permutes once on leaving Absorbing mode, and the later absorb(2) calls (from
Squeezing mode, lanes 0-1) permute not at all.  Per call kind: the median time of the _dev call (CUDA events) and, for the kinds
that permute, the permutations per second; the same n through cpb_poseidon_permute_batch_dev, alternated with the duplex calls in
the same run, so the two compare one permutation per sponge with the same state traffic.  Then the same
transcript for 16 sponges one after the other through PoseidonSponge (one host-form call per absorb or squeeze) and through one
cpb_poseidon_permute_batch call of n = 1 per permutation (the permutations alone of the Python duplex loop PoseidonSponge ran
before; its big-int additions are not counted, so that figure is a lower bound of the old cost).
Prints one JSON object with the card's name, power limit and SM clock read in the same run; --out also writes it.
Usage: python tools/perf_duplex.py [--log-n 20] [--reps 5] [--out FILE]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    import numpy as np
    import torch
    import bench
    import crypto_primitives_b200 as cp
    from crypto_primitives_b200 import _native as N

    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream().cuda_stream
    n = 1 << a.log_n
    configs = {"bn254_t3": bench.poseidon_params(cp, "bn254"),
               "bls12_381_r2": cp.get_default_poseidon_parameters(cp.BLS12_381_FR, 2, False)}
    res = {"card": None, "n": n, "configs": {}}
    for name, cfg in configs.items():
        ctx = cfg.context(0)
        t = cfg.rate + cfg.capacity
        f = cfg.field
        g = torch.Generator(device="cpu").manual_seed(1)
        msg = torch.randint(0, 256, (n, 64), dtype=torch.uint8, generator=g).to(dev)
        el = torch.from_numpy(np.tile(f.elements([3, 5]), (n, 1, 1)).view(np.int64)).to(dev)
        states = torch.zeros((n, t, 4), dtype=torch.int64, device=dev)
        out = torch.empty((n, 1, 4), dtype=torch.int64, device=dev)
        pin, pout = torch.zeros_like(states), torch.empty_like(states)

        def transcript(times):
            states.zero_()
            m = N.SpongeMode(0, 0)
            calls = [("absorb_bytes", lambda: N.lib.cpb_poseidon_duplex_absorb_bytes_dev(ctx, states.data_ptr(), C.byref(m), msg.data_ptr(), 64, 64, n, st))]
            for r in range(8):
                calls.append(("absorb2_first" if r == 0 else "absorb2_no_perm", lambda: N.lib.cpb_poseidon_duplex_absorb_dev(ctx, states.data_ptr(), C.byref(m), el.data_ptr(), 2, n, st)))
                calls.append(("squeeze1", lambda: N.lib.cpb_poseidon_duplex_squeeze_dev(ctx, states.data_ptr(), C.byref(m), out.data_ptr(), 1, 0, n, st)))
            for kind, fn in calls:
                for arm, call in ((kind, fn), ("permute_batch_dev", lambda: N.lib.cpb_poseidon_permute_batch_dev(ctx, pin.data_ptr(), pout.data_ptr(), n, st))):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    N.check(call())
                    e1.record()
                    torch.cuda.synchronize()
                    times.setdefault(arm, []).append(e0.elapsed_time(e1))

        transcript({})                                     # warm-up
        times = {}
        for _ in range(a.reps):
            transcript(times)
        perms = {"absorb_bytes": 1, "absorb2_first": 1, "absorb2_no_perm": 0, "squeeze1": 1, "permute_batch_dev": 1}
        r = {k: {"median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v), "calls": len(v), "perms_per_call": perms[k],
                 "perms_per_s": perms[k] * n / (statistics.median(v) * 1e-3)} for k, v in times.items()}
        r["duplex_vs_permute"] = {k: r[k]["median_ms"] / r["permute_batch_dev"]["median_ms"] for k in ("absorb_bytes", "absorb2_first", "squeeze1")}

        # 16 transcripts one after the other: the new PoseidonSponge, and one n = 1 permute call per permutation
        msg16 = [bytes(range(i, i + 64)) for i in range(16)]
        x2 = f.elements([3, 5])

        def single():
            for i in range(16):
                s = cp.PoseidonSponge(cfg)
                s.absorb(msg16[i])
                for _ in range(8):
                    s.absorb(x2)
                    s.squeeze_native_field_elements(1)

        st1 = np.zeros((t, 4), dtype=np.uint64)
        o1 = np.empty_like(st1)

        def old_perms():
            for _ in range(16 * 10):                       # 10 permutations per transcript
                N.check(N.lib.cpb_poseidon_permute_batch(ctx, st1.ctypes.data_as(N.u64p), o1.ctypes.data_as(N.u64p), 1))

        for fn, key in ((single, "sponge_16_transcripts_ms"), (old_perms, "permute_n1_16_transcripts_ms")):
            fn()
            ts = []
            for _ in range(3):
                t0 = time.perf_counter()
                fn()
                ts.append((time.perf_counter() - t0) * 1e3)
            r[key] = statistics.median(ts)
        res["configs"][name] = r
    res["card"] = _card()
    s = json.dumps(res)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(s + "\n")


if __name__ == "__main__":
    main()
