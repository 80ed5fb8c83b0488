"""Latency of the host-pointer entry points (include/cpb200.h): one form of each family at n = 1 (the fixed cost of staging),
2^10 and 2^20 (the copies), for two builds of the library loaded through CPB_LIB_NAME and alternated in the same run.  Each
(library, round) is a process of its own that times every family; a timing is the host clock around calls that end in the
library's own synchronisation, median of --reps calls after one warm-up call.  The card name, power limit and SM clock are read
in the same run.  Inputs are seeded random bytes: the forms copy and hash them whatever they hold.

    python tools/perf_host_forms.py --libs libcpb200_parent.so libcpb200.so [--rounds 3] [--reps 5] [--out FILE]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = (1, 1 << 10, 1 << 20)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def child(reps: int) -> dict:
    sys.path.insert(0, ROOT)
    import numpy as np
    import crypto_primitives_b200 as cp
    from crypto_primitives_b200 import _native as N
    from crypto_primitives_b200.crh import bowe_hopwood as bh, pedersen as ped
    from crypto_primitives_b200.commitment import pedersen as pcom
    from oracle import fields as OF

    L = N.lib
    g = np.random.default_rng(7)
    u64 = lambda a: a.ctypes.data_as(N.u64p)          # noqa: E731
    u8 = lambda a: a.ctypes.data_as(N.u8p)            # noqa: E731

    def elems(*shape):                                # field elements below 2^252: valid in every field
        a = g.integers(0, 1 << 63, (*shape, 4), dtype=np.uint64)
        a[..., 3] >>= 4
        return a

    f = cp.BLS12_381_FR
    cfg = cp.get_default_poseidon_parameters(f, 2, False)
    pc = cfg.context(0)
    t = cfg.rate + cfg.capacity
    rng = OF.SplitMix64(3)
    ped_prm = pcom.Commitment.setup(rng, ped.Window(4, 256), cp.curves.JUBJUB)     # 128-byte inputs; its two-to-one takes 128
    pd = ped_prm.context(0)
    bh_prm = bh.CRH.setup(rng, ped.Window(32, 8), cp.curves.JUBJUB)
    bc = bh_prm.context(0)
    sig = cp.Schnorr.setup(rng, cp.curves.JUBJUB)
    sc = sig.context(0)
    salt = sig.salt_arg()
    depth = 20
    tree_n = 1 << depth
    tree_leaves, tree_nodes = elems(tree_n), elems(tree_n - 1)
    applied = C.c_int(0)

    def family(n):
        """name -> zero-argument call of one host form over n items (buffers allocated here, outside the timing)."""
        F = {}
        x2, out1 = elems(n, 2), elems(n)
        F["poseidon_crh"] = lambda: L.cpb_poseidon_crh_batch(pc, u64(x2), 2, u64(out1), n)
        out3 = elems(n, 3)
        F["poseidon_sponge"] = lambda: L.cpb_poseidon_sponge_batch(pc, u64(x2), 2, u64(out3), 3, n)
        lens = g.integers(1, 5, n)
        off = np.zeros(n + 1, dtype=np.uint64)
        off[1:] = np.cumsum(lens)
        vals = elems(int(off[-1]))
        F["poseidon_crh_ragged"] = lambda: L.cpb_poseidon_crh_ragged_batch(pc, u64(vals), u64(off), u64(out1), n)
        root, sib, paths, idx = elems(1), elems(n), elems(n, depth - 1), np.zeros(n, dtype=np.uint64)
        ok = np.zeros(n, dtype=np.uint8)
        F["poseidon_verify"] = lambda: L.cpb_merkle_poseidon_verify_batch(pc, pc, u64(root), u64(x2), 2, u64(sib), u64(paths), depth - 1,
                                                                          u64(idx), u8(ok), n)
        states = elems(n, t)
        mode = N.SpongeMode(0, 0)
        F["duplex_absorb"] = lambda: L.cpb_poseidon_duplex_absorb(pc, u64(states), C.byref(mode), u64(x2), 2, n)
        modes = (N.SpongeMode * n)()
        F["duplex_absorb_ragged"] = lambda: L.cpb_poseidon_duplex_absorb_ragged(pc, u64(states), modes, u64(vals), u64(off), n)
        msg = g.integers(0, 256, (n, 128), dtype=np.uint8)
        pts = elems(n, 2)
        F["pedersen_crh"] = lambda: L.cpb_pedersen_crh_batch(pd, u8(msg), 128, 128, u64(pts), n)
        rnd = g.integers(0, 256, (n, 32), dtype=np.uint8)
        rnd[:, 31] = 0
        F["pedersen_commit"] = lambda: L.cpb_pedersen_commit_batch(pd, u8(msg), 128, 128, u8(rnd), u64(pts), n)
        F["bowe_hopwood_crh"] = lambda: L.cpb_bowe_hopwood_crh_batch(bc, u8(msg), 64, 64, u64(out1), n)
        k_idx = g.integers(0, tree_n, n, dtype=np.uint64)
        new = elems(n)
        F["poseidon_update"] = lambda: L.cpb_merkle_poseidon_update_digests(pc, u64(tree_leaves), u64(tree_nodes), tree_n, u64(k_idx),
                                                                             u64(new), n, None, C.byref(applied))
        psib, ppaths, proot = elems(n, 2), elems(n, depth - 1, 2), elems(2)
        F["pedersen_verify"] = lambda: L.cpb_merkle_pedersen_verify_batch(pd, pd, u64(proot), u8(msg), 128, u64(psib), u64(ppaths), depth - 1,
                                                                          u64(idx), u8(ok), n)
        F["mixed_verify"] = lambda: L.cpb_merkle_mixed_verify_batch(pd, pc, u64(root), u8(msg), 128, u64(sib), u64(paths), depth - 1,
                                                                    u64(idx), u8(ok), n)
        sks = elems(n)
        mo = np.arange(n + 1, dtype=np.uint64) * 64
        sigs, signed = elems(n, 2), np.zeros(n, dtype=np.uint8)
        F["schnorr_sign"] = lambda: L.cpb_schnorr_sign_batch(sc, salt, u64(sks), u64(sks), u8(msg), u64(mo), u64(sigs), u8(signed), n)
        F["schnorr_verify"] = lambda: L.cpb_schnorr_verify_batch(sc, salt, u64(pts), u8(msg), u64(mo), u64(sigs), u8(ok), n)
        F["field_to_montgomery"] = lambda: L.cpb_field_to_montgomery(f.id, 0, u64(sks), u64(out1), n)
        return F

    res = {}
    for n in SIZES:
        for name, fn in family(n).items():
            N.check(fn())                                  # warm-up: module load, arena growth
            ts = []
            for _ in range(reps):
                a = time.perf_counter()
                N.check(fn())
                ts.append((time.perf_counter() - a) * 1e3)
            res[f"{name}/{n}"] = sorted(ts)[len(ts) // 2]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--libs", nargs="+", default=["libcpb200.so"])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_host_forms_perf.json"))
    ap.add_argument("--child", action="store_true")
    args = ap.parse_args()
    if args.child:
        print(json.dumps(child(args.reps)))
        return
    runs = {lib: [] for lib in args.libs}
    gpu = [gpu_info()]
    for _ in range(args.rounds):
        for lib in args.libs:
            env = dict(os.environ, CPB_LIB_NAME=lib)
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--reps", str(args.reps)], env=env,
                               capture_output=True, text=True, check=True)
            runs[lib].append(json.loads(r.stdout.strip().splitlines()[-1]))
            gpu.append(gpu_info())
    keys = list(runs[args.libs[0]][0])
    table = {k: {lib: [r[k] for r in runs[lib]] for lib in args.libs} for k in keys}
    for k, v in table.items():
        print(f"{k:32s} " + "  ".join(f"{lib}: " + " ".join(f"{x:9.3f}" for x in xs) for lib, xs in v.items()) + "  (ms)")
    with open(args.out, "w") as fh:
        json.dump({"gpu (name, power limit, sm clock, max sm clock)": gpu, "unit": "ms, median of reps, per round", "rounds": args.rounds,
                   "reps": args.reps, "results": table}, fh, indent=1)
    print("wrote", args.out)


if __name__ == "__main__":
    main()
