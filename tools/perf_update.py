"""Merkle update on one GPU: the 2^24-leaf BN254 bench tree, k distinct random leaves replaced (DESIGN §4.4).

For k in {1, 16, 2^10, 2^16, 2^20} it times, with CUDA events around each call (median of --iters after a warm-up):
  dev        cpb_merkle_poseidon_update_dev on the device-resident tree, in place (CudaPoseidonBackend.update);
  host       cpb_merkle_poseidon_update on a host-resident copy of the tree (only touched nodes and read siblings cross PCIe);
  level_loop the previous Python path of MerkleTree.update_batch for the same k: per level, np.unique / stack on the host and one
             host-pointer two-to-one call (kept in merkle_tree.py for the Configs without a Poseidon inner hash); run in the same
             process and alternated with `host` call by call;
and once per run the full device rebuild (cpb_merkle_poseidon_build_dev).  For each case it reports the permutations the update
needs (k leaf hashes + the touched inner nodes, counted from the indexes), the achieved permutations/s, and the kernel launches of
one `dev` call (torch.profiler, a separate pass).  The card's name, power limit and sampled SM clock are read in the same run.
Usage: python tools/perf_update.py [--iters 5] [--out FILE]   (profiles/h100_update_perf.json is one run)
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


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, sm, smax = [x.strip() for x in q.split(",")]
        return {"gpu": name, "power_limit": pl, "sm_clock_now": sm, "sm_clock_max": smax}
    except Exception as e:                                 # the numbers are still reported, without the card's settings
        return {"gpu_info_error": repr(e)}


def touched_inner(idx, h):
    import numpy as np
    u, total = np.unique(idx), 0
    for _ in range(h):
        u = np.unique(u >> 1)
        total += u.size
    return total


def timed(fn, iters, warm=1):
    import torch
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1))
    return out


def count_launches(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "emcpy" not in e.name and "emset" not in e.name)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--log2n", type=int, default=24)
    ap.add_argument("--ks", default="0,4,10,16,20", help="log2 of k")
    ap.add_argument("--out")
    a = ap.parse_args()
    import numpy as np
    import torch
    import bench
    import bench_inputs as BI
    import crypto_primitives_b200 as cp
    from crypto_primitives_b200 import _native as N
    from crypto_primitives_b200.distributed import CudaPoseidonBackend
    from crypto_primitives_b200.merkle_tree import MerkleTree, PoseidonFieldConfig

    class LevelLoopConfig(PoseidonFieldConfig):
        """The same hashes through the generic per-level loop (a subclass, so MerkleTree does not take the one-call path)."""

    res = {"gpu_info": gpu_info(), "log2_leaves": a.log2n, "field": "bn254_fr", "iters": a.iters, "cases": []}
    prm = bench.poseidon_params(cp, "bn254")
    n, h = 1 << a.log2n, a.log2n
    leaves = BI.field_elements_torch(torch, N, prm.field.id, BI.SEED_CONFIG4, 0, 2 * n, 0).view(n, 2, 4)
    be = CudaPoseidonBackend(prm, prm, 0)
    ln, nn = be.build_local(leaves)
    res["rebuild_ms"] = statistics.median(timed(lambda: be.build_local(leaves), a.iters))
    dl, dn = ln.clone(), nn.clone()
    hl, hn = ln.cpu().numpy().view(np.uint64).copy(), nn.cpu().numpy().view(np.uint64).copy()
    loop_tree = MerkleTree(LevelLoopConfig(), hl.copy(), hn.copy(), prm, prm, 0)
    host_tree = MerkleTree(PoseidonFieldConfig(), hl, hn, prm, prm, 0)
    rng = np.random.default_rng(24)
    for lk in [int(x) for x in a.ks.split(",")]:
        k = 1 << lk
        idx = np.sort(rng.choice(n, size=k, replace=False)).astype(np.int64)
        rng.shuffle(idx)
        new = BI.field_elements_torch(torch, N, prm.field.id, 900 + lk, 0, 2 * k, 0).view(k, 2, 4)
        new_np = new.cpu().numpy().view(np.uint64)
        d_idx = torch.from_numpy(idx).cuda()
        perms = k + touched_inner(idx, h)
        case = {"k": k, "permutations": int(perms)}
        dev_ms = timed(lambda: be.update(dl, dn, d_idx, new), a.iters)
        case["dev_ms"] = statistics.median(dev_ms)
        case["dev_launches"] = count_launches(lambda: be.update(dl, dn, d_idx, new))
        iters = a.iters if k <= (1 << 16) else 2
        host_ms, loop_ms = [], []
        for it in range(iters + 1):                             # alternated call by call; the first pair is the warm-up
            for name, tree, acc in (("host", host_tree, host_ms), ("level_loop", loop_tree, loop_ms)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                tree.update_batch(idx, new_np)
                torch.cuda.synchronize()
                if it:
                    acc.append(1e3 * (time.perf_counter() - t0))
        case["host_ms"], case["level_loop_ms"] = statistics.median(host_ms), statistics.median(loop_ms)
        case["level_loop_launches"] = 1 + h                      # one leaf-hash call, then one two-to-one call per level
        for key in ("dev", "host", "level_loop"):
            case[f"{key}_perm_per_s"] = perms / (case[f"{key}_ms"] * 1e-3)
        # every path left the same tree
        case["trees_agree"] = bool(np.array_equal(dn.cpu().numpy().view(np.uint64), host_tree.non_leaf_nodes)
                                   and np.array_equal(loop_tree.non_leaf_nodes, host_tree.non_leaf_nodes))
        res["cases"].append(case)
        print(json.dumps(case), flush=True)
    res["gpu_info_after"] = gpu_info()
    print(json.dumps({"rebuild_ms": res["rebuild_ms"], **res["gpu_info"]}))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
