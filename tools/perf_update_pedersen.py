"""Merkle update on one GPU for the Pedersen byte tree: 2^20 Jubjub leaves of 128 bytes, window 4 x 256 (the reference's Merkle
bench size), k distinct random leaves replaced (DESIGN §4.4).

For the default (18-bit) and the 8-bit table context, and k in {1, 16, 2^10, 2^16, 2^20}, it times with CUDA events (median of
--iters after a warm-up):
  dev        cpb_merkle_pedersen_update_dev on the device-resident tree, in place (CudaPedersenBackend.update);
  host       cpb_merkle_pedersen_update on a host-resident copy of the tree (MerkleTree.update_batch);
  level_loop the previous Python path of MerkleTree.update_batch (per level np.unique / stack on the host and one host-pointer
             two-to-one call), run in the same process and alternated with `host` call by call;
and once per context the full device rebuild (cpb_merkle_pedersen_build_dev).  For k in {1, 16} it also times `dev` with the narrow
levels on the per-level grids instead of the warp launch (a child process with CPB_PED_UPD_WARP_MAX=0: `dev_level_grids_ms`).  For each case it reports the hashes the update needs
(k leaf hashes + the touched inner nodes, counted from the indexes), the kernel launches of one `dev` call (torch.profiler, a
separate pass) and whether the three paths left the same tree.  The card's name, power limit and sampled SM clock are read in the
same run, and the SM clock is sampled every 0.5 s while the cases run (`sm_clock_during_mhz`).
Usage: python tools/perf_update_pedersen.py [--iters 5] [--out FILE]   (profiles/h100_update_pedersen_perf.json is one run)
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.perf_update import count_launches, gpu_info, timed, touched_inner  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--log2n", type=int, default=20)
    ap.add_argument("--ks", default="0,4,10,16,20", help="log2 of k")
    ap.add_argument("--chunk-bits", default="0,8", help="table contexts (0 = the library default)")
    ap.add_argument("--dev-only", action="store_true", help="time the _dev form only (the per-level-grid pass)")
    ap.add_argument("--out")
    a = ap.parse_args()
    clocks, stop = [], threading.Event()

    def sample():
        while not stop.is_set():
            try:
                q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                                   timeout=10).stdout.split()
                clocks.append(int(q[0]))
            except Exception:
                pass
            stop.wait(0.5)
    sampler = threading.Thread(target=sample, daemon=True)
    sampler.start()
    import numpy as np
    import torch
    import crypto_primitives_b200 as cp
    from crypto_primitives_b200.crh.pedersen import Parameters, Window
    from crypto_primitives_b200.distributed import CudaPedersenBackend
    from crypto_primitives_b200.merkle_tree import MerkleTree, PedersenByteConfig
    from oracle import pedersen as OPD

    class LevelLoopConfig(PedersenByteConfig):
        """The same hashes through the generic per-level loop (a subclass, so MerkleTree does not take the one-call path)."""

    res = {"gpu_info": gpu_info(), "log2_leaves": a.log2n, "curve": "jubjub", "window": [4, 256], "leaf_len": 128, "iters": a.iters,
           "contexts": []}
    oprm = OPD.setup(OPD.Window(4, 256), 5)
    gens = cp.BLS12_381_FR.elements([c for w in oprm.generators for pt in w for c in pt]).reshape(256, 4, 2, 4)
    n, h, L = 1 << a.log2n, a.log2n, 128
    g = torch.Generator(device="cuda").manual_seed(20)
    leaves = torch.randint(0, 256, (n, L), dtype=torch.uint8, device="cuda", generator=g)
    for cb in [int(x) for x in a.chunk_bits.split(",")]:
        prm = Parameters(cp.curves.JUBJUB, Window(4, 256), gens, chunk_bits=cb)
        be = CudaPedersenBackend(prm, prm, 0)
        ln, nn = be.build_local(leaves)
        ctx = {"chunk_bits_requested": cb, "rebuild_ms": statistics.median(timed(lambda: be.build_local(leaves), a.iters)), "cases": []}
        ln, nn = be.build_local(leaves)
        dl, dn = ln.clone(), nn.clone()
        hl = ln.cpu().numpy().view(np.uint64).reshape(n, 2, 4).copy()
        hn = nn.cpu().numpy().view(np.uint64).reshape(n - 1, 2, 4).copy()
        loop_tree = MerkleTree(LevelLoopConfig(), hl.copy(), hn.copy(), prm, prm, 0)
        host_tree = MerkleTree(PedersenByteConfig(), hl, hn, prm, prm, 0)
        rng = np.random.default_rng(20 + cb)
        for lk in [int(x) for x in a.ks.split(",")]:
            k = 1 << lk
            idx = np.sort(rng.choice(n, size=k, replace=False)).astype(np.int64)
            rng.shuffle(idx)
            new = torch.randint(0, 256, (k, L), dtype=torch.uint8, device="cuda", generator=g)
            new_np = new.cpu().numpy()
            d_idx = torch.from_numpy(idx).cuda()
            hashes = k + touched_inner(idx, h)
            case = {"k": k, "hashes": int(hashes)}
            case["dev_ms"] = statistics.median(timed(lambda: be.update(dl, dn, d_idx, new), a.iters))
            case["dev_launches"] = count_launches(lambda: be.update(dl, dn, d_idx, new))
            if a.dev_only:
                ctx["cases"].append(case)
                continue
            iters = a.iters if k <= (1 << 16) else 2
            host_ms, loop_ms = [], []
            for it in range(iters + 1):                         # alternated call by call; the first pair is the warm-up
                for tree, acc in ((host_tree, host_ms), (loop_tree, loop_ms)):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    tree.update_batch(idx, new_np)
                    torch.cuda.synchronize()
                    if it:
                        acc.append(1e3 * (time.perf_counter() - t0))
            case["host_ms"], case["level_loop_ms"] = statistics.median(host_ms), statistics.median(loop_ms)
            case["dev_over_rebuild"] = case["dev_ms"] / ctx["rebuild_ms"]
            for key in ("dev", "host", "level_loop"):
                case[f"{key}_hashes_per_s"] = hashes / (case[f"{key}_ms"] * 1e-3)
            dev_nodes = dn.cpu().numpy().view(np.uint64).reshape(n - 1, 2, 4)
            dev_leaves = dl.cpu().numpy().view(np.uint64).reshape(n, 2, 4)
            case["trees_agree"] = bool(np.array_equal(dev_nodes, host_tree.non_leaf_nodes) and np.array_equal(dev_leaves, host_tree.leaf_nodes)
                                       and np.array_equal(loop_tree.non_leaf_nodes, host_tree.non_leaf_nodes)
                                       and np.array_equal(loop_tree.leaf_nodes, host_tree.leaf_nodes))
            ctx["cases"].append(case)
            print(json.dumps({"chunk_bits_requested": cb, **case}), flush=True)
        del be
        res["contexts"].append(ctx)
        print(json.dumps({"chunk_bits_requested": cb, "rebuild_ms": ctx["rebuild_ms"]}), flush=True)
        del prm
        torch.cuda.empty_cache()
    stop.set()
    sampler.join()
    res["sm_clock_during_mhz"] = {"samples": len(clocks), "min": min(clocks, default=None), "median": statistics.median(clocks) if clocks else None,
                                  "max": max(clocks, default=None)}
    if not a.dev_only:                                        # the narrow levels on per-level grids, k in {1, 16}
        with tempfile.TemporaryDirectory() as td:
            out = os.path.join(td, "grids.json")
            env = dict(os.environ, CPB_PED_UPD_WARP_MAX="0")
            subprocess.run([sys.executable, os.path.abspath(__file__), "--dev-only", "--ks", "0,4", "--iters", str(a.iters), "--log2n",
                            str(a.log2n), "--chunk-bits", a.chunk_bits, "--out", out], env=env, check=True)
            with open(out) as f:
                grids = json.load(f)
        for ctx, gctx in zip(res["contexts"], grids["contexts"]):
            for gc in gctx["cases"]:
                for case in ctx["cases"]:
                    if case["k"] == gc["k"]:
                        case["dev_level_grids_ms"] = gc["dev_ms"]
                        case["dev_level_grids_launches"] = gc["dev_launches"]
                        case["warp_launch_wins"] = case["dev_ms"] < gc["dev_ms"]
                        print(json.dumps({"chunk_bits_requested": ctx["chunk_bits_requested"], "k": case["k"], "dev_ms": case["dev_ms"],
                                          "dev_level_grids_ms": gc["dev_ms"]}), flush=True)
    res["gpu_info_after"] = gpu_info()
    print(json.dumps(res["gpu_info"]))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
