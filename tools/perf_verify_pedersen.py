"""Merkle path verification on one GPU for the two trees with a Pedersen leaf hash (DESIGN §4.4):
  byte   2^20 Jubjub leaves of 128 bytes, window 4 x 256, default (18-bit) tables, pedersen::TwoToOneCRH nodes;
  mixed  2^20 leaves of 128 bytes with the Pedersen and Poseidon parameters of bench config 5 (BLS12-381 Fr, rate 2).
For n in {1, 16, 2^10, 2^16, 2^20} proofs of random leaves it times
  dev        cpb_merkle_*_verify_batch_dev on device-resident proofs (CUDA events, median of --iters after a warm-up);
  host       cpb_merkle_*_verify_batch through MerkleTree.verify_proofs_batch on host arrays (host clock around a synchronised call);
  level_loop verify_paths_batch, the level-synchronous Python path (one host-pointer two-to-one call per level), median of --iters,
             2 at n >= 2^16; `host` and `level_loop` alternate call by call;
asserts that every verdict is true and that the three forms agree, and counts the kernel launches of one `dev` call for n in {1, 2^10}
(torch.profiler, one child process per tree: repeated profiler sessions in the timing process dropped kernel records).  The card's
name, power limit and SM clock are read in the same run, and the SM clock is sampled every 0.5 s while the cases run
(`sm_clock_during_mhz`).
Usage: python tools/perf_verify_pedersen.py [--iters 5] [--out FILE]   (profiles/h100_verify_pedersen_perf.json is one run)
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

from tools.perf_update import count_launches, gpu_info, timed  # noqa: E402


class _Proof:
    """A Path over rows of the proof arrays (no copies), for verify_paths_batch."""
    __slots__ = ("leaf_sibling_hash", "auth_path", "leaf_index")

    def __init__(self, sib, path, index):
        self.leaf_sibling_hash, self.auth_path, self.leaf_index = sib, path, index


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--log2n", type=int, default=20)
    ap.add_argument("--ns", default="0,4,10,16,20", help="log2 of the number of proofs")
    ap.add_argument("--trees", default="byte,mixed")
    ap.add_argument("--count-only", action="store_true", help="only count the launches of one dev call (the profiler pass)")
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
    import bench_inputs as BI
    import crypto_primitives_b200 as cp
    from crypto_primitives_b200 import _native as N
    from crypto_primitives_b200.commitment.pedersen import Commitment
    from crypto_primitives_b200.crh.pedersen import Parameters, Window
    from crypto_primitives_b200.distributed import CudaMixedBackend, CudaPedersenBackend
    from crypto_primitives_b200.merkle_tree import MerkleTree, PedersenByteConfig, PedersenPoseidonConfig, verify_paths_batch
    from oracle import pedersen as OPD

    res = {"gpu_info": gpu_info(), "log2_leaves": a.log2n, "leaf_len": 128, "iters": a.iters, "trees": []}
    n_leaves, L = 1 << a.log2n, 128
    g = torch.Generator(device="cuda").manual_seed(30)
    leaves = torch.randint(0, 256, (n_leaves, L), dtype=torch.uint8, device="cuda", generator=g)
    leaves_np = leaves.cpu().numpy()
    stream = lambda: torch.cuda.current_stream().cuda_stream                      # noqa: E731
    for kind in a.trees.split(","):
        if kind == "byte":
            oprm = OPD.setup(OPD.Window(4, 256), 5)
            gens = cp.BLS12_381_FR.elements([c for w in oprm.generators for pt in w for c in pt]).reshape(256, 4, 2, 4)
            leaf_prm = node_prm = Parameters(cp.curves.JUBJUB, Window(4, 256), gens)
            be, cfg, w = CudaPedersenBackend(leaf_prm, node_prm, 0), PedersenByteConfig(), 8
            fn = N.lib.cpb_merkle_pedersen_verify_batch_dev
            desc = {"tree": "byte", "curve": "jubjub", "window": [4, 256], "chunk_bits": "library default (18)"}
        else:
            leaf_prm = Commitment.setup(BI.StreamRng(BI.SEED_CONFIG3_PARAMS), Window(4, 256))
            node_prm = cp.get_default_poseidon_parameters(cp.BLS12_381_FR, 2, False)
            be, cfg, w = CudaMixedBackend(leaf_prm, node_prm, 0), PedersenPoseidonConfig(), 4
            fn = N.lib.cpb_merkle_mixed_verify_batch_dev
            desc = {"tree": "mixed", "curve": "jubjub", "window": [4, 256], "poseidon": "BLS12-381 Fr default, rate 2 (bench config 5)"}
        ln, nn = be.build_local(leaves)
        torch.cuda.synchronize()
        hl = ln.cpu().numpy().view(np.uint64).reshape((n_leaves,) + ((2, 4) if w == 8 else (4,))).copy()
        hn = nn.cpu().numpy().view(np.uint64).reshape((n_leaves - 1,) + hl.shape[1:]).copy()
        del ln, nn
        tree = MerkleTree(cfg, hl, hn, leaf_prm, node_prm, 0)
        plen = tree.height() - 2
        lctx, nctx = leaf_prm.context(0), node_prm.context(0)
        d_root = torch.from_numpy(tree.root().reshape(-1).view(np.int64)).cuda()
        rng = np.random.default_rng(31)
        entry = {**desc, "path_len": plen, "cases": []}
        for lg in [int(x) for x in a.ns.split(",")]:
            n = 1 << lg
            ix = rng.integers(0, n_leaves, size=n).astype(np.int64)
            sib, paths, idx = tree.generate_proofs_batch(ix)
            lv = np.ascontiguousarray(leaves_np[ix])
            d_lv = torch.from_numpy(lv).cuda()
            d_sib = torch.from_numpy(np.ascontiguousarray(sib).view(np.int64)).cuda()
            d_paths = torch.from_numpy(np.ascontiguousarray(paths).view(np.int64)).cuda()
            d_idx = torch.from_numpy(idx.view(np.int64)).cuda()
            d_ok = torch.zeros(n, dtype=torch.uint8, device="cuda")

            def dev():
                N.check(fn(lctx, nctx, d_root.data_ptr(), d_lv.data_ptr(), L, L, d_sib.data_ptr(), d_paths.data_ptr(), plen, d_idx.data_ptr(),
                           d_ok.data_ptr(), n, stream()))
            if a.count_only:
                dev()
                entry["cases"].append({"n": n, "dev_launches": count_launches(dev)})
                continue
            case = {"n": n, "dev_ms": statistics.median(timed(dev, a.iters))}
            dev_ok = d_ok.cpu().numpy().astype(bool)
            proofs = [_Proof(sib[i], paths[i], int(idx[i])) for i in range(n)]
            iters, warm = (a.iters, 1) if n < (1 << 16) else (2, 0)   # alternated call by call; below 2^16 the first pair is a warm-up
            host_ms, loop_ms, verdicts = [], [], {}
            for it in range(warm + iters):
                for key, call, acc in (("host", lambda: tree.verify_proofs_batch((sib, paths, idx), lv), host_ms),
                                       ("level_loop", lambda: verify_paths_batch(leaf_prm, node_prm, tree.root(), lv, proofs, cfg), loop_ms)):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    verdicts[key] = np.asarray(call())
                    torch.cuda.synchronize()
                    if it >= warm:
                        acc.append(1e3 * (time.perf_counter() - t0))
            case["host_ms"], case["level_loop_ms"] = statistics.median(host_ms), statistics.median(loop_ms)
            case["level_loop_over_dev"] = case["level_loop_ms"] / case["dev_ms"]
            case["all_true"] = bool(dev_ok.all() and verdicts["host"].all() and verdicts["level_loop"].all())
            case["forms_agree"] = bool(np.array_equal(dev_ok, verdicts["host"]) and np.array_equal(dev_ok, verdicts["level_loop"]))
            assert case["all_true"] and case["forms_agree"], case
            entry["cases"].append(case)
            print(json.dumps({"tree": kind, **case}), flush=True)
            del proofs, d_lv, d_sib, d_paths, d_idx, d_ok
        res["trees"].append(entry)
        del be, tree
        torch.cuda.empty_cache()
    stop.set()
    sampler.join()
    res["sm_clock_during_mhz"] = {"samples": len(clocks), "min": min(clocks, default=None), "median": statistics.median(clocks) if clocks else None,
                                  "max": max(clocks, default=None)}
    if not a.count_only:
        for entry in res["trees"]:                            # one child per tree: a few profiler sessions each
            with tempfile.TemporaryDirectory() as td:
                out = os.path.join(td, "launches.json")
                subprocess.run([sys.executable, os.path.abspath(__file__), "--count-only", "--ns", "0,10", "--log2n", str(a.log2n), "--trees",
                                entry["tree"], "--out", out], check=True)
                with open(out) as f:
                    cases = json.load(f)["trees"][0]["cases"]
            entry["dev_launches"] = {str(c["n"]): c["dev_launches"] for c in cases}
            print(json.dumps({"tree": entry["tree"], "path_len": entry["path_len"], "dev_launches": entry["dev_launches"]}), flush=True)
    res["gpu_info_after"] = gpu_info()
    print(json.dumps(res["gpu_info"]))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
