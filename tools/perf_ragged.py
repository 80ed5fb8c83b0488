"""Ragged Poseidon batches on one GPU: what the ordering by permutation count buys (DESIGN §4.2).

  (a) 2^24 BN254 inputs of length 2: the ragged CRH against the uniform leaf kernel (cpb_poseidon_crh_batch_dev).
  (b) 2^22 BN254 inputs with lengths uniform on 0..8 (1-4 absorb permutations at rate 2):
      (i)   the ragged call;
      (ii)  the ideal: one uniform call per length on inputs grouped by length in advance on the device (grouping not timed);
      (iii) the ragged kernels in input order, no ordering step (CPB_RAGGED_ORDER=0, read once, so a process of its own).
  (c) the ordering step alone (histogram + scan + scatter kernels, torch.profiler device time) at 2^22 and 2^24 items.
  (d) a 2^24-leaf ragged tree with every leaf of length 2 against cpb_merkle_poseidon_build_dev on the same leaves; both roots
      are checked against the bench golden root.

The parent process only spawns children, alternating the ordered and unordered ones, `--runs` of each; every child times its
arms alternately (CUDA events around each call, median of `--iters` after a warm-up) and prints one JSON line.  The parent
prints the summary with the card's name, power limit and SM clock read in the same run, and with --out also writes every run
to that file (profiles/h100_ragged_perf.json is one).
Usage: python tools/perf_ragged.py [--runs 3] [--iters 5] [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _time(fn, iters, warm=1):
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
    return statistics.median(out)


def child(mode, iters):
    import torch
    import bench
    import bench_inputs as BI
    import crypto_primitives_b200 as cp
    from crypto_primitives_b200 import _native as N

    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream().cuda_stream
    cfg = bench.poseidon_params(cp, "bn254")
    ctx = cfg.context(0)
    fid = cfg.field.id
    res = {"mode": mode}

    # (b) 2^22 inputs, lengths uniform on 0..8
    nb = 1 << 22
    g = torch.Generator(device=dev)
    g.manual_seed(2024)
    lens = torch.randint(0, 9, (nb,), generator=g, device=dev, dtype=torch.int64)
    offb = torch.zeros(nb + 1, dtype=torch.int64, device=dev)
    offb[1:] = torch.cumsum(lens, 0)
    vb = BI.field_elements_torch(torch, N, fid, BI.SEED_CONFIG4, 0, int(offb[-1].item()), 0).view(-1, 4)
    outb = torch.empty((nb, 4), dtype=torch.int64, device=dev)

    def ragged_b():
        N.check(N.lib.cpb_poseidon_crh_ragged_batch_dev(ctx, vb.data_ptr(), offb.data_ptr(), outb.data_ptr(), nb, st))

    if mode == "unordered":
        res["b_iii_input_order_ms"] = _time(ragged_b, iters)
        ref = outb.clone()
        return res | {"b_outputs_sha": _digest(ref)}

    # (ii) grouped in advance: one contiguous (n_L, L, 4) tensor per length
    groups = []
    for L in range(9):
        idx = torch.nonzero(lens == L).flatten()
        if L:
            x = vb[(offb[idx].unsqueeze(1) + torch.arange(L, device=dev)).flatten()].view(-1, L, 4).contiguous()
        else:
            x = torch.zeros((idx.numel(), 0, 4), dtype=torch.int64, device=dev)
        groups.append((L, idx.numel(), x, torch.empty((idx.numel(), 4), dtype=torch.int64, device=dev)))

    def grouped_b():
        for L, m, x, o in groups:
            N.check(N.lib.cpb_poseidon_crh_batch_dev(ctx, x.data_ptr() if L else vb.data_ptr(), L, o.data_ptr(), m, st))

    # (a) 2^24 inputs of length 2, the bench leaves
    na = 1 << 24
    xa = BI.field_elements_torch(torch, N, fid, BI.SEED_CONFIG4, 0, 2 * na, 0).view(na, 2, 4)
    offa = torch.arange(0, na + 1, dtype=torch.int64, device=dev) * 2
    outa_u = torch.empty((na, 4), dtype=torch.int64, device=dev)
    outa_r = torch.empty((na, 4), dtype=torch.int64, device=dev)

    def uniform_a():
        N.check(N.lib.cpb_poseidon_crh_batch_dev(ctx, xa.data_ptr(), 2, outa_u.data_ptr(), na, st))

    def ragged_a():
        N.check(N.lib.cpb_poseidon_crh_ragged_batch_dev(ctx, xa.data_ptr(), offa.data_ptr(), outa_r.data_ptr(), na, st))

    # (d) trees over the same leaves
    ln_u = torch.empty((na, 4), dtype=torch.int64, device=dev)
    nn_u = torch.empty((na - 1, 4), dtype=torch.int64, device=dev)
    ln_r = torch.empty_like(ln_u)
    nn_r = torch.empty_like(nn_u)

    def tree_u():
        N.check(N.lib.cpb_merkle_poseidon_build_dev(ctx, ctx, xa.data_ptr(), 2, na, ln_u.data_ptr(), nn_u.data_ptr(), st))

    def tree_r():
        N.check(N.lib.cpb_merkle_poseidon_build_ragged_dev(ctx, ctx, xa.data_ptr(), offa.data_ptr(), na, ln_r.data_ptr(), nn_r.data_ptr(), st))

    a_u, a_r, b_i, b_ii, d_u, d_r = [], [], [], [], [], []
    for _ in range(2):                                     # arms alternate inside the child as well
        a_u.append(_time(uniform_a, iters)); a_r.append(_time(ragged_a, iters))
        b_i.append(_time(ragged_b, iters)); b_ii.append(_time(grouped_b, iters))
        d_u.append(_time(tree_u, iters)); d_r.append(_time(tree_r, iters))
    res |= {"a_uniform_ms": min(a_u), "a_ragged_ms": min(a_r), "b_i_ragged_ms": min(b_i), "b_ii_grouped_ms": min(b_ii),
            "d_tree_uniform_ms": min(d_u), "d_tree_ragged_ms": min(d_r)}
    torch.cuda.synchronize()
    res["a_outputs_equal"] = bool(torch.equal(outa_u, outa_r))
    res["b_outputs_sha"] = _digest(outb)
    gold = bench.goldens()["merkle_2^24_poseidon_bn254"]["root"]
    to_list = lambda t: [int(v) & 0xFFFFFFFFFFFFFFFF for v in t.cpu().tolist()]     # noqa: E731
    res["d_roots_match_golden"] = to_list(nn_u[0]) == gold and to_list(nn_r[0]) == gold
    res["d_trees_equal"] = bool(torch.equal(nn_u, nn_r) and torch.equal(ln_u, ln_r))

    # (c) the ordering kernels' device time per call, from the profiler (after all timing above)
    from torch.profiler import ProfilerActivity, profile
    for name, fn, n in (("c_order_2^22_ms", ragged_b, nb), ("c_order_2^24_ms", ragged_a, na)):
        reps = 3
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                fn()
            torch.cuda.synchronize()
        us = sum(e.device_time_total for e in prof.key_averages() if "k_ragged_" in e.key)
        res[name] = us / reps / 1000.0
    return res


def _digest(t):
    import hashlib
    return hashlib.sha256(t.cpu().numpy().tobytes()).hexdigest()[:16]


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, sm, smax = [x.strip() for x in q.split(",")]
        return {"gpu": name, "power_limit": pl, "sm_clock_now": sm, "sm_clock_max": smax}
    except Exception as e:                                 # the numbers are still reported, without the card's settings
        return {"gpu_info_error": repr(e)}


def spread(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs), "runs": xs}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--child", choices=["ordered", "unordered"])
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--out", help="write the summary and every run as JSON to this file")
    a = ap.parse_args()
    if a.child:
        print(json.dumps(child(a.child, a.iters)), flush=True)
        return
    info = gpu_info()
    runs = []
    for r in range(a.runs):
        for mode in ("ordered", "unordered"):
            env = dict(os.environ)
            if mode == "unordered":
                env["CPB_RAGGED_ORDER"] = "0"
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", mode, "--iters", str(a.iters)], env=env,
                               capture_output=True, text=True)
            if p.returncode != 0:
                sys.stderr.write(p.stdout + p.stderr)
                raise SystemExit(f"child {mode} failed")
            runs.append(json.loads(p.stdout.strip().splitlines()[-1]))
            print(json.dumps(runs[-1]), flush=True)
    info_after = gpu_info()
    ordered = [x for x in runs if x["mode"] == "ordered"]
    unordered = [x for x in runs if x["mode"] == "unordered"]
    summary = {k: spread([x[k] for x in ordered]) for k in ordered[0] if k.endswith("_ms")}
    summary["b_iii_input_order_ms"] = spread([x["b_iii_input_order_ms"] for x in unordered])
    m = lambda k: summary[k]["median"]                     # noqa: E731
    summary["ratios"] = {"a_ragged_over_uniform": m("a_ragged_ms") / m("a_uniform_ms"),
                         "b_ragged_over_grouped": m("b_i_ragged_ms") / m("b_ii_grouped_ms"),
                         "b_input_order_over_ragged": m("b_iii_input_order_ms") / m("b_i_ragged_ms"),
                         "d_ragged_tree_over_uniform": m("d_tree_ragged_ms") / m("d_tree_uniform_ms")}
    summary["checks"] = {"a_outputs_equal": all(x["a_outputs_equal"] for x in ordered),
                         "b_outputs_identical_across_arms": len({x["b_outputs_sha"] for x in runs}) == 1,
                         "d_roots_match_golden": all(x["d_roots_match_golden"] for x in ordered),
                         "d_trees_equal": all(x["d_trees_equal"] for x in ordered)}
    out = {"card_before": info, "card_after": info_after, "iters": a.iters, "summary": summary, "runs": runs}
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps({"summary": summary, "card": info}, indent=1))


if __name__ == "__main__":
    main()
