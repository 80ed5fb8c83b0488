"""Ragged duplex calls on one GPU (DESIGN §4.2): what a mode per sponge costs, and what the ordering by permutation count buys.

For the bench's BN254 Fr t = 3 config and BLS12-381 Fr default rate 2, at n = 2^20 sponges (--log-n):
  (a) equal spans: the calls of tools/perf_duplex.py's transcript (64-byte absorb_bytes from Absorbing{0}; absorb(2) from
      Absorbing{1}, one permutation; squeeze(1) from Absorbing{1}, one permutation; absorb(2) from Squeezing{1}, none), each as the
      uniform call (cpb_poseidon_duplex_*_dev) and as the ragged call with every span equal, alternated.
  (b) mixed spans: every sponge runs absorb_bytes(L), absorb(k1), squeeze(m1), absorb(k2), squeeze(m2) with L uniform on 0..128
      bytes, k uniform on 1..6 and m on 1..3, from a fresh state:
      (i)   the ragged calls;
      (ii)  the grouped ideal: per call, the sponges grouped by their count in that call in advance, one uniform call per group on a
            contiguous slice of states, in the mode the group's first sponge holds there (grouping not timed), summed per call;
      (iii) the ragged kernels in input order without the ordering step (CPB_RAGGED_ORDER=0, read once, so a process of its own).
The parent process only spawns children, alternating the ordered and unordered ones, `--runs` of each; every child times its arms
alternately (CUDA events around each call, median of `--iters` after a warm-up) and prints one JSON line.  The parent prints the
summary with the card's name, power limit and SM clock read in the same run, and with --out also writes every run to that file.
Usage: python tools/perf_duplex_ragged.py [--log-n 20] [--runs 3] [--iters 5] [--out FILE]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CALLS_B = ("bytes", "absorb1", "squeeze1", "absorb2", "squeeze2")


def _ev():
    import torch
    return torch.cuda.Event(enable_timing=True)


def _timed(fn, prep=None):
    """Device time of fn() in ms (CUDA events); prep() runs before, untimed."""
    import torch
    if prep:
        prep()
    e0, e1 = _ev(), _ev()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def _digest(*ts):
    import hashlib
    h = hashlib.sha256()
    for t in ts:
        h.update(t.cpu().numpy().tobytes())
    return h.hexdigest()[:16]


def child(mode, iters, log_n):
    import numpy as np
    import torch
    import bench
    import crypto_primitives_b200 as cp
    from crypto_primitives_b200 import _native as N

    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream().cuda_stream
    n = 1 << log_n
    L = N.lib
    configs = {"bn254_t3": bench.poseidon_params(cp, "bn254"),
               "bls12_381_r2": cp.get_default_poseidon_parameters(cp.BLS12_381_FR, 2, False)}
    res = {"mode": mode, "n": n, "configs": {}}
    for name, cfg in configs.items():
        ctx = cfg.context(0)
        t = cfg.rate + cfg.capacity
        f = cfg.field
        g = torch.Generator(device="cpu").manual_seed(1)
        msg = torch.randint(0, 256, (n, 128), dtype=torch.uint8, generator=g).to(dev)
        el = torch.from_numpy(np.tile(f.elements([3, 5, 7, 11, 13, 17]), (n, 1, 1)).view(np.int64)).to(dev)   # (n, 6, 4)
        states = torch.zeros((n, t, 4), dtype=torch.int64, device=dev)
        modes = torch.zeros((n, 2), dtype=torch.int64, device=dev)
        out = torch.empty((3 * n, 4), dtype=torch.int64, device=dev)
        ar = torch.arange(n + 1, dtype=torch.int64, device=dev)
        r = {}

        # (a) equal spans, uniform against ragged, from the transcript's modes
        if mode == "ordered":
            msg64 = msg[:, :64].contiguous()
            el2 = el[:, :2].contiguous()
            off64, off2 = ar * 64, ar * 2
            a_kinds = {
                "absorb_bytes": ((0, 0), lambda m: L.cpb_poseidon_duplex_absorb_bytes_dev(ctx, states.data_ptr(), C.byref(m), msg64.data_ptr(), 64, 64, n, st),
                                 lambda: L.cpb_poseidon_duplex_absorb_bytes_ragged_dev(ctx, states.data_ptr(), modes.data_ptr(), msg64.data_ptr(), off64.data_ptr(), n, st)),
                "absorb2_first": ((0, 1), lambda m: L.cpb_poseidon_duplex_absorb_dev(ctx, states.data_ptr(), C.byref(m), el2.data_ptr(), 2, n, st),
                                  lambda: L.cpb_poseidon_duplex_absorb_ragged_dev(ctx, states.data_ptr(), modes.data_ptr(), el2.data_ptr(), off2.data_ptr(), n, st)),
                "squeeze1": ((0, 1), lambda m: L.cpb_poseidon_duplex_squeeze_dev(ctx, states.data_ptr(), C.byref(m), out.data_ptr(), 1, 0, n, st),
                             lambda: L.cpb_poseidon_duplex_squeeze_ragged_dev(ctx, states.data_ptr(), modes.data_ptr(), out.data_ptr(), ar.data_ptr(), 0, n, st)),
                "absorb2_no_perm": ((1, 1), lambda m: L.cpb_poseidon_duplex_absorb_dev(ctx, states.data_ptr(), C.byref(m), el2.data_ptr(), 2, n, st),
                                    lambda: L.cpb_poseidon_duplex_absorb_ragged_dev(ctx, states.data_ptr(), modes.data_ptr(), el2.data_ptr(), off2.data_ptr(), n, st)),
            }
            a = {}
            for kind, (m0, uni, rag) in a_kinds.items():
                set_modes = lambda m0=m0: (modes[:, 0].fill_(m0[0]), modes[:, 1].fill_(m0[1]))          # noqa: E731
                tu, tr = [], []
                for it in range(iters + 1):                # the first round warms up
                    x = _timed(lambda: N.check(uni(N.SpongeMode(*m0))))
                    y = _timed(lambda: N.check(rag()), set_modes)
                    if it:
                        tu.append(x)
                        tr.append(y)
                a[kind] = {"uniform_ms": statistics.median(tu), "ragged_ms": statistics.median(tr)}
            r["a"] = a

        # (b) mixed spans
        gen = torch.Generator(device="cpu").manual_seed(2)
        Ls = torch.randint(0, 129, (n,), generator=gen)
        k1, k2 = (torch.randint(1, 7, (n,), generator=gen) for _ in range(2))
        m1, m2 = (torch.randint(1, 4, (n,), generator=gen) for _ in range(2))
        counts = {"bytes": Ls, "absorb1": k1, "squeeze1": m1, "absorb2": k2, "squeeze2": m2}

        def offs(c):
            o = torch.zeros(n + 1, dtype=torch.int64)
            torch.cumsum(c, 0, out=o[1:])
            return o.to(dev)

        offb = {k: offs(v) for k, v in counts.items()}
        mask = torch.arange(128, device=dev)[None, :] < Ls.to(dev)[:, None]
        bflat = msg[mask].contiguous()
        eflat = {k: el[torch.arange(6, device=dev)[None, :] < counts[k].to(dev)[:, None]].contiguous() for k in ("absorb1", "absorb2")}
        sout = torch.empty((3 * n, 4), dtype=torch.int64, device=dev)
        rcall = {
            "bytes": lambda: L.cpb_poseidon_duplex_absorb_bytes_ragged_dev(ctx, states.data_ptr(), modes.data_ptr(), bflat.data_ptr(), offb["bytes"].data_ptr(), n, st),
            "absorb1": lambda: L.cpb_poseidon_duplex_absorb_ragged_dev(ctx, states.data_ptr(), modes.data_ptr(), eflat["absorb1"].data_ptr(), offb["absorb1"].data_ptr(), n, st),
            "squeeze1": lambda: L.cpb_poseidon_duplex_squeeze_ragged_dev(ctx, states.data_ptr(), modes.data_ptr(), sout.data_ptr(), offb["squeeze1"].data_ptr(), 0, n, st),
            "absorb2": lambda: L.cpb_poseidon_duplex_absorb_ragged_dev(ctx, states.data_ptr(), modes.data_ptr(), eflat["absorb2"].data_ptr(), offb["absorb2"].data_ptr(), n, st),
            "squeeze2": lambda: L.cpb_poseidon_duplex_squeeze_ragged_dev(ctx, states.data_ptr(), modes.data_ptr(), sout.data_ptr(), offb["squeeze2"].data_ptr(), 0, n, st),
        }

        def ragged_transcript(times=None, modes_before=None):
            states.zero_()
            modes.zero_()
            for c in CALLS_B:
                if modes_before is not None:
                    modes_before[c] = modes.cpu()
                x = _timed(lambda: N.check(rcall[c]()))
                if times is not None:
                    times.setdefault(c, []).append(x)

        mb = {}
        ragged_transcript(modes_before=mb)                 # warm-up, and the modes each call starts from
        digest = _digest(states, modes, sout[:int(offb["squeeze2"][-1])])
        tb = {}
        if mode == "unordered":
            for _ in range(iters):
                ragged_transcript(tb)
        else:
            # the grouped ideal: per call, one contiguous group per count, in its first sponge's mode
            groups = {}
            for c in CALLS_B:
                gl = []
                for v in sorted(set(counts[c].tolist())):
                    idx = torch.nonzero(counts[c] == v).flatten()
                    m0 = mb[c][idx[0]]
                    ng = idx.numel()
                    gs = torch.zeros((ng, t, 4), dtype=torch.int64, device=dev)
                    if c == "bytes":
                        data = msg[idx.to(dev), :v].contiguous() if v else msg
                    elif c.startswith("absorb"):
                        data = el[idx.to(dev), :v].contiguous()
                    else:
                        data = torch.empty((ng * v, 4), dtype=torch.int64, device=dev)
                    gl.append((v, ng, int(m0[0]), int(m0[1]), gs, data))
                groups[c] = gl

            def grouped(c):
                for v, ng, sq, ix, gs, data in groups[c]:
                    m = N.SpongeMode(sq, ix)
                    if c == "bytes":
                        N.check(L.cpb_poseidon_duplex_absorb_bytes_dev(ctx, gs.data_ptr(), C.byref(m), data.data_ptr(), v, v, ng, st))
                    elif c.startswith("absorb"):
                        N.check(L.cpb_poseidon_duplex_absorb_dev(ctx, gs.data_ptr(), C.byref(m), data.data_ptr(), v, ng, st))
                    else:
                        N.check(L.cpb_poseidon_duplex_squeeze_dev(ctx, gs.data_ptr(), C.byref(m), data.data_ptr(), v, 0, ng, st))

            for c in CALLS_B:
                grouped(c)                                 # warm-up
            tg = {}
            for _ in range(iters):
                ragged_transcript(tb)
                for c in CALLS_B:
                    tg.setdefault(c, []).append(_timed(lambda: grouped(c)))
            r["b_grouped_ms"] = {c: statistics.median(v) for c, v in tg.items()}
            r["b_grouped_total_ms"] = sum(r["b_grouped_ms"].values())
        r["b_ragged_ms"] = {c: statistics.median(v) for c, v in tb.items()}
        r["b_ragged_total_ms"] = sum(r["b_ragged_ms"].values())
        r["b_digest"] = digest
        res["configs"][name] = r
    return res


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, sm, smax = [x.strip() for x in q.split(",")]
        return {"gpu": name, "power_limit": pl, "sm_clock_now": sm, "sm_clock_max": smax}
    except Exception as e:                                 # the numbers are still reported, without the card's settings
        return {"gpu_info_error": repr(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--child", choices=["ordered", "unordered"])
    ap.add_argument("--log-n", type=int, default=20)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--out", help="write the summary and every run as JSON to this file")
    a = ap.parse_args()
    if a.child:
        print(json.dumps(child(a.child, a.iters, a.log_n)), flush=True)
        return
    info = gpu_info()
    runs = []
    for _ in range(a.runs):
        for mode in ("ordered", "unordered"):
            env = dict(os.environ)
            if mode == "unordered":
                env["CPB_RAGGED_ORDER"] = "0"
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", mode, "--iters", str(a.iters), "--log-n", str(a.log_n)],
                               env=env, capture_output=True, text=True)
            if p.returncode != 0:
                sys.stderr.write(p.stdout + p.stderr)
                raise SystemExit(f"child {mode} failed")
            runs.append(json.loads(p.stdout.strip().splitlines()[-1]))
            print(json.dumps(runs[-1]), flush=True)
    info_after = gpu_info()
    med = statistics.median
    summary = {}
    for name in runs[0]["configs"]:
        o = [x["configs"][name] for x in runs if x["mode"] == "ordered"]
        u = [x["configs"][name] for x in runs if x["mode"] == "unordered"]
        s = {"a": {k: {"uniform_ms": med([x["a"][k]["uniform_ms"] for x in o]), "ragged_ms": med([x["a"][k]["ragged_ms"] for x in o])}
                   for k in o[0]["a"]}}
        for k, v in s["a"].items():
            v["ragged_over_uniform"] = v["ragged_ms"] / v["uniform_ms"]
        s["b_ragged_ms"] = {c: med([x["b_ragged_ms"][c] for x in o]) for c in CALLS_B}
        s["b_grouped_ms"] = {c: med([x["b_grouped_ms"][c] for x in o]) for c in CALLS_B}
        s["b_input_order_ms"] = {c: med([x["b_ragged_ms"][c] for x in u]) for c in CALLS_B}
        tot = {k: med([x[k] for x in o]) for k in ("b_ragged_total_ms", "b_grouped_total_ms")}
        tot["b_input_order_total_ms"] = med([x["b_ragged_total_ms"] for x in u])
        s |= tot
        s["b_ragged_over_grouped"] = tot["b_ragged_total_ms"] / tot["b_grouped_total_ms"]
        s["b_input_order_over_ragged"] = tot["b_input_order_total_ms"] / tot["b_ragged_total_ms"]
        s["b_results_identical_across_arms"] = len({x["b_digest"] for x in o + u}) == 1
        summary[name] = s
    out = {"card_before": info, "card_after": info_after, "n": runs[0]["n"], "iters": a.iters, "summary": summary, "runs": runs}
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps({"summary": summary, "card": info}, indent=1))


if __name__ == "__main__":
    main()
