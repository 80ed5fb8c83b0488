"""Development probe: CRH throughput for every default-parameter width (rate 2..8, t = 3..9; BLS12-381 Fr) and the
Bowe-Hopwood CRH, device-resident.  One permutation per hash (input length = rate)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import crypto_primitives_b200 as cp
from crypto_primitives_b200 import _native as N
from tools.quick_perf import timeit

dev = torch.device("cuda:0")
f = cp.BLS12_381_FR
n = 1 << 20
for rate in range(2, 9):
    cfg = cp.get_default_poseidon_parameters(f, rate, False)
    ctx = cfg.context(0)
    x = torch.randint(0, 2**59, (n, rate, 4), dtype=torch.int64).to(dev)
    out = torch.empty((n, 4), dtype=torch.int64, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    def go():
        N.check(N.lib.cpb_poseidon_crh_batch_dev(ctx, x.data_ptr(), rate, out.data_ptr(), n, st))
    ms = timeit(go, iters=3, warm=1)
    t = rate + 1
    rf, rp = cfg.full_rounds, cfg.partial_rounds
    # wide multiply-adds per permutation with the sparse schedule: S-boxes (4 sqr + 1 mul for alpha 17), dense rows, sparse rows
    sbox = 4 * 84 + 112
    dot = lambda k: 8 * (6 * k + 6)          # BLS12-381: 6 wides per row per term + 6 per reduction row
    wides = rf * (t * sbox + t * dot(t)) + rp * (sbox + dot(t) + (t - 1) * 112)
    print(f"t={t} (rate {rate}, {rf}+{rp} rounds, sparse={cp._native.lib.cpb_poseidon_ctx_is_sparse(ctx)}): {ms:.3f} ms  {n / ms / 1e3:.2f} M perms/s"
          f"  ~{wides / 1e3:.1f}k wide madds/perm -> {n * wides / (ms * 1e-3) / (132 * 32 * 1.98e9):.2f} of the issue peak", flush=True)
