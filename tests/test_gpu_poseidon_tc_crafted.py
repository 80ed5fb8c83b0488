"""The BN254 Fr tensor-core hash kernel (k_poseidon_crh_tc) at S-box operands chosen on the host.

Random inputs reach the carry-sensitive states of the kernel's arithmetic -- the u8 IMMA column sums of the R^-1 product at their
maximum, a packed column pair that carries into the next, tc_finish's carry chains running their whole length -- at rates like
2^-32 or less, so neither random tests nor the benchmark's root check can see a defect that lives only there.  Here the inputs
are solved with exact field algebra from the schedule's own constants so that a chosen S-box operand inside the kernel takes a
chosen Montgomery-form integer s < p:

  * full round 1, lanes 1 and 2 at once (lane 0's S-box there is the schedule constant S(c0));
  * full round 2, every pair of its three lanes (RF = 8: neither the entry round nor touched by the sparse factorisation): the
    round-2 operands are affine in (b^5, c^5) with b, c lanes 1, 2 of round 1, so a 2 x 2 system gives b^5, c^5 and a fifth
    root (exponent 5^-1 mod p - 1; 5 does not divide p - 1) gives b, c;
  * partial round 0's S-box operand, the first pos_sbox5_tc of the partial-round loop: at RF = 2 affine in b^5 for a fixed c; at
    RF = 4 a degree-5 polynomial in b^5, whose roots over F_p come from gcd(f, X^p - X) and equal-degree splitting (another c
    when it has none).  The kernel squares the canonical lane-0 value after phase 0 plus Cp0, and row 0 of Mpre is row 0 of M
    and Cp0[0] = ark[RF/2][0], so that value is the reference's lane 0 of round RF/2 after its constant; a CPU test checks both
    facts on the product's schedule.

The target families: squares whose upper 32-bit limbs hold all-ones runs (helpers.crafted_sbox_inputs), squares whose low half
ends in a long run of 0xFF bytes (s = sqrt(-7) mod 2^k by Hensel lifting, bits above k free: the R^-1 product's byte columns at
their largest sums), and 0, 1, p - 1.  A CPU test checks with a round-by-round trace in Python integers that every steered input
produces its targeted operand; the GPU test runs each (position, family) on 4096 hashes against the C oracle and against the
alpha = 5 integer kernel (CPB_POS_TC=0, in a child process).  A reduction that drops a carry only these operands produce (a
column sum that overflows a packed pair, a carry chain cut short, a byte lane mapped to the wrong row) gives wrong digests.

The second part (tests/device/tc_probe.cu) runs the kernel's tensor-core pieces themselves on one warp at a time and compares
them bit for bit with the CPU emulation of tests/test_poseidon_tc.py."""
import ctypes as C
import multiprocessing
import os
import random
import subprocess
import sys
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import pytest

from helpers import ROOT, build_host_shim, crafted_sbox_inputs, oracle_config
from oracle import cref, fields as OF, poseidon as OP
from test_poseidon_lane1_basis import random_config, regions
from test_poseidon_scaled_lane0 import FID, schedule

P = OF.BN254_FR
R = 1 << 256
RINV = pow(R, -1, P)
INV5 = pow(5, -1, P - 1)
THREADS = os.cpu_count() or 8


# ------------------------------------------------------------------------------------------------------------- configurations
def steer_config(name):
    if name == "bench":                                        # RF = 8, RP = 57, Grain LFSR constants
        return oracle_config("bn254_r2")[1]
    rf = {"rf2": 2, "rf4": 4}[name]
    return random_config(P, 3, rf, 57, 5, seed=5200 + rf)


def trace(cfg, x):
    """The permutation of a fresh sponge that absorbed x (field integers), round by round in Python integers (arkworks order:
    constants, S-boxes, MDS).  Returns (ops, out): ops[r][i] is lane i after round r's constants -- the S-box operand -- and
    out the final state."""
    p, t, half = cfg.p, cfg.rate + cfg.capacity, cfg.full_rounds // 2
    s = [0] * t
    for j, v in enumerate(x):
        s[cfg.capacity + j] = v % p
    ops = []
    for r in range(cfg.full_rounds + cfg.partial_rounds):
        s = [(a + c) % p for a, c in zip(s, cfg.ark[r])]
        ops.append(list(s))
        full = r < half or r >= half + cfg.partial_rounds
        s = [pow(a, cfg.alpha, p) for a in s] if full else [pow(s[0], cfg.alpha, p)] + s[1:]
        s = [sum(m * a for m, a in zip(row, s)) % p for row in cfg.mds]
    return ops, s


# ------------------------------------------------------------------------------------------------------------- target operands
def hensel_sqrt_m7(k):
    """r with r^2 = -7 (mod 2^k), k >= 3: -7 = 1 (mod 8), and each further bit is fixed by adding 2^(i-1)."""
    r = 1
    for i in range(3, k):
        if ((r * r + 7) >> i) & 1:
            r += 1 << (i - 1)
    return r


def target(family, rnd):
    """A Montgomery-form integer s < p of the family."""
    if family == "ones":
        # helpers.crafted_sbox_inputs builds in0 = s - ark[0][1] (Montgomery integers) with s^2's all-ones limbs: take s back
        cfg = steer_config("bench")
        in0 = OF.from_limbs(crafted_sbox_inputs(cfg, 1, seed=rnd.getrandbits(32))[0, 0])
        return (in0 + cfg.ark[0][1] * R) % P
    if family == "hensel":
        k = rnd.choice((64, 128, 192, 224, 248, 252))
        r = hensel_sqrt_m7(k)
        r = rnd.choice((r, -r, r + (1 << (k - 1)), -r + (1 << (k - 1)))) % (1 << k)
        while True:
            s = r + (rnd.randrange(1 << (P.bit_length() - k)) << k)
            if s < P:
                return s
    if family == "fixed":
        return rnd.choice((0, 1, P - 1))
    raise KeyError(family)


# ------------------------------------------------------------------------------------------------------------- F_p[X], degree <= 5
def _trim(a):
    a = [v % P for v in a]
    while a and a[-1] == 0:
        a.pop()
    return a


def _rem(a, f):
    """a mod f for a monic f."""
    a = list(a)
    d = len(f) - 1
    for i in range(len(a) - 1, d - 1, -1):
        c = a[i] % P
        if c:
            for j in range(d + 1):
                a[i - d + j] -= c * f[j]
    return [v % P for v in a[:d]]


def _monic(a):
    inv = pow(a[-1], -1, P)
    return [v * inv % P for v in a]


def _mulmod(a, b, f):
    out = [0] * (len(a) + len(b) - 1)
    for i, x in enumerate(a):
        if x:
            for j, y in enumerate(b):
                out[i + j] += x * y
    return _rem(out, f)


def _powmod(base, e, f):
    r, b = _rem([1], f), _rem(base, f)
    for bit in bin(e)[2:]:
        r = _mulmod(r, r, f)
        if bit == "1":
            r = _mulmod(r, b, f)
    return r


def _minus(a, k, c=1):
    """a - c X^k."""
    a = a + [0] * (k + 1 - len(a))
    a[k] = (a[k] - c) % P
    return a


def _gcd(a, b):
    a, b = _trim(a), _trim(b)
    while b:
        b = _monic(b)
        a, b = b, _trim(_rem(a, b))
    return _monic(a) if a else a


def poly_root(f, rnd):
    """One root in F_p of f (coefficients low to high), or None: g = gcd(f, X^p - X) keeps the linear factors, and equal-degree
    splitting with gcd(g, (X + d)^((p-1)/2) - 1) halves g until it is linear."""
    f = _monic(_trim(f))
    if len(f) < 2:
        return None
    xp = _powmod([0, 1], P, f)
    g = _gcd(f, _minus(xp, 1))
    while len(g) > 2:
        d = rnd.randrange(P)
        w = _powmod([d, 1], (P - 1) // 2, g)
        h = _gcd(g, _minus(w, 0))
        if 1 < len(h) < len(g):
            g = h
    return (-g[0]) % P if len(g) == 2 else None


# ------------------------------------------------------------------------------------------------------------- the solvers
POSITIONS = {                        # position -> (config, round, lanes)
    "fr1-12": ("bench", 0, (1, 2)),
    "fr2-01": ("bench", 1, (0, 1)),
    "fr2-02": ("bench", 1, (0, 2)),
    "fr2-12": ("bench", 1, (1, 2)),
    "pr0-rf2": ("rf2", 1, (0, )),
    "pr0-rf4": ("rf4", 2, (0, )),
}
FAMILIES = ("ones", "hensel", "fixed")


def solve(cfg, position, targets, rnd):
    """Inputs (x0, x1) (field integers) whose S-box operands at `position` are the field elements with Montgomery integers
    `targets` (one per lane of the position), or None when this draw has no solution."""
    p, M, ark = cfg.p, cfg.mds, cfg.ark
    f = [s * RINV % p for s in targets]
    S0 = pow(ark[0][0], 5, p)                                  # lane 0 of round 0: S(c0), the capacity entering as zero
    _, rnd_, lanes = POSITIONS[position]
    if position == "fr1-12":
        return (f[0] - ark[0][1]) % p, (f[1] - ark[0][2]) % p
    if position.startswith("fr2"):
        # ops[1][i] = M[i][0] S0 + M[i][1] B + M[i][2] C + ark[1][i] with B = b^5, C = c^5
        i, j = lanes
        a11, a12, a21, a22 = M[i][1], M[i][2], M[j][1], M[j][2]
        r1 = (f[0] - M[i][0] * S0 - ark[1][i]) % p
        r2 = (f[1] - M[j][0] * S0 - ark[1][j]) % p
        det = (a11 * a22 - a12 * a21) % p
        inv = pow(det, -1, p)
        B = (r1 * a22 - a12 * r2) * inv % p
        Cc = (a11 * r2 - a21 * r1) * inv % p
        return (pow(B, INV5, p) - ark[0][1]) % p, (pow(Cc, INV5, p) - ark[0][2]) % p
    c = rnd.randrange(p)
    Cc = pow(c, 5, p)
    if position == "pr0-rf2":
        # ops[1][0] = M[0][0] S0 + M[0][1] B + M[0][2] C + ark[1][0]
        B = (f[0] - M[0][0] * S0 - M[0][2] * Cc - ark[1][0]) * pow(M[0][1], -1, p) % p
    else:
        # ops[2][0] = sum_l M[0][l] (M[l][1] B + d_l)^5 + ark[2][0], d_l = M[l][0] S0 + M[l][2] C + ark[1][l]
        poly = [0] * 6
        poly[0] = (ark[2][0] - f[0]) % p
        for l in range(3):
            a, d = M[l][1], (M[l][0] * S0 + M[l][2] * Cc + ark[1][l]) % p
            for k, binom in enumerate((1, 5, 10, 10, 5, 1)):
                poly[k] += M[0][l] * binom * pow(a, k, p) * pow(d, 5 - k, p)
        B = poly_root(poly, rnd)
        if B is None:
            return None
    return (pow(B, INV5, p) - ark[0][1]) % p, (c - ark[0][2]) % p


def steered(position, family, count, seed):
    """count rows (x0, x1, s-targets) for the position and family."""
    cfg = steer_config(POSITIONS[position][0])
    rnd = random.Random(seed)
    rows = []
    while len(rows) < count:
        ts = [target(family, rnd) for _ in POSITIONS[position][2]]
        x = solve(cfg, position, ts, rnd)
        if x is not None:
            rows.append((x[0], x[1], ts))
    return rows


def _steered_job(args):
    return steered(*args)


def steered_rows(position, family, count, seed, workers=1):
    """steered() split over worker processes (the RF = 4 root finding costs a few milliseconds a row).  Spawned, not forked: the
    test process holds a CUDA context and the library's threads."""
    if workers <= 1 or count < 256:
        return steered(position, family, count, seed)
    per = -(-count // workers)
    jobs = [(position, family, min(per, count - w * per), seed * 1000 + w) for w in range(workers) if count > w * per]
    with ProcessPoolExecutor(len(jobs), mp_context=multiprocessing.get_context("spawn")) as ex:
        return [r for part in ex.map(_steered_job, jobs) for r in part]


def as_inputs(rows):
    return np.ascontiguousarray(cref.ints_to_mont([v for x0, x1, _ in rows for v in (x0, x1)], P).reshape(len(rows), 2, 4))


def _seed(position, family):
    return 8800 + 10 * list(POSITIONS).index(position) + FAMILIES.index(family)


# ------------------------------------------------------------------------------------------------------------- CPU checks
def test_trace_is_the_oracle_permutation():
    for name in ("bench", "rf2", "rf4"):
        cfg = steer_config(name)
        rnd = random.Random(3)
        for _ in range(4):
            x = [rnd.randrange(P), rnd.randrange(P)]
            st = cref.ints_to_mont([0] + x, P)
            assert trace(cfg, x)[1] == cref.mont_to_ints(cref.Poseidon(cfg).permute(st), P)


def test_hensel_roots_square_to_minus_7():
    for k in (3, 8, 64, 128, 192, 248, 252):
        r = hensel_sqrt_m7(k)
        assert (r * r + 7) % (1 << k) == 0
    rnd = random.Random(1)
    for _ in range(50):
        s = target("hensel", rnd)
        lo = (s * s) % R
        assert s < P and lo.to_bytes(32, "little")[1:8] == b"\xff" * 7        # at least k = 64: T_lo ends ...ff f9


@pytest.mark.parametrize("name", ["rf2", "rf4"])
def test_partial_round_0_operand_is_the_reference_lane_0(name):
    """The two facts the partial-round steering rests on, on the product's schedule: after phase 0 the kernel adds Cp0 to the
    entry round's rows, whose row 0 comes from Mpre, so its first partial-round operand is the reference's lane 0 of round RF/2
    after that round's constant exactly when row 0 of Mpre is row 0 of M and Cp0[0] = ark[RF/2][0]."""
    cfg = steer_config(name)
    o, v = schedule(FID["bn254_fr"], cfg)
    assert o["sparse"] == 1
    reg = regions(o, v, 3, cfg.full_rounds, cfg.partial_rounds)
    assert reg["Mpre"][:3] == reg["M"][:3] == cfg.mds[0]
    assert reg["Cp0"][0] == cfg.ark[cfg.full_rounds // 2][0]


@pytest.mark.parametrize("position", list(POSITIONS))
@pytest.mark.parametrize("family", FAMILIES)
def test_steered_inputs_reach_their_operands(position, family):
    """Every steered input's targeted operands in a round-by-round trace of the reference permutation: the field element whose
    Montgomery integer is the target, at the round and lanes of the position (full round 2 at RF = 8 and the partial rounds'
    first operand are neither the entry round nor lanes the kernel loads from the schedule)."""
    cfg_name, rnd_, lanes = POSITIONS[position]
    cfg = steer_config(cfg_name)
    half = cfg.full_rounds // 2
    assert rnd_ < half - 1 or rnd_ == half                     # not the entry round (Mpre), or the first partial round
    rows = steered(position, family, 12 if position == "pr0-rf4" else 48, _seed(position, family) + 1)
    for x0, x1, ts in rows:
        ops, _ = trace(cfg, [x0, x1])
        for lane, s in zip(lanes, ts):
            assert ops[rnd_][lane] * R % P == s, (position, family, lane)


# ------------------------------------------------------------------------------------------------------------- GPU
COUNT = 4096
_CHILD = """
import sys
import numpy as np
sys.path.insert(0, {root!r}); sys.path.insert(0, {tests!r})
from test_gpu_poseidon_tc_crafted import product_of
from crypto_primitives_b200.crh.poseidon import CRH
d = np.load({inp!r})
np.savez({out!r}, **{{k: CRH.evaluate_batch(product_of(k), d[k]) for k in d.files}})
"""


def product_of(cfg_name):
    import crypto_primitives_b200 as cp
    c = steer_config(cfg_name)
    return cp.PoseidonConfig.from_ints(cp.BN254_FR, c.full_rounds, c.partial_rounds, c.alpha, c.mds, c.ark, c.rate, c.capacity)


@pytest.mark.gpu
def test_steered_operands_through_the_tc_kernel(tmp_path):
    """4096 hashes per (position, family) through CRH.evaluate_batch on the tensor-core kernel, against the C oracle and the
    alpha = 5 integer kernel."""
    from crypto_primitives_b200 import _native as N
    from crypto_primitives_b200.crh.poseidon import CRH
    batches = {name: [] for name in ("bench", "rf2", "rf4")}
    for position in POSITIONS:
        for family in FAMILIES:
            rows = steered_rows(position, family, COUNT, _seed(position, family), workers=THREADS)
            batches[POSITIONS[position][0]].append(as_inputs(rows))
    xs = {name: np.ascontiguousarray(np.concatenate(b)) for name, b in batches.items()}
    inp, out = str(tmp_path / "in.npz"), str(tmp_path / "out.npz")
    np.savez(inp, **xs)
    subprocess.run([sys.executable, "-c", _CHILD.format(root=ROOT, tests=os.path.join(ROOT, "tests"), inp=inp, out=out)],
                   env=dict(os.environ, CPB_POS_TC="0"), check=True)
    ref = np.load(out)
    for name, x in xs.items():
        cfg = product_of(name)
        assert N.lib.cpb_poseidon_ctx_is_sparse(cfg.context(0)) == 1
        got = CRH.evaluate_batch(cfg, x)
        assert np.array_equal(got, cref.Poseidon(steer_config(name)).crh_batch(x, threads=THREADS)), ("oracle", name)
        assert np.array_equal(got, ref[name]), ("integer kernel", name)


# ============================================================================================================= the device probe
# tests/device/tc_probe.cu runs tc_redc, pos_sbox5_tc, tc_partial_round, tc_full_round and tc_finish on the device on operands
# chosen per lane, and each result -- the unreduced value, not only its residue -- is compared bit for bit with the CPU emulation
# of tests/test_poseidon_tc.py (ldmatrix, IMMA and the C buffer in Python from the PTX ISA's fragment tables, the product's own
# tc_finish built for the host), with the exact value mod p, and with the documented bound.  A warp's 32 lanes take 32 different
# operand kinds, and warp w puts kind (lane + w) mod 32 on each lane, so over 32 warps every kind sits on every lane: a fragment,
# row or lane mapped wrongly on the device (where the emulation cannot reach: nvcc's code for the real mma.sync and ldmatrix, the
# 128-bit C-buffer stores) shows as a lane whose result differs.
PROBE_WARPS = 32
PROBE_DEPS = [os.path.join(ROOT, "tests", "device", "tc_probe.cu")] + [
    os.path.join(ROOT, "crypto_primitives_b200", "csrc", f) for f in os.listdir(os.path.join(ROOT, "crypto_primitives_b200", "csrc"))
    if f.endswith(("cuh", "hpp"))]
u32p = C.POINTER(C.c_uint32)


def build_probe():
    """nvcc build of tests/device/tc_probe.cu with the library's flags into tests/host/_build/, redone when a source is newer."""
    out_dir = os.path.join(ROOT, "tests", "host", "_build")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "tc_probe.so")
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in PROBE_DEPS):
        nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
        tmp = so + f".{os.getpid()}.tmp"
        subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-shared", "-Xcompiler", "-fPIC",
                               PROBE_DEPS[0], "-o", tmp, "-lcudart_static", "-lpthread", "-ldl", "-lrt"])
        os.replace(tmp, so)
    return so


def test_probe_compiles_for_sm_90a():
    lib = C.CDLL(build_probe())
    assert lib.probe_threads_per_cta() == 128


def _words(vals, n):
    """Integers -> uint32 limbs, n per value."""
    return np.array([(v >> (32 * i)) & 0xFFFFFFFF for v in vals for i in range(n)], dtype=np.uint32)


def _ints(words, n):
    w = words.reshape(-1, n)
    return [sum(int(x) << (32 * i) for i, x in enumerate(row)) for row in w]


def _fit(pattern, top):
    """The longest low-end prefix of a little-endian byte pattern whose value is below top."""
    for nb in range(32, 0, -1):
        v = int.from_bytes(pattern[:nb], "little")
        if v < top:
            return v
    return 0


def kinds(top, rnd):
    """32 operand kinds below top: 0, 1, p - 1, p, 2p - 1 and the contract's maximum where they are below it, the byte patterns
    0xFF.., 0x80.., 0x7F.., 0xFF00.. and 0x00FF.. (their longest prefix below top), the two crafted-square families, then random
    values below top and below p."""
    p = P
    vals = [v for v in (0, 1, 2, p - 1, p, p + 1, 2 * p - 1, 2 * p, top - 1, top - 2, (1 << 255) - 1, 1 << 255, (1 << 254) - 1)
            if v < top]
    vals += [_fit(b, top) for b in (b"\xff" * 32, b"\x80" * 32, b"\x7f" * 32, b"\xff\x00" * 16, b"\x00\xff" * 16)]
    vals += [target("ones", rnd), target("ones", rnd), target("hensel", rnd), target("hensel", rnd)]
    out = []
    for v in vals:
        if v not in out:
            out.append(v)
    while len(out) < 32:
        out.append(rnd.randrange(top) if len(out) % 2 else rnd.randrange(p))
    return out[:32]


def rotated(kind_list, offset=0):
    """Per thread of PROBE_WARPS warps: kind (lane + warp + offset) mod 32."""
    return [kind_list[(lane + w + offset) % 32] for w in range(PROBE_WARPS) for lane in range(32)]


HI_MAX = (2 * P - 1) ** 2 >> 256                               # T_hi of a product of operands below 2p (the S-box's widest)


def redc_kinds(rnd):
    """32 kinds of 512-bit T for tc_redc: T_hi up to HI_MAX with T_lo = 0, R - 1 and the byte patterns, the crafted squares of
    both families, squares and products of the edge operands, and random T."""
    lo = [0, R - 1] + [_fit(b, R) for b in (b"\x80" * 32, b"\x7f" * 32, b"\xff\x00" * 16, b"\x00\xff" * 16)]
    Ts = [HI_MAX * R + l for l in lo]
    Ts += [rnd.randrange(HI_MAX + 1) * R, rnd.randrange(HI_MAX + 1) * R + R - 1, 0, 1, R - 1, R]
    Ts += [s * s for s in (target("ones", rnd), target("ones", rnd), target("hensel", rnd), target("hensel", rnd),
                           P - 1, P, 2 * P - 1, 2 * P - 2, (1 << 254) - 1)]
    Ts += [(2 * P - 1) * (P - 1), (2 * P - 1) * (P + 1), (R - 1) * 2 % (HI_MAX * R)]
    while len(Ts) < 32:
        Ts.append(rnd.randrange(2 * P) * rnd.randrange(2 * P))
    assert all(T >> 256 <= HI_MAX for T in Ts)
    return Ts[:32]


MONT = (1 << 32) - pow(P, -1, 1 << 32)                         # -p^-1 mod 2^32


def finish_exact(h, y, u):
    """tc_finish's value: V = sum h[m] 2^(16m) (+ y 2^32), then one Montgomery row (V + m p) / 2^32, not reduced."""
    V = sum(x << (16 * i) for i, x in enumerate(h)) + (y << 32 if u else 0)
    m = (V & 0xFFFFFFFF) * MONT & 0xFFFFFFFF
    return (V + m * P) >> 32, V + m * P


def finish_ok(h, y, u):
    """tc_finish's preconditions: h[m] < 2^31, V + m p < 2^288, and with the addend y + (V_h >> 32) < 2^256."""
    Vh = sum(x << (16 * i) for i, x in enumerate(h))
    return all(0 <= x < 1 << 31 for x in h) and finish_exact(h, y, u)[1] < 1 << 288 and (not u or y + (Vh >> 32) < R)


def y_limit(h):
    """The largest addend the preconditions allow with these h (y 2^32 leaves V mod 2^32, hence m, unchanged)."""
    Vh = sum(x << (16 * i) for i, x in enumerate(h))
    m = (Vh & 0xFFFFFFFF) * MONT & 0xFFFFFFFF
    return min(R - 1 - (Vh >> 32), ((1 << 288) - 1 - Vh - m * P) >> 32)


def _odd_words(h):
    """O of tc_finish: limbs 1.. of sum_L h[2L+1] 2^(32L+16)."""
    return [((h[2 * L + 3] << 16) | (h[2 * L + 1] >> 16)) & 0xFFFFFFFF for L in range(7)] + [h[15] >> 16]


def finish_kinds(rnd):
    """32 (h, y) kinds meeting tc_finish's preconditions: zero, every packed pair at 2^31 - 1 or at the IMMA's largest column
    pair, with y zero or at its limit; E[0]'s carry (h[0] + (h[1] << 16) >= 2^32) -- the later E limbs cannot carry, h < 2^31 --;
    every add_cc of the U chain carrying out (y limbs 0..6 all ones over nonzero O limbs); V = p (mod 2^32), so that m = 2^32 - 1,
    and V = 0 (mod 2^32), m = 0; then random packed pairs with random or limit addends."""
    hmax, col = (1 << 31) - 1, 3 * 32 * 255 * 255 * 257
    out = [([0] * 16, 0), ([hmax] * 16, 0), ([col] * 16, 0), ([0] * 16, R - 1)]
    out += [([hmax] * 16, y_limit([hmax] * 16)), ([col] * 16, y_limit([col] * 16))]
    carry_e = [hmax, 0xFFFF] + [rnd.randrange(1 << 31) for _ in range(14)]
    out += [(carry_e, 0), (carry_e, y_limit(carry_e))]
    for _ in range(4):
        h = [rnd.randrange(1, 1 << 31) | 0x10001 for _ in range(16)]
        assert all(_odd_words(h)[L] for L in range(7))
        out.append((h, (1 << 224) - 1))                        # O[L] + 0xffffffff carries for L = 0..6
        out.append((h, y_limit(h)))
    for h0, h1 in ((0x70000001, 0x8000), (0, 0)):              # V mod 2^32 = p mod 2^32 (m = 2^32 - 1), then 0 (m = 0)
        h = [h0, h1] + [rnd.randrange(1 << 31) for _ in range(14)]
        out += [(h, 0), (h, y_limit(h))]
    while len(out) < 32:
        h = [rnd.randrange(1 << 31) for _ in range(16)]
        out.append((h, rnd.choice((rnd.randrange(y_limit(h) + 1), y_limit(h)))))
    return out[:32]


def host_finish(tc_lib, h, y, u):
    out = (C.c_uint32 * 8)()
    tc_lib.host_tc_finish((C.c_uint32 * 16)(*h), (C.c_uint32 * 8)(*[(y >> (32 * i)) & 0xFFFFFFFF for i in range(8)]), u, out)
    return sum(int(x) << (32 * i) for i, x in enumerate(out))


def test_finish_kinds_meet_the_preconditions():
    """The probe's tc_finish inputs: every one meets the preconditions (with and without the addend), each limit is exact (one
    more breaks a precondition), the carry kinds carry where they claim to, and the host build of tc_finish gives the exact
    value on all of them."""
    tc_lib = build_host_shim("poseidon_tc_shim")
    for seed in range(3):
        ks = finish_kinds(random.Random(seed))
        assert len(ks) == 32
        e_carry = u_carry = at_limit = 0
        for i, (h, y) in enumerate(ks):
            for u in (0, 1):
                yy = y if u else 0
                assert finish_ok(h, yy, u), (seed, i, u)
                assert host_finish(tc_lib, h, yy, u) == finish_exact(h, yy, u)[0], (seed, i, u)
            if y == y_limit(h):
                assert not finish_ok(h, y + 1, 1), (seed, i)
                at_limit += 1
            e_carry += h[0] + ((h[1] << 16) & 0xFFFFFFFF) >= 1 << 32
            O, c, carries = _odd_words(h), 0, 0
            for L in range(7):
                c = (O[L] + ((y >> (32 * L)) & 0xFFFFFFFF) + c) >> 32
                carries += c
            u_carry += carries == 7
        assert e_carry >= 2 and u_carry >= 4 and at_limit >= 6, (e_carry, u_carry, at_limit)


# ------------------------------------------------------------------------------------------------------------- GPU probe runs
@pytest.fixture(scope="module")
def probe():
    lib = C.CDLL(build_probe())
    return lib


@pytest.fixture(scope="module")
def shims():
    return {"tc": build_host_shim("poseidon_tc_shim"), "redc": build_host_shim("poseidon_tc_redc_shim"),
            "full": build_host_shim("poseidon_tc_full_shim")}


def _call(fn, *arrays_and_ints):
    args = [a.ctypes.data_as(u32p) if isinstance(a, np.ndarray) else a for a in arrays_and_ints]
    rc = fn(*args)
    assert rc == 0, f"CUDA error {rc}"


def _rinv(shims):
    from test_poseidon_tc_redc import as_round_words, rinv_table
    tab, words = rinv_table(shims["redc"])
    return np.array(tab, dtype=np.uint32), as_round_words(tab, words)


def _warps(vals):
    return [vals[32 * w:32 * w + 32] for w in range(PROBE_WARPS)]


@pytest.mark.gpu
def test_probe_tc_finish(probe, shims):
    """tc_finish on the device, per thread, against its host build and the exact value, with and without the addend."""
    ks = finish_kinds(random.Random(11))
    hy = rotated(ks)
    n = len(hy)
    for u in (0, 1):
        inp = np.concatenate([np.concatenate([_words(h, 1), _words([y if u else 0], 8)]) for h, y in hy])
        out = np.zeros(8 * n, dtype=np.uint32)
        _call(probe.probe_finish, inp, u, out, n)
        got = _ints(out, 8)
        for i, ((h, y), r) in enumerate(zip(hy, got)):
            yy = y if u else 0
            assert r == finish_exact(h, yy, u)[0] == host_finish(shims["tc"], h, yy, u), (u, i // 32, i % 32)


@pytest.mark.gpu
def test_probe_tc_redc(probe, shims):
    """tc_redc over the R^-1 table in shared memory against the warp emulation, T / R mod p, and T_hi + p (1 + 32 * 255 / 2^32)."""
    from test_poseidon_tc_redc import EXTRA, reduce_warp
    tab, tab4 = _rinv(shims)
    Ts = rotated(redc_kinds(random.Random(12)))
    out = np.zeros(8 * len(Ts), dtype=np.uint32)
    _call(probe.probe_redc, _words(Ts, 16), tab, out, len(Ts))
    got = _ints(out, 8)
    for w, (Tw, gw) in enumerate(zip(_warps(Ts), _warps(got))):
        assert gw == reduce_warp(shims["tc"], tab4, Tw), w
        for lane, (T, r) in enumerate(zip(Tw, gw)):
            assert r % P == T * RINV % P and r < (T >> 256) + P * (1 + EXTRA), (w, lane)


@pytest.mark.gpu
def test_probe_sbox5_tc(probe, shims):
    """pos_sbox5_tc (three 512-bit products, each reduced on the tensor cores) on operands below 2p, the partial rounds' S-box
    input contract, against three emulated reductions, x^5 / R^4 mod p, and its bound x^5 < 1.60p."""
    from test_poseidon_tc_redc import reduce_warp
    tab, tab4 = _rinv(shims)
    xs = rotated(kinds(2 * P, random.Random(13)))
    out = np.zeros(8 * len(xs), dtype=np.uint32)
    _call(probe.probe_sbox5, _words(xs, 8), tab, out, len(xs))
    got = _ints(out, 8)
    r4 = pow(RINV, 4, P)
    for w, (xw, gw) in enumerate(zip(_warps(xs), _warps(got))):
        x2 = reduce_warp(shims["tc"], tab4, [x * x for x in xw])
        x4 = reduce_warp(shims["tc"], tab4, [v * v for v in x2])
        x5 = reduce_warp(shims["tc"], tab4, [a * b for a, b in zip(x4, xw)])
        assert gw == x5, w
        for lane, (x, r) in enumerate(zip(xw, gw)):
            assert r % P == pow(x, 5, P) * r4 % P and 100 * r < 160 * P, (w, lane)


@pytest.mark.gpu
def test_probe_tc_partial_round(probe, shims):
    """tc_partial_round over a round's table in shared memory, at y < 1.60p, any a below 2^256 and s2 < 2p (the contracts'
    maxima included), against the warp emulation (an unreduced; s2 after reduce8<F, 1, 1>), the field algebra and the bounds."""
    from test_poseidon_tc import emulate_output, tc_round_tables
    from test_poseidon_scaled_lane0 import schedule as sched
    cfg = steer_config("bench")
    lp = regions(*sched(FID["bn254_fr"], cfg), 3, cfg.full_rounds, cfg.partial_rounds)["lp"]
    tabs = tc_round_tables(shims["tc"], cfg)
    rnd = random.Random(14)
    ys, az, s2s = rotated(kinds(16 * P // 10, rnd)), rotated(kinds(R, rnd), 11), rotated(kinds(2 * P, rnd), 21)
    n = len(ys)
    inp = np.concatenate([_words([y, a, s2], 8) for y, a, s2 in zip(ys, az, s2s)])
    for k in (0, cfg.partial_rounds - 1):
        out = np.zeros(16 * n, dtype=np.uint32)
        _call(probe.probe_partial_round, inp, np.ascontiguousarray(tabs[k]), out, n)
        res = _ints(out, 8)
        an, s2n = res[0::2], res[1::2]
        gam, alp, bet, vv = (x * R % P for x in lp[k][:4])
        for w in range(PROBE_WARPS):
            sl = slice(32 * w, 32 * w + 32)
            ops = [[y, a, s] for y, a, s in zip(ys[sl], az[sl], s2s[sl])]
            e_an = emulate_output(shims["tc"], ops, tabs[k], [0, 1, 2])
            e_s2 = [v - 2 * P if v >= 2 * P else v for v in emulate_output(shims["tc"], [[y] for y in ys[sl]], tabs[k], [3], y=s2s[sl])]
            assert an[sl] == e_an and s2n[sl] == e_s2, (k, w)
            for lane, (y, a, s, r1, r2) in enumerate(zip(ys[sl], az[sl], s2s[sl], an[sl], s2n[sl])):
                assert r1 % P == (gam * y + alp * a + bet * s) * RINV % P and r1 < P + P * 3 * 255 // (1 << 27) + 1, (k, w, lane)
                assert r2 % P == (s + vv * y * RINV) % P and r2 < 2 * P, (k, w, lane)


@pytest.mark.gpu
def test_probe_tc_full_round(probe, shims):
    """tc_full_round over row tables in global memory, any operands below 2^256, for every matrix with all rows, the entry round
    (Mpre with the entry row) and the last round's partial `need` masks, against the warp emulation, the field algebra and the
    row bound; rows outside `need` are zero."""
    from test_poseidon_tc import emulate_output
    from test_poseidon_tc_full import EXTRA, ROW_WORDS, as_round_words, full_tables, row_constants, row_words
    cfg = steer_config("bench")
    tabs, words = full_tables(shims["full"], cfg), row_words(shims["full"])
    tabs4 = [as_round_words(tabs[row], words) for row in range(10)]
    rows = row_constants(cfg)
    rnd = random.Random(15)
    ops = list(zip(rotated(kinds(R, rnd)), rotated(kinds(R, rnd), 11), rotated(kinds(R, rnd), 21)))
    n = len(ops)
    inp = np.concatenate([_words(list(o), 8) for o in ops])
    for m, entry, need in ((0, False, 0b111), (1, True, 0b111), (2, False, 0b111), (0, False, 0b010), (0, False, 0b110)):
        table = np.ascontiguousarray(np.concatenate([tabs[3 * m], tabs[3 * m + 1], tabs[3 * m + 2], tabs[9] if entry else tabs[3 * m + 1]]))
        assert table.size == 4 * ROW_WORDS
        out = np.zeros(24 * n, dtype=np.uint32)
        _call(probe.probe_full_round, inp, table, C.c_uint(need), out, n)
        res = _ints(out, 8)
        for i in range(3):
            got = res[i::3]
            if not (need >> i) & 1:
                assert got == [0] * n, (m, i)
                continue
            consts = rows[9] if entry and i == 1 else rows[3 * m + i]
            tab4 = tabs4[9] if entry and i == 1 else tabs4[3 * m + i]
            mont = [c * R % P for c in consts]
            for w in range(PROBE_WARPS):
                sl = slice(32 * w, 32 * w + 32)
                raw = emulate_output(shims["tc"], [list(o) for o in ops[sl]], tab4, [0, 1, 2])
                assert got[sl] == [v - P if v >= P else v for v in raw], (m, i, w)
                for lane, (o, v) in enumerate(zip(ops[sl], raw)):
                    assert v < P * (1 + EXTRA) and got[32 * w + lane] == sum(c * s for c, s in zip(mont, o)) * RINV % P, (m, i, w, lane)
