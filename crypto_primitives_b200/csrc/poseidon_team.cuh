// poseidon_team.cuh -- latency-oriented two-to-one compression for t = 3: FOUR WARPS cooperate on 32 hashes.
//
// The top ~13 levels of a Merkle tree have fewer nodes than the GPU has warp schedulers; with one hash per thread each
// such level costs one full single-warp permutation (~0.23 ms for BLS12-381 Fr), all of it on one scheduler: what bounds
// a level there is the length of the dependent chain of field multiplications (~730 cycles each for a lone warp), not
// throughput.  Here warp w (w = 0, 1, 2) of a 128-thread CTA owns state lane w of 32 hashes and warp 3 is a helper, so the
// chain per round is as short as the algebra allows:
//
//   full round (dense layer)    phase 1: lane w adds its constant and computes its S-box            (k squarings + 1 product)
//                               phase 2: lane w forms row w of the matrix as one lazy dot product   (~2 products)
//   sparse partial round k      x = lane 0, alpha = e + 1:
//                               phase 1: warp 0: y = x^e  (for alpha = 2^k + 1: k squarings)
//                                        warp j = 1, 2: u_j = w^_j * s_j, then t_j = v_j * x       (x published by warp 0 earlier)
//                                        warp 3: a = m00 * x, then u = u_1 + u_2 (+ constant)      (named barrier with warps 1, 2)
//                               phase 2: warp 0: lane 0 <- a * y + u                               = m00 * x^alpha + sum w^_j s_j
//                                        warp j: s_j <- s_j + t_j * y                               = s_j + v_j * x^alpha
//
// i.e. the S-box's last product is merged with the multiplication by m00 and by v_j -- (m00 * x) * x^e == m00 * x^alpha
// exactly, every fp_mul returns the canonical representative -- so a partial round costs k + 1 multiplication times
// instead of k + 2 (alpha = 5: 3 instead of 4; alpha = 17: 5 instead of 6; the three-warp version of round 1 needed
// S-box + one product).  BN254 Fr (8 + 57 rounds): 8*5 + 57*3 = 211 multiplication times per level instead of 268.
// Values are exchanged through single-buffered shared-memory slots with one __syncthreads after each phase: a slot
// written in phase p of a round is read only in the following phase and rewritten no earlier than phase p of the next
// round, two barriers later.  Same schedule (poseidon_host.hpp) and field values as poseidon.cuh => identical outputs.  (Sparse
// schedules carry lane 0 scaled and store m00 as one, so a = x here; the product is off the critical path and is kept.)
// The phase functions are CPB_HD: tests/host runs them for w = 0..3 in sequence as the CPU model of the kernel.
#pragma once
#include "poseidon.cuh"

namespace cpb {

// exchange slots, each [32 hashes] x 8 words: lanes 0..2 of the state (full rounds), then x, y, a, u1, u2 (partial rounds)
enum { TS_L0 = 0, TS_L1 = 1, TS_L2 = 2, TS_X = 3, TS_Y = 4, TS_A = 5, TS_U1 = 6, TS_U2 = 7, TS_U = 8, TS_COUNT = 9 };
CPB_HD u32* team_slot(u32* xb, int slot, int lane) { return xb + ((slot * 32 + lane) * 8); }
constexpr int kTeamXbWords = TS_COUNT * 32 * 8;
constexpr int kTeamThreads = 128;

// Named barrier among the three helper warps (1, 2, 3) inside phase 1 of a sparse partial round: warps 1, 2 arrive after
// publishing u_j, warp 3 after publishing a; warp 3 then sums u_1 + u_2 (+ constant) while warps 1, 2 go on with t_j, so that
// warp 0 needs one product and ONE addition in phase 2 (-2.5 % per level).  On the host (sequential model: w = 0, 1, 2, 3 in
// order) it is a no-op.  Four warps = one per scheduler is the sweet spot: a variant with two more helper warps (t_j = v_j * x
// off warps 1, 2) measured 5 % SLOWER -- a second active warp on the critical warp's scheduler competes for its multiplier
// pipe, which is what bounds a lone warp.
#if defined(__CUDA_ARCH__)
#define CPB_TEAM_HELPER_BARRIER() asm volatile("bar.sync 1, 96;" ::: "memory")
#else
#define CPB_TEAM_HELPER_BARRIER() ((void)0)
#endif

struct TeamRound {
    bool full, sparse_partial;
    int fr, k;            // index among the full rounds / among the partial rounds
};
CPB_HD TeamRound team_round(const PoseidonDev& P, int r) {
    const int half = P.rf / 2;
    TeamRound R;
    R.full = r < half || r >= half + P.rp;
    R.sparse_partial = !R.full && P.sparse;
    R.fr = r < half ? r : r - P.rp;
    R.k = r - half;
    return R;
}

// x^e by left-to-right square-and-multiply (e >= 1; top_bit = index of its leading one).  x0 = x is kept for the products.
template <class F> CPB_HD void team_pow(u32* x, u64 e, int top_bit, const u32* pm) {
    u32 x0[8];
    fp_copy(x0, x);
#pragma unroll 1
    for (int i = top_bit - 1; i >= 0; i--) {
        fp_sqr<F>(x, x, pm);
        if ((e >> i) & 1) fp_mul<F>(x, x, x0, pm);
    }
}

// Registers of one thread: s = its state lane (w < 3), t = v_j * x carried from phase 1 to phase 2 (w = 1, 2).
template <class F>
CPB_HD void team_phase1(u32* s, u32* t, int w, int lane, int r, const PoseidonDev& P, const u32* cs, const u32* pm, u32* xb,
                        int top_bit_alpha, int top_bit_e) {
    const TeamRound R = team_round(P, r);
    u32 c[8];
    if (!R.sparse_partial) {
        if (w > 2) return;
        if (R.full) ld_elem(c, cs + 8 * (P.off_c + R.fr * 3 + w));
        else ld_elem(c, cs + 8 * (P.off_arkp + R.k * 3 + w));
        fp_add<F>(s, s, c);
        if (R.full || w == 0) pos_sbox<F>(s, P.alpha, top_bit_alpha, pm);
        st_elem(team_slot(xb, TS_L0 + w, lane), s);
        return;
    }
    const u32* row = cs + 8 * (P.off_sp + R.k * 5);             // [m00, w^1, w^2 | v1, v2]
    if (w == 0) {
        u32 y[8];
        fp_copy(y, s);
        team_pow<F>(y, P.alpha - 1, top_bit_e, pm);             // x^(alpha-1); s keeps x (not needed afterwards)
        st_elem(team_slot(xb, TS_Y, lane), y);
    } else if (w == 3) {
        u32 x[8], a[8], u1[8], u2[8];
        ld_elem(x, team_slot(xb, TS_X, lane));
        ld_elem(c, row);
        fp_mul<F>(a, x, c, pm);
        st_elem(team_slot(xb, TS_A, lane), a);
        CPB_TEAM_HELPER_BARRIER();                              // u_1, u_2 are published
        ld_elem(u1, team_slot(xb, TS_U1, lane));
        ld_elem(u2, team_slot(xb, TS_U2, lane));
        fp_add<F>(u1, u1, u2);
        if (R.k + 1 < P.rp) {                                   // the lane-0 constant of the next round rides along
            ld_elem(c, cs + 8 * (P.off_pc + R.k + 1));
            fp_add<F>(u1, u1, c);
        }
        st_elem(team_slot(xb, TS_U, lane), u1);
    } else {
        u32 x[8], u[8];
        ld_elem(c, row + 8 * w);
        fp_mul<F>(u, s, c, pm);                                 // w^_j * s_j: needs nothing from this round, goes first
        st_elem(team_slot(xb, TS_U1 + (w - 1), lane), u);
        CPB_TEAM_HELPER_BARRIER();
        ld_elem(x, team_slot(xb, TS_X, lane));
        ld_elem(c, row + 8 * (3 + (w - 1)));
        fp_mul<F>(t, x, c, pm);                                 // v_j * x
    }
}

template <class F>
CPB_HD void team_phase2(u32* s, const u32* t, int w, int lane, int r, const PoseidonDev& P, const u32* cs, const u32* pm, u32* xb) {
    const TeamRound R = team_round(P, r);
    u32 c[8];
    if (!R.sparse_partial) {
        if (w > 2) return;
        u32 v[3][8];
#pragma unroll
        for (int j = 0; j < 3; j++) ld_elem(v[j], team_slot(xb, TS_L0 + j, lane));
        const u32* M = cs + 8 * (R.full ? pos_full_matrix(P, R.fr) : P.off_m);
        u32 d[8];
        fp_dot<F, 3>(d, v, M + 8 * 3 * w, pm);
        fp_copy(s, d);
        return;
    }
    if (w == 0) {
        u32 a[8], y[8], u[8], d[8];
        ld_elem(a, team_slot(xb, TS_A, lane));
        ld_elem(y, team_slot(xb, TS_Y, lane));
        ld_elem(u, team_slot(xb, TS_U, lane));                  // u_1 + u_2 (+ next constant), summed by warp 3
        fp_mul<F>(d, a, y, pm);
        fp_add<F>(s, d, u);
        (void)c;
    } else if (w < 3) {
        u32 y[8], tmp[8];
        ld_elem(y, team_slot(xb, TS_Y, lane));
        fp_mul<F>(tmp, t, y, pm);
        fp_add<F>(s, s, tmp);
    }
}

// What must be visible in the slots BEFORE phase 1 of round r+1 starts (runs after phase 2 of round r, before its barrier):
// a sparse partial round reads x = lane 0 from slot TS_X; the first one also needs the pre-constants Cp0 on every lane.
template <class F>
CPB_HD void team_publish(u32* s, int w, int lane, int r, const PoseidonDev& P, const u32* cs, u32* xb) {
    if (w > 2 || !P.sparse || P.rp == 0) return;
    const int half = P.rf / 2;
    const int next = r + 1;
    if (next < half || next >= half + P.rp) return;             // next round is not a partial one
    if (next == half) {                                         // entering the partial rounds: constants of round k = 0
        u32 c[8];
        ld_elem(c, cs + 8 * (P.off_cp0 + w));
        fp_add<F>(s, s, c);
    }
    if (w == 0) st_elem(team_slot(xb, TS_X, lane), s);   // its own slot: other warps may still be reading TS_L0 in phase 2
}

}  // namespace cpb
