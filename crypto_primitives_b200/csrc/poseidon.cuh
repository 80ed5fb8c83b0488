// poseidon.cuh -- the Poseidon permutation and the CRH / two-to-one evaluation built on it,
// one hash per thread, whole state in registers.
//
// Device counterpart of PoseidonSponge::permute (R/sponge/poseidon/mod.rs:66-121) and of
// crh::poseidon::{CRH::evaluate, TwoToOneCRH::compress} (R/crh/poseidon/mod.rs:30-40,66-79),
// i.e. new sponge -> absorb (mod.rs:124-153) -> squeeze one native element (mod.rs:323-345).
// Executes the schedule produced by host::derive_schedule (poseidon_host.hpp): same function,
// sparse partial rounds.  Everything here is CPB_HD so tests/host can run the identical code
// on the CPU (PTX primitives emulated) against the oracle before any GPU time is spent.
#pragma once
#include "fp.cuh"

namespace cpb {

struct PoseidonDev {
    int t, rate, cap, rf, rp, sparse;
    u64 alpha;
    int off_c, off_m, off_mpre, off_cp0, off_pc, off_sp, off_arkp, off_mod, off_sc0, n_elems;
    // Always 0.  Kernels add threadIdx.x * zero to the shared-memory address of every constant so
    // that ptxas keeps multiplier operands in ordinary registers: values loaded from a
    // warp-uniform address are promoted to uniform registers, and a multiply-add with a
    // uniform-register factor is emitted as IMAD.X + IMAD.HI.U32.X instead of one IMAD.WIDE.U32.X.
    int zero;
    // Digit tables of the sparse schedule (PoseidonSchedule::tabs) in global memory: pos_permute_split multiplies by its
    // constants through them (fp_dot_tab).  Every device context has them; a CPU build of this code driven without them
    // (nullptr) multiplies by the Montgomery rows of `cs` instead, as the merged loop and the team kernel always do.
    const u32* tab = nullptr;
};

// This thread's pointer to P.tab.  On the device it is offset by threadIdx.x * zero for the reason given at `zero`.
CPB_HD const u32* pos_tables(const PoseidonDev& P) {
#if defined(__CUDA_ARCH__)
    return P.tab + (int)threadIdx.x * P.zero;
#else
    return P.tab;
#endif
}
// Whether pos_permute_split takes the table path: always on the device (the fallback is not compiled there).
CPB_HD bool pos_has_tables(const PoseidonDev& P) {
#if defined(__CUDA_ARCH__)
    return true;
#else
    return P.tab != nullptr;
#endif
}
// Element offsets (x 8 limbs) of the digit tables of the full-round matrix of round fr, of the per-round partial constants and
// of the entry row (PoseidonSchedule::tabs): M, Mpre, Mpost, then the off_sc0 + 1 region; 8 elements per constant.
CPB_HD int pos_full_table(const PoseidonDev& P, int fr) {
    const int half = P.rf / 2;
    return 8 * P.t * P.t * (fr == half - 1 ? 1 : fr == half ? 2 : 0);
}

template <class F, int T> CPB_HD void pos_add_vec(u32 (&s)[T][8], const u32* c) {
#pragma unroll
    for (int i = 0; i < T; i++) {
        u32 k[8];
        ld_elem(k, c + 8 * i);
        fp_add<F>(s[i], s[i], k);
    }
}

// Offset of the matrix of full round fr (0 .. rf-1): Mpre for the last first-half round, Mpost (stored right after Mpre) for the
// first second-half round, M otherwise.  Dense schedules store M in both slots.
CPB_HD int pos_full_matrix(const PoseidonDev& P, int fr) {
    const int half = P.rf / 2;
    return fr == half - 1 ? P.off_mpre : fr == half ? P.off_mpre + P.t * P.t : P.off_m;
}

// (s0, s1, ..., s_{T-1}) <- (s1, ..., s_{T-1}, s0).  Lets a rolled loop visit every lane while
// the state stays in registers (register files cannot be indexed dynamically); a rotation is
// 8T moves against ~900 instructions of work per visit.
template <int T> CPB_HD void pos_rotl(u32 (&s)[T][8]) {
    u32 tmp[8];
    fp_copy(tmp, s[0]);
#pragma unroll
    for (int i = 0; i + 1 < T; i++) fp_copy(s[i], s[i + 1]);
    fp_copy(s[T - 1], tmp);
}

// x^alpha, left-to-right binary.  For the arkworks S-box exponents (3, 5, 17, 257 = 2^k+1)
// this is k squarings and one multiplication -- the optimal chain -- from a single pair of
// inlined multiplier bodies, which keeps the kernel's instruction footprint small.
// lazy (F::LAZY5 fields, alpha = 5, canonical x): the three products skip their conditional subtraction; x^2 < 1.19p, x^4 < 1.27p,
// x^5 < 1.24p for p/R < 0.19 -- what the dense rows take with EX = 1 (3 * 1.24 p < 4p).
template <class F> CPB_HD void pos_sbox(u32* x, u64 alpha, int top_bit, const u32* pm, bool lazy = false) {
    u32 x0[8];
    fp_copy(x0, x);
#pragma unroll 1
    for (int i = top_bit - 1; i >= 0; i--) {
        if constexpr (F::LAZY5) {
            fp_sqr_rt<F>(x, x, pm, lazy);
            if ((alpha >> i) & 1) fp_mul_rt<F>(x, x, x0, pm, lazy);
        } else {
            fp_sqr<F>(x, x, pm);
            if ((alpha >> i) & 1) fp_mul<F>(x, x, x0, pm);
        }
    }
}

// x^5 as sqr, sqr, mul.  LAZY (F::LAZY5 fields): the three products skip their conditional subtractions (bounds at pos_sbox and
// pos_permute_split).
template <class F, bool LAZY> CPB_HD void pos_sbox5(u32* x, const u32* pm) {
    u32 x2[8];
    fp_sqr<F, LAZY>(x2, x, pm);
    fp_sqr<F, LAZY>(x2, x2, pm);
    fp_mul<F, LAZY>(x, x2, x, pm);
}

// The permutation, one rolled loop over all RF+RP rounds with a single instance of each
// arithmetic body:  [add round constants] -> S-box on T lanes or lane 0 -> linear layer as
// lazy dot products (T rows of a dense matrix, or the one dense row of the sparse form
// followed by the rank-one column update).
// 1: every field uses pos_permute_split; 0: none; unset: per field (F::SPLIT_ROUNDS).  Measured on the t = 3 kernels:
// BN254 Fr (57 partial rounds, alpha = 5) +3 %; BLS12-381 Fr (31 partial rounds, alpha = 17) -1 % before and +0.9 %
// after the squaring lost 51 instructions -- so every field uses the split form now.
#ifdef CPB_POS_SPLIT
#define CPB_POS_SPLIT_FOR(F) (CPB_POS_SPLIT != 0)
#else
#define CPB_POS_SPLIT_FOR(F) (F::SPLIT_ROUNDS)
#endif
#ifndef CPB_SBOX5
#define CPB_SBOX5 1        // straight-line x^5 in the partial-round loop (+0.6 % on BN254 Fr; other exponents use the bit loop)
#endif
#ifndef CPB_COL_UNROLL_MAX
#define CPB_COL_UNROLL_MAX 4
#endif

// Sparse schedules only: the same permutation with the partial rounds in a loop of their own.  The two
// halves of the full rounds share one body through a two-trip outer loop, so there is still a single
// instance of the dense round; the partial-round loop has no full/partial selection and no lane
// rotation, i.e. none of the register shuffles the merged loop pays at its control-flow joins.
//
// Two things the sponge knows and a bare permutation does not (PermuteHint): (i) in the first permutation of a fresh sponge the
// capacity lane 0 is zero, so its first S-box input is the round constant itself and S(c) comes from the schedule (off_sc0);
// (ii) when the permutation's result is only squeezed (no further permutation), the last round needs just the rows of the lanes
// that are read -- one of t for CRH::evaluate / TwoToOneCRH::compress.  Both leave every value that is used bit-identical.
struct PermuteHint {
    int lane0_zero;        // != 0: state lane 0 is zero on entry
    unsigned need;         // bit i set: lane i of the result is read; everything else is dead
};

// A5: the exponent is 5, known at compile time (P.alpha is not read).  Every S-box is then the straight-line pos_sbox5, with no
// run-time exponent test and no generic square-and-multiply body in either loop.
template <class F, int T, bool A5 = false>
CPB_HD void pos_permute_split(u32 (&s)[T][8], const PoseidonDev& P, const u32* cs, const u32* pm, const PermuteHint& H) {
    const int half = P.rf / 2;
    int top_bit = 0;
    if (!A5)
        for (int i = 63; i > 0; i--)
            if ((P.alpha >> i) & 1) { top_bit = i; break; }
    const bool alpha_zero = !A5 && P.alpha == 0;
    // Lazy reduction (F::LAZY5: p/2^256 <= 0.19, i.e. BN254 Fr; alpha = 5; widths whose (T+1)-term rows need no overflow word).
    // Full rounds: the S-box of a canonical x skips its three conditional subtractions (x^5 < 1.24p, see pos_sbox) and the dense
    // rows take the T unreduced lanes as EX = 1 (T * 1.24p < (T+1)*p for T <= 4), returning canonical values.
    constexpr bool LZ = F::LAZY5 && !detail::dot_needs_x<F, T + 1>() && T <= 4;
    static_assert(!F::LAZY5 || 100 * ((u64)F::P(7) + 1) <= 19 * ((u64)1 << LIMB_BITS), "LAZY5 needs p/2^256 <= 0.19");
    const bool lazy = LZ && (A5 || (CPB_SBOX5 && P.alpha == 5));
    // Lane 1 is carried as a = w_hat . s through the partial rounds (poseidon_host.hpp).  Its coefficients follow S(c0) in the
    // schedule (so PoseidonDev needs no field): per round [gamma, alpha, beta | v[2..T-1]], then the Mpre row and Cp0 entry that
    // put lane 1 into that basis on entry.
    const u32* lp = cs + 8 * (P.off_sc0 + 1);
    const u32* lp_entry = lp + 8 * P.rp * (2 * T - 2);
    // Digit tables (fp_dot_tab): every product by a schedule constant below goes through them -- two reduction rows per output
    // instead of eight -- and takes any operand below 2^256, so the lazy lanes need no EX term.  tk: the lp region's tables.
    const bool tabs = pos_has_tables(P);
    const u32* tb = pos_tables(P);
    const u32* tk = tb + 64 * 3 * T * T;
    const u32* tk_entry = tk + 64 * P.rp * (2 * T - 2);
#pragma unroll 1
    for (int phase = 0; phase < 2; phase++) {
        const int cnt = phase == 0 ? half : P.rf - half;   // odd RF: floor(RF/2) rounds before, ceil(RF/2) after (mod.rs:98-121)
#pragma unroll 1
        for (int q = 0; q < cnt; q++) {
            pos_add_vec<F, T>(s, cs + 8 * (P.off_c + (phase * half + q) * T));
            const int first_j = (H.lane0_zero != 0 && phase == 0 && q == 0) ? 0 : -1;     // the lane whose S-box is the schedule constant
            const unsigned need = (phase == 1 && q == cnt - 1) ? H.need : ~0u;            // rows of this round that are used
#pragma unroll 1
            for (int j = 0; j < T; j++) {
                if (j == first_j) ld_elem(s[0], cs + 8 * P.off_sc0);         // S(0 + c) of the schedule
                else if constexpr (A5) pos_sbox5<F, LZ>(s[0], pm);
                else if (alpha_zero) fp_one<F>(s[0]);
                else pos_sbox<F>(s[0], P.alpha, top_bit, pm, lazy);
                pos_rotl<T>(s);
            }
            const u32* rows = cs + 8 * pos_full_matrix(P, phase * half + q);
            const u32* trows = tb + 8 * pos_full_table(P, phase * half + q);
            const bool entry = phase == 0 && q == cnt - 1;                                 // Mpre: row 1 of the split form
            // Row collector, zeroed per round so that it is dead in the partial-round loop (24 registers at t = 3, which the
            // table rows of fp_dot_tab need there) and the shift below never reads an indeterminate value.
            u32 n[T][8];
#pragma unroll
            for (int i = 0; i < T; i++) fp_zero(n[i]);
#pragma unroll 1
            for (int i = 0; i < T; i++) {
                u32 d[8];
                fp_zero(d);
                if ((need >> i) & 1u) {
                    if (tabs) fp_dot_tab<F, T>(d, s, (entry && i == 1) ? tk_entry : trows + 64 * T * i, pm);
                    else fp_dot<F, T, LZ ? 1 : 0>(d, s, (entry && i == 1) ? lp_entry : rows + 8 * T * i, pm);
                }
#pragma unroll
                for (int k = 0; k + 1 < T; k++) fp_copy(n[k], n[k + 1]);
                fp_copy(n[T - 1], d);
            }
#pragma unroll
            for (int i = 0; i < T; i++) fp_copy(s[i], n[i]);
        }
        if (phase == 0 && P.rp > 0) {
#pragma unroll
            for (int i = 0; i < T; i++) {                                  // Cp0, lane 1's entry in the w_hat_0 basis
                u32 c[8];
                ld_elem(c, i == 1 ? lp_entry + 8 * T : cs + 8 * (P.off_cp0 + i));
                fp_add<F>(s[i], s[i], c);
            }
            const u32* row = lp;
            const u32* pc = cs + 8 * (P.off_pc + 1);
            // Lane 0 is carried scaled and lane 1 as a = w_hat . s (poseidon_host.hpp): the row is L' = y + a, additions only, and
            // lane 1 moves on with one T-term dot a' = gamma*y + alpha*a + sum_{j>=2} beta_j*s_j over the state as it stands.
            // Lazy lane 0 (LZ): lane 0 lives in [0, 2p) from the constant
            // addition to the S-box output.  With a, b < 2p the Montgomery product (a*b + M*p)/R is below p*(4p/R + 1) <= 2p,
            // so x^2, x^4, x^5 need no conditional subtraction, nor does x = d + c (d, c < p).  Consumers of y < 1.60p: the dot
            // takes it as its one unreduced term (EX = 1) and returns a canonical a'; d = y + a < 2.60p is made canonical by two
            // conditional subtractions (fp_add_lazy); the column products v_j * y are ordinary multiplications whose full operand
            // y + p stays below 2^256 and whose results are reduced, so lanes 2.. stay canonical.  Bit-identical outputs.
            // With the digit tables the dot takes y like any operand below 2^256, and the column update s_j' = s_j + v_j * y is one
            // fp_dot_tab term with s_j as its unit addend.
            // Wide lanes (table path; every bound in tests/test_poseidon_bn254_alu.py).  The tables take any operand below 2^256, so
            // lanes 1.. need not be canonical inside the loop; only the additions that follow them and the exit care:
            //   lanes j >= 2 in [0, 2p) (WC: fields whose accumulator holds a unit addend below 2p, tab_fits -- not BLS12-381 Fr): the
            //     column update takes s_j < 2p as its unit addend (U = 2, result < p*(3 + 2^-29)) and one conditional subtraction of
            //     2p brings it back below 2p (the pass by p is skipped).
            //   lane 1 (LZ only): a' = the dot's result below p*(1 + T*2^-29) with its one conditional subtraction skipped.  Its one
            //     addition is d = y + a' < 1.60p + 1.01p < 3p, which fp_add_lazy brings to [0, p) as before.
            // After the last round lanes 1.. are made canonical (one pass by p), so the second-half constant additions see [0, p).
            constexpr bool WC = detail::tab_fits<F, 1, 2>();
            constexpr int UC = WC ? 2 : 1;
            const u32* trow = tk;
#pragma unroll 1
            for (int k = 0; k < P.rp; k++, row += 8 * (2 * T - 2), trow += 64 * (2 * T - 2), pc += 8) {
                if constexpr (A5) {
                    pos_sbox5<F, LZ>(s[0], pm);
                } else {
#if CPB_SBOX5
                    if (P.alpha == 5) pos_sbox5<F, LZ>(s[0], pm);     // straight-line x^5
                    else
#endif
                    if (alpha_zero) fp_one<F>(s[0]);
                    else pos_sbox<F>(s[0], P.alpha, top_bit, pm);
                }
                u32 an[8];
                if (tabs) fp_dot_tab<F, T, 0, LZ>(an, s, trow, pm);      // row = [gamma, alpha, beta[2..T-1]]
                else fp_dot<F, T, LZ ? 1 : 0>(an, s, row, pm);
                if constexpr (LZ) fp_add_lazy<F>(s[1], s[0], s[1]);      // s[1] <- d = y + a
                else fp_add<F>(s[1], s[0], s[1]);
                const u32* v = row + 8 * T;                               // v[2..T-1]
                const u32* tv = trow + 64 * T;
                if (T <= CPB_COL_UNROLL_MAX) {
#pragma unroll
                    for (int j = 2; j < T; j++) {
                        if (tabs) {
                            fp_dot_tab<F, 1, UC, WC>(s[j], &s[0], tv + 64 * (j - 2), pm, s[j]);
                            continue;
                        }
                        u32 c[8], tmp[8];
                        ld_elem(c, v + 8 * (j - 2));
                        fp_mul<F>(tmp, s[0], c, pm);
                        fp_add<F>(s[j], s[j], tmp);
                    }
                } else {
#pragma unroll 1
                    for (int j = 2; j < T; j++) {
                        u32 c[8], tmp[8];
                        if (tabs) {
                            fp_dot_tab<F, 1, UC, WC>(s[2], &s[0], tv + 64 * (j - 2), pm, s[2]);
                        } else {
                            ld_elem(c, v + 8 * (j - 2));
                            fp_mul<F>(tmp, s[0], c, pm);
                            fp_add<F>(s[2], s[2], tmp);
                        }
                        fp_copy(tmp, s[2]);                               // rotate lanes 2..T-1
#pragma unroll
                        for (int q = 2; q + 1 < T; q++) fp_copy(s[q], s[q + 1]);
                        fp_copy(s[T - 1], tmp);
                    }
                }
                if (k + 1 < P.rp) {
                    u32 c[8];
                    ld_elem(c, pc);
                    if (lazy) fp_add_noreduce(s[0], s[1], c);
                    else fp_add<F>(s[0], s[1], c);
                } else {
                    fp_copy(s[0], s[1]);
                }
                fp_copy(s[1], an);
            }
#pragma unroll
            for (int i = 1; i < T; i++) fp_final_sub<F>(s[i]);
        }
    }
}

// A5: see pos_permute_split; dense schedules take the merged loop, which reads P.alpha.
template <class F, int T, bool A5 = false>
CPB_HD void pos_permute(u32 (&s)[T][8], const PoseidonDev& P, const u32* cs, const u32* pm, const PermuteHint& H = PermuteHint{0, ~0u}) {
    if constexpr (CPB_POS_SPLIT_FOR(F)) {
        if (P.sparse) {
            pos_permute_split<F, T, A5>(s, P, cs, pm, H);
            return;
        }
    }
    const int half = P.rf / 2, total = P.rf + P.rp;
    int top_bit = 0;
    for (int i = 63; i > 0; i--)
        if ((P.alpha >> i) & 1) { top_bit = i; break; }
    const bool alpha_zero = P.alpha == 0;
    // row collector of the dense layers; defined once so that the shift below never reads an
    // indeterminate value (with the array declared inside the loop nvcc miscompiled t >= 5)
    u32 n[T][8];
#pragma unroll
    for (int i = 0; i < T; i++) fp_zero(n[i]);
#pragma unroll 1
    for (int r = 0; r < total; r++) {
        const bool full = r < half || r >= half + P.rp;
        const int k = r - half;                       // partial-round index when !full
        // --- round constants
        if (full) {
            const int fr = r < half ? r : r - P.rp;
            pos_add_vec<F, T>(s, cs + 8 * (P.off_c + fr * T));
        } else if (!P.sparse) {
            pos_add_vec<F, T>(s, cs + 8 * (P.off_arkp + k * T));
        } else if (k == 0) {
            pos_add_vec<F, T>(s, cs + 8 * P.off_cp0);
        }
        // --- S-box
        const int lanes = full ? T : 1;
#pragma unroll 1
        for (int j = 0; j < lanes; j++) {
            if (alpha_zero) fp_one<F>(s[0]);
            else pos_sbox<F>(s[0], P.alpha, top_bit, pm);
            if (full) pos_rotl<T>(s);
        }
        // --- linear layer
        const bool dense = full || !P.sparse;
        const u32* rows = dense ? cs + 8 * (full ? pos_full_matrix(P, r < half ? r : r - P.rp) : P.off_m)
                                : cs + 8 * (P.off_sp + k * (2 * T - 1));
        const int nrows = dense ? T : 1;
        u32 d[8];
#pragma unroll 1
        for (int i = 0; i < nrows; i++) {
            fp_dot<F, T>(d, s, rows + 8 * T * i, pm);
            if (dense) {                        // collect row i; after T iterations n[i] holds row i
#pragma unroll
                for (int q = 0; q + 1 < T; q++) fp_copy(n[q], n[q + 1]);
                fp_copy(n[T - 1], d);
            }
        }
        if (dense) {
#pragma unroll
            for (int i = 0; i < T; i++) fp_copy(s[i], n[i]);
        } else {
            // s_j += v_j * s_0 for j >= 1 (old s_0), then s_0 <- row product d (+ next lane-0 constant)
            const u32* v = rows + 8 * T;
            if (T <= CPB_COL_UNROLL_MAX) {
#pragma unroll
                for (int j = 1; j < T; j++) {
                    u32 c[8], tmp[8];
                    ld_elem(c, v + 8 * (j - 1));
                    fp_mul<F>(tmp, s[0], c, pm);
                    fp_add<F>(s[j], s[j], tmp);
                }
            } else {
#pragma unroll 1
                for (int j = 1; j < T; j++) {
                    u32 c[8], tmp[8];
                    ld_elem(c, v + 8 * (j - 1));
                    fp_mul<F>(tmp, s[0], c, pm);
                    fp_add<F>(s[1], s[1], tmp);
                    fp_copy(tmp, s[1]);        // rotate lanes 1..T-1
#pragma unroll
                    for (int q = 1; q + 1 < T; q++) fp_copy(s[q], s[q + 1]);
                    fp_copy(s[T - 1], tmp);
                }
            }
            if (k + 1 < P.rp) {
                u32 c[8];
                ld_elem(c, cs + 8 * (P.off_pc + k + 1));
                fp_add<F>(s[0], d, c);
            } else {
                fp_copy(s[0], d);
            }
        }
    }
}

// New sponge -> absorb `len` elements at `in` -> squeeze `n_out` native elements to `out` (8 limbs each).
// n_out == 1 is crh::poseidon::CRH::evaluate (R/crh/poseidon/mod.rs:30-40).  Absorb semantics of
// R/sponge/poseidon/mod.rs:124-153: fill `rate` lanes, permute while more input remains; the squeeze
// (mod.rs:156-186, 323-345) permutes once from Absorbing mode (so an empty input still costs one
// permutation), then emits `rate` lanes per permutation.
template <class F, int T>
CPB_HD void pos_sponge(u32* out, long n_out, const u32* in, long len, const PoseidonDev& P, const u32* cs, const u32* pm) {
    u32 s[T][8];
#pragma unroll
    for (int i = 0; i < T; i++) fp_zero(s[i]);
    const int rate = P.rate, cap = P.cap;
    const long nblocks = len <= rate ? 1 : (len + rate - 1) / rate;
    const long nsq = n_out <= rate ? 1 : (n_out + rate - 1) / rate;
#pragma unroll 1
    for (long b = 0; b < nblocks + nsq - 1; b++) {
        if (b < nblocks) {
            const long pos = b * rate;
            const long rem = len - pos;
            const int cnt = rem > rate ? rate : (int)rem;
#pragma unroll
            for (int i = 0; i < T; i++) {
                int lane = i - cap;
                if (lane >= 0 && lane < cnt) {
                    u32 e[8];
                    ld_elem(e, in + 8 * (pos + lane));
                    fp_add<F>(s[i], s[i], e);
                }
            }
        }
        pos_permute<F, T>(s, P, cs, pm);
        if (b >= nblocks - 1) {
            const long q = b - (nblocks - 1);          // squeeze block index
            const long left = n_out - q * rate;
            const int cnt = left > rate ? rate : (int)left;
#pragma unroll
            for (int i = 0; i < T; i++) {
                int lane = i - cap;
                if (lane >= 0 && lane < cnt) st_elem(out + 8 * (q * rate + lane), s[i]);
            }
        }
    }
}

// The one-permutation case of pos_sponge (len <= rate, 1 <= n_out <= rate, capacity >= 1) -- every hash of a Merkle build and
// every CRH::evaluate / TwoToOneCRH::compress of up to `rate` elements -- with the permutation told what the sponge knows
// (PermuteHint): lane 0 enters as zero, and only lanes cap .. cap+n_out-1 of the result are read.  A5: P.alpha == 5 (pos_permute_split).
template <class F, int T, bool A5 = false>
CPB_HD void pos_hash_single(u32* out, int n_out, const u32* in, int len, const PoseidonDev& P, const u32* cs, const u32* pm) {
    u32 s[T][8];
    const int cap = P.cap;
#pragma unroll
    for (int i = 0; i < T; i++) {
        const int lane = i - cap;
        if (lane >= 0 && lane < len) ld_elem(s[i], in + 8 * lane);
        else fp_zero(s[i]);
    }
    pos_permute<F, T, A5>(s, P, cs, pm, PermuteHint{1, ((1u << n_out) - 1u) << cap});
#pragma unroll
    for (int i = 0; i < T; i++) {
        const int lane = i - cap;
        if (lane >= 0 && lane < n_out) st_elem(out + 8 * lane, s[i]);
    }
}

template <class F, int T> CPB_HD void pos_crh(u32* out, const u32* in, long len, const PoseidonDev& P, const u32* cs, const u32* pm) {
    pos_sponge<F, T>(out, 1, in, len, P, cs, pm);
}

// Path::verify (R/merkle_tree/mod.rs:172-212) for the field-leaf Config: hash the leaf, fold the
// authentication path bottom-up choosing sides by the index bits, compare with the root.
// auth_path: plen elements ordered root side first (as Path.auth_path).  PL/PN, cl/cn: leaf / node schedules.
template <class F, int T>
CPB_HD bool pos_verify_path(const u32* leaf, long leaf_len, const u32* sibling, const u32* auth_path, int plen, unsigned long long index,
                            const u32* root, const PoseidonDev& PL, const u32* cl, const PoseidonDev& PN, const u32* cn, const u32* pm) {
    alignas(16) u32 pair[16];        // read back through 128-bit loads
    u32 cur[8];
    pos_crh<F, T>(cur, leaf, leaf_len, PL, cl, pm);
    u32 sib[8];
    ld_elem(sib, sibling);
#pragma unroll 1
    for (int level = plen; level >= 0; level--) {
        const bool right = (index & 1ull) != 0;       // computed node is the right child
#pragma unroll
        for (int j = 0; j < 8; j++) {
            pair[j] = right ? sib[j] : cur[j];
            pair[8 + j] = right ? cur[j] : sib[j];
        }
        pos_crh<F, T>(cur, pair, 2, PN, cn, pm);
        index >>= 1;
        if (level > 0) ld_elem(sib, auth_path + 8 * (level - 1));
    }
    u32 r[8];
    ld_elem(r, root);
    return fp_eq(cur, r);
}

// ---- ragged batches: input i is values[offsets[i] .. offsets[i+1]), n + 1 offsets, offsets[0] not necessarily 0.
// The hash launches walk the items sorted by their absorb-permutation count (a counting sort, cpb_poseidon.cu), so that a warp
// runs items of one length class instead of as many permutations as its longest input.  Keys are clamped at kRaggedBuckets:
// inputs of kRaggedBuckets or more blocks share the last bucket, and warps there may diverge.
constexpr int kRaggedBuckets = 64;

// Item i's slot range, clamped to [offsets[0], offsets[n]): a decreasing pair, or one outside that window, is an empty input, so
// no thread reads outside the caller's values whatever the offsets hold.
struct RaggedSpan {
    u64 lo;
    long len;
};
CPB_HD RaggedSpan ragged_span(const u64* offsets, long i, long n) {
    const u64 a = offsets[0], b = offsets[n];
    u64 lo = offsets[i], hi = offsets[i + 1];
    if (lo < a) lo = a;
    if (hi > b) hi = b;
    if (hi <= lo) return RaggedSpan{a, 0};
    return RaggedSpan{lo, (long)(hi - lo)};
}
// Absorb permutations of a `len`-element input (pos_sponge: an empty input still costs one) and its sort key, 0 .. kRaggedBuckets-1.
CPB_HD long ragged_blocks(long len, int rate) { return len <= rate ? 1 : (len + rate - 1) / rate; }
CPB_HD int ragged_key(long len, int rate) {
    const long b = ragged_blocks(len, rate);
    return (int)(b < kRaggedBuckets ? b : kRaggedBuckets) - 1;
}
// Exclusive scan of the key histogram: bucket b occupies order[starts[b] .. starts[b+1]); starts[kRaggedBuckets] = n.
CPB_HD void ragged_scan(const unsigned* hist, unsigned* starts) {
    unsigned s = 0;
    for (int b = 0; b < kRaggedBuckets; b++) {
        starts[b] = s;
        s += hist[b];
    }
    starts[kRaggedBuckets] = s;
}
// The two hash launches' slices of `order`: range[0..1] for the one-permutation kernel (bucket 0, when the squeeze fits one
// permutation too), range[2..3] for the general sponge kernel (everything else).
CPB_HD void ragged_ranges(const unsigned* starts, bool single, unsigned* range) {
    const unsigned split = single ? starts[1] : 0u;
    range[0] = 0;
    range[1] = split;
    range[2] = split;
    range[3] = starts[kRaggedBuckets];
}

}  // namespace cpb
