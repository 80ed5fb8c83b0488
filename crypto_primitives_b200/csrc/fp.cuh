// fp.cuh -- 256-bit prime-field arithmetic in Montgomery form (R = 2^256) on 8 x 32-bit
// limbs held in registers; compile-time modulus per field tag.
//
// Replaces, for the device hot path, what the reference gets from ark-ff's
// Fp<MontBackend<_,4>,4> (third-party; call sites R/sponge/poseidon/mod.rs:70,75,81,90-91,
// R/crh/pedersen/mod.rs:116-124).  The memory image of an element is identical to ark-ff's:
// 4 x u64 little-endian limbs == 8 x u32 little-endian limbs, Montgomery form, fully reduced.
//
// mont_mul is CIOS with the even/odd accumulator split: products a[j]*b_i for even j are
// 64-bit values at even limb offsets and form one carry chain (one IMAD.WIDE.U32.X each);
// odd j form a second chain one limb higher.  Dividing by 2^32 after each reduction row swaps
// the roles of the two accumulators, so the shift costs no instructions.
#pragma once
#include "ptx.cuh"

namespace cpb {

// ---------------------------------------------------------------------------------------
// Field tags.  limb(i) getters fold to immediates once loops are unrolled.
// ---------------------------------------------------------------------------------------
#define CPB_FIELD_TABLE(NAME, ...)                                   \
    static CPB_HD constexpr u32 NAME(int i) {                        \
        constexpr u32 v[8] = {__VA_ARGS__};                          \
        return v[i];                                                 \
    }

struct Bls12_381_Fr {
    static constexpr bool LAZY5 = false;
    static constexpr bool SPLIT_ROUNDS = true;   // Poseidon: partial rounds in a loop of their own (poseidon.cuh)
    static constexpr int P0_POW = 0;          // k > 0: p[0] == 2^32 - 2^k + 1
    static constexpr bool P0_ONE = true;       // p[0] == 1  (then -p^-1 mod 2^32 == -1)
    static constexpr bool P1_ALLONES = true;   // p[1] == 0xffffffff
    static constexpr int ID = 0;
    static constexpr u32 NINV = 0xffffffffu;
    static constexpr int BITS = 255;
    CPB_FIELD_TABLE(P, 0x00000001u, 0xffffffffu, 0xfffe5bfeu, 0x53bda402u, 0x09a1d805u, 0x3339d808u, 0x299d7d48u, 0x73eda753u)
    CPB_FIELD_TABLE(ONE, 0xfffffffeu, 0x00000001u, 0x00034802u, 0x5884b7fau, 0xecbc4ff5u, 0x998c4fefu, 0xacc5056fu, 0x1824b159u)
    CPB_FIELD_TABLE(R2, 0xf3f29c6du, 0xc999e990u, 0x87925c23u, 0x2b6cedcbu, 0x7254398fu, 0x05d31496u, 0x9f59ff11u, 0x0748d9d9u)
};
struct Bn254_Fr {
    static constexpr bool LAZY5 = true;          // Poseidon alpha = 5 partial rounds keep lane 0 in [0, 2p) (poseidon.cuh; bounds there)
    static constexpr bool SPLIT_ROUNDS = true;   // Poseidon: partial rounds in a loop of their own (poseidon.cuh)
    static constexpr int P0_POW = 0;           // p[0] = 2^32 - 2^28 + 1, but the shift/add form measured slower (see DESIGN.md)          // k > 0: p[0] == 2^32 - 2^k + 1
    static constexpr bool P0_ONE = false;       // p[0] == 1  (then -p^-1 mod 2^32 == -1)
    static constexpr bool P1_ALLONES = false;   // p[1] == 0xffffffff
    static constexpr int ID = 1;
    static constexpr u32 NINV = 0xefffffffu;
    static constexpr int BITS = 254;
    CPB_FIELD_TABLE(P, 0xf0000001u, 0x43e1f593u, 0x79b97091u, 0x2833e848u, 0x8181585du, 0xb85045b6u, 0xe131a029u, 0x30644e72u)
    CPB_FIELD_TABLE(ONE, 0x4ffffffbu, 0xac96341cu, 0x9f60cd29u, 0x36fc7695u, 0x7879462eu, 0x666ea36fu, 0x9a07df2fu, 0x0e0a77c1u)
    CPB_FIELD_TABLE(R2, 0xae216da7u, 0x1bb8e645u, 0xe35c59e3u, 0x53fe3ab1u, 0x53bb8085u, 0x8c49833du, 0x7f4e44a5u, 0x0216d0b1u)
};
struct Jubjub_Fr {
    static constexpr bool LAZY5 = false;
    static constexpr bool SPLIT_ROUNDS = true;   // Poseidon: partial rounds in a loop of their own (poseidon.cuh)
    static constexpr int P0_POW = 0;          // k > 0: p[0] == 2^32 - 2^k + 1
    static constexpr bool P0_ONE = false;       // p[0] == 1  (then -p^-1 mod 2^32 == -1)
    static constexpr bool P1_ALLONES = false;   // p[1] == 0xffffffff
    static constexpr int ID = 2;
    static constexpr u32 NINV = 0xef788ef9u;
    static constexpr int BITS = 252;
    CPB_FIELD_TABLE(P, 0xd6f72cb7u, 0xd0970e5eu, 0xccc81082u, 0xa6682093u, 0x01343b00u, 0x06673b01u, 0x6533afa9u, 0x0e7db4eau)
    CPB_FIELD_TABLE(ONE, 0xb99607d9u, 0x25f80bb3u, 0x66b6e750u, 0xf315d62fu, 0xeb8814f4u, 0x932514eeu, 0x479155c6u, 0x09a6fc6fu)
    CPB_FIELD_TABLE(R2, 0x95e57731u, 0x67719aa4u, 0x9ce3fc26u, 0x51b0cef0u, 0xc026e9a5u, 0x69dab7fau, 0x8d127688u, 0x04f6547bu)
};
struct Bls12_377_Fr {
    static constexpr bool LAZY5 = false;
    static constexpr bool SPLIT_ROUNDS = true;   // Poseidon: partial rounds in a loop of their own (poseidon.cuh)
    static constexpr int P0_POW = 0;          // k > 0: p[0] == 2^32 - 2^k + 1
    static constexpr bool P0_ONE = true;       // p[0] == 1  (then -p^-1 mod 2^32 == -1)
    static constexpr bool P1_ALLONES = false;   // p[1] == 0xffffffff
    static constexpr int ID = 3;
    static constexpr u32 NINV = 0xffffffffu;
    static constexpr int BITS = 253;
    CPB_FIELD_TABLE(P, 0x00000001u, 0x0a118000u, 0xd0000001u, 0x59aa76feu, 0x5c37b001u, 0x60b44d1eu, 0x9a2ca556u, 0x12ab655eu)
    CPB_FIELD_TABLE(ONE, 0xfffffff3u, 0x7d1c7fffu, 0x6ffffff2u, 0x7257f50fu, 0x512c0feeu, 0x16d81575u, 0x2bbb9a9du, 0x0d4bda32u)
    CPB_FIELD_TABLE(R2, 0xb861857bu, 0x25d577bau, 0x8860591fu, 0xcc2c27b5u, 0xe5dc8593u, 0xa7cc008fu, 0xeff1c939u, 0x011fdae7u)
};

// ---------------------------------------------------------------------------------------
// Element-wise helpers (all loops fully unrolled: limbs live in registers).
// ---------------------------------------------------------------------------------------
CPB_HD void fp_copy(u32* r, const u32* a) {
#pragma unroll
    for (int i = 0; i < 8; i++) r[i] = a[i];
}
CPB_HD void fp_zero(u32* r) {
#pragma unroll
    for (int i = 0; i < 8; i++) r[i] = 0;
}
template <class F> CPB_HD void fp_one(u32* r) {
#pragma unroll
    for (int i = 0; i < 8; i++) r[i] = F::ONE(i);
}
// Load one element (32 B, 16-byte aligned) as two 128-bit accesses.
CPB_HD void ld_elem(u32* r, const u32* p) {
#if defined(__CUDA_ARCH__)
    uint4 a = *reinterpret_cast<const uint4*>(p);
    uint4 b = *reinterpret_cast<const uint4*>(p + 4);
    r[0] = a.x; r[1] = a.y; r[2] = a.z; r[3] = a.w;
    r[4] = b.x; r[5] = b.y; r[6] = b.z; r[7] = b.w;
#else
    for (int i = 0; i < 8; i++) r[i] = p[i];
#endif
}
CPB_HD void st_elem(u32* p, const u32* r) {
#if defined(__CUDA_ARCH__)
    *reinterpret_cast<uint4*>(p) = make_uint4(r[0], r[1], r[2], r[3]);
    *reinterpret_cast<uint4*>(p + 4) = make_uint4(r[4], r[5], r[6], r[7]);
#else
    for (int i = 0; i < 8; i++) p[i] = r[i];
#endif
}

CPB_HD bool fp_eq(const u32* a, const u32* b) {
    u32 d = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) d |= a[i] ^ b[i];
    return d == 0;
}

// The multiplier takes the modulus limbs as a register array `pm` (loaded once per kernel from
// shared memory): ptxas fuses mad.lo.cc/madc.hi.cc into one IMAD.WIDE.U32.X only when both
// factors are ordinary registers -- with an immediate or constant-bank factor it emits
// IMAD.X + IMAD.HI.U32.X, doubling the reduction cost (seen in cuobjdump -sass).  Additive
// paths keep the modulus as immediates (F::P), which costs no registers.
template <class F> CPB_HD void fp_modulus(u32* pm) {
#pragma unroll
    for (int i = 0; i < 8; i++) pm[i] = F::P(i);
}

// r in [0, 2p) -> [0, p).  Requires 2p < 2^256 (true for every field tag above).
template <class F> CPB_HD void fp_final_sub(u32* r) {
    u32 t[8];
    t[0] = sub_cc(r[0], F::P(0));
#pragma unroll
    for (int i = 1; i < 8; i++) t[i] = subc_cc(r[i], F::P(i));
    u32 borrow = subc(0, 0);   // 0xffffffff when r < p
#pragma unroll
    for (int i = 0; i < 8; i++) r[i] = borrow ? r[i] : t[i];
}

template <class F> CPB_HD void fp_add(u32* r, const u32* a, const u32* b) {
    r[0] = add_cc(a[0], b[0]);
#pragma unroll
    for (int i = 1; i < 7; i++) r[i] = addc_cc(a[i], b[i]);
    r[7] = addc(a[7], b[7]);   // a+b < 2p < 2^256
    fp_final_sub<F>(r);
}

// r = a + b without reduction (callers guarantee a + b < 2^256).
CPB_HD void fp_add_noreduce(u32* r, const u32* a, const u32* b) {
    r[0] = add_cc(a[0], b[0]);
#pragma unroll
    for (int i = 1; i < 7; i++) r[i] = addc_cc(a[i], b[i]);
    r[7] = addc(a[7], b[7]);
}

template <class F> CPB_HD void fp_sub(u32* r, const u32* a, const u32* b) {
    u32 t[8];
    t[0] = sub_cc(a[0], b[0]);
#pragma unroll
    for (int i = 1; i < 8; i++) t[i] = subc_cc(a[i], b[i]);
    u32 borrow = subc(0, 0);
    r[0] = add_cc(t[0], F::P(0) & borrow);
#pragma unroll
    for (int i = 1; i < 7; i++) r[i] = addc_cc(t[i], F::P(i) & borrow);
    r[7] = addc(t[7], F::P(7) & borrow);
}

template <class F> CPB_HD void fp_double(u32* r, const u32* a) { fp_add<F>(r, a, a); }

// ---------------------------------------------------------------------------------------
// Montgomery multiplication.
// ---------------------------------------------------------------------------------------
namespace detail {

// V += m*p with m chosen so the low limb of V = E + 2^32*O becomes zero.
// A 32x32->64 multiply-add (IMAD.WIDE / IMAD.HI) occupies the integer multiply pipe longer than a
// 32-bit IMAD or an ALU op, and the ALU pipe is mostly idle in this code, so moduli with
// trivial low limbs trade multiplies for adds:
//   p[0] == 1          : m = -E[0];  E[0] + m*1 is exactly 2^32 when E[0] != 0, i.e. just a carry.
//   p[1] == 2^32 - 1   : m*(2^32-1) = (m - [m!=0]) * 2^32 + E[0]   (two adds, no multiply).
// BLS12-381 Fr has both (6 wide multiply-adds per row instead of 8), BLS12-377 Fr the first.
template <class F, bool WITH_X> CPB_HD void redc_row_impl(u32* E, u32* O, u32* X, const u32* pm) {
    if (F::P0_ONE) {
        const u32 e0 = E[0];
        const u32 m = sub_cc(0u, e0);                 // CF = (e0 != 0)
        if (F::P1_ALLONES) {
            const u32 hi1 = subc(m, 0u);              // m - [m != 0]
            O[0] = add_cc(O[0], e0);
            O[1] = addc_cc(O[1], hi1);
        } else {
            mad_wide_cc(O[0], O[1], pm[1], m);
        }
        madc_wide_cc(O[2], O[3], pm[3], m);
        madc_wide_cc(O[4], O[5], pm[5], m);
        madc_wide_cc(O[6], O[7], pm[7], m);
        if (WITH_X) *X = addc(*X, 0);
        (void)add_cc(e0, LIMB_MASK);                  // CF = (e0 != 0): the carry out of E[0] + m
        E[1] = addc_cc(E[1], 0u);
        madc_wide_cc(E[2], E[3], pm[2], m);
        madc_wide_cc(E[4], E[5], pm[4], m);
        madc_wide_cc(E[6], E[7], pm[6], m);
    } else if (F::P0_POW > 0) {
        // p[0] = 2^32 - 2^k + 1 (BN254 Fr, k = 28): -p^-1 = -(1 + 2^k) mod 2^32 and m*p[0] are shifts and
        // adds on the idle ALU pipe instead of an IMAD and an IMAD.HI on the saturated multiply pipe.
        constexpr int K = F::P0_POW > 0 ? F::P0_POW : 1;   // (branch is dead when P0_POW == 0)
        const u32 e0 = E[0];
        const u32 m = (0u - (e0 + (e0 << K))) & LIMB_MASK;
        // B = m * (2^k - 1);  m*p[0] = m*2^32 - B;  hi(m*p[0] + e0) = m - B_hi - [B_lo != 0] + [e0 != 0]
        const u32 b_lo = sub_cc((m << K) & LIMB_MASK, m);
        const u32 b_hi = subc(m >> (LIMB_BITS - K), 0u);
        (void)sub_cc(0u, b_lo);                       // CF = (b_lo != 0)
        u32 hw = subc(m, b_hi);
        (void)add_cc(e0, LIMB_MASK);                  // CF = (e0 != 0)
        hw = addc(hw, 0u);
        mad_wide_cc(O[0], O[1], pm[1], m);
        madc_wide_cc(O[2], O[3], pm[3], m);
        madc_wide_cc(O[4], O[5], pm[5], m);
        madc_wide_cc(O[6], O[7], pm[7], m);
        if (WITH_X) *X = addc(*X, 0);
        E[1] = add_cc(E[1], hw);
        madc_wide_cc(E[2], E[3], pm[2], m);
        madc_wide_cc(E[4], E[5], pm[4], m);
        madc_wide_cc(E[6], E[7], pm[6], m);
    } else {
        const u32 m = mul_lo(E[0], F::NINV);
        mad_wide_cc(O[0], O[1], pm[1], m);
        madc_wide_cc(O[2], O[3], pm[3], m);
        madc_wide_cc(O[4], O[5], pm[5], m);
        madc_wide_cc(O[6], O[7], pm[7], m);           // without X: no carry out, V < 2^288
        if (WITH_X) *X = addc(*X, 0);
        mad_wide_cc(E[0], E[1], pm[0], m);
        madc_wide_cc(E[2], E[3], pm[2], m);
        madc_wide_cc(E[4], E[5], pm[4], m);
        madc_wide_cc(E[6], E[7], pm[6], m);
    }
    if (WITH_X) {
        O[7] = addc_cc(O[7], 0);
        *X = addc(*X, 0);
    } else {
        O[7] = addc(O[7], 0);
    }
}
template <class F> CPB_HD void redc_row(u32* E, u32* O, const u32* pm) { redc_row_impl<F, false>(E, O, nullptr, pm); }

// First row: V = a*b0, then reduce.
template <class F> CPB_HD void first_row(u32* E, u32* O, const u32* a, u32 bi, const u32* pm) {
#pragma unroll
    for (int j = 0; j < 8; j += 2) {
        mul_wide(E[j], E[j + 1], a[j], bi);
        mul_wide(O[j], O[j + 1], a[j + 1], bi);
    }
    redc_row<F>(E, O, pm);
}

// Later rows.  On entry `O` is the previous row's even accumulator (low limb zero) and `E`
// the previous odd one: V/2^32 = E + O[1] + 2^32 * (O >> 64).  Adds a*bi, then reduces.
template <class F> CPB_HD void next_row(u32* E, u32* O, const u32* a, u32 bi, const u32* pm) {
    E[0] = add_cc(E[0], O[1]);
    madc_wide_cc_from(O[0], O[1], a[1], bi, O[2], O[3]);
    madc_wide_cc_from(O[2], O[3], a[3], bi, O[4], O[5]);
    madc_wide_cc_from(O[4], O[5], a[5], bi, O[6], O[7]);
    madc_wide_end(O[6], O[7], a[7], bi);
    mad_wide_cc(E[0], E[1], a[0], bi);
    madc_wide_cc(E[2], E[3], a[2], bi);
    madc_wide_cc(E[4], E[5], a[4], bi);
    madc_wide_cc(E[6], E[7], a[6], bi);
    O[7] = addc(O[7], 0);
    redc_row<F>(E, O, pm);
}

}  // namespace detail

// r = a*b/R mod p, fully reduced.  a, b in [0,p).  r may alias a or b.
// LAZY (fields with slack, see F::LAZY5): the conditional subtraction is skipped and r = (a*b + M*p)/R < p*(a*b/(R*p) + 1) is
// returned as it is.  Operand ranges of the row accumulators: `a` (the full operand of every row) may be any value with
// a + p < 2^256 -- the running value stays below a + p --, `b` (scanned limb by limb) any 256-bit value.
template <class F, bool LAZY = false> CPB_HD void fp_mul(u32* r, const u32* a, const u32* b, const u32* pm) {
    u32 ev[8], od[8];
    detail::first_row<F>(ev, od, a, b[0], pm);
    detail::next_row<F>(od, ev, a, b[1], pm);
    detail::next_row<F>(ev, od, a, b[2], pm);
    detail::next_row<F>(od, ev, a, b[3], pm);
    detail::next_row<F>(ev, od, a, b[4], pm);
    detail::next_row<F>(od, ev, a, b[5], pm);
    detail::next_row<F>(ev, od, a, b[6], pm);
    detail::next_row<F>(od, ev, a, b[7], pm);
    // last row used E = od (low limb zero), O = ev:  result = (od >> 32) + ev
    r[0] = add_cc(ev[0], od[1]);
#pragma unroll
    for (int i = 1; i < 7; i++) r[i] = addc_cc(ev[i], od[i + 1]);
    r[7] = addc(ev[7], 0);
    if (!LAZY) fp_final_sub<F>(r);
}

template <class F, bool LAZY = false> CPB_HD void fp_sqr(u32* r, const u32* a, const u32* pm);

// ---------------------------------------------------------------------------------------
// Lazy dot product: r = (sum_j a_j * b_j) / R mod p with ONE Montgomery reduction.
// One CIOS pass adds all T partial products of a row before reducing it, so a T-term dot
// product costs 8*(8T+8) wide multiply-adds instead of T*136.  The running value can reach
// (T+1)*p*2^32, which for a 255-bit p no longer fits the 9 limbs of (E, O); X catches the
// carries out of the top limb (it sits at 2^288 before the per-row shift, 2^256 after).
// ---------------------------------------------------------------------------------------
namespace detail {

template <class F> CPB_HD void redc_row_x(u32* E, u32* O, u32& X, const u32* pm) { redc_row_impl<F, true>(E, O, &X, pm); }

// Reduction row of the squaring: V <- V/2^32 + tin*2^256, then V += m*p as in redc_row_impl.
// On entry O is the previous row's even accumulator (low limb zero after its reduction), E the previous odd one,
// X the previous overflow word (it sat at 2^288, now at 2^256) and tin the limb of the square that enters the
// window at 2^256.  The two-limb shift of the old even accumulator is folded into the addend operand of the odd
// chain's multiply-adds (as next_row does for a product row), so it costs no instructions.
// tin + X may carry (X = 1 is common, tin = 0xffffffff a 2^-32 event): both are added with carry-out into the new X.
template <class F> CPB_HD void redc_row_shift_x(u32* E, u32* O, u32& X, u32 tin, const u32* pm) {
    E[0] = add_cc(E[0], O[1]);
    u32 xn;
    if (F::P0_ONE) {
        const u32 c0 = addc(0u, 0u);                  // carry into 2^32; joins the even chain below
        const u32 e0 = E[0];
        const u32 m = sub_cc(0u, e0);                 // CF = (e0 != 0)
        if (F::P1_ALLONES) {
            const u32 hi1 = subc(m, 0u);              // m - [m != 0]
            O[0] = add_cc(O[2], e0);
            O[1] = addc_cc(O[3], hi1);
        } else {
            mad_wide_cc_from(O[0], O[1], pm[1], m, O[2], O[3]);
        }
        madc_wide_cc_from(O[2], O[3], pm[3], m, O[4], O[5]);
        madc_wide_cc_from(O[4], O[5], pm[5], m, O[6], O[7]);
        madc_wide_cc_from(O[6], O[7], pm[7], m, 0u, tin);
        xn = addc(0u, 0u);
        O[7] = add_cc(O[7], X);
        xn = addc(xn, 0u);
        (void)add_cc(e0, LIMB_MASK);                  // CF = (e0 != 0): the carry out of E[0] + m
        E[1] = addc_cc(E[1], c0);
        madc_wide_cc(E[2], E[3], pm[2], m);
        madc_wide_cc(E[4], E[5], pm[4], m);
        madc_wide_cc(E[6], E[7], pm[6], m);
    } else {
        const u32 m = mul_lo(E[0], F::NINV);          // (does not touch the carry flag)
        madc_wide_cc_from(O[0], O[1], pm[1], m, O[2], O[3]);
        madc_wide_cc_from(O[2], O[3], pm[3], m, O[4], O[5]);
        madc_wide_cc_from(O[4], O[5], pm[5], m, O[6], O[7]);
        madc_wide_cc_from(O[6], O[7], pm[7], m, 0u, tin);
        xn = addc(0u, 0u);
        O[7] = add_cc(O[7], X);
        xn = addc(xn, 0u);
        mad_wide_cc(E[0], E[1], pm[0], m);
        madc_wide_cc(E[2], E[3], pm[2], m);
        madc_wide_cc(E[4], E[5], pm[4], m);
        madc_wide_cc(E[6], E[7], pm[6], m);
    }
    O[7] = addc_cc(O[7], 0u);
    X = addc(xn, 0u);
}

// The same row without an overflow word, for a window that provably stays below 2^288 (fp_sqr, the second row of fp_dot_tab):
// t7 and t8 enter at 2^224 and 2^256 after the shift, through the addend of the odd chain's top multiply-add, and the chains end
// without a carry out.
template <class F> CPB_HD void redc_row_shift(u32* E, u32* O, u32 t7, u32 t8, const u32* pm) {
    E[0] = add_cc(E[0], O[1]);
    if (F::P0_ONE) {
        const u32 c0 = addc(0u, 0u);                  // carry into 2^32; joins the even chain below
        const u32 e0 = E[0];
        const u32 m = sub_cc(0u, e0);                 // CF = (e0 != 0)
        if (F::P1_ALLONES) {
            const u32 hi1 = subc(m, 0u);              // m - [m != 0]
            O[0] = add_cc(O[2], e0);
            O[1] = addc_cc(O[3], hi1);
        } else {
            mad_wide_cc_from(O[0], O[1], pm[1], m, O[2], O[3]);
        }
        madc_wide_cc_from(O[2], O[3], pm[3], m, O[4], O[5]);
        madc_wide_cc_from(O[4], O[5], pm[5], m, O[6], O[7]);
        madc_wide_end_from(O[6], O[7], pm[7], m, t7, t8);
        (void)add_cc(e0, LIMB_MASK);                  // CF = (e0 != 0): the carry out of E[0] + m
        E[1] = addc_cc(E[1], c0);
        madc_wide_cc(E[2], E[3], pm[2], m);
        madc_wide_cc(E[4], E[5], pm[4], m);
        madc_wide_cc(E[6], E[7], pm[6], m);
    } else {
        const u32 m = mul_lo(E[0], F::NINV);          // (does not touch the carry flag)
        madc_wide_cc_from(O[0], O[1], pm[1], m, O[2], O[3]);
        madc_wide_cc_from(O[2], O[3], pm[3], m, O[4], O[5]);
        madc_wide_cc_from(O[4], O[5], pm[5], m, O[6], O[7]);
        madc_wide_end_from(O[6], O[7], pm[7], m, t7, t8);
        mad_wide_cc(E[0], E[1], pm[0], m);
        madc_wide_cc(E[2], E[3], pm[2], m);
        madc_wide_cc(E[4], E[5], pm[4], m);
        madc_wide_cc(E[6], E[7], pm[6], m);
    }
    O[7] = addc(O[7], 0u);
}

// V += a * bi   (no shift).  WX: keep the overflow word X up to date (see fp_dot for when it is needed).
template <bool WX> CPB_HD void acc_row_x(u32* E, u32* O, u32& X, const u32* a, u32 bi) {
    mad_wide_cc(O[0], O[1], a[1], bi);
    madc_wide_cc(O[2], O[3], a[3], bi);
    madc_wide_cc(O[4], O[5], a[5], bi);
    madc_wide_cc(O[6], O[7], a[7], bi);
    if (WX) X = addc(X, 0);
    mad_wide_cc(E[0], E[1], a[0], bi);
    madc_wide_cc(E[2], E[3], a[2], bi);
    madc_wide_cc(E[4], E[5], a[4], bi);
    madc_wide_cc(E[6], E[7], a[6], bi);
    if (WX) {
        O[7] = addc_cc(O[7], 0);
        X = addc(X, 0);
    } else {
        O[7] = addc(O[7], 0);
    }
}

// V = V/2^32 + a * bi  (E/O are the swapped accumulators, see next_row)
template <bool WX> CPB_HD void shift_acc_row_x(u32* E, u32* O, u32& X, const u32* a, u32 bi) {
    E[0] = add_cc(E[0], O[1]);
    madc_wide_cc_from(O[0], O[1], a[1], bi, O[2], O[3]);
    madc_wide_cc_from(O[2], O[3], a[3], bi, O[4], O[5]);
    madc_wide_cc_from(O[4], O[5], a[5], bi, O[6], O[7]);
    madc_wide_end(O[6], O[7], a[7], bi);
    if (WX) O[7] += X;   // old overflow limb lands on the new top limb; cannot overflow (V/2^32 < 2^288)
    mad_wide_cc(E[0], E[1], a[0], bi);
    madc_wide_cc(E[2], E[3], a[2], bi);
    madc_wide_cc(E[4], E[5], a[4], bi);
    madc_wide_cc(E[6], E[7], a[6], bi);
    if (WX) {
        O[7] = addc_cc(O[7], 0);
        X = addc(0, 0);
    } else {
        O[7] = addc(O[7], 0);
    }
}

// limb i (0..8) of p << k
template <class F> CPB_HD constexpr u32 p_shl(int k, int i) {
    return (u32)(((((i < 8) ? (u64)F::P(i < 8 ? i : 0) : 0ull) << k) |
                  ((i > 0 && k > 0) ? ((u64)F::P(i - 1) >> (LIMB_BITS - k)) : 0ull)) & LIMB_MASK);
}

// r (N = 9 limbs) < 2^(K+1) * p  ->  r[0..7] in [0, 2^KLO * p): conditional subtractions of 2^K p, ..., 2^KLO p.  N = 8: r < 2^256.
template <class F, int K, int KLO = 0, int N = 9> CPB_HD void reduce9(u32* r) {
    static_assert(N == 9 || N == 8, "9 limbs, or 8 for a value below 2^256");
    static_assert(N == 9 || p_shl<F>(K, 8) == 0, "2^K p must fit 8 limbs");
#pragma unroll
    for (int k = K; k >= KLO; k--) {
        u32 t[N];
        t[0] = sub_cc(r[0], p_shl<F>(k, 0));
#pragma unroll
        for (int i = 1; i < N; i++) t[i] = subc_cc(r[i], p_shl<F>(k, i));
        u32 borrow = subc(0, 0);
#pragma unroll
        for (int i = 0; i < N; i++) r[i] = borrow ? r[i] : t[i];
    }
}
template <class F, int K, int KLO = 0> CPB_HD void reduce8(u32* r) { reduce9<F, K, KLO, 8>(r); }

// The running value of a T-term dot product stays below (T+1) * p * 2^32.  When (T+1) * p <= 2^256 that fits the 9 limbs
// of (E, O) and the overflow word is dead weight: 5 ALU instructions per row.  Decided on the top limb (p < (p[7]+1) * 2^224):
// BN254 Fr up to T = 4, BLS12-377 Fr up to 12, Jubjub Fr up to 16; BLS12-381 Fr (p/2^256 = 0.453) needs X from T = 2.
template <class F, int T> CPB_HD constexpr bool dot_needs_x() {
    return (u64)(T + 1) * ((u64)F::P(7) + 1) > ((u64)1 << LIMB_BITS);
}
// The reduced value is (sum_j a_j*b_j + M*p) / R with M < R and a_j, b_j < p, i.e. below p * (T*p/R + 1): the number of
// conditional subtractions reduce9 needs is the smallest K with T*p <= (2^(K+1) - 1) * R (again on the top limb).  One pass
// for BN254 Fr up to T = 5 (three-term rows: 1.57 p), two for BLS12-381 Fr at T = 3 (2.36 p).  U > 0: a term below U*p is added
// to the reduced value (fp_dot_unit), i.e. the smallest K with T*p <= (2^(K+1) - 1 - U) * R.
template <class F, int T, int U = 0> CPB_HD constexpr int dot_reduce_passes() {
    int k = 0;
    while ((long long)T * ((long long)F::P(7) + 1) > (((long long)2 << k) - 1 - U) * ((long long)1 << LIMB_BITS)) k++;
    return k;
}

// One CIOS row over the terms J0 .. T-1 of a (b holds their T - J0 constants).
template <class F, int T, int I, int EX, int J0 = 0>
CPB_HD void dot_row(u32* E, u32* O, u32& X, const u32 (&a)[T][8], const u32* b, const u32* pm) {
    constexpr bool WX = dot_needs_x<F, T - J0 + EX>();
    // b: T - J0 constants of 8 limbs each (shared memory); this row uses limb I of each
    if (I == 0) {
        u32 bi = b[0];
#pragma unroll
        for (int j = 0; j < 8; j += 2) {
            mul_wide(E[j], E[j + 1], a[J0][j], bi);
            mul_wide(O[j], O[j + 1], a[J0][j + 1], bi);
        }
    } else {
        shift_acc_row_x<WX>(E, O, X, a[J0], b[I]);
    }
#pragma unroll
    for (int t = J0 + 1; t < T; t++) acc_row_x<WX>(E, O, X, a[t], b[8 * (t - J0) + I]);
    if (WX) redc_row_x<F>(E, O, X, pm);
    else redc_row<F>(E, O, pm);
}

}  // namespace detail

// r = sum_{j<T} a[j] * b[j] / R mod p, fully reduced.  a[j], b[j] in [0,p).  r must not alias a.
// EX > 0: the a[j] may be unreduced as long as sum_j a[j] < (T + EX) * p (outputs of the LAZY multiplier); the overflow word
// and the number of conditional subtractions are then decided for T + EX terms.
template <class F, int T, int EX = 0> CPB_HD void fp_dot(u32* r, const u32 (&a)[T][8], const u32* b, const u32* pm) {
    u32 ev[8], od[8], X = 0;
    detail::dot_row<F, T, 0, EX>(ev, od, X, a, b, pm);
    detail::dot_row<F, T, 1, EX>(od, ev, X, a, b, pm);
    detail::dot_row<F, T, 2, EX>(ev, od, X, a, b, pm);
    detail::dot_row<F, T, 3, EX>(od, ev, X, a, b, pm);
    detail::dot_row<F, T, 4, EX>(ev, od, X, a, b, pm);
    detail::dot_row<F, T, 5, EX>(od, ev, X, a, b, pm);
    detail::dot_row<F, T, 6, EX>(ev, od, X, a, b, pm);
    detail::dot_row<F, T, 7, EX>(od, ev, X, a, b, pm);
    u32 w[9];
    w[0] = add_cc(ev[0], od[1]);
#pragma unroll
    for (int i = 1; i < 7; i++) w[i] = addc_cc(ev[i], od[i + 1]);
    w[7] = addc_cc(ev[7], 0);
    w[8] = addc(X, 0);
    // value < p * (T*p/R + 1) <= 2^(K+1) * p
    constexpr int K = detail::dot_reduce_passes<F, T + EX>();
    detail::reduce9<F, K>(w);
#pragma unroll
    for (int i = 0; i < 8; i++) r[i] = w[i];
}

// r = a[0] + sum_{1<=j<T} a[j] * b[j-1] / R mod p, fully reduced: a row whose coefficient of a[0] is one (R in Montgomery form),
// as the sparse partial rounds with a scaled lane 0 have (poseidon_host.hpp).  The unit term costs additions, not a product:
// a[0]*R/R is added to the reduced (T-1)-term sum before the final conditional subtractions, value < XI*p + p*((T-1)*p/R + 1).
// a[1..T-1], b[j] in [0,p); a[0] < XI * p (XI = 2: an output of the LAZY multiplier).  r must not alias a.
template <class F, int T, int XI> CPB_HD void fp_dot_unit(u32* r, const u32 (&a)[T][8], const u32* b, const u32* pm) {
    static_assert(T >= 2, "fp_dot_unit needs at least one product term");
    u32 ev[8], od[8], X = 0;
    detail::dot_row<F, T, 0, 0, 1>(ev, od, X, a, b, pm);
    detail::dot_row<F, T, 1, 0, 1>(od, ev, X, a, b, pm);
    detail::dot_row<F, T, 2, 0, 1>(ev, od, X, a, b, pm);
    detail::dot_row<F, T, 3, 0, 1>(od, ev, X, a, b, pm);
    detail::dot_row<F, T, 4, 0, 1>(ev, od, X, a, b, pm);
    detail::dot_row<F, T, 5, 0, 1>(od, ev, X, a, b, pm);
    detail::dot_row<F, T, 6, 0, 1>(ev, od, X, a, b, pm);
    detail::dot_row<F, T, 7, 0, 1>(od, ev, X, a, b, pm);
    u32 w[9];
    w[0] = add_cc(ev[0], od[1]);
#pragma unroll
    for (int i = 1; i < 7; i++) w[i] = addc_cc(ev[i], od[i + 1]);
    w[7] = addc_cc(ev[7], 0);
    w[8] = addc(X, 0);
    w[0] = add_cc(w[0], a[0][0]);
#pragma unroll
    for (int i = 1; i < 8; i++) w[i] = addc_cc(w[i], a[0][i]);
    w[8] = addc(w[8], 0);
    constexpr int K = detail::dot_reduce_passes<F, T - 1, XI>();
    detail::reduce9<F, K>(w);
#pragma unroll
    for (int i = 0; i < 8; i++) r[i] = w[i];
}

// ---------------------------------------------------------------------------------------
// Dot product with fixed coefficients through digit tables: r = sum_{j<T} a[j] * c_j (+ y) mod p with TWO reduction rows.
// The coefficient c_j (Montgomery form) is known ahead of time, so instead of reducing each of the 8 rows of a[j] * c_j the
// host pre-reduces its digit multiples K_i(c_j) = c_j * 2^(32 i) * 2^64 / R mod p (i = 0..7, canonical plain integers; the
// schedule's digit tables, poseidon_host.hpp).  Then  V = sum_j sum_i a[j][i] * K_i(c_j) == (sum_j a[j] * c_j / R) * 2^64  and
// two Montgomery rows divide by 2^64.  The rows are 8T scalar x vector products at the same limb offset (a[j]'s limb is the
// scalar, the table row the vector): 64T + 16 wide multiply-adds (64T + 12 for BLS12-381 Fr) instead of fp_dot's 64T + 64.
//   V < 8T * 2^32 * p = T * 2^35 * p, for ANY a[j] < 2^256 (lazy outputs included), plus y * 2^64 for the unit addend (U > 0,
//   y in [0, U*p), added at limbs 2..9 with additions only).  The accumulator is E, O (limbs 0..8) and the overflow word X (limb 9);
//   U = 2 needs the slack tab_fits checks.
//   Result = (V + M*p) / 2^64 with M < 2^64: below p * (1 + U + T * 2^-29), brought to [0,p) by conditional subtractions of
//   2^K p, ..., p (K = 1 for U = 1, 2: below 4p).  LAZY: the last one, by p, is skipped and the result left in [0, 2p) -- below
//   p * (1 + T * 2^-29) when U = 0.  With w-bit limbs (the toy-field model) read 2^32, 2^64 as 2^w, 2^2w.
// tab: T tables of 8 rows of 8 limbs (K_0(c_j) .. K_7(c_j)), read with 128-bit loads.  r must not alias a; it may alias y.
// ---------------------------------------------------------------------------------------
namespace detail {

// Overflow word needed by the product rows (without the unit addend): the 8T rows plus a reduction row stay below 2^288 iff
// (8T + 1) * p <= 2^256 (decided on the top limb, as dot_needs_x).  The unit addend's top limb lands on limb 9 itself.
template <class F, int T, int U> CPB_HD constexpr bool tab_needs_x() { return U > 0 || dot_needs_x<F, 8 * T>(); }

// The accumulator's ten limbs (E, O, X) hold V + M*p < p * (8T * 2^32 + (1 + U) * 2^64) iff
// (p[7] + 1) * (1 + U + 8T * 2^-32) <= 2^32 (on the top limb): a unit addend below 2p (U = 2) needs about 3p < 2^256 -- every
// field tag but BLS12-381 Fr.
template <class F, int T, int U> CPB_HD constexpr bool tab_fits() {
    return ((u64)F::P(7) + 1) * (1 + U) + ((((u64)F::P(7) + 1) * 8 * T + LIMB_MASK) >> LIMB_BITS) <= ((u64)1 << LIMB_BITS);
}

// Overflow word of the second reduction row: after it (before the final shift) the value is (V + m0*p)/2^32 + m1*p, below
// p * (8T + 1 + (1 + U) * 2^32).  That stays below 2^288 -- so X is dead in the second row -- when
// (p[7] + 1) * (8T + 1 + (1 + U) * 2^32) <= 2^64 (on the top limb, p < (p[7] + 1) * 2^224), and the result is then below 2^256.
// BN254 Fr for U <= 2, BLS12-381 Fr for U <= 1.
template <class F, int T, int U> CPB_HD constexpr bool tab_row2_needs_x() {
    return ((u64)F::P(7) + 1) * (1 + U) + ((((u64)F::P(7) + 1) * (8 * T + 1) + LIMB_MASK) >> LIMB_BITS) > ((u64)1 << LIMB_BITS);
}

// Conditional subtractions after the two rows: the smallest K with (1 + U) * 2^29 + T <= 2^(K + 30) (result bound above; the
// limb width enters as 2^29 = 2^32 / 8).
template <int T, int U> CPB_HD constexpr int tab_reduce_passes() {
    int k = 0;
    while (((long long)(1 + U) << (LIMB_BITS - 3)) + T > ((long long)1 << (k + 1 + LIMB_BITS - 3))) k++;
    return k;
}

// A table row is stored odd limbs first (K[1], K[3], K[5], K[7], K[0], K[2], K[4], K[6]): each 128-bit load feeds one of the
// two carry chains of acc_row_x.
CPB_HD void ld_tab_row(u32* r, const u32* p) {
#if defined(__CUDA_ARCH__)
    const uint4 o = __ldg(reinterpret_cast<const uint4*>(p));
    const uint4 e = __ldg(reinterpret_cast<const uint4*>(p + 4));
    r[1] = o.x; r[3] = o.y; r[5] = o.z; r[7] = o.w;
    r[0] = e.x; r[2] = e.y; r[4] = e.z; r[6] = e.w;
#else
    for (int i = 0; i < 4; i++) {
        r[2 * i + 1] = p[i];
        r[2 * i] = p[4 + i];
    }
#endif
}

}  // namespace detail

template <class F, int T, int U = 0, bool LAZY = false>
CPB_HD void fp_dot_tab(u32* r, const u32 (*a)[8], const u32* tab, const u32* pm, const u32* y = nullptr) {
    static_assert(U >= 0 && U <= 2, "fp_dot_tab takes one unit addend below 2p at most");
    static_assert(U < 2 || detail::tab_fits<F, T, U>(), "the accumulator does not hold a unit addend below 2p");
    constexpr bool WX = detail::tab_needs_x<F, T, U>();
    u32 ev[8], od[8], X = 0, k[8];
    detail::ld_tab_row(k, tab);
#pragma unroll
    for (int j = 0; j < 8; j += 2) {
        mul_wide(ev[j], ev[j + 1], k[j], a[0][0]);
        mul_wide(od[j], od[j + 1], k[j + 1], a[0][0]);
    }
#pragma unroll
    for (int q = 1; q < 8 * T; q++) {
        detail::ld_tab_row(k, tab + 8 * q);                    // K_i(c_j), q = 8j + i
        detail::acc_row_x<WX>(ev, od, X, k, a[q / 8][q % 8]);
    }
    if (U) {                                                   // + y * 2^64: limbs 2..7 in ev, 8 in od[7], 9 in X
        ev[2] = add_cc(ev[2], y[0]);
#pragma unroll
        for (int i = 3; i < 8; i++) ev[i] = addc_cc(ev[i], y[i - 2]);
        od[7] = addc_cc(od[7], y[6]);
        X = addc(X, y[7]);
    }
    constexpr int K = detail::tab_reduce_passes<T, U>(), KLO = LAZY ? 1 : 0;
    if (WX) detail::redc_row_x<F>(ev, od, X, pm);
    else detail::redc_row<F>(ev, od, pm);
    // as fp_dot: the last row used E = od (low limb zero), O = ev
    if constexpr (detail::tab_row2_needs_x<F, T, U>()) {
        detail::redc_row_shift_x<F>(od, ev, X, 0u, pm);
        u32 w[9];
        w[0] = add_cc(ev[0], od[1]);
#pragma unroll
        for (int i = 1; i < 7; i++) w[i] = addc_cc(ev[i], od[i + 1]);
        w[7] = addc_cc(ev[7], 0);
        w[8] = addc(X, 0);
        detail::reduce9<F, K, KLO>(w);
#pragma unroll
        for (int i = 0; i < 8; i++) r[i] = w[i];
    } else {                                                   // result < 2^256: 8 limbs
        detail::redc_row_shift<F>(od, ev, 0u, WX ? X : 0u, pm);
        u32 w[8];
        w[0] = add_cc(ev[0], od[1]);
#pragma unroll
        for (int i = 1; i < 7; i++) w[i] = addc_cc(ev[i], od[i + 1]);
        w[7] = addc(ev[7], 0);
        detail::reduce8<F, K, KLO>(w);
#pragma unroll
        for (int i = 0; i < 8; i++) r[i] = w[i];
    }
}

// r = a + b mod p, fully reduced, for a + b < 3p (a < 2p an output of the LAZY multiplier, b in [0,p) or slightly above, as a
// LAZY fp_dot_tab leaves it): brought to [0,p) by two conditional subtractions, 2p then p.  Needs 3p < 2^256 (the F::LAZY5
// fields).  r may alias a or b.
template <class F> CPB_HD void fp_add_lazy(u32* r, const u32* a, const u32* b) {
    static_assert(3 * ((u64)F::P(7) + 1) <= ((u64)1 << LIMB_BITS), "fp_add_lazy needs 3p < 2^256");
    fp_add_noreduce(r, a, b);
    u32 t[8];
    t[0] = sub_cc(r[0], detail::p_shl<F>(1, 0));
#pragma unroll
    for (int i = 1; i < 8; i++) t[i] = subc_cc(r[i], detail::p_shl<F>(1, i));
    u32 borrow = subc(0, 0);   // 0xffffffff when r < 2p
#pragma unroll
    for (int i = 0; i < 8; i++) r[i] = borrow ? r[i] : t[i];
    fp_final_sub<F>(r);
}


// r = a*a/R mod p.  Dedicated squaring: the 28 cross products are computed once and doubled with
// adds (the ALU pipe has slack, the multiply pipe does not), then the 8 diagonal squares are added
// and the 512-bit value goes through 8 Montgomery reduction rows.  100 wide multiply-adds (84 for
// BLS12-381 Fr) against 128 (112) for fp_mul(a, a).
// LAZY: a < 2^256 with a^2 < R*p; the result (a^2 + M*p)/R < p*(a^2/(R*p) + 1) is returned without the conditional subtraction.
template <class F, bool LAZY> CPB_HD void fp_sqr(u32* r, const u32* a, const u32* pm) {
    // Cross products a_i*a_j (i<j) sit at limb i+j.  Even positions accumulate in E (index = limb),
    // odd positions in O (index = limb-1), so every product is an aligned 64-bit multiply-add and each
    // row is one carry chain per array.  A chain's carry-out always lands on a limb no earlier row
    // has touched, so it is simply materialised there.
    u32 E[14], O[14];
    // row 0
    mul_wide(O[0], O[1], a[0], a[1]);
    mul_wide(E[2], E[3], a[0], a[2]);
    mul_wide(O[2], O[3], a[0], a[3]);
    mul_wide(E[4], E[5], a[0], a[4]);
    mul_wide(O[4], O[5], a[0], a[5]);
    mul_wide(E[6], E[7], a[0], a[6]);
    mul_wide(O[6], O[7], a[0], a[7]);
    // row 1
    mad_wide_cc(O[2], O[3], a[1], a[2]);
    madc_wide_cc(O[4], O[5], a[1], a[4]);
    madc_wide_cc(O[6], O[7], a[1], a[6]);
    O[8] = addc(0, 0);
    mad_wide_cc(E[4], E[5], a[1], a[3]);
    madc_wide_cc(E[6], E[7], a[1], a[5]);
    madc_wide_end(E[8], E[9], a[1], a[7]);
    // row 2
    mad_wide_cc(O[4], O[5], a[2], a[3]);
    madc_wide_cc(O[6], O[7], a[2], a[5]);
    madc_wide_end_from(O[8], O[9], a[2], a[7], O[8]);
    mad_wide_cc(E[6], E[7], a[2], a[4]);
    madc_wide_cc(E[8], E[9], a[2], a[6]);
    E[10] = addc(0, 0);
    // row 3
    mad_wide_cc(O[6], O[7], a[3], a[4]);
    madc_wide_cc(O[8], O[9], a[3], a[6]);
    O[10] = addc(0, 0);
    mad_wide_cc(E[8], E[9], a[3], a[5]);
    madc_wide_end_from(E[10], E[11], a[3], a[7], E[10]);
    // row 4
    mad_wide_cc(O[8], O[9], a[4], a[5]);
    madc_wide_end_from(O[10], O[11], a[4], a[7], O[10]);
    mad_wide_cc(E[10], E[11], a[4], a[6]);
    E[12] = addc(0, 0);
    // row 5
    mad_wide_cc(O[10], O[11], a[5], a[6]);
    O[12] = addc(0, 0);
    mad_wide_end_from(E[12], E[13], a[5], a[7], E[12]);
    // row 6
    mad_wide_end_from(O[12], O[13], a[6], a[7], O[12]);
    // T = E + (O << 32)        (E[0] = E[1] = 0, nothing above E[13] / O[13])
    u32 T[16];
    T[0] = 0;
    T[1] = O[0];
    T[2] = add_cc(E[2], O[1]);
#pragma unroll
    for (int i = 3; i < 14; i++) T[i] = addc_cc(E[i], O[i - 1]);
    T[14] = addc_cc(O[13], 0);
    T[15] = addc(0, 0);
    // T = 2T + sum a_i^2 * 2^(64 i)
    T[0] = add_cc(T[0], T[0]);
#pragma unroll
    for (int i = 1; i < 15; i++) T[i] = addc_cc(T[i], T[i]);
    T[15] = addc(T[15], T[15]);
    mad_wide_cc(T[0], T[1], a[0], a[0]);
#pragma unroll
    for (int i = 1; i < 8; i++) madc_wide_cc(T[2 * i], T[2 * i + 1], a[i], a[i]);
    // Montgomery reduction of the 16-limb T with a rolling 9-limb window (ev, od) and no overflow word.  Limb i + 7 of T enters at
    // row i (i >= 1), limb 15 after the last row, so after row i the window holds (T mod 2^(32(i+8)) + M*p) / 2^(32i) with
    // M < 2^(32(i+1)): below 2^256 + 2^32*p < 2^288 for ANY a < 2^256 whenever p < 2^256 - 2^224 (every field tag).  The
    // result (T + M*p)/R is the same value the per-row entry at 2^256 computes.
    static_assert(F::P(7) < LIMB_MASK, "fp_sqr's window bound needs p < 2^256 - 2^224");
    u32 ev[8], od[8];
#pragma unroll
    for (int i = 0; i < 8; i++) { ev[i] = T[i]; od[i] = 0; }
    detail::redc_row<F>(ev, od, pm);
#pragma unroll
    for (int i = 1; i < 8; i++) {
        // shift the window by one limb: roles of ev/od swap each row
        u32* Ea = (i & 1) ? od : ev;    // new even accumulator (previous odd)
        u32* Oa = (i & 1) ? ev : od;    // previous even accumulator: low limb is zero, limb 1 moves into Ea[0]
        detail::redc_row_shift<F>(Ea, Oa, T[i + 7], 0u, pm);
    }
    // 8 rows: the last used E = od (low limb zero), O = ev; T[15] lands on limb 7.  The result is below 2p < 2^256 (a < p, or
    // a^2 < R*p when LAZY), so nothing carries out of limb 7.
    u32 w[8];
    w[0] = add_cc(ev[0], od[1]);
#pragma unroll
    for (int i = 1; i < 7; i++) w[i] = addc_cc(ev[i], od[i + 1]);
    w[7] = addc(ev[7], T[15]);
    if (!LAZY) fp_final_sub<F>(w);     // T < p^2  =>  result < 2p
#pragma unroll
    for (int i = 0; i < 8; i++) r[i] = w[i];
}

// Multiplier / squarer whose conditional subtraction is skipped when `lazy` (uniform at run time): one code instance serves
// both modes in rolled loops.
template <class F> CPB_HD void fp_mul_rt(u32* r, const u32* a, const u32* b, const u32* pm, bool lazy) {
    fp_mul<F, true>(r, a, b, pm);
    if (!lazy) fp_final_sub<F>(r);
}
template <class F> CPB_HD void fp_sqr_rt(u32* r, const u32* a, const u32* pm, bool lazy) {
    fp_sqr<F, true>(r, a, pm);          // a < p: result < 2p either way
    if (!lazy) fp_final_sub<F>(r);
}

// x^alpha for the S-box.  5 and 17 get fixed addition chains; anything else falls back to
// left-to-right square-and-multiply (alpha is uniform across the grid: no divergence).
template <class F> CPB_HD void fp_pow_alpha(u32* x, u64 alpha, const u32* pm) {
    u32 t[8];
    if (alpha == 5) {
        fp_sqr<F>(t, x, pm);
        fp_sqr<F>(t, t, pm);
        fp_mul<F>(x, t, x, pm);
    } else if (alpha == 17) {
        fp_sqr<F>(t, x, pm);
        fp_sqr<F>(t, t, pm);
        fp_sqr<F>(t, t, pm);
        fp_sqr<F>(t, t, pm);
        fp_mul<F>(x, t, x, pm);
    } else if (alpha == 3) {
        fp_sqr<F>(t, x, pm);
        fp_mul<F>(x, t, x, pm);
    } else {
        if (alpha == 0) { fp_one<F>(x); return; }
        int top = 63;
        while (!((alpha >> top) & 1)) top--;
        fp_copy(t, x);
        for (int i = top - 1; i >= 0; i--) {
            fp_sqr<F>(t, t, pm);
            if ((alpha >> i) & 1) fp_mul<F>(t, t, x, pm);
        }
        fp_copy(x, t);
    }
}

// Fermat inversion x^(p-2); 0 -> 0.  Only on cold paths (table build, batch normalisation).
template <class F> CPB_HD void fp_inv(u32* r, const u32* x, const u32* pm) {
    u32 acc[8], base[8], e[8];
    fp_one<F>(acc);
    fp_copy(base, x);
    e[0] = sub_cc(F::P(0), 2u);
#pragma unroll
    for (int i = 1; i < 8; i++) e[i] = subc_cc(F::P(i), 0u);
    // right-to-left binary exponentiation over the 8 limbs of p-2
#pragma unroll 1
    for (int k = 0; k < 8 * LIMB_BITS; k++) {
        u32 w = 0;
#pragma unroll
        for (int i = 0; i < 8; i++) w = (k / LIMB_BITS) == i ? e[i] : w;
        if ((w >> (k % LIMB_BITS)) & 1) fp_mul<F>(acc, acc, base, pm);
        fp_sqr<F>(base, base, pm);
    }
    fp_copy(r, acc);
}

}  // namespace cpb
