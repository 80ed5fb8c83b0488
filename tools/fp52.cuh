// fp52.cuh -- EXPERIMENT, not part of the library: 256-bit Montgomery arithmetic on the FP64 pipe (5 limbs of 52 bits,
// radix R' = 2^260).  Bit-exact; tools/ubench_modmul.cu times it against the IMAD.WIDE path of csrc/fp.cuh.  A DFMA takes two issue
// cycles and a 52x52-bit product needs three FP64 instructions plus four integer ones (two 64-bit adds): 2704 bit-products
// per ~10 issue cycles against 1024 per 4 for IMAD.WIDE -- the same multiplier throughput per issue slot, and the SM
// issues one instruction per cycle per scheduler whichever pipe it goes to.  Kept because the emulation / range-assertion
// scaffolding is reusable.
//
// Idea: a 32x32->64 multiply-add (IMAD.WIDE) issues at 32 lanes/clk/SM, a double-precision FMA at 64, and a
// DFMA delivers a 52x52-bit product half where the IMAD delivers 32x32 (tools/ubench_fp64.cu):
// about 2.5x the multiplier throughput for big-integer work, on a pipe fp.cuh leaves idle.
//
// How (the double-precision technique of Emmart, Zheng & Weems): for integers a, b < 2^52 held exactly in doubles,
//     h = fma_rz(a, b, 2^104)                 = 2^104 + floor(a*b / 2^52) * 2^52        (exact: truncation only)
//     l = fma_rz(a, b, (2^104 + 2^52) - h)    = 2^52  + (a*b mod 2^52)                  (exact)
// The mantissa field of h is the high half of the product and that of l the low half, so column sums are formed by
// adding the raw 64-bit patterns with integer adds; the exponent fields add up to a constant per column that is known
// at compile time and is subtracted by initialising the column with its negative.  No carry flags anywhere: columns
// are 64-bit integers with > 6 bits of headroom, carries are explicit shifts.
//
// Values are kept LAZILY reduced: R' = 2^260 exceeds p by >= 5 bits, so a product of operands < 2p is < 1.34 p without
// any conditional subtraction; additions subtract 2p when the sum's top limb says so.  Only f52_canon() produces the
// canonical representative.  Element = 5 x u64 integer limbs (each < 2^52, value < 2p); multiplication operands are
// converted to doubles on demand (one LOP3 + one DADD per limb).
//
// Everything is CPB_HD: off the device fma_rz is emulated exactly with 128-bit integers (with range assertions when
// CPB_F52_CHECK is defined), so the code is verified bit-for-bit against Python integers on the CPU
// (tests/test_fp52_host.py) before any GPU time is spent.
#pragma once
#include "../crypto_primitives_b200/csrc/fp.cuh"

namespace cpb {
namespace f52 {

typedef long long s64;
constexpr u64 M52 = (1ull << 52) - 1;
constexpr u64 K_LO = 0x4330000000000000ull;   // bit pattern of 2^52  (exponent of every "l")
constexpr u64 K_HI = 0x4670000000000000ull;   // bit pattern of 2^104 (exponent of every "h")

#if defined(__CUDA_ARCH__)
CPB_D double fma_rz(double a, double b, double c) { return __fma_rz(a, b, c); }
CPB_D double sub_rz(double a, double b) { return __dsub_rz(a, b); }
CPB_D u64 dbits(double x) { return (u64)__double_as_longlong(x); }
CPB_D double from_bits(u64 b) { return __longlong_as_double((long long)b); }
#define CPB_F52_ASSERT(c) ((void)0)
#else
}  // namespace f52
}  // namespace cpb
#include <cassert>
#include <cstring>
namespace cpb {
namespace f52 {
#ifdef CPB_F52_CHECK
#define CPB_F52_ASSERT(c) assert(c)
#else
#define CPB_F52_ASSERT(c) ((void)0)
#endif
namespace detail {
typedef __int128 i128;
inline double rz53(i128 t) {                    // round an integer toward zero to 53 significant bits
    const bool neg = t < 0;
    unsigned __int128 m = neg ? (unsigned __int128)(-t) : (unsigned __int128)t;
    int len = 0;
    for (unsigned __int128 x = m; x; x >>= 1) len++;
    if (len > 53) m = (m >> (len - 53)) << (len - 53);
    const double d = (double)m;                 // <= 53 significant bits: exact
    return neg ? -d : d;
}
}  // namespace detail
inline double fma_rz(double a, double b, double c) { return detail::rz53((detail::i128)a * (detail::i128)b + (detail::i128)c); }
inline double sub_rz(double a, double b) { return detail::rz53((detail::i128)a - (detail::i128)b); }
inline u64 dbits(double x) { u64 b; memcpy(&b, &x, 8); return b; }
inline double from_bits(u64 b) { double x; memcpy(&x, &b, 8); return x; }
#endif

// ---- per-field constants, derived at compile time from the 32-bit limb table of fp.cuh
template <class F> CPB_HD constexpr u64 p52(int i) {
    u64 v = 0;
    for (int b = 0; b < 52; b++) {
        const int bit = 52 * i + b;
        if (bit < 256) v |= (u64)((F::P(bit / 32) >> (bit % 32)) & 1u) << b;
    }
    return v;
}
template <class F> CPB_HD constexpr u64 ninv52() {   // -p^-1 mod 2^52
    const u64 p0 = p52<F>(0) | (p52<F>(1) << 52);     // low 64 bits of p
    u64 inv = 1;
    for (int i = 0; i < 6; i++) inv *= 2 - p0 * inv;
    return (0 - inv) & M52;
}
template <class F> CPB_HD constexpr u64 twop52(int i) {   // limbs of 2p (2p < 2^257: fits 5 limbs)
    const u64 lo = i > 0 ? (p52<F>(i - 1) >> 51) : 0;
    return ((p52<F>(i) << 1) & M52) | lo;
}

// integer limb -> the same integer as a double
CPB_HD double to_dbl(u64 x) { return sub_rz(from_bits(x | K_LO), 4503599627370496.0); }
CPB_HD void to_dbl5(double* d, const u64* x) {
#pragma unroll
    for (int i = 0; i < 5; i++) d[i] = to_dbl(x[i]);
}

// one 52x52-bit product into two columns: lo += bits(l), hi += bits(h)  (each add carries the exponent constant)
CPB_HD void mac(u64& lo, u64& hi, double a, double b) {
    CPB_F52_ASSERT(a >= 0 && a < 4503599627370496.0 && b >= 0 && b < 4503599627370496.0);
    const double h = fma_rz(a, b, 0x1p104);
    const double l = fma_rz(a, b, sub_rz(0x1p104 + 0x1p52, h));
    hi += dbits(h);
    lo += dbits(l);
}
// the same product counted twice (cross terms of a square)
CPB_HD void mac2(u64& lo, u64& hi, double a, double b) {
    CPB_F52_ASSERT(a >= 0 && a < 4503599627370496.0 && b >= 0 && b < 4503599627370496.0);
    const double h = fma_rz(a, b, 0x1p104);
    const double l = fma_rz(a, b, sub_rz(0x1p104 + 0x1p52, h));
    hi += dbits(h) << 1;
    lo += dbits(l) << 1;
}

// number of index pairs (i, j), 0 <= i, j < 5, with i + j == k
CPB_HD constexpr int cnt5(int k) { return (k < 0 || k > 8) ? 0 : (k < 5 ? k + 1 : 9 - k); }
// columns start at minus the exponent constants they are going to receive: NP full 5x5 products (the reduction is one)
template <int NP> CPB_HD void cols_init(u64* c) {
#pragma unroll
    for (int k = 0; k < 10; k++) c[k] = 0 - ((u64)(NP * cnt5(k)) * K_LO + (u64)(NP * cnt5(k - 1)) * K_HI);
}
CPB_HD void acc_product(u64* c, const double* a, const double* b) {
#pragma unroll
    for (int i = 0; i < 5; i++)
#pragma unroll
        for (int j = 0; j < 5; j++) mac(c[i + j], c[i + j + 1], a[i], b[j]);
}
CPB_HD void acc_square(u64* c, const double* a) {
#pragma unroll
    for (int i = 0; i < 5; i++) {
        mac(c[2 * i], c[2 * i + 1], a[i], a[i]);
#pragma unroll
        for (int j = i + 1; j < 5; j++) mac2(c[i + j], c[i + j + 1], a[i], a[j]);
    }
}

// Montgomery reduction of the 10 columns (radix 2^52, five steps) and carry normalisation: r = V / 2^260 mod p, lazily
// reduced (r < V/2^260 + p), limbs < 2^52.  pd = the modulus as doubles, kept in registers by the caller.
template <class F> CPB_HD void reduce(u64* r, u64* c, const double* pd) {
    const double ninv = (double)ninv52<F>();
#pragma unroll
    for (int k = 0; k < 5; k++) {
        // q = (c[k] mod 2^52) * ninv mod 2^52   (the exponent constants are multiples of 2^52: the low bits are true)
        const double t = to_dbl(c[k] & M52);
        const double h = fma_rz(t, ninv, 0x1p104);
        const double l = fma_rz(t, ninv, sub_rz(0x1p104 + 0x1p52, h));
        const double q = sub_rz(l, 0x1p52);
#pragma unroll
        for (int j = 0; j < 5; j++) mac(c[k + j], c[k + j + 1], q, pd[j]);
        CPB_F52_ASSERT((c[k] & M52) == 0 && (c[k] >> 63) == 0);
        c[k + 1] += c[k] >> 52;
    }
#pragma unroll
    for (int i = 5; i < 9; i++) {
        CPB_F52_ASSERT((c[i] >> 63) == 0);
        c[i + 1] += c[i] >> 52;
        r[i - 5] = c[i] & M52;
    }
    CPB_F52_ASSERT(c[9] < (1ull << 52));
    r[4] = c[9];
}

template <class F> CPB_HD void load_modulus(double* pd) {
#pragma unroll
    for (int i = 0; i < 5; i++) pd[i] = (double)p52<F>(i);
}

// r = a*b / 2^260 (mod p), lazily reduced.  a, b: doubles holding limbs < 2^52 of values < 4p.
template <class F> CPB_HD void mul(u64* r, const double* a, const double* b, const double* pd) {
    u64 c[10];
    cols_init<2>(c);
    acc_product(c, a, b);
    reduce<F>(r, c, pd);
}
template <class F> CPB_HD void sqr(u64* r, const double* a, const double* pd) {
    u64 c[10];
    cols_init<2>(c);            // a square carries the same exponent constants as a product (cross terms count twice)
    acc_square(c, a);
    reduce<F>(r, c, pd);
}
// r = (sum_j a[j]*b[j] + addend * 2^260) / 2^260, lazily reduced; addend (integer limbs, may be null) costs 5 adds.
template <class F, int T> CPB_HD void dot(u64* r, const double (&a)[T][5], const double* b, const u64* addend, const double* pd) {
    u64 c[10];
    cols_init<T + 1>(c);
#pragma unroll
    for (int t = 0; t < T; t++) acc_product(c, a[t], b + 5 * t);
    if (addend) {
#pragma unroll
        for (int i = 0; i < 5; i++) c[5 + i] += addend[i];
    }
    reduce<F>(r, c, pd);
}

// r = a + b, brought back below 2p + 2^208 by subtracting 2p when the top limb reaches that of 2p.  Limbs < 2^52.
template <class F> CPB_HD void add(u64* r, const u64* a, const u64* b) {
    s64 t[5];
#pragma unroll
    for (int i = 0; i < 5; i++) t[i] = (s64)(a[i] + b[i]);
    const bool big = (u64)t[4] > twop52<F>(4);          // then a + b > 2p for certain (lower limbs cannot borrow that much)
#pragma unroll
    for (int i = 0; i < 5; i++) t[i] -= big ? (s64)twop52<F>(i) : 0;
#pragma unroll
    for (int i = 0; i < 4; i++) {                       // signed carries
        t[i + 1] += t[i] >> 52;
        t[i] &= (s64)M52;
    }
    CPB_F52_ASSERT(t[4] >= 0 && t[4] < (1ll << 52));
#pragma unroll
    for (int i = 0; i < 5; i++) r[i] = (u64)t[i];
}

// canonical representative: value < 4p -> [0, p)
template <class F> CPB_HD void canon(u64* r) {
#pragma unroll
    for (int round = 0; round < 3; round++) {
        s64 t[5];
        s64 borrow = 0;
#pragma unroll
        for (int i = 0; i < 5; i++) {
            t[i] = (s64)r[i] - (s64)p52<F>(i) + borrow;
            borrow = t[i] >> 52;                        // 0 or -1 (limbs are < 2^52: the difference is > -2^53)
            t[i] &= (s64)M52;
        }
        if (borrow == 0) {
#pragma unroll
            for (int i = 0; i < 5; i++) r[i] = (u64)t[i];
        }
    }
}

// 8 x u32 (256 bits, little endian) <-> 5 x 52-bit limbs
CPB_HD void from_words(u64* x, const u32* w) {
    u64 q[4];
#pragma unroll
    for (int i = 0; i < 4; i++) q[i] = (u64)w[2 * i] | ((u64)w[2 * i + 1] << 32);
    x[0] = q[0] & M52;
    x[1] = ((q[0] >> 52) | (q[1] << 12)) & M52;
    x[2] = ((q[1] >> 40) | (q[2] << 24)) & M52;
    x[3] = ((q[2] >> 28) | (q[3] << 36)) & M52;
    x[4] = q[3] >> 16;
}
CPB_HD void to_words(u32* w, const u64* x) {
    u64 q[4];
    q[0] = x[0] | (x[1] << 52);
    q[1] = (x[1] >> 12) | (x[2] << 40);
    q[2] = (x[2] >> 24) | (x[3] << 28);
    q[3] = (x[3] >> 36) | (x[4] << 16);
#pragma unroll
    for (int i = 0; i < 4; i++) { w[2 * i] = (u32)q[i]; w[2 * i + 1] = (u32)(q[i] >> 32); }
}

}  // namespace f52
}  // namespace cpb
