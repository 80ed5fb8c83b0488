// te_ops.cuh -- the twisted-Edwards (a = -1) operations behind signature::schnorr (R/signature/schnorr/mod.rs) and
// encryption::elgamal (R/encryption/elgamal/mod.rs), on top of pedersen.cuh's TePoint and mixed addition:
// doubling, full extended addition, negation, affine normalisation, point compression, variable-base scalar
// multiplication, and the scalar-field glue (Fr Montgomery limbs <-> integers, Fp::from_random_bytes).
//
// Formulas: Hisil-Wong-Carter-Dawson 2008, extended coordinates, a = -1 ("dbl-2008-hwcd", "add-2008-hwcd-3").  The
// doubling's denominators are F = y^2 - x^2 - 2 = d x^2 y^2 - 1 and G = 1 + d x^2 y^2 (affine, Z = 1), never zero when d
// is a non-square, so it agrees with the complete law on every point, the 8-torsion included (tests check it).
#pragma once
#include "pedersen.cuh"

namespace cpb {

// 2p: A = X^2, B = Y^2, C = 2 Z^2, D = -A, E = (X+Y)^2 - A - B, G = D + B, F = G - C, H = D - B.  4M + 4S.
template <class F> CPB_HD void te_dbl(TePoint& p, const u32* pm) {
    u32 a[8], b[8], c[8], e[8], g[8], f[8], h[8];
    fp_sqr<F>(a, p.X, pm);
    fp_sqr<F>(b, p.Y, pm);
    fp_sqr<F>(c, p.Z, pm);
    fp_add<F>(c, c, c);
    fp_add<F>(e, p.X, p.Y);
    fp_sqr<F>(e, e, pm);
    fp_sub<F>(e, e, a);
    fp_sub<F>(e, e, b);
    fp_sub<F>(g, b, a);                                  // D + B = B - A
    fp_sub<F>(f, g, c);
    fp_add<F>(h, a, b);                                  // H = D - B = -(A + B)
    fp_zero(c);
    fp_sub<F>(h, c, h);
    fp_mul<F>(p.X, e, f, pm);
    fp_mul<F>(p.Y, g, h, pm);
    fp_mul<F>(p.T, e, h, pm);
    fp_mul<F>(p.Z, f, g, pm);
}

// Projective Niels form of a point: (Y + X, Y - X, 2Z, 2d T).  Adding it costs 8M.
struct TeNiels {
    u32 yp[8], ym[8], z2[8], t2d[8];
};

template <class F> CPB_HD void te_to_niels(TeNiels& n, const TePoint& p, const u32* d2, const u32* pm) {
    fp_add<F>(n.yp, p.Y, p.X);
    fp_sub<F>(n.ym, p.Y, p.X);
    fp_add<F>(n.z2, p.Z, p.Z);
    fp_mul<F>(n.t2d, p.T, d2, pm);
}

// p += q (q in Niels form), negated first when `neg`: -(x, y) = (-x, y) swaps Y+X and Y-X and negates T.
template <class F> CPB_HD void te_add_niels(TePoint& p, const TeNiels& q, bool neg, const u32* pm) {
    u32 a[8], b[8], c[8], d[8], e[8], f[8], g[8], h[8], z[8];
    fp_sub<F>(a, p.Y, p.X);
    fp_mul<F>(a, a, neg ? q.yp : q.ym, pm);
    fp_add<F>(b, p.Y, p.X);
    fp_mul<F>(b, b, neg ? q.ym : q.yp, pm);
    fp_mul<F>(c, p.T, q.t2d, pm);
    if (neg) {
        fp_zero(z);
        fp_sub<F>(c, z, c);
    }
    fp_mul<F>(d, p.Z, q.z2, pm);
    fp_sub<F>(e, b, a);
    fp_sub<F>(f, d, c);
    fp_add<F>(g, d, c);
    fp_add<F>(h, b, a);
    fp_mul<F>(p.X, e, f, pm);
    fp_mul<F>(p.Y, g, h, pm);
    fp_mul<F>(p.T, e, h, pm);
    fp_mul<F>(p.Z, f, g, pm);
}

// Full extended addition p += q.  9M.
template <class F> CPB_HD void te_add(TePoint& p, const TePoint& q, const u32* d2, const u32* pm) {
    TeNiels n;
    te_to_niels<F>(n, q, d2, pm);
    te_add_niels<F>(p, n, false, pm);
}

template <class F> CPB_HD void te_neg(TePoint& p) {
    u32 z[8];
    fp_zero(z);
    fp_sub<F>(p.X, z, p.X);
    fp_sub<F>(p.T, z, p.T);
}

template <class F> CPB_HD void te_from_affine(TePoint& p, const u32* x, const u32* y, const u32* pm) {
    fp_copy(p.X, x);
    fp_copy(p.Y, y);
    fp_one<F>(p.Z);
    fp_mul<F>(p.T, x, y, pm);
}

// (X : Y : Z) -> affine (x, y), one Fermat inversion.
template <class F> CPB_HD void te_to_affine(u32* x, u32* y, const TePoint& p, const u32* pm) {
    u32 zi[8];
    fp_inv<F>(zi, p.Z, pm);
    fp_mul<F>(x, p.X, zi, pm);
    fp_mul<F>(y, p.Y, zi, pm);
}

// Montgomery -> canonical integer (multiply by 1).
template <class F> CPB_HD void fp_to_canonical(u32* r, const u32* a, const u32* pm) {
    u32 one[8];
    fp_zero(one);
    one[0] = 1;
    fp_mul<F>(r, a, one, pm);
}

// a > b as 256-bit integers
CPB_HD bool u256_gt(const u32* a, const u32* b) {
    int r = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) r = a[i] > b[i] ? 1 : a[i] < b[i] ? -1 : r;
    return r > 0;
}

// Compressed serialisation of an affine point (ark-serialize 0.4, *dep*; same rule as cpb_point_serialize): 32-byte LE
// canonical y, bit 7 of the last byte set when x > -x.  out = 8 little-endian words.
template <class F> CPB_HD void te_compress(u32* out, const u32* x, const u32* y, const u32* pm) {
    u32 xc[8], nx[8], z[8];
    fp_to_canonical<F>(xc, x, pm);
    fp_zero(z);
    fp_sub<F>(nx, z, xc);                                // q - x, or 0 for x = 0
    fp_to_canonical<F>(out, y, pm);
    if (u256_gt(xc, nx)) out[7] |= 0x80000000u;
}

// ark-ff 0.4 `Fp::from_random_bytes` on a 32-byte digest (*dep*): the LE integer with every bit at or above
// MODULUS_BIT_SIZE cleared; None (false) when that value is >= the modulus.  On success `mont` = the element.
template <class S> CPB_HD bool fr_from_random_bytes(u32* mont, const u32* digest, const u32* sm) {
    u32 v[8], r2[8];
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const int lo = 32 * i;
        v[i] = lo + 32 <= S::BITS ? digest[i] : lo >= S::BITS ? 0u : digest[i] & ((1u << (S::BITS - lo)) - 1u);
    }
    u32 pmod[8];
#pragma unroll
    for (int i = 0; i < 8; i++) pmod[i] = S::P(i);
    if (!u256_gt(pmod, v)) return false;
#pragma unroll
    for (int i = 0; i < 8; i++) r2[i] = S::R2(i);
    fp_mul<S>(mont, v, r2, sm);
    return true;
}

CPB_HD u32 bitrev8(u32 b) {
    b = ((b & 0xF0u) >> 4) | ((b & 0x0Fu) << 4);
    b = ((b & 0xCCu) >> 2) | ((b & 0x33u) << 2);
    return ((b & 0xAAu) >> 1) | ((b & 0x55u) << 1);
}

// ---- variable-base scalar multiplication ------------------------------------------------------------------------------
// Signed 4-bit windows (Booth recoding): with n_k the k-th nibble of the scalar and b_k its top bit,
// digit_k = n_k - 16 b_k + b_{k-1} lies in [-8, 8] and sum_k digit_k 16^k equals the scalar (the b terms telescope; one
// extra top digit b_{K-1}).  Each digit depends on two adjacent nibbles only, so the digits are produced left to right
// straight from the scalar, with no recoding pass and no digit array.  Table: 0P..8P in Niels form (0P = identity keeps
// the loop free of branches), read with a data-dependent index: 9 x 128 B per thread in local memory.
// A scalar is a nibble source: `nibble(k)` for k < `nibbles()`.
constexpr int kVarWindow = 4;
constexpr int kVarTable = 9;

template <class F, class Scalar>
CPB_HD void te_mul_var(TePoint& acc, const u32* bx, const u32* by, const Scalar& s, const u32* d2, const u32* pm) {
    TeNiels tab[kVarTable];
    TePoint p, q;
    te_identity<F>(q);
    te_to_niels<F>(tab[0], q, d2, pm);
    te_from_affine<F>(p, bx, by, pm);
    te_to_niels<F>(tab[1], p, d2, pm);
    q = p;
#pragma unroll 1
    for (int j = 2; j < kVarTable; j++) {                // jP = (j-1)P + P
        te_add_niels<F>(q, tab[1], false, pm);
        te_to_niels<F>(tab[j], q, d2, pm);
    }
    const int K = s.nibbles();
    auto digit = [&](int k) -> int {                     // n_k - 16 b_k + b_{k-1}
        const int n = k < K ? (int)s.nibble(k) : 0;
        const int lo = k > 0 ? (int)(s.nibble(k - 1) >> 3) : 0;
        return n - ((n >> 3) << 4) + lo;
    };
    te_identity<F>(acc);
#pragma unroll 1
    for (int k = K; k >= 0; k--) {
        if (k != K)
            for (int i = 0; i < kVarWindow; i++) te_dbl<F>(acc, pm);
        const int dg = digit(k);
        const int ad = dg < 0 ? -dg : dg;
        te_add_niels<F>(acc, tab[ad], dg < 0, pm);
    }
}

// A canonical integer of 8 LE words (up to 256 bits).
struct ScalarWords {
    const u32* w;
    int n;                                               // nibbles used: 64 for 256 bits, 63 for scalars below 2^252
    CPB_HD int nibbles() const { return n; }
    CPB_HD u32 nibble(int k) const { return (w[k >> 3] >> (4 * (k & 7))) & 15u; }
};

// The integer sum_b bitrev8(bytes[b]) 2^(8b) of a byte string (R/signature/schnorr/mod.rs:185-194 `bytes_to_bits` read as
// little-endian bits), of any length.
struct ScalarBitrevBytes {
    const uint8_t* p;
    u64 len;
    CPB_HD int nibbles() const { return (int)(2 * len); }
    CPB_HD u32 nibble(int k) const { return (bitrev8(p[k >> 1]) >> (4 * (k & 1))) & 15u; }
};

}  // namespace cpb
