// pedersen.cuh -- twisted-Edwards group arithmetic and the bit-selected fixed-base sum behind
// crh::pedersen::CRH::evaluate (R/crh/pedersen/mod.rs:76-129) and
// commitment::pedersen::Commitment::commit (R/commitment/pedersen/mod.rs:62-105).
//
// The reference walks the input bit by bit and adds generators[w][j] (projective +=) when the bit
// is set.  A group element has one affine representative, so any evaluation order gives the same
// output; here the flattened generator list is cut into chunks of 8 consecutive bits and each
// chunk's 256 subset sums are tabulated once per context (on the GPU, k_pedersen_table).  A hash is
// then one table lookup + one mixed addition per input BYTE: 7 field multiplications per 8 bits
// instead of ~9 per set bit.  No assumption is made about the generators (the reference's
// Parameters.generators is a public field, :28-31): the table is built from whatever points the
// caller supplies.
//
// Curve: a*x^2 + y^2 = 1 + d*x^2*y^2 with a = -1 (Jubjub / ed-on-bls12-377).  Points are kept in
// extended coordinates (X:Y:Z:T), x=X/Z, y=Y/Z, T=XY/Z; table entries are "affine Niels"
// (y+x, y-x, 2d*x*y).  The addition below is the unified a=-1 law (Hisil-Wong-Carter-Dawson 2008,
// sec. 3.1): complete when a is a square and d a non-square, i.e. valid for doubling, inverses,
// the identity and low-order points alike (checked against the affine oracle in tests).
#pragma once
#include "fp.cuh"

namespace cpb {

struct TePoint {
    u32 X[8], Y[8], Z[8], T[8];
};

template <class F> CPB_HD void te_identity(TePoint& p) {
    fp_zero(p.X);
    fp_one<F>(p.Y);
    fp_one<F>(p.Z);
    fp_zero(p.T);
}

// p += (yp, ym, t2d) where the entry is (y+x, y-x, 2d*x*y) of an affine point.  7M.
template <class F> CPB_HD void te_madd(TePoint& p, const u32* yp, const u32* ym, const u32* t2d, const u32* pm) {
    u32 a[8], b[8], c[8], d[8], e[8], f[8], g[8], h[8];
    fp_sub<F>(a, p.Y, p.X);
    fp_mul<F>(a, a, ym, pm);
    fp_add<F>(b, p.Y, p.X);
    fp_mul<F>(b, b, yp, pm);
    fp_mul<F>(c, p.T, t2d, pm);
    fp_add<F>(d, p.Z, p.Z);
    fp_sub<F>(e, b, a);
    fp_sub<F>(f, d, c);
    fp_add<F>(g, d, c);
    fp_add<F>(h, b, a);
    fp_mul<F>(p.X, e, f, pm);
    fp_mul<F>(p.Y, g, h, pm);
    fp_mul<F>(p.T, e, h, pm);
    fp_mul<F>(p.Z, f, g, pm);
}

// affine (x, y) -> Niels entry; d2 = 2d (Montgomery).
template <class F>
CPB_HD void te_niels(u32* yp, u32* ym, u32* t2d, const u32* x, const u32* y, const u32* d2, const u32* pm) {
    u32 t[8];
    fp_add<F>(yp, y, x);
    fp_sub<F>(ym, y, x);
    fp_mul<F>(t, x, y, pm);
    fp_mul<F>(t2d, t, d2, pm);
}

// a*x^2 + y^2 == 1 + d*x^2*y^2 with a = -1
template <class F> CPB_HD bool te_on_curve(const u32* x, const u32* y, const u32* d, const u32* pm) {
    u32 xx[8], yy[8], l[8], r[8], one[8];
    fp_sqr<F>(xx, x, pm);
    fp_sqr<F>(yy, y, pm);
    fp_sub<F>(l, yy, xx);
    fp_mul<F>(r, xx, yy, pm);
    fp_mul<F>(r, r, d, pm);
    fp_one<F>(one);
    fp_add<F>(r, r, one);
    return fp_eq(l, r);
}

// Table index of lookup c of a `len`-byte message at `cb` bits per lookup (cb <= 22): bits [c cb, (c + 1) cb) of the message,
// zero beyond len, little-endian -- up to four bytes, the value k_pedersen_hash_gather computes (for cb = 8, byte c).
CPB_HD u32 te_lookup_value(const uint8_t* msg, long len, int c, int cb) {
    const long bit = (long)c * cb, byte = bit >> 3;
    u64 v = 0;
#pragma unroll
    for (int k = 0; k < 4; k++)
        if (byte + k < len) v |= (u64)msg[byte + k] << (8 * k);
    return (u32)(v >> (bit & 7)) & ((1u << cb) - 1u);
}

// One lane's share of a hash split over `lanes` lanes: the mixed additions of lookups c = lane, lane + lanes, ... < n_chunks, from
// the identity.  entry(c, value, yp, ym, t2d) fetches the table entry.  The lanes' sums are then added in any order (the group is
// abelian): the warp kernel of the Pedersen-node update (cpb_merkle_update_pedersen.cu) reduces them with shuffles and te_add.
template <class F, class Entry>
CPB_HD void te_lane_sum(TePoint& acc, const uint8_t* msg, long len, int cb, int n_chunks, int lane, int lanes, Entry&& entry, const u32* pm) {
    te_identity<F>(acc);
#pragma unroll 1
    for (int c = lane; c < n_chunks; c += lanes) {
        u32 yp[8], ym[8], t2d[8];
        entry(c, te_lookup_value(msg, len, c, cb), yp, ym, t2d);
        te_madd<F>(acc, yp, ym, t2d, pm);
    }
}

// TwoToOneCRH::compress input of one node (R/crh/pedersen/mod.rs:187-197): the two children (affine x, y in Montgomery form)
// serialised uncompressed -- canonical little-endian x_l || y_l || x_r || y_r, 32 words.  The same bytes as k_points_to_bytes
// (cpb_pedersen.cu) writes for the build.
template <class F> CPB_HD void te_node_row(u32* row, const u32* left, const u32* right) {
    u32 pm[8], one[8], a[8];
    fp_modulus<F>(pm);
    fp_zero(one);
    one[0] = 1;
#pragma unroll 1
    for (int j = 0; j < 4; j++) {
        ld_elem(a, (j < 2 ? left : right) + 8 * (j & 1));
        fp_mul<F>(a, a, one, pm);
        st_elem(row + 8 * j, a);
    }
}

}  // namespace cpb
