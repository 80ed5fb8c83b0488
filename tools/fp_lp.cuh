// fp_lp.cuh -- PROTOTYPE (not used by the library): LIMB-PARALLEL 256-bit Montgomery arithmetic, one field element
// per 8 lanes of a warp, lane g holds limb g -- the "one warp per permutation, warp-shuffle" mapping BASELINE.json's
// north_star sketches.  tools/ubench_lp.cu checks it bit for bit against csrc/fp.cuh and times it: about 25
// dependent shuffle / ballot steps per multiplication replace the multiplier-pipe time they save.  Kept as the record of
// that experiment.
//
// Idea: the small levels of a Merkle tree are bound by the dependent chain of multiplications, and a lone warp needs
// one fp_mul (136 IMAD.WIDE at 4 issue cycles each on ONE scheduler, fp.cuh).  Spreading the 64 limb products of
// a multiplication over 8 lanes makes the chain short instead: every lane does 8 wide multiply-adds per 256x256 product,
// and carries are resolved across lanes a few times per multiplication instead of once per instruction.
//
// Algorithm (product scanning, no interleaving -- the word-by-word CIOS form needs two dependent shuffles per reduction
// step): lane g accumulates column g (low half) and column g+8 (high half) of a 16-limb number in three words each
// (c0 + c1*2^32 + c2*2^64; c2 counts carries), from 8 products a_k * b_((g-k) mod 8):
//     X  = a*b                                  8 products per lane
//     q  = (X mod 2^256) * (-p^-1) mod 2^256    <= 8 products per lane, needs the low half of X as proper limbs (1 resolve)
//     X += q*p                                  8 products per lane, on top of the unresolved accumulators
//     r  = X / 2^256                            resolve (low half: only its carry-out matters), then r >= p ? r - p : r
// `resolve` turns redundant columns into limbs: neighbours' c1 / c2 words by shuffle, the small carries by one more shuffle,
// and the remaining 0/1 ripple by a carry-lookahead on ballot masks (generate = my addition overflowed, propagate = my limb
// is all ones; the carries INTO each lane are (A + B) ^ A ^ B for A = G | P, B = G, per 8-lane group).
// Values are canonical (< p) Montgomery residues, bit-identical to fp.cuh's (tests: lp self-test kernel against fp_mul /
// fp_add / fp_sub on pattern-limb operands -- limbs drawn from {0, 1, 2^32-1, 2^31, random} so that every carry path is hit
// constantly -- and the tree-top parity tests).
//
// All 32 lanes of the warp must execute every function (full-mask shuffles / ballots): 4 elements per warp.
#pragma once
#include "../crypto_primitives_b200/csrc/ptx.cuh"

namespace cpb {

#if defined(__CUDACC__)

struct LpLane {
    u32 p;        // limb g of the modulus
    u32 ninv;     // limb g of -p^-1 mod 2^256
    int g;        // lane & 7
    int sh;       // 8 * (lane >> 3): position of this group's byte in a ballot mask
};

struct LpCol {
    u32 c0, c1, c2;
};

__device__ __forceinline__ u32 lp_shfl(u32 v, int src) { return __shfl_sync(0xffffffffu, v, src, 8); }

// (L or H) += a * b, L when to_low
__device__ __forceinline__ void lp_mad(LpCol& L, LpCol& H, u32 a, u32 b, bool to_low) {
    u32 lo, hi;
    asm("mul.lo.u32 %0, %2, %3; mul.hi.u32 %1, %2, %3;" : "=r"(lo), "=r"(hi) : "r"(a), "r"(b));
    const u32 m = to_low ? 0xffffffffu : 0u;
    asm("add.cc.u32 %0, %0, %3; addc.cc.u32 %1, %1, %4; addc.u32 %2, %2, 0;" : "+r"(L.c0), "+r"(L.c1), "+r"(L.c2) : "r"(lo & m), "r"(hi & m));
    asm("add.cc.u32 %0, %0, %3; addc.cc.u32 %1, %1, %4; addc.u32 %2, %2, 0;" : "+r"(H.c0), "+r"(H.c1), "+r"(H.c2) : "r"(lo & ~m), "r"(hi & ~m));
}

// X(L,H) += a * b for lane-distributed a, b (8 products per lane)
__device__ __forceinline__ void lp_mul_acc(LpCol& L, LpCol& H, u32 a, u32 b, const LpLane& C) {
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const u32 ak = lp_shfl(a, k);
        const u32 bk = lp_shfl(b, (C.g - k) & 7);
        lp_mad(L, H, ak, bk, k <= C.g);
    }
}
// low half only: L += (a * b) mod 2^256 columns
__device__ __forceinline__ void lp_mul_lo_acc(LpCol& L, u32 a, u32 b, const LpLane& C) {
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const u32 ak = lp_shfl(a, k);
        const u32 bk = lp_shfl(b, (C.g - k) & 7);
        u32 lo, hi;
        asm("mul.lo.u32 %0, %2, %3; mul.hi.u32 %1, %2, %3;" : "=r"(lo), "=r"(hi) : "r"(ak), "r"(bk));
        const u32 m = k <= C.g ? 0xffffffffu : 0u;
        asm("add.cc.u32 %0, %0, %3; addc.cc.u32 %1, %1, %4; addc.u32 %2, %2, 0;" : "+r"(L.c0), "+r"(L.c1), "+r"(L.c2) : "r"(lo & m), "r"(hi & m));
    }
}

// Carries INTO every lane of an 8-lane chain, given per lane: gen = "my limb addition overflowed" and prop = "my limb is all
// ones" (mutually exclusive), and a carry into lane 0.  Returns (carry into my lane, carry out of lane 7).
__device__ __forceinline__ void lp_lookahead(bool gen, bool prop, u32 cin0, const LpLane& C, u32& cin, u32& cout) {
    const u32 G = (__ballot_sync(0xffffffffu, gen) >> C.sh) & 0xffu;
    const u32 P = (__ballot_sync(0xffffffffu, prop) >> C.sh) & 0xffu;
    const u32 A = G | P, B = G;
    const u32 S = A + B + cin0;
    const u32 X = S ^ A ^ B;             // bit j: carry into lane j; bit 8: carry out of the group
    cin = (X >> C.g) & 1u;
    cout = (X >> 8) & 1u;
}

// Columns (c0, c1, c2) of one 8-lane half -> proper limbs.  in1 / in2: what enters limb 0 and limb 1 of this half from below
// (the c1 / c2 spill of the half underneath, already shuffled into lanes 0 and 1 by the caller: pass per lane the value that
// must be added to ITS limb from outside the half, 0 elsewhere), kin: small carry into limb 0, cin0: 0/1 ripple into limb 0.
// Returns the limb; kout = small carry out of limb 7 (lane 7's k), cout = 0/1 ripple carry out of limb 7.
__device__ __forceinline__ u32 lp_resolve_half(const LpCol& c, u32 ext1, u32 ext2, u32 kin, u32 cin0, const LpLane& C, u32& kout, u32& cout) {
    const u32 up1 = lp_shfl(c.c1, (C.g - 1) & 7);
    const u32 up2 = lp_shfl(c.c2, (C.g - 2) & 7);
    const u32 t1 = C.g >= 1 ? up1 : ext1;          // lane 0 takes the spill of the half below
    const u32 t2 = C.g >= 2 ? up2 : ext2;          // lanes 0, 1 likewise
    u32 w, k;
    asm("add.cc.u32 %0, %2, %3; addc.u32 %1, 0, 0;" : "=r"(w), "=r"(k) : "r"(c.c0), "r"(t1));
    asm("add.cc.u32 %0, %0, %2; addc.u32 %1, %1, 0;" : "+r"(w), "+r"(k) : "r"(t2));
    // small carries one lane up, then the 0/1 ripple by look-ahead
    const u32 kup = lp_shfl(k, (C.g - 1) & 7);
    const u32 kadd = C.g >= 1 ? kup : kin;
    u32 s, g1;
    asm("add.cc.u32 %0, %2, %3; addc.u32 %1, 0, 0;" : "=r"(s), "=r"(g1) : "r"(w), "r"(kadd));
    u32 cin;
    lp_lookahead(g1 != 0, s == 0xffffffffu, cin0, C, cin, cout);
    kout = lp_shfl(k, 7);
    return s + cin;
}

// r = (a + b) mod p, r = (a - b) mod p on canonical inputs
__device__ __forceinline__ u32 lp_cond_sub_p(u32 r, u32 carry_top, const LpLane& C) {
    // r (plus carry_top * 2^256) >= p ?  compare by masks: highest differing limb decides
    const u32 GT = (__ballot_sync(0xffffffffu, r > C.p) >> C.sh) & 0xffu;
    const u32 LT = (__ballot_sync(0xffffffffu, r < C.p) >> C.sh) & 0xffu;
    const bool ge = carry_top != 0 || GT >= LT;            // GT > LT: greater; both 0: equal
    // d = r - p with borrow look-ahead: generate = r_g < p_g, propagate = r_g == p_g
    const u32 d = r - C.p;
    const u32 A = LT | (~(GT | LT) & 0xffu), B = LT;
    const u32 S = A + B;
    const u32 X = S ^ A ^ B;
    const u32 bin = (X >> C.g) & 1u;
    return ge ? d - bin : r;
}
__device__ __forceinline__ u32 lp_add(u32 a, u32 b, const LpLane& C) {
    u32 s, g1;
    asm("add.cc.u32 %0, %2, %3; addc.u32 %1, 0, 0;" : "=r"(s), "=r"(g1) : "r"(a), "r"(b));
    u32 cin, cout;
    lp_lookahead(g1 != 0, s == 0xffffffffu, 0u, C, cin, cout);
    return lp_cond_sub_p(s + cin, cout, C);
}
__device__ __forceinline__ u32 lp_sub(u32 a, u32 b, const LpLane& C) {
    // a - b, + p when negative
    const u32 GT = (__ballot_sync(0xffffffffu, a > b) >> C.sh) & 0xffu;
    const u32 LT = (__ballot_sync(0xffffffffu, a < b) >> C.sh) & 0xffu;
    const u32 A = LT | (~(GT | LT) & 0xffu), B = LT;
    const u32 X = (A + B) ^ A ^ B;
    const u32 d = a - b - ((X >> C.g) & 1u);
    const bool neg = LT > GT;
    // + p
    u32 s, g1;
    asm("add.cc.u32 %0, %2, %3; addc.u32 %1, 0, 0;" : "=r"(s), "=r"(g1) : "r"(d), "r"(C.p));
    u32 cin, cout;
    lp_lookahead(g1 != 0, s == 0xffffffffu, 0u, C, cin, cout);
    return neg ? s + cin : d;
}

// Montgomery reduction of the accumulators X(L,H) (+ optional addend E: a canonical element added to the RESULT, i.e.
// E * 2^256 added to X): returns limb g of  X / 2^256 + E  mod p.  Needs X / 2^256 + E < 2^256 (true for sums of at most
// 3 products of canonical values plus one canonical addend when 5p < 2^256, else callers add separately).
__device__ __forceinline__ u32 lp_redc(LpCol L, LpCol H, const LpLane& C) {
    // low half of X as limbs
    u32 k0, c0;
    const u32 xlo = lp_resolve_half(L, 0u, 0u, 0u, 0u, C, k0, c0);
    // q = xlo * ninv mod 2^256
    LpCol Q = {0u, 0u, 0u};
    lp_mul_lo_acc(Q, xlo, C.ninv, C);
    u32 kq, cq;
    const u32 q = lp_resolve_half(Q, 0u, 0u, 0u, 0u, C, kq, cq);
    // X += q * p
    lp_mul_acc(L, H, q, C.p, C);
    // low half: all limbs are zero by construction, only what leaves it matters
    u32 kL, cL;
    (void)lp_resolve_half(L, 0u, 0u, 0u, 0u, C, kL, cL);
    // spill of the low half into limbs 8 and 9: c1 of column 7 and c2 of column 6 -> limb 8; c2 of column 7 -> limb 9
    const u32 l1_7 = lp_shfl(L.c1, 7), l2_6 = lp_shfl(L.c2, 6), l2_7 = lp_shfl(L.c2, 7);
    // lane 0 of the high half receives l1_7 (as its "c1 from below") and l2_6 (as "c2 from two below"); lane 1 receives l2_7
    u32 kH, cH;
    const u32 r = lp_resolve_half(H, l1_7, C.g == 0 ? l2_6 : l2_7, kL, cL, C, kH, cH);
    return lp_cond_sub_p(r, kH + cH, C);
}

__device__ __forceinline__ u32 lp_mul(u32 a, u32 b, const LpLane& C) {
    LpCol L = {0u, 0u, 0u}, H = {0u, 0u, 0u};
    lp_mul_acc(L, H, a, b, C);
    return lp_redc(L, H, C);
}

#endif  // __CUDACC__

}  // namespace cpb
