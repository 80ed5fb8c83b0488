// poseidon_tc.cuh -- products by schedule constants on the tensor cores (u8 IMMA): the partial rounds' linear layer of the
// BN254 Fr t = 3 one-permutation hash kernel (k_poseidon_crh_tc, pos_permute_split with TC).
//
// Byte-digit tables.  For a constant c (Montgomery form) K8_i(c) = c * 2^(8i) * 2^32 / R mod p, i = 0..31, canonical plain
// integers.  A sum of products sum_j a_j * c_j over operands a_j < 2^256 is then a u8 GEMM over the operands' bytes:
//   V = sum_n C[n] * 2^(8n),  C[n] = sum_{j,i} byte_i(a_j) * byte_n(K8_i(c_j))  ==  (sum_j a_j * c_j / R) * 2^32  (mod p),
// every column sum C[n] <= 32 NT * 255^2 < 2^23 (s32 accumulators), V < 32 NT * 255 * p, and ONE Montgomery row (8 wide
// multiply-adds) divides by 2^32: result (V + m*p) / 2^32 < p * (1 + 32 NT * 255 * 2^-32).  A unit addend y enters as y * 2^32.
// Across a warp's 32 hashes A is 32 x 32NT (one row of operand bytes per lane) and B (32NT x 32, the table) is shared by every
// hash: mma.m16n8k32.row.col.s32.u8.u8.s32 over 2 m-tiles, 4 n-tiles and NT k-chunks.  A partial round (t = 3) needs
//   a' = gamma*y + alpha*a + beta*s2   (NT = 3, 24 IMMA)   and   s2' = s2 + v*y   (NT = 1, 8 IMMA).
// The same product reduces the S-box's products (tc_redc): for T = a*b = T_lo + R*T_hi, T/R == T_hi + T_lo * R^-1 (mod p), and
// T_lo * R^-1 is a product by the constant R^-1, through the byte-digit table of the plain constant 1 (K8_i = 2^(8i) * 2^32 / R).
// A full round's dense rows (tc_full_round) are NT = 3 products of the three S-box outputs, one per row, brought to [0, p) by one
// conditional subtraction.
// Every bound is checked with exact rationals in tests/test_poseidon_tc.py, tests/test_poseidon_tc_redc.py and
// tests/test_poseidon_tc_full.py.
#pragma once
#include "fp.cuh"

namespace cpb {

constexpr int kTcTerms = 4;                              // k-chunks of a round's table: gamma, alpha, beta, then v
constexpr int kTcRoundWords = 4 * kTcTerms * 32 * 2;     // u32 per partial round: [n-tile][k-chunk][lane][b0, b1], 4 KB
constexpr int kTcStageStride = 28;                       // u32 per staged row: 96 operand bytes + 16 B so ldmatrix rows miss
                                                         // each other's banks
constexpr int kTcCbufWords = 32 * 16;                    // C buffer: 32 rows of 16 packed column pairs
constexpr int kTcWarpWords = 32 * kTcStageStride + kTcCbufWords;   // per-warp shared memory, 5632 B
constexpr int kTcRinvWords = 4 * 32 * 2;                 // the R^-1 table: one constant, [n-tile][lane][b0, b1], 1 KB
constexpr int kTcRowWords = 4 * 3 * 32 * 2;              // a full-round row's table: 3 constants, [n-tile][k-chunk][lane][b0, b1], 3 KB
constexpr int kTcFullRows = 10;                          // the rows of M, Mpre, Mpost (3 each), then the entry row

// The per-CTA ring of the partial rounds' tables (k_poseidon_crh_tc).  The CTA's four warps run the same partial rounds in the same
// order, batch after batch, so they share one shared-memory copy of each round's table instead of each fetching it from L2.  Round
// g of the CTA -- counted over all of its batches, so g mod rp is the partial round -- reads slot g mod kTcRingSlots once that
// slot's "full" mbarrier has completed phase g / kTcRingSlots (one bulk copy of kTcRoundWords, verbatim from P.tab8).  A warp
// releases round g when its last read of the slot is done; the kTcRingWarps-th release (a per-slot count) refills the slot with
// round g + kTcRingSlots's table, unless the CTA runs no such round.  Two slots keep the CTA's shared memory under 6 CTAs per SM.
constexpr int kTcRingSlots = 2;
constexpr int kTcRingWarps = 4;                          // warps per CTA (kBlock / 32) that read every slot
CPB_HD int tc_ring_slot(unsigned g) { return (int)(g % kTcRingSlots); }
CPB_HD unsigned tc_ring_parity(unsigned g) { return (g / kTcRingSlots) & 1u; }
// The partial round whose table the refill after partial round k brings: the one kTcRingSlots rounds later, wrapping into the
// next hash of the batch loop.
CPB_HD int tc_ring_next(int k, int rp) { return (k + kTcRingSlots) % rp; }
struct TcRing {
    u32* slots;                    // kTcRingSlots x kTcRoundWords, shared memory
    unsigned long long* full;      // kTcRingSlots mbarriers, arrival count 1 (the refill's expect_tx), completed by the copy
    unsigned* released;            // kTcRingSlots counters of releases; a multiple of kTcRingWarps when every warp is done
    const u32* src;                // the partial rounds' tables (P.tab8)
    int rp;
    unsigned g;                    // this warp's next round
    unsigned g_end;                // the CTA's number of rounds: batches x rp (below 2^32 for any n the grid can stride over)
};

// Fragment maps of mma.m16n8k32 with .u8 operands (PTX ISA, "Matrix Fragments for mma.m16n8k32"), g = lane >> 2, t = lane & 3:
//   A (16 x 32, .row): register r (0..3), byte q  ->  row g + 8 (r & 1),  k 4t + q + 16 (r >> 1)
//   B (32 x 8, .col):  register r (0..1), byte q  ->  k 4t + q + 16 r,    column g
//   C (16 x 8, .s32):  register r (0..3)          ->  row g + 8 (r >> 1), column 2t + (r & 1)
CPB_HD int tc_a_row(int lane, int r) { return (lane >> 2) + 8 * (r & 1); }
CPB_HD int tc_a_k(int lane, int r, int q) { return 4 * (lane & 3) + q + 16 * (r >> 1); }
CPB_HD int tc_b_k(int lane, int r, int q) { return 4 * (lane & 3) + q + 16 * r; }
CPB_HD int tc_b_col(int lane) { return lane >> 2; }
CPB_HD int tc_c_row(int lane, int r) { return (lane >> 2) + 8 * (r >> 1); }
CPB_HD int tc_c_col(int lane, int r) { return 2 * (lane & 3) + (r & 1); }
// ldmatrix.x4: lane supplies the address of row lane & 7 of matrix lane >> 3, and destination register m receives row g, bytes
// 4t .. 4t+3 of matrix m.  Matrix m is rows 8 (m & 1) .. +7, bytes 16 (m >> 1) .. +15 of the 16 x 32 tile, so register m is A's.
CPB_HD int tc_ldsm_row(int lane) { return (lane & 7) + 8 * ((lane >> 3) & 1); }
CPB_HD int tc_ldsm_half(int lane) { return lane >> 4; }
// u32 index, in a table of `terms` constants (a partial round's kTcTerms, a full-round row's 3, or the R^-1 table's one), of lane's
// B register r for n-tile nt and k-chunk kc (host::tc_tables, host::tc_full_tables and host::tc_rinv_table write, the kernel reads).
CPB_HD int tc_tab_word(int nt, int kc, int lane, int r, int terms = kTcTerms) { return ((nt * terms + kc) * 32 + lane) * 2 + r; }
// C buffer: row `row` keeps the packed column pairs of thread-in-group t (one word per n-tile) in 16-byte chunk
// t ^ ((row >> 1) & 3), so that the 128-bit stores by fragment and the 128-bit loads by row are both free of bank conflicts.
CPB_HD int tc_cbuf_chunk(int row, int t) { return t ^ ((row >> 1) & 3); }

// V = sum_m h[m] * 2^(16 m) (+ y * 2^32 when U), then one Montgomery row: r = (V + m*p) / 2^32, not reduced.
// h[m] < 2^31 (a packed column pair C[2m] + 256 C[2m+1]); V + m*p < 2^288 (the caller's bound), y + (V >> 32) < 2^256.
// V is held as E + 2^32 * O (the accumulators of redc_row): E = sum_L h[2L] 2^(32L) + (h[1] << 16 mod 2^32), which cannot carry
// out (h[14] < 2^31), and O[L] = limb L + 1 of sum_L h[2L+1] 2^(32L+16), a funnel shift of two packed values.
template <class F, bool U> CPB_HD void tc_finish(u32* r, const u32 (&h)[16], const u32* y, const u32* pm) {
    u32 E[8], O[8];
    E[0] = add_cc(h[0], h[1] << 16);
#pragma unroll
    for (int L = 1; L < 7; L++) E[L] = addc_cc(h[2 * L], 0u);
    E[7] = addc(h[14], 0u);
#pragma unroll
    for (int L = 0; L < 7; L++) O[L] = (h[2 * L + 3] << 16) | (h[2 * L + 1] >> 16);
    O[7] = h[15] >> 16;
    if (U) {
        O[0] = add_cc(O[0], y[0]);
#pragma unroll
        for (int L = 1; L < 7; L++) O[L] = addc_cc(O[L], y[L]);
        O[7] = addc(O[7], y[7]);
    }
    detail::redc_row<F>(E, O, pm);
    r[0] = add_cc(O[0], E[1]);
#pragma unroll
    for (int i = 1; i < 7; i++) r[i] = addc_cc(O[i], E[i + 1]);
    r[7] = addc(O[7], 0u);
}

#if defined(__CUDACC__)
CPB_D unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}

// Bulk copy of partial round k's table into `slot`, completing the slot's next phase (one thread).  The proxy fence orders the
// warps' reads of the slot, which the release count has ordered before this thread, before the copy's writes.
CPB_D void tc_ring_fill(const TcRing& R, int slot, int k) {
    const unsigned mb = (unsigned)__cvta_generic_to_shared(R.full + slot);
    const unsigned dst = (unsigned)__cvta_generic_to_shared(R.slots + slot * kTcRoundWords);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mb), "r"(kTcRoundWords * 4) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
                 "l"(R.src + (size_t)k * kTcRoundWords), "r"(kTcRoundWords * 4), "r"(mb)
                 : "memory");
}

// This warp's round R.g: waits (every lane) until its table has landed and returns the slot.  Bounded: trap after ~4 s.
CPB_D const u32* tc_ring_acquire(const TcRing& R) {
    const int slot = tc_ring_slot(R.g);
    const unsigned mb = (unsigned)__cvta_generic_to_shared(R.full + slot), par = tc_ring_parity(R.g);
    unsigned done = 0;
    unsigned long long t0 = 0;
    for (;;) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done) : "r"(mb), "r"(par) : "memory");
        if (done) break;
        if (t0 == 0) t0 = globaltimer_ns();
        else if (globaltimer_ns() - t0 > 4000000000ull) __trap();
    }
    return R.slots + slot * kTcRoundWords;
}

// This warp is done with round R.g (partial round k of its hash): lane 0 counts the release, and the last of the CTA's warps
// refills the slot with round R.g + kTcRingSlots's table.  The block fences make the count a release / acquire pair, so every
// warp's reads of the slot come before the refill.
CPB_D void tc_ring_release(TcRing& R, int k) {
    __syncwarp();
    if ((threadIdx.x & 31) == 0) {
        const int slot = tc_ring_slot(R.g);
        __threadfence_block();
        if (atomicAdd(R.released + slot, 1u) % kTcRingWarps == kTcRingWarps - 1 && R.g + kTcRingSlots < R.g_end) {
            __threadfence_block();
            tc_ring_fill(R, slot, tc_ring_next(k, R.rp));
        }
    }
    R.g++;
}
#endif

#if defined(__CUDA_ARCH__)
CPB_D void tc_ldsm_x4(u32 (&d)[4], const u32* smem) {
    const unsigned a = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(d[0]), "=r"(d[1]), "=r"(d[2]), "=r"(d[3]) : "r"(a) : "memory");
}
CPB_D void tc_mma(u32 (&c)[4], const u32 (&a)[4], uint2 b) {
    asm("mma.sync.aligned.m16n8k32.row.col.s32.u8.u8.s32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
        : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b.x), "r"(b.y));
}

// Where tc_output reads its B fragments: tables of NT constants in global memory through the read-only path (a full-round row's 3),
// or in shared memory (a partial round's kTcTerms in a slot of the ring, the R^-1 table's one).
template <int NT> struct TcTabGlobal {
    static constexpr int kTerms = NT;
    static CPB_D uint2 ld(const u32* p) { return __ldg(reinterpret_cast<const uint2*>(p)); }
};
template <int NT> struct TcTabShared {
    static constexpr int kTerms = NT;
    static CPB_D uint2 ld(const u32* p) { return *reinterpret_cast<const uint2*>(p); }
};

// One output for lane's hash: the GEMM over k-chunks KC0 .. KC0+NT-1 of the table (read through B) against the staged operands
// 0 .. NT-1, packed, moved to one row per lane through the C buffer, rebuilt and reduced by tc_finish.  Both m-tiles at once, so
// each B fragment is loaded once for two IMMA (DESIGN §4.2).  Every lane has read the stage when it returns.
template <class F, class B, int NT, int KC0, bool U>
CPB_D void tc_output(u32* r, const u32* stage, u32* cbuf, const u32* tab, int lane, const u32* y, const u32* pm) {
    const int g = lane >> 2, t = lane & 3;
    u32 a[2][NT][4];
#pragma unroll
    for (int mt = 0; mt < 2; mt++)
#pragma unroll
        for (int kc = 0; kc < NT; kc++)
            tc_ldsm_x4(a[mt][kc], stage + (16 * mt + tc_ldsm_row(lane)) * kTcStageStride + 8 * kc + 4 * tc_ldsm_half(lane));
    u32 pk[2][2][4];                                    // [m-tile][C row g / g + 8 of it][n-tile]
#pragma unroll
    for (int nt = 0; nt < 4; nt++) {
        u32 c[2][4] = {{0u, 0u, 0u, 0u}, {0u, 0u, 0u, 0u}};
#pragma unroll
        for (int kc = 0; kc < NT; kc++) {
            const uint2 b = B::ld(tab + tc_tab_word(nt, KC0 + kc, lane, 0, B::kTerms));   // one load for both m-tiles
            tc_mma(c[0], a[0][kc], b);
            tc_mma(c[1], a[1][kc], b);
        }
#pragma unroll
        for (int mt = 0; mt < 2; mt++) {
            pk[mt][0][nt] = c[mt][0] + (c[mt][1] << 8);  // columns 2t, 2t + 1: 16-bit digit 4 nt + t of the row's V
            pk[mt][1][nt] = c[mt][2] + (c[mt][3] << 8);
        }
    }
#pragma unroll
    for (int mt = 0; mt < 2; mt++)
#pragma unroll
        for (int u = 0; u < 2; u++) {
            const int row = 16 * mt + 8 * u + g;
            *reinterpret_cast<uint4*>(cbuf + 16 * row + 4 * tc_cbuf_chunk(row, t)) =
                make_uint4(pk[mt][u][0], pk[mt][u][1], pk[mt][u][2], pk[mt][u][3]);
        }
    __syncwarp();
    u32 h[16];
#pragma unroll
    for (int tt = 0; tt < 4; tt++) {
        const uint4 v = *reinterpret_cast<const uint4*>(cbuf + 16 * lane + 4 * tc_cbuf_chunk(lane, tt));
        h[tt] = v.x; h[4 + tt] = v.y; h[8 + tt] = v.z; h[12 + tt] = v.w;
    }
    __syncwarp();                                       // the buffer is free for the next output
    tc_finish<F, U>(r, h, y, pm);
}

// The partial round's products by constants for the 32 hashes of a converged warp, lane's hash in s = (y, a, s2):
//   an = gamma*y + alpha*a + beta*s2, below p * (1 + 3 * 255 * 2^-27) (the LAZY fp_dot_tab contract: not reduced);
//   s2 <- s2 + v*y for s2 in [0, 2p): below p * (3 + 255 * 2^-27) after the row, one conditional subtraction of 2p (WC).
// tab: this round's kTcRoundWords in shared memory (a slot of the ring), buf: the warp's kTcWarpWords of shared memory.
// Stages lane's three operands s[0..2] as its row of the A operand (bytes 32 j .. 32 j + 31: s[j]) for the warp's products.
CPB_D void tc_stage3(u32* stage, const u32 (&s)[3][8], int lane) {
#pragma unroll
    for (int j = 0; j < 3; j++) {
        *reinterpret_cast<uint4*>(stage + lane * kTcStageStride + 8 * j) = make_uint4(s[j][0], s[j][1], s[j][2], s[j][3]);
        *reinterpret_cast<uint4*>(stage + lane * kTcStageStride + 8 * j + 4) = make_uint4(s[j][4], s[j][5], s[j][6], s[j][7]);
    }
    __syncwarp();
}

template <class F> CPB_D void tc_partial_round(u32 (&an)[8], u32 (&s)[3][8], const u32* tab, u32* buf, const u32* pm) {
    const int lane = threadIdx.x & 31;
    u32* stage = buf;
    u32* cbuf = buf + 32 * kTcStageStride;
    tc_stage3(stage, s, lane);
    tc_output<F, TcTabShared<kTcTerms>, 3, 0, false>(an, stage, cbuf, tab, lane, nullptr, pm);
    u32 w[8];
    tc_output<F, TcTabShared<kTcTerms>, 1, 3, true>(w, stage, cbuf, tab, lane, s[2], pm);
    detail::reduce8<F, 1, 1>(w);
    fp_copy(s[2], w);
    __syncwarp();                                       // every lane has read the staged operands: the next round may restage
}

// A full round's dense rows for the 32 hashes of a converged warp, lane's S-box outputs in s (any values below 2^256, so the lazy
// outputs below 1.24p enter as they are): s[i] <- row_i . s, canonical, for every row i with bit i of need set, and zero for the
// others.  rows: the round matrix's three row tables, kTcRowWords apart (host::tc_full_tables); row1: the table row 1 reads (rows +
// kTcRowWords, or the entry row).  A row's product is below p * (1 + 3 * 255 * 2^-27) < 2p, so one conditional subtraction makes it
// canonical.  need must be the same in every lane.  buf: the warp's kTcWarpWords; the stage is free again when this returns.
template <class F> CPB_D void tc_full_round(u32 (&s)[3][8], const u32* rows, const u32* row1, unsigned need, u32* buf, const u32* pm) {
    const int lane = threadIdx.x & 31;
    tc_stage3(buf, s, lane);
#pragma unroll
    for (int i = 0; i < 3; i++) {
        if ((need >> i) & 1u) {
            tc_output<F, TcTabGlobal<3>, 3, 0, false>(s[i], buf, buf + 32 * kTcStageStride, i == 1 ? row1 : rows + i * kTcRowWords,
                                                      lane, nullptr, pm);
            fp_final_sub<F>(s[i]);
        } else {
            fp_zero(s[i]);
        }
    }
}

// r == T/R (mod p) for the 32 hashes of a converged warp, lane's 512-bit T (fp_sqr_wide, fp_mul_wide): T_lo * R^-1 on the tensor
// cores over the R^-1 table rinv (shared memory, host::tc_rinv_table), with T_hi as the unit addend of its reduction row.
//   r < T_hi + p * (1 + 32 * 255 * 2^-32) <= T/R + p * (1 + 32 * 255 * 2^-32), not reduced (the CIOS rows: below T/R + p).
// tc_finish needs T_hi + p * (1 + 2^-19) < 2^256.  buf: the warp's kTcWarpWords; the stage is free again when this returns.
template <class F> CPB_D void tc_redc(u32* r, const u32 (&T)[16], const u32* rinv, u32* buf, const u32* pm) {
    const int lane = threadIdx.x & 31;
    *reinterpret_cast<uint4*>(buf + lane * kTcStageStride) = make_uint4(T[0], T[1], T[2], T[3]);
    *reinterpret_cast<uint4*>(buf + lane * kTcStageStride + 4) = make_uint4(T[4], T[5], T[6], T[7]);
    __syncwarp();
    tc_output<F, TcTabShared<1>, 1, 0, true>(r, buf, buf + 32 * kTcStageStride, rinv, lane, T + 8, pm);
}
#endif

}  // namespace cpb
