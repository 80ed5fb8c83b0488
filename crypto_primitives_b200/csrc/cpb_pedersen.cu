// cpb_pedersen.cu -- CUDA kernels + C-ABI for Pedersen CRH / two-to-one / commitment over a
// twisted-Edwards curve and the Merkle builds that use them (include/cpb200.h).
//
// Kernels (sm_90a, integer pipe):
//   k_pedersen_table   once per context: 256 subset sums per 8-bit chunk of the flattened generator
//                      list, normalised to affine-Niels entries (96 B each).
//   k_pedersen_hash    one hash per thread: for every input byte, one table lookup + one 7M mixed
//                      addition; the chunk's 24 KB table slice is staged in shared memory by TMA
//                      bulk copies, double-buffered against the additions; output projective.
//   k_pedersen_normalise projective -> affine with one field inversion per 32 points (Montgomery's trick along
//                      each thread's own sequence of points).
//   k_points_to_bytes  serialize_uncompressed of child digests for TwoToOneCRH::compress
//                      (R/crh/pedersen/mod.rs:187-197, R/macros.rs:3-13): canonical x || y.
#include <vector>

#include "common.cuh"
#include "hostfp.hpp"
#include "pedersen.cuh"
#include "pedersen_internal.cuh"

namespace cpb {

constexpr int kPedBlock = 256;
constexpr int kEntryWords = 24;                    // 3 field elements
constexpr int kChunkWords = 256 * kEntryWords;     // one 8-bit chunk: 24576 B
constexpr unsigned kChunkBytes = kChunkWords * 4;
#ifndef CPB_PEDERSEN_CHUNK_BITS
#define CPB_PEDERSEN_CHUNK_BITS 8
#endif
constexpr int kDefaultChunkBits = CPB_PEDERSEN_CHUNK_BITS;

// consts layout (u32 words): [0..8) modulus limbs, [8..16) 2d (Montgomery), [16..24) d (Montgomery)
template <class F>
__global__ void __launch_bounds__(256)
k_pedersen_table(const u32* __restrict__ consts, const u32* __restrict__ gens_xy, int n_gens, int n_chunks, int chunk_bits,
                 u32* __restrict__ table, int zero) {
    long e = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= ((long)n_chunks << chunk_bits)) return;
    const int chunk = (int)(e >> chunk_bits), mask = (int)(e & ((1 << chunk_bits) - 1));
    const u32* ct = consts + (int)threadIdx.x * zero;
    u32 pm[8], d2[8];
    ld_elem(pm, ct);
    ld_elem(d2, ct + 8);
    TePoint acc;
    te_identity<F>(acc);
#pragma unroll 1
    for (int j = 0; j < chunk_bits; j++) {
        int g = chunk * chunk_bits + j;
        if (!((mask >> j) & 1) || g >= n_gens) continue;
        u32 x[8], y[8], yp[8], ym[8], t2d[8];
        ld_elem(x, gens_xy + 16 * (long)g);
        ld_elem(y, gens_xy + 16 * (long)g + 8);
        te_niels<F>(yp, ym, t2d, x, y, d2, pm);
        te_madd<F>(acc, yp, ym, t2d, pm);
    }
    // projective (X, Y, Z) into the entry's 96 bytes; k_pedersen_table_finish normalises in place
    u32* o = table + e * kEntryWords;
    st_elem(o, acc.X);
    st_elem(o + 8, acc.Y);
    st_elem(o + 16, acc.Z);
}

// Second pass of the table build: entries (X, Y, Z) -> affine-Niels (y+x, y-x, 2d*x*y), with ONE field inversion per
// kFinishBatch entries (Montgomery's trick along the thread's own sequence of entries; prefix products in local memory).
// The first version inverted per entry: 4.2 M Fermat inversions (~380 products each) for the 16-bit tables of a 4x256 window.
constexpr int kFinishBatch = 16;
template <class F>
__global__ void __launch_bounds__(128)
k_pedersen_table_finish(const u32* __restrict__ consts, u32* __restrict__ table, long n_entries, int zero) {
    const long stride = (n_entries + kFinishBatch - 1) / kFinishBatch;
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= stride) return;
    const u32* ct = consts + (int)threadIdx.x * zero;
    u32 pm[8], d2[8], acc[8], z[8];
    ld_elem(pm, ct);
    ld_elem(d2, ct + 8);
    u32 pref[kFinishBatch][8];
    fp_one<F>(acc);
#pragma unroll 1
    for (int j = 0; j < kFinishBatch; j++) {
        const long i = t + j * stride;
        if (i >= n_entries) break;
        fp_copy(pref[j], acc);
        ld_elem(z, table + i * kEntryWords + 16);
        fp_mul<F>(acc, acc, z, pm);                        // Z != 0: the addition law is complete
    }
    u32 inv[8];
    fp_inv<F>(inv, acc, pm);
#pragma unroll 1
    for (int j = kFinishBatch - 1; j >= 0; j--) {
        const long i = t + j * stride;
        if (i >= n_entries) continue;
        u32* o = table + i * kEntryWords;
        u32 zi[8], x[8], y[8], yp[8], ym[8], t2d[8];
        fp_mul<F>(zi, inv, pref[j], pm);                   // 1 / Z_i
        ld_elem(z, o + 16);
        fp_mul<F>(inv, inv, z, pm);
        ld_elem(x, o);
        ld_elem(y, o + 8);
        fp_mul<F>(x, x, zi, pm);
        fp_mul<F>(y, y, zi, pm);
        te_niels<F>(yp, ym, t2d, x, y, d2, pm);
        st_elem(o, yp);
        st_elem(o + 8, ym);
        st_elem(o + 16, t2d);
    }
}

// 16 input bytes starting at `off` of a `len`-byte message (zero beyond len), as 4 LE words.
__device__ __forceinline__ void load16(u32* w, const uint8_t* base, long off, long len) {
    const uint8_t* p = base + off;
    if (off + 16 <= len && ((reinterpret_cast<uintptr_t>(p) & 15) == 0)) {
        uint4 v = *reinterpret_cast<const uint4*>(p);
        w[0] = v.x; w[1] = v.y; w[2] = v.z; w[3] = v.w;
        return;
    }
    w[0] = w[1] = w[2] = w[3] = 0;
#pragma unroll 1
    for (int k = 0; k < 16; k++) {
        u32 b = (off + k < len) ? (u32)p[k] : 0u;
        u32 sh = b << (8 * (k & 3));
        w[0] |= (k >> 2) == 0 ? sh : 0u;
        w[1] |= (k >> 2) == 1 ? sh : 0u;
        w[2] |= (k >> 2) == 2 ? sh : 0u;
        w[3] |= (k >> 2) == 3 ? sh : 0u;
    }
}

// out = n x (X, Y, Z, -) projective, 32 words per hash (normalised by k_pedersen_normalise)
template <class F>
__global__ void __launch_bounds__(kPedBlock)
k_pedersen_hash(PedersenDev P, const u32* __restrict__ consts, const u32* __restrict__ table,
                const uint8_t* __restrict__ in, long len, long stride, const uint8_t* __restrict__ rand32,
                u32* __restrict__ out, long n) {
    extern __shared__ __align__(128) u32 sm[];          // 2 x kChunkWords
    __shared__ __align__(8) unsigned long long full[2];
    const int tid = threadIdx.x;
    const int total = P.n_in_chunks + (rand32 ? P.n_rand_chunks : 0);
    const unsigned full_s[2] = {(unsigned)__cvta_generic_to_shared(&full[0]), (unsigned)__cvta_generic_to_shared(&full[1])};
    const unsigned buf_s[2] = {(unsigned)__cvta_generic_to_shared(sm), (unsigned)__cvta_generic_to_shared(sm + kChunkWords)};
    if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(full_s[0]));
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(full_s[1]));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const u32* ct = consts + tid * P.zero;
    u32 pm[8];
    ld_elem(pm, ct);
    unsigned uses0 = 0, uses1 = 0;                      // completed phases per buffer (CTA-uniform)

    auto issue = [&](int chunk, int b) {                // thread 0 only
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(full_s[b]), "r"(kChunkBytes) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(buf_s[b]),
                     "l"(table + (long)chunk * kChunkWords), "r"(kChunkBytes), "r"(full_s[b])
                     : "memory");
    };

    const long nblocks = (n + kPedBlock - 1) / kPedBlock;
    for (long blk = blockIdx.x; blk < nblocks; blk += gridDim.x) {
        const long i = blk * kPedBlock + tid;
        const bool active = i < n;
        const uint8_t* msg = in + (active ? i : 0) * stride;
        const uint8_t* rnd = rand32 ? rand32 + (active ? i : 0) * 32 : nullptr;
        TePoint acc;
        te_identity<F>(acc);
        if (tid == 0 && total > 0) {
            issue(0, 0);
            if (total > 1) issue(1, 1);
        }
        u32 w[4] = {0, 0, 0, 0};
#pragma unroll 1
        for (int c = 0; c < total; c++) {
            const bool is_rand = c >= P.n_in_chunks;
            const int bidx = is_rand ? c - P.n_in_chunks : c;
            if ((bidx & 15) == 0) {
                if (is_rand) load16(w, rnd, bidx, 32);
                else load16(w, msg, bidx, len);
            }
            const int wi = (bidx >> 2) & 3;
            u32 word = wi == 0 ? w[0] : wi == 1 ? w[1] : wi == 2 ? w[2] : w[3];
            u32 byte = active ? (word >> (8 * (bidx & 3))) & 0xffu : 0u;
            const int b = c & 1;
            const unsigned parity = (b ? uses1 : uses0) & 1u;
            unsigned done = 0;
            while (!done) {
                asm volatile(
                    "{\n\t.reg .pred p;\n\t"
                    "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                    "selp.u32 %0, 1, 0, p;\n\t}"
                    : "=r"(done) : "r"(full_s[b]), "r"(parity) : "memory");
            }
            if (b) uses1++; else uses0++;
            const u32* e = sm + b * kChunkWords + byte * kEntryWords;
            u32 yp[8], ym[8], t2d[8];
            ld_elem(yp, e);
            ld_elem(ym, e + 8);
            ld_elem(t2d, e + 16);
            te_madd<F>(acc, yp, ym, t2d, pm);
            __syncthreads();                            // every thread is done with buffer b
            if (tid == 0 && c + 2 < total) issue(c + 2, b);
        }
        // projective result; k_pedersen_normalise turns it into the affine output (crh/pedersen/mod.rs:128 `result.into()`)
        if (active) {
            u32* o = out + 32 * i;
            st_elem(o, acc.X);
            st_elem(o + 8, acc.Y);
            st_elem(o + 16, acc.Z);
        }
    }
}


// Wide-chunk variant: `chunk_bits` (9..16) consecutive input bits select one of 2^chunk_bits subset sums per
// lookup, so a hash needs bits/chunk_bits mixed additions instead of bits/8.  The tables no longer fit shared
// memory (12 bits: 33 MB for a 1024-bit input, within the H100's 50 MB L2; 16 bits: 400 MB in HBM); each thread gathers
// its 96-byte entry with read-only 128-bit loads.  Trades L2/HBM capacity for integer-pipe work.
template <class F>
__global__ void __launch_bounds__(kPedBlock)
k_pedersen_hash_gather(PedersenDev P, const u32* __restrict__ consts, const u32* __restrict__ table,
                       const uint8_t* __restrict__ in, long len, long stride, const uint8_t* __restrict__ rand32,
                       u32* __restrict__ out, long n) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const u32* ct = consts + (int)threadIdx.x * P.zero;
    u32 pm[8];
    ld_elem(pm, ct);
    const int cb = P.chunk_bits;
    const u32 vmask = (1u << cb) - 1u;
    const uint8_t* msg = in + i * stride;
    const uint8_t* rnd = rand32 ? rand32 + i * 32 : nullptr;
    const int total = P.n_in_chunks + (rand32 ? P.n_rand_chunks : 0);
    TePoint acc;
    te_identity<F>(acc);
    // table entry of lookup c for this message (the lookup value comes from up to 3 input bytes)
    auto entry = [&](int c) -> const uint4* {
        const bool is_rand = c >= P.n_in_chunks;
        const uint8_t* src = is_rand ? rnd : msg;
        const long slen = is_rand ? 32 : len;
        const long bit = (long)(is_rand ? c - P.n_in_chunks : c) * cb;
        const long byte = bit >> 3;
        u64 v64 = 0;
#pragma unroll
        for (int k = 0; k < 4; k++)                      // chunk_bits + 7 <= 29 bits: four bytes always cover a lookup value
            if (byte + k < slen) v64 |= (u64)__ldg(src + byte + k) << (8 * k);
        const u32 v = (u32)(v64 >> (bit & 7)) & vmask;
        return reinterpret_cast<const uint4*>(table + (((long)c << cb) + v) * kEntryWords);
    };
    // Software pipeline over the gathers: the entry of lookup c+1 is loaded into registers and the entry of lookup
    // c+kPrefetchAhead is pulled into L2 while the mixed addition of lookup c (7 field products) runs, so the
    // ~1 us DRAM latency of a 96-byte random access is off the critical path (ncu round 1: long_scoreboard 0.87 / issue).
    constexpr int kPrefetchAhead = 4;
    uint4 q0, q1, q2, q3, q4, q5;
    if (total > 0) {
        const uint4* e4 = entry(0);
        q0 = __ldg(e4); q1 = __ldg(e4 + 1); q2 = __ldg(e4 + 2); q3 = __ldg(e4 + 3); q4 = __ldg(e4 + 4); q5 = __ldg(e4 + 5);
    }
#pragma unroll 1
    for (int c = 1; c < kPrefetchAhead && c < total; c++) asm volatile("prefetch.global.L2 [%0];" ::"l"(entry(c)));
#pragma unroll 1
    for (int c = 0; c < total; c++) {
        u32 yp[8], ym[8], t2d[8];
        yp[0] = q0.x; yp[1] = q0.y; yp[2] = q0.z; yp[3] = q0.w; yp[4] = q1.x; yp[5] = q1.y; yp[6] = q1.z; yp[7] = q1.w;
        ym[0] = q2.x; ym[1] = q2.y; ym[2] = q2.z; ym[3] = q2.w; ym[4] = q3.x; ym[5] = q3.y; ym[6] = q3.z; ym[7] = q3.w;
        t2d[0] = q4.x; t2d[1] = q4.y; t2d[2] = q4.z; t2d[3] = q4.w; t2d[4] = q5.x; t2d[5] = q5.y; t2d[6] = q5.z; t2d[7] = q5.w;
        if (c + kPrefetchAhead < total) asm volatile("prefetch.global.L2 [%0];" ::"l"(entry(c + kPrefetchAhead)));
        if (c + 1 < total) {
            const uint4* e4 = entry(c + 1);
            q0 = __ldg(e4); q1 = __ldg(e4 + 1); q2 = __ldg(e4 + 2); q3 = __ldg(e4 + 3); q4 = __ldg(e4 + 4); q5 = __ldg(e4 + 5);
        }
        te_madd<F>(acc, yp, ym, t2d, pm);
    }
    u32* o = out + 32 * i;
    st_elem(o, acc.X);
    st_elem(o + 8, acc.Y);
    st_elem(o + 16, acc.Z);
}

// Projective -> affine for n points with one field inversion per 32 points (Montgomery's trick along a
// thread's own sequence of points: prefix products, one Fermat inversion, back-substitution).  A warp
// pays for an inversion once whether its lanes invert the same or different values, so batching has to
// be sequential inside a thread; thread t owns points t, t + stride, t + 2*stride, ... (coalesced).
// proj: n x (X, Y, Z, scratch) of 8 words; mode 0: out = n x (x, y), mode 1: out = n x x.
template <class F>
__global__ void __launch_bounds__(128)
k_pedersen_normalise(const u32* __restrict__ consts, u32* __restrict__ proj, u32* __restrict__ out, long n, int mode, int zero) {
    constexpr int B = 32;
    const long stride = (n + B - 1) / B;
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= stride) return;
    u32 pm[8], acc[8], z[8], tmp[8];
    ld_elem(pm, consts + (int)threadIdx.x * zero);
    fp_one<F>(acc);
#pragma unroll 1
    for (int j = 0; j < B; j++) {
        const long i = t + j * stride;
        if (i >= n) break;
        st_elem(proj + 32 * i + 24, acc);              // prefix product of the Z's before this one
        ld_elem(z, proj + 32 * i + 16);
        fp_mul<F>(acc, acc, z, pm);
    }
    u32 inv[8];
    fp_inv<F>(inv, acc, pm);
#pragma unroll 1
    for (int j = B - 1; j >= 0; j--) {
        const long i = t + j * stride;
        if (i >= n) continue;
        u32 zi[8], c[8];
        ld_elem(tmp, proj + 32 * i + 24);
        fp_mul<F>(zi, inv, tmp, pm);                   // 1 / Z_i
        ld_elem(z, proj + 32 * i + 16);
        fp_mul<F>(inv, inv, z, pm);
        ld_elem(c, proj + 32 * i);
        fp_mul<F>(c, c, zi, pm);
        if (mode == 0) {
            st_elem(out + 16 * i, c);
            ld_elem(c, proj + 32 * i + 8);
            fp_mul<F>(c, c, zi, pm);
            st_elem(out + 16 * i + 8, c);
        } else {
            st_elem(out + 8 * i, c);
        }
    }
}

// n x 2 child points (Montgomery x,y each) -> n x 128 bytes: canonical LE x_l || y_l || x_r || y_r
template <class F>
__global__ void k_points_to_bytes(const u32* __restrict__ children, u32* __restrict__ bytes_out, long n_elems) {
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_elems) return;
    u32 a[8], one[8], pm[8];
    ld_elem(a, children + 8 * i);
    fp_zero(one);
    one[0] = 1;
    fp_modulus<F>(pm);
    fp_mul<F>(a, a, one, pm);
    st_elem(bytes_out + 8 * i, a);
}


// ======================================================================= Bowe-Hopwood Pedersen CRH
// bowe_hopwood::CRH::evaluate (R/crh/bowe_hopwood/mod.rs:115-185): 3-bit chunk k of the input selects
// (1 + c0 + 2*c1) * (-1)^c2 * generators[k / WS][k % WS]; only the chunks the input covers contribute
// (an all-zero chunk still adds its generator once).  Same table idea as above: m consecutive chunks
// (3m bits) select one of 2^(3m) precomputed sums; the chunks left over at the end of an input use
// per-chunk 8-entry tables.

// table3[k][v], v = c0 + 2*c1 + 4*c2: affine-Niels of the encoded multiple of generator k
template <class F>
__global__ void __launch_bounds__(128)
k_bh_table3(const u32* __restrict__ consts, const u32* __restrict__ gens_xy, int n_gens, u32* __restrict__ table3, int zero) {
    long e = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (long)n_gens * 8) return;
    const int k = (int)(e >> 3), v = (int)(e & 7);
    const u32* ct = consts + (int)threadIdx.x * zero;
    u32 pm[8], d2[8], x[8], y[8], yp[8], ym[8], t2d[8];
    ld_elem(pm, ct);
    ld_elem(d2, ct + 8);
    ld_elem(x, gens_xy + 16 * (long)k);
    ld_elem(y, gens_xy + 16 * (long)k + 8);
    te_niels<F>(yp, ym, t2d, x, y, d2, pm);
    TePoint acc;
    te_identity<F>(acc);
    const int mult = 1 + (v & 1) + 2 * ((v >> 1) & 1);
#pragma unroll 1
    for (int r = 0; r < mult; r++) te_madd<F>(acc, yp, ym, t2d, pm);
    u32 zi[8];
    fp_inv<F>(zi, acc.Z, pm);
    fp_mul<F>(x, acc.X, zi, pm);
    fp_mul<F>(y, acc.Y, zi, pm);
    if (v & 4) {                                   // -(x, y) = (-x, y)
        u32 z0[8];
        fp_zero(z0);
        fp_sub<F>(x, z0, x);
    }
    te_niels<F>(yp, ym, t2d, x, y, d2, pm);
    u32* o = table3 + e * kEntryWords;
    st_elem(o, yp);
    st_elem(o + 8, ym);
    st_elem(o + 16, t2d);
}

// table[g][value]: sum over the m chunks of group g of table3[g*m + j][(value >> 3j) & 7]
template <class F>
__global__ void __launch_bounds__(128)
k_bh_table_group(const u32* __restrict__ consts, const u32* __restrict__ table3, int n_gens, int n_groups, int m,
                 u32* __restrict__ table, int zero) {
    long e = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const int gb = 3 * m;
    if (e >= ((long)n_groups << gb)) return;
    const int g = (int)(e >> gb);
    const u32 value = (u32)(e & ((1L << gb) - 1));
    const u32* ct = consts + (int)threadIdx.x * zero;
    u32 pm[8], d2[8];
    ld_elem(pm, ct);
    ld_elem(d2, ct + 8);
    TePoint acc;
    te_identity<F>(acc);
#pragma unroll 1
    for (int j = 0; j < m; j++) {
        int k = g * m + j;
        if (k >= n_gens) break;
        const u32* t = table3 + ((long)k * 8 + ((value >> (3 * j)) & 7u)) * kEntryWords;
        u32 yp[8], ym[8], t2d[8];
        ld_elem(yp, t);
        ld_elem(ym, t + 8);
        ld_elem(t2d, t + 16);
        te_madd<F>(acc, yp, ym, t2d, pm);
    }
    u32 zi[8], x[8], y[8], yp[8], ym[8], t2d[8];
    fp_inv<F>(zi, acc.Z, pm);
    fp_mul<F>(x, acc.X, zi, pm);
    fp_mul<F>(y, acc.Y, zi, pm);
    te_niels<F>(yp, ym, t2d, x, y, d2, pm);
    u32* o = table + e * kEntryWords;
    st_elem(o, yp);
    st_elem(o + 8, ym);
    st_elem(o + 16, t2d);
}

__device__ __forceinline__ u32 bits_at(const uint8_t* src, long slen, long bit, int nbits) {
    const long byte = bit >> 3;
    u32 v = 0;
#pragma unroll
    for (int k = 0; k < 3; k++)
        if (byte + k < slen) v |= (u32)__ldg(src + byte + k) << (8 * k);
    return (v >> (bit & 7)) & ((1u << nbits) - 1u);
}

__device__ __forceinline__ void gather_entry(u32* yp, u32* ym, u32* t2d, const u32* e) {
    const uint4* e4 = reinterpret_cast<const uint4*>(e);
    uint4 q0 = __ldg(e4), q1 = __ldg(e4 + 1), q2 = __ldg(e4 + 2), q3 = __ldg(e4 + 3), q4 = __ldg(e4 + 4), q5 = __ldg(e4 + 5);
    yp[0] = q0.x; yp[1] = q0.y; yp[2] = q0.z; yp[3] = q0.w; yp[4] = q1.x; yp[5] = q1.y; yp[6] = q1.z; yp[7] = q1.w;
    ym[0] = q2.x; ym[1] = q2.y; ym[2] = q2.z; ym[3] = q2.w; ym[4] = q3.x; ym[5] = q3.y; ym[6] = q3.z; ym[7] = q3.w;
    t2d[0] = q4.x; t2d[1] = q4.y; t2d[2] = q4.z; t2d[3] = q4.w; t2d[4] = q5.x; t2d[5] = q5.y; t2d[6] = q5.z; t2d[7] = q5.w;
}

// one hash per thread; out = n x (X, Y, Z, -) projective (normalised by k_pedersen_normalise, mode 1 = x only)
template <class F>
__global__ void __launch_bounds__(kPedBlock)
k_bh_hash(const u32* __restrict__ consts, const u32* __restrict__ table, const u32* __restrict__ table3, int m, int n_full,
          int n_tail, const uint8_t* __restrict__ in, long len, long stride, u32* __restrict__ out, long n, int zero) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    u32 pm[8];
    ld_elem(pm, consts + (int)threadIdx.x * zero);
    const uint8_t* msg = in + i * stride;
    const int gb = 3 * m;
    TePoint acc;
    te_identity<F>(acc);
    u32 yp[8], ym[8], t2d[8];
#pragma unroll 1
    for (int g = 0; g < n_full; g++) {
        u32 v = bits_at(msg, len, (long)g * gb, gb);
        gather_entry(yp, ym, t2d, table + (((long)g << gb) + v) * kEntryWords);
        te_madd<F>(acc, yp, ym, t2d, pm);
    }
#pragma unroll 1
    for (int j = 0; j < n_tail; j++) {
        const long k = (long)n_full * m + j;
        u32 v = bits_at(msg, len, 3 * k, 3);
        gather_entry(yp, ym, t2d, table3 + (k * 8 + v) * kEntryWords);
        te_madd<F>(acc, yp, ym, t2d, pm);
    }
    u32* o = out + 32 * i;
    st_elem(o, acc.X);
    st_elem(o + 8, acc.Y);
    st_elem(o + 16, acc.Z);
}

// n x (left, right) base-field elements -> n x stride bytes: canonical LE left || right (64 bytes), rest untouched (zeroed by the caller)
template <class F>
__global__ void k_bh_children_to_bytes(const u32* __restrict__ children, uint8_t* __restrict__ out, long n, long stride, long keep) {
    long e = (long)blockIdx.x * blockDim.x + threadIdx.x;     // element index: 2 per node
    if (e >= 2 * n) return;
    u32 a[8], one[8], pm[8];
    ld_elem(a, children + 8 * e);
    fp_zero(one);
    one[0] = 1;
    fp_modulus<F>(pm);
    fp_mul<F>(a, a, one, pm);
    uint8_t* o = out + (e >> 1) * stride + (e & 1) * 32;
    const long base = (e & 1) * 32;
#pragma unroll 1
    for (int b = 0; b < 32; b++)
        if (base + b < keep) o[b] = (uint8_t)(a[b >> 2] >> (8 * (b & 3)));
}

}  // namespace cpb

using namespace cpb;

extern "C" cpb_status cpb_pedersen_ctx_create_ex(int, int, int, const uint64_t*, size_t, const uint64_t*, int, int, cpb_pedersen_ctx**);
extern "C" int cpb_poseidon_ctx_field(const cpb_poseidon_ctx* ctx);
extern "C" int cpb_poseidon_ctx_device(const cpb_poseidon_ctx* ctx);

namespace {


struct CurveInfo {
    int field_id;
    bool d_is_ratio;      // d = -(num/den) when true, else d = num
    uint64_t num, den;
};
bool curve_info(int curve_id, CurveInfo& ci) {
    switch (curve_id) {
        case CPB_JUBJUB: ci = {CPB_BLS12_381_FR, true, 10240, 10241}; return true;          // ark-ed-on-bls12-381: a=-1, d=-(10240/10241)
        case CPB_ED_ON_BLS12_377: ci = {CPB_BLS12_377_FR, false, 3021, 1}; return true;     // ark-ed-on-bls12-377: a=-1, d=3021
    }
    return false;
}

template <class K> cpb_status ped_grid(K kernel, size_t smem, int sms, long n, int& grid) {
    static thread_local const void* last = nullptr;
    static thread_local int occ = 0, last_dev = -1;          // the attribute and the occupancy belong to (kernel, device)
    int dev = -1;
    CPB_CUDA(cudaGetDevice(&dev));
    if (last != (const void*)kernel || last_dev != dev) {
        CPB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        CPB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, kPedBlock, smem));
        if (occ < 1) return fail(CPB_CUDA_ERROR, "pedersen kernel does not fit on an SM");
        last = (const void*)kernel; last_dev = dev;
    }
    long need = (n + kPedBlock - 1) / kPedBlock, cap = (long)sms * occ;
    grid = (int)(need < cap ? need : cap);
    if (grid < 1) grid = 1;
    return CPB_OK;
}

}  // namespace

namespace cpb {

template <class F>
cpb_status launch_hash_f(cpb_pedersen_ctx* c, const uint8_t* in, size_t len, size_t stride, const uint8_t* rand32,
                         u32* out, size_t n, int mode, cudaStream_t st) {
    size_t smem = 2 * (size_t)kChunkBytes;
    int grid = 1;
    CPB_TRY(ped_grid(k_pedersen_hash<F>, smem, c->sms, (long)n, grid));
    u32* proj = nullptr;
    CPB_CUDA(cudaMallocAsync((void**)&proj, n * 128, st));           // stream-ordered scratch: n x (X, Y, Z, prefix)
    if (c->dev.chunk_bits == 8)
        k_pedersen_hash<F><<<grid, kPedBlock, smem, st>>>(c->dev, c->d_consts, c->d_table, in, (long)len, (long)stride, rand32,
                                                          proj, (long)n);
    else
        k_pedersen_hash_gather<F><<<(int)((n + kPedBlock - 1) / kPedBlock), kPedBlock, 0, st>>>(
            c->dev, c->d_consts, c->d_table, in, (long)len, (long)stride, rand32, proj, (long)n);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) {
        long threads = ((long)n + 31) / 32;
        k_pedersen_normalise<F><<<(int)((threads + 127) / 128), 128, 0, st>>>(c->d_consts, proj, out, (long)n, mode, 0);
        e = cudaGetLastError();
    }
    cudaFreeAsync(proj, st);
    if (e != cudaSuccess) return fail(CPB_CUDA_ERROR, "pedersen launch failed: %s", cudaGetErrorString(e));
    return CPB_OK;
}

cpb_status check_len(const cpb_pedersen_ctx* c, size_t len, bool commit) {
    if (commit && len > c->nbits) return fail(CPB_BAD_LENGTH, "incorrect input length: %zu", len);
    if (len * 8 > c->nbits)
        return fail(CPB_BAD_LENGTH, "incorrect input length %zu for window params %dx%d", len, c->window_size, c->num_windows);
    return CPB_OK;
}

cpb_status launch_hash(cpb_pedersen_ctx* c, const uint8_t* in, size_t len, size_t stride, const uint8_t* rand32, u32* out,
                       size_t n, int mode, cudaStream_t st) {
    if (n == 0) return CPB_OK;
    if (rand32 && c->n_rand == 0) return fail(CPB_BAD_PARAMS, "context has no randomness generators");
    switch (c->field_id) {
        case CPB_BLS12_381_FR: return launch_hash_f<Bls12_381_Fr>(c, in, len, stride, rand32, out, n, mode, st);
        case CPB_BLS12_377_FR: return launch_hash_f<Bls12_377_Fr>(c, in, len, stride, rand32, out, n, mode, st);
    }
    return fail(CPB_UNSUPPORTED, "no kernel for base field %d", c->field_id);
}

size_t two_to_one_len(const cpb_pedersen_ctx* c) {
    size_t half = c->nbits / 2, buf = (half + half) / 8;
    return buf < 128 ? buf : 128;
}

}  // namespace cpb

namespace {

cpb_status launch_points_to_bytes(cpb_pedersen_ctx* c, const u32* children, u32* bytes, size_t n_nodes, cudaStream_t st) {
    long elems = (long)n_nodes * 4;
    int grid = (int)((elems + 255) / 256);
    switch (c->field_id) {
        case CPB_BLS12_381_FR: k_points_to_bytes<Bls12_381_Fr><<<grid, 256, 0, st>>>(children, bytes, elems); break;
        case CPB_BLS12_377_FR: k_points_to_bytes<Bls12_377_Fr><<<grid, 256, 0, st>>>(children, bytes, elems); break;
        default: return fail(CPB_UNSUPPORTED, "no kernel for base field %d", c->field_id);
    }
    CPB_CUDA(cudaGetLastError());
    return CPB_OK;
}

cpb_status two_to_one_dev(cpb_pedersen_ctx* c, const u32* children, u32* out, size_t n, u32* scratch_bytes, cudaStream_t st) {
    if (n == 0) return CPB_OK;
    CPB_TRY(check_len(c, two_to_one_len(c), false));
    CPB_TRY(launch_points_to_bytes(c, children, scratch_bytes, n, st));
    return launch_hash(c, (const uint8_t*)scratch_bytes, two_to_one_len(c), 128, nullptr, out, n, 0, st);
}

cpb_status ped_check(const cpb_pedersen_ctx* c) {
    if (!c) return fail(CPB_NULL_POINTER, "null context");
    return CPB_OK;
}
bool pow2_gt1(size_t n) { return n > 1 && (n & (n - 1)) == 0; }

// heap-ordered inner levels of a byte tree (ByteDigestConverter + pedersen::TwoToOneCRH)
cpb_status pedersen_levels(cpb_pedersen_ctx* node, const u32* leaf_xy, size_t n, u32* nodes_xy, u32* scratch_bytes,
                           cudaStream_t st) {
    size_t start = n / 2 - 1;
    CPB_TRY(two_to_one_dev(node, leaf_xy, nodes_xy + 16 * start, n / 2, scratch_bytes, st));
    while (start > 0) {
        size_t upper = start;
        start = (start - 1) / 2;
        CPB_TRY(two_to_one_dev(node, nodes_xy + 16 * upper, nodes_xy + 16 * start, upper - start, scratch_bytes, st));
    }
    return CPB_OK;
}

}  // namespace

extern "C" {

cpb_status cpb_pedersen_ctx_create(int curve_id, int window_size, int num_windows, const uint64_t* generators_xy,
                                   size_t n_rand, const uint64_t* rand_generators_xy, int device, cpb_pedersen_ctx** out) {
    return cpb::guarded([&]() -> cpb_status {
    return cpb_pedersen_ctx_create_ex(curve_id, window_size, num_windows, generators_xy, n_rand, rand_generators_xy, device, 0, out);
    });
}

cpb_status cpb_pedersen_ctx_create_ex(int curve_id, int window_size, int num_windows, const uint64_t* generators_xy,
                                      size_t n_rand, const uint64_t* rand_generators_xy, int device, int chunk_bits,
                                      cpb_pedersen_ctx** out) {
    return cpb::guarded([&]() -> cpb_status {
    if (!out) return fail(CPB_NULL_POINTER, "null out");
    if (chunk_bits == 0) {
        // default: the widest lookup whose tables stay under 2 GiB -- 18 bits for a 1024-bit input + 252 randomness
        // generators (1.8 GB; one gathered 96-byte entry and one mixed addition per 18 input bits: HBM capacity traded for
        // integer-pipe work), else 16, else 12 (L2-resident), else 8 (shared memory)
        const size_t bits_total = (size_t)window_size * num_windows + n_rand;
        chunk_bits = kDefaultChunkBits;
        for (int cand : {18, 16, 12}) {
            size_t chunks = (bits_total + cand - 1) / cand + 1;
            if (chunks * (((size_t)kEntryWords * 4) << cand) <= ((size_t)2 << 30)) { chunk_bits = cand; break; }
        }
    }
    if (chunk_bits < 8 || chunk_bits > 22) return fail(CPB_BAD_PARAMS, "chunk_bits must be 8..22 (0 = default)");
    *out = nullptr;
    CurveInfo ci;
    if (!curve_info(curve_id, ci)) return fail(CPB_BAD_PARAMS, "unknown curve id %d", curve_id);
    if (window_size < 1 || num_windows < 1 || (size_t)window_size * num_windows > (1u << 20))
        return fail(CPB_BAD_PARAMS, "bad window %dx%d", window_size, num_windows);
    if (!generators_xy || (n_rand && !rand_generators_xy)) return fail(CPB_NULL_POINTER, "null generators");
    if (n_rand > 256) return fail(CPB_BAD_PARAMS, "at most 256 randomness generators");
    host::Field F(host::field_modulus(ci.field_id));
    host::Fe d = ci.d_is_ratio ? F.neg(F.mul(F.from_u64(ci.num), F.inv(F.from_u64(ci.den)))) : F.from_u64(ci.num);
    host::Fe d2 = F.add(d, d);
    const size_t nbits = (size_t)window_size * num_windows;
    auto on_curve = [&](const uint64_t* xy) {
        host::Fe x, y;
        memcpy(x.l, xy, 32);
        memcpy(y.l, xy + 4, 32);
        if (!F.is_canonical(x) || !F.is_canonical(y)) return false;
        host::Fe xx = F.mul(x, x), yy = F.mul(y, y);
        return F.sub(yy, xx) == F.add(F.one(), F.mul(d, F.mul(xx, yy)));
    };
    for (size_t i = 0; i < nbits; i++)
        if (!on_curve(generators_xy + 8 * i)) return fail(CPB_BAD_PARAMS, "generator %zu is not a reduced point on the curve", i);
    for (size_t i = 0; i < n_rand; i++)
        if (!on_curve(rand_generators_xy + 8 * i)) return fail(CPB_BAD_PARAMS, "randomness generator %zu is not on the curve", i);

    DeviceGuard g(device);
    if (!g.ok) { cudaGetLastError(); return fail(CPB_NO_DEVICE, "cudaSetDevice(%d) failed: no usable CUDA device", device); }
    CPB_TRY(check_device_arch(device));

    keep_pool_memory(device);
    cpb_pedersen_ctx* c = new cpb_pedersen_ctx();
    c->curve_id = curve_id; c->field_id = ci.field_id; c->device = device; c->sms = sm_count(device);
    c->window_size = window_size; c->num_windows = num_windows; c->n_rand = (int)n_rand; c->nbits = nbits;
    c->dev.chunk_bits = chunk_bits;
    const size_t settable = (nbits / 8) * 8;          // input bits that can ever be set (padding rule, crh/pedersen/mod.rs:94-99)
    c->dev.n_in_chunks = (int)((settable + chunk_bits - 1) / chunk_bits);
    c->dev.n_rand_chunks = (int)((n_rand + chunk_bits - 1) / chunk_bits);
    const size_t chunk_words = ((size_t)kEntryWords) << chunk_bits;
    c->dev.zero = 0;
    const int total_chunks = c->dev.n_in_chunks + c->dev.n_rand_chunks;
    uint64_t consts[12];
    memcpy(consts, F.p, 32);
    memcpy(consts + 4, d2.l, 32);
    memcpy(consts + 8, d.l, 32);
    u32 *d_gens = nullptr, *d_rgens = nullptr;
    cudaError_t e = cudaMalloc(&c->d_consts, sizeof consts);
    if (e == cudaSuccess) e = cudaMemcpy(c->d_consts, consts, sizeof consts, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMalloc(&c->d_table, (size_t)(total_chunks > 0 ? total_chunks : 1) * chunk_words * 4);
    if (e == cudaSuccess) e = cudaMalloc(&d_gens, nbits * 64);
    if (e == cudaSuccess) e = cudaMemcpy(d_gens, generators_xy, nbits * 64, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && n_rand) e = cudaMalloc(&d_rgens, n_rand * 64);
    if (e == cudaSuccess && n_rand) e = cudaMemcpy(d_rgens, rand_generators_xy, n_rand * 64, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) {
        auto build = [&](const u32* gens, int n_gens, int n_chunks, u32* table) {
            if (n_chunks <= 0) return;
            long entries = (long)n_chunks << chunk_bits;
            int grid = (int)((entries + 255) / 256);
            long fin_threads = (entries + kFinishBatch - 1) / kFinishBatch;
            int fgrid = (int)((fin_threads + 127) / 128);
            if (c->field_id == CPB_BLS12_381_FR) {
                k_pedersen_table<Bls12_381_Fr><<<grid, 256>>>(c->d_consts, gens, n_gens, n_chunks, chunk_bits, table, 0);
                k_pedersen_table_finish<Bls12_381_Fr><<<fgrid, 128>>>(c->d_consts, table, entries, 0);
            } else {
                k_pedersen_table<Bls12_377_Fr><<<grid, 256>>>(c->d_consts, gens, n_gens, n_chunks, chunk_bits, table, 0);
                k_pedersen_table_finish<Bls12_377_Fr><<<fgrid, 128>>>(c->d_consts, table, entries, 0);
            }
        };
        build(d_gens, (int)settable, c->dev.n_in_chunks, c->d_table);
        build(d_rgens, (int)n_rand, c->dev.n_rand_chunks, c->d_table + (size_t)c->dev.n_in_chunks * chunk_words);
        e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaDeviceSynchronize();
    }
    if (d_gens) cudaFree(d_gens);
    if (d_rgens) cudaFree(d_rgens);
    if (e != cudaSuccess) {
        if (c->d_consts) cudaFree(c->d_consts);
        if (c->d_table) cudaFree(c->d_table);
        if (c->stream) cudaStreamDestroy(c->stream);
        delete c;
        return fail(CPB_CUDA_ERROR, "pedersen context build failed: %s", cudaGetErrorString(e));
    }
    *out = c;
    return CPB_OK;
    });
}

void cpb_pedersen_ctx_destroy(cpb_pedersen_ctx* c) {
    if (!c) return;
    DeviceGuard g(c->device);
    if (c->stream) { cudaStreamSynchronize(c->stream); cudaStreamDestroy(c->stream); }
    if (c->d_consts) cudaFree(c->d_consts);
    if (c->d_table) cudaFree(c->d_table);
    c->s_in.release(); c->s_out.release(); c->s_aux.release(); c->s_rand.release();
    delete c;
}

// ---- device-pointer entry points
cpb_status cpb_pedersen_crh_batch_dev(cpb_pedersen_ctx* c, const uint8_t* in, size_t len, size_t stride, uint64_t* out_xy,
                                      size_t n, void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(ped_check(c));
    CPB_TRY(check_len(c, len, false));
    DeviceGuard g(c->device);
    return launch_hash(c, in, len, stride, nullptr, (u32*)out_xy, n, 0, (cudaStream_t)stream);
    });
}
cpb_status cpb_pedersen_crh_x_batch_dev(cpb_pedersen_ctx* c, const uint8_t* in, size_t len, size_t stride, uint64_t* out_x,
                                        size_t n, void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(ped_check(c));
    CPB_TRY(check_len(c, len, false));
    DeviceGuard g(c->device);
    return launch_hash(c, in, len, stride, nullptr, (u32*)out_x, n, 1, (cudaStream_t)stream);
    });
}
cpb_status cpb_pedersen_commit_batch_dev(cpb_pedersen_ctx* c, const uint8_t* in, size_t len, size_t stride,
                                         const uint8_t* randomness_le32, uint64_t* out_xy, size_t n, void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(ped_check(c));
    if (c->n_rand == 0) return fail(CPB_BAD_PARAMS, "context has no randomness generators");
    if (!randomness_le32 && n) return fail(CPB_NULL_POINTER, "null randomness");
    CPB_TRY(check_len(c, len, true));
    DeviceGuard g(c->device);
    return launch_hash(c, in, len, stride, randomness_le32, (u32*)out_xy, n, 0, (cudaStream_t)stream);
    });
}
cpb_status cpb_pedersen_two_to_one_batch_dev(cpb_pedersen_ctx* c, const uint64_t* children_xy, uint64_t* out_xy, size_t n,
                                             void* scratch_128n, void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(ped_check(c));
    if (n && !scratch_128n) return fail(CPB_NULL_POINTER, "null scratch");
    DeviceGuard g(c->device);
    return two_to_one_dev(c, (const u32*)children_xy, (u32*)out_xy, n, (u32*)scratch_128n, (cudaStream_t)stream);
    });
}
cpb_status cpb_merkle_pedersen_build_dev(cpb_pedersen_ctx* leaf, cpb_pedersen_ctx* node, const uint8_t* leaves,
                                         size_t leaf_len, size_t leaf_stride, size_t n, uint64_t* leaf_nodes_xy,
                                         uint64_t* non_leaf_nodes_xy, void* scratch_64n, void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(ped_check(leaf));
    CPB_TRY(ped_check(node));
    if (leaf->device != node->device || leaf->field_id != node->field_id)
        return fail(CPB_BAD_PARAMS, "leaf and node contexts must share device and curve");
    if (!pow2_gt1(n)) return fail(CPB_NOT_POW2, "leaves.len() should be power of two and greater than one (got %zu)", n);
    if (!scratch_64n) return fail(CPB_NULL_POINTER, "null scratch");
    CPB_TRY(check_len(leaf, leaf_len, false));
    DeviceGuard g(leaf->device);
    cudaStream_t st = (cudaStream_t)stream;
    CPB_TRY(launch_hash(leaf, leaves, leaf_len, leaf_stride, nullptr, (u32*)leaf_nodes_xy, n, 0, st));
    return pedersen_levels(node, (const u32*)leaf_nodes_xy, n, (u32*)non_leaf_nodes_xy, (u32*)scratch_64n, st);
    });
}
cpb_status cpb_merkle_mixed_build_dev(cpb_pedersen_ctx* leaf, cpb_poseidon_ctx* node, const uint8_t* leaves, size_t leaf_len,
                                      size_t leaf_stride, size_t n, uint64_t* leaf_nodes, uint64_t* non_leaf_nodes,
                                      void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(ped_check(leaf));
    if (!node) return fail(CPB_NULL_POINTER, "null context");
    if (cpb_poseidon_ctx_field(node) != leaf->field_id || cpb_poseidon_ctx_device(node) != leaf->device)
        return fail(CPB_BAD_PARAMS, "the Poseidon field must be the curve's base field, on the same device");
    if (!pow2_gt1(n)) return fail(CPB_NOT_POW2, "leaves.len() should be power of two and greater than one (got %zu)", n);
    CPB_TRY(check_len(leaf, leaf_len, false));
    DeviceGuard g(leaf->device);
    cudaStream_t st = (cudaStream_t)stream;
    CPB_TRY(launch_hash(leaf, leaves, leaf_len, leaf_stride, nullptr, (u32*)leaf_nodes, n, 1, st));
    return cpb_merkle_poseidon_from_digests_dev(node, leaf_nodes, n, non_leaf_nodes, stream);
    });
}

// Sharded form of the mixed build (include/cpb200.h, "Merkle tree across several GPUs"): this rank's leaves, then the
// Poseidon levels with the fused root exchange.
cpb_status cpb_merkle_mixed_build_sharded_dev(cpb_pedersen_ctx* leaf, cpb_poseidon_ctx* node, cpb_exchange* ex, const uint8_t* leaves,
                                              size_t leaf_len, size_t leaf_stride, size_t n_local, uint64_t* leaf_nodes,
                                              uint64_t* non_leaf_nodes, uint64_t* top_nodes, void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(ped_check(leaf));
    if (!node) return fail(CPB_NULL_POINTER, "null context");
    if (cpb_poseidon_ctx_field(node) != leaf->field_id || cpb_poseidon_ctx_device(node) != leaf->device)
        return fail(CPB_BAD_PARAMS, "the Poseidon field must be the curve's base field, on the same device");
    if (!pow2_gt1(n_local)) return fail(CPB_NOT_POW2, "the local leaf count should be a power of two greater than one (got %zu)", n_local);
    CPB_TRY(check_len(leaf, leaf_len, false));
    {
        DeviceGuard g(leaf->device);
        CPB_TRY(launch_hash(leaf, leaves, leaf_len, leaf_stride, nullptr, (u32*)leaf_nodes, n_local, 1, (cudaStream_t)stream));
    }
    return cpb_merkle_poseidon_from_digests_sharded_dev(node, ex, leaf_nodes, n_local, non_leaf_nodes, top_nodes, stream);
    });
}

// ---- host-pointer entry points
static cpb_status ped_host_hash(cpb_pedersen_ctx* c, const uint8_t* in, size_t len, size_t stride, const uint8_t* rnd,
                                uint64_t* out, size_t n, int mode, bool commit) {
    CPB_TRY(ped_check(c));
    CPB_TRY(check_len(c, len, commit));
    if (n == 0) return CPB_OK;
    if ((!in && len) || !out) return fail(CPB_NULL_POINTER, "null buffer");
    if (stride < len) return fail(CPB_BAD_PARAMS, "stride < len");
    std::lock_guard<std::mutex> lk(c->mu);
    DeviceGuard g(c->device);
    size_t in_b = (n - 1) * stride + len, out_b = n * (mode == 0 ? 64 : 32);
    CPB_TRY(c->s_in.reserve(in_b ? in_b : 16));
    CPB_TRY(c->s_out.reserve(out_b));
    if (in_b) CPB_CUDA(cudaMemcpyAsync(c->s_in.ptr, in, in_b, cudaMemcpyHostToDevice, c->stream));
    const uint8_t* d_rnd = nullptr;
    if (rnd) {
        CPB_TRY(c->s_rand.reserve(n * 32));
        CPB_CUDA(cudaMemcpyAsync(c->s_rand.ptr, rnd, n * 32, cudaMemcpyHostToDevice, c->stream));
        d_rnd = (const uint8_t*)c->s_rand.ptr;
    }
    CPB_TRY(launch_hash(c, (const uint8_t*)c->s_in.ptr, len, stride, d_rnd, (u32*)c->s_out.ptr, n, mode, c->stream));
    CPB_CUDA(cudaMemcpyAsync(out, c->s_out.ptr, out_b, cudaMemcpyDeviceToHost, c->stream));
    CPB_CUDA(cudaStreamSynchronize(c->stream));
    return CPB_OK;
}
cpb_status cpb_pedersen_crh_batch(cpb_pedersen_ctx* c, const uint8_t* in, size_t len, size_t stride, uint64_t* out_xy, size_t n) {
    return cpb::guarded([&]() -> cpb_status {
    return ped_host_hash(c, in, len, stride, nullptr, out_xy, n, 0, false);
    });
}
cpb_status cpb_pedersen_crh_x_batch(cpb_pedersen_ctx* c, const uint8_t* in, size_t len, size_t stride, uint64_t* out_x, size_t n) {
    return cpb::guarded([&]() -> cpb_status {
    return ped_host_hash(c, in, len, stride, nullptr, out_x, n, 1, false);
    });
}
cpb_status cpb_pedersen_commit_batch(cpb_pedersen_ctx* c, const uint8_t* in, size_t len, size_t stride,
                                     const uint8_t* randomness_le32, uint64_t* out_xy, size_t n) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(ped_check(c));
    if (c->n_rand == 0) return fail(CPB_BAD_PARAMS, "context has no randomness generators");
    if (!randomness_le32 && n) return fail(CPB_NULL_POINTER, "null randomness");
    return ped_host_hash(c, in, len, stride, randomness_le32, out_xy, n, 0, true);
    });
}
cpb_status cpb_pedersen_two_to_one_batch(cpb_pedersen_ctx* c, const uint64_t* children_xy, uint64_t* out_xy, size_t n) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(ped_check(c));
    if (n == 0) return CPB_OK;
    if (!children_xy || !out_xy) return fail(CPB_NULL_POINTER, "null buffer");
    std::lock_guard<std::mutex> lk(c->mu);
    DeviceGuard g(c->device);
    CPB_TRY(c->s_in.reserve(n * 128));
    CPB_TRY(c->s_aux.reserve(n * 128));
    CPB_TRY(c->s_out.reserve(n * 64));
    CPB_CUDA(cudaMemcpyAsync(c->s_in.ptr, children_xy, n * 128, cudaMemcpyHostToDevice, c->stream));
    CPB_TRY(two_to_one_dev(c, (const u32*)c->s_in.ptr, (u32*)c->s_out.ptr, n, (u32*)c->s_aux.ptr, c->stream));
    CPB_CUDA(cudaMemcpyAsync(out_xy, c->s_out.ptr, n * 64, cudaMemcpyDeviceToHost, c->stream));
    CPB_CUDA(cudaStreamSynchronize(c->stream));
    return CPB_OK;
    });
}
cpb_status cpb_merkle_pedersen_build(cpb_pedersen_ctx* leaf, cpb_pedersen_ctx* node, const uint8_t* leaves, size_t leaf_len,
                                     size_t n, uint64_t* leaf_nodes_xy, uint64_t* non_leaf_nodes_xy) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(ped_check(leaf));
    CPB_TRY(ped_check(node));
    if (!pow2_gt1(n)) return fail(CPB_NOT_POW2, "leaves.len() should be power of two and greater than one (got %zu)", n);
    if ((!leaves && leaf_len) || !leaf_nodes_xy || !non_leaf_nodes_xy) return fail(CPB_NULL_POINTER, "null buffer");
    std::lock_guard<std::mutex> lk(leaf->mu);
    DeviceGuard g(leaf->device);
    CPB_TRY(leaf->s_in.reserve(n * leaf_len ? n * leaf_len : 16));
    CPB_TRY(leaf->s_out.reserve(n * 64 + (n - 1) * 64));
    CPB_TRY(leaf->s_aux.reserve(n * 64));
    cudaStream_t st = leaf->stream;
    u32* d_leaf = (u32*)leaf->s_out.ptr;
    u32* d_nodes = d_leaf + 16 * n;
    if (n * leaf_len) CPB_CUDA(cudaMemcpyAsync(leaf->s_in.ptr, leaves, n * leaf_len, cudaMemcpyHostToDevice, st));
    CPB_TRY(cpb_merkle_pedersen_build_dev(leaf, node, (const uint8_t*)leaf->s_in.ptr, leaf_len, leaf_len, n, (uint64_t*)d_leaf,
                                          (uint64_t*)d_nodes, leaf->s_aux.ptr, st));
    CPB_CUDA(cudaMemcpyAsync(leaf_nodes_xy, d_leaf, n * 64, cudaMemcpyDeviceToHost, st));
    CPB_CUDA(cudaMemcpyAsync(non_leaf_nodes_xy, d_nodes, (n - 1) * 64, cudaMemcpyDeviceToHost, st));
    CPB_CUDA(cudaStreamSynchronize(st));
    return CPB_OK;
    });
}
cpb_status cpb_merkle_mixed_build(cpb_pedersen_ctx* leaf, cpb_poseidon_ctx* node, const uint8_t* leaves, size_t leaf_len,
                                  size_t n, uint64_t* leaf_nodes, uint64_t* non_leaf_nodes) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(ped_check(leaf));
    if (!node) return fail(CPB_NULL_POINTER, "null context");
    if (!pow2_gt1(n)) return fail(CPB_NOT_POW2, "leaves.len() should be power of two and greater than one (got %zu)", n);
    if ((!leaves && leaf_len) || !leaf_nodes || !non_leaf_nodes) return fail(CPB_NULL_POINTER, "null buffer");
    std::lock_guard<std::mutex> lk(leaf->mu);
    DeviceGuard g(leaf->device);
    CPB_TRY(leaf->s_in.reserve(n * leaf_len ? n * leaf_len : 16));
    CPB_TRY(leaf->s_out.reserve(n * 32 + (n - 1) * 32));
    cudaStream_t st = leaf->stream;
    u32* d_leaf = (u32*)leaf->s_out.ptr;
    u32* d_nodes = d_leaf + 8 * n;
    if (n * leaf_len) CPB_CUDA(cudaMemcpyAsync(leaf->s_in.ptr, leaves, n * leaf_len, cudaMemcpyHostToDevice, st));
    CPB_TRY(cpb_merkle_mixed_build_dev(leaf, node, (const uint8_t*)leaf->s_in.ptr, leaf_len, leaf_len, n, (uint64_t*)d_leaf,
                                       (uint64_t*)d_nodes, st));
    CPB_CUDA(cudaMemcpyAsync(leaf_nodes, d_leaf, n * 32, cudaMemcpyDeviceToHost, st));
    CPB_CUDA(cudaMemcpyAsync(non_leaf_nodes, d_nodes, (n - 1) * 32, cudaMemcpyDeviceToHost, st));
    CPB_CUDA(cudaStreamSynchronize(st));
    return CPB_OK;
    });
}

}  // extern "C"

// ======================================================================= Bowe-Hopwood C ABI
struct cpb_bowe_hopwood_ctx {
    int curve_id = 0, field_id = 0, device = 0, sms = 132;
    int window_size = 0, num_windows = 0, m = 4;
    size_t n_gens = 0;
    u32* d_consts = nullptr;
    u32* d_table3 = nullptr;
    u32* d_table = nullptr;
    cudaStream_t stream = nullptr;
    std::mutex mu;
    Scratch s_in, s_out, s_aux;
};

namespace {

template <class F>
cpb_status bh_launch_f(cpb_bowe_hopwood_ctx* c, const uint8_t* in, size_t len, size_t stride, u32* out_x, size_t n, cudaStream_t st) {
    const size_t nc3 = (8 * len + 2) / 3;                         // chunks the (zero-padded) input covers, mod.rs:133-140
    const int n_full = (int)(nc3 / c->m), n_tail = (int)(nc3 % c->m);
    u32* proj = nullptr;
    CPB_CUDA(cudaMallocAsync((void**)&proj, n * 128, st));
    k_bh_hash<F><<<(int)((n + kPedBlock - 1) / kPedBlock), kPedBlock, 0, st>>>(c->d_consts, c->d_table, c->d_table3, c->m, n_full, n_tail,
                                                                               in, (long)len, (long)stride, proj, (long)n, 0);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) {
        long threads = ((long)n + 31) / 32;
        k_pedersen_normalise<F><<<(int)((threads + 127) / 128), 128, 0, st>>>(c->d_consts, proj, out_x, (long)n, 1, 0);
        e = cudaGetLastError();
    }
    cudaFreeAsync(proj, st);
    if (e != cudaSuccess) return fail(CPB_CUDA_ERROR, "bowe-hopwood launch failed: %s", cudaGetErrorString(e));
    return CPB_OK;
}
cpb_status bh_launch(cpb_bowe_hopwood_ctx* c, const uint8_t* in, size_t len, size_t stride, u32* out_x, size_t n, cudaStream_t st) {
    if (n == 0) return CPB_OK;
    if (len * 8 > c->n_gens * 3)   // R/crh/bowe_hopwood/mod.rs:121-129 (panic)
        return fail(CPB_BAD_LENGTH, "incorrect input bitlength %zu for window params %dx%dx3", len * 8, c->window_size, c->num_windows);
    switch (c->field_id) {
        case CPB_BLS12_381_FR: return bh_launch_f<Bls12_381_Fr>(c, in, len, stride, out_x, n, st);
        case CPB_BLS12_377_FR: return bh_launch_f<Bls12_377_Fr>(c, in, len, stride, out_x, n, st);
    }
    return fail(CPB_UNSUPPORTED, "no kernel for base field %d", c->field_id);
}
// TwoToOneCRH::evaluate buffer: INPUT_SIZE_BITS / 8 bytes with INPUT_SIZE_BITS = WINDOW_SIZE * NUM_WINDOWS (mod.rs:69, 218)
size_t bh_two_to_one_len(const cpb_bowe_hopwood_ctx* c) { return c->n_gens / 8; }
size_t bh_two_to_one_stride(const cpb_bowe_hopwood_ctx* c) {
    size_t l = bh_two_to_one_len(c);
    if (l < 64) l = 64;
    return (l + 15) & ~(size_t)15;
}
cpb_status bh_two_to_one_dev(cpb_bowe_hopwood_ctx* c, const u32* children, u32* out_x, size_t n, uint8_t* scratch, cudaStream_t st) {
    if (n == 0) return CPB_OK;
    const size_t len = bh_two_to_one_len(c), stride = bh_two_to_one_stride(c);
    CPB_CUDA(cudaMemsetAsync(scratch, 0, n * stride, st));
    int grid = (int)((2 * n + 255) / 256);
    if (c->field_id == CPB_BLS12_381_FR) k_bh_children_to_bytes<Bls12_381_Fr><<<grid, 256, 0, st>>>(children, scratch, (long)n, (long)stride, (long)len);
    else k_bh_children_to_bytes<Bls12_377_Fr><<<grid, 256, 0, st>>>(children, scratch, (long)n, (long)stride, (long)len);
    CPB_CUDA(cudaGetLastError());
    return bh_launch(c, scratch, len, stride, out_x, n, st);
}

}  // namespace

extern "C" {

cpb_status cpb_bowe_hopwood_ctx_create(int curve_id, int window_size, int num_windows, const uint64_t* generators_xy, int device,
                                       cpb_bowe_hopwood_ctx** out) {
    return cpb::guarded([&]() -> cpb_status {
    if (!out) return fail(CPB_NULL_POINTER, "null out");
    *out = nullptr;
    CurveInfo ci;
    if (!curve_info(curve_id, ci)) return fail(CPB_BAD_PARAMS, "unknown curve id %d", curve_id);
    if (window_size < 1 || num_windows < 1 || (size_t)window_size * num_windows > (1u << 16))
        return fail(CPB_BAD_PARAMS, "bad window %dx%d", window_size, num_windows);
    if (!generators_xy) return fail(CPB_NULL_POINTER, "null generators");
    host::Field F(host::field_modulus(ci.field_id));
    host::Fe d = ci.d_is_ratio ? F.neg(F.mul(F.from_u64(ci.num), F.inv(F.from_u64(ci.den)))) : F.from_u64(ci.num);
    host::Fe d2 = F.add(d, d);
    const size_t n_gens = (size_t)window_size * num_windows;
    for (size_t i = 0; i < n_gens; i++) {
        host::Fe x, y;
        memcpy(x.l, generators_xy + 8 * i, 32);
        memcpy(y.l, generators_xy + 8 * i + 4, 32);
        host::Fe xx = F.mul(x, x), yy = F.mul(y, y);
        if (!F.is_canonical(x) || !F.is_canonical(y) || !(F.sub(yy, xx) == F.add(F.one(), F.mul(d, F.mul(xx, yy)))))
            return fail(CPB_BAD_PARAMS, "generator %zu is not a reduced point on the curve", i);
    }
    DeviceGuard g(device);
    if (!g.ok) { cudaGetLastError(); return fail(CPB_NO_DEVICE, "cudaSetDevice(%d) failed: no usable CUDA device", device); }
    CPB_TRY(check_device_arch(device));

    keep_pool_memory(device);
    cpb_bowe_hopwood_ctx* c = new cpb_bowe_hopwood_ctx();
    c->curve_id = curve_id; c->field_id = ci.field_id; c->device = device; c->sms = sm_count(device);
    c->window_size = window_size; c->num_windows = num_windows; c->n_gens = n_gens;
    c->m = 5;                                                    // 15-bit lookups unless the tables would exceed 1 GiB
    if (((n_gens + 4) / 5) * (((size_t)kEntryWords * 4) << 15) > ((size_t)1 << 30)) c->m = 4;
    const size_t n_groups = (n_gens + c->m - 1) / c->m;
    uint64_t consts[12];
    memcpy(consts, F.p, 32);
    memcpy(consts + 4, d2.l, 32);
    memcpy(consts + 8, d.l, 32);
    u32* d_gens = nullptr;
    cudaError_t e = cudaMalloc(&c->d_consts, sizeof consts);
    if (e == cudaSuccess) e = cudaMemcpy(c->d_consts, consts, sizeof consts, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMalloc(&c->d_table3, n_gens * 8 * kEntryWords * 4);
    if (e == cudaSuccess) e = cudaMalloc(&c->d_table, (n_groups << (3 * c->m)) * kEntryWords * 4);
    if (e == cudaSuccess) e = cudaMalloc(&d_gens, n_gens * 64);
    if (e == cudaSuccess) e = cudaMemcpy(d_gens, generators_xy, n_gens * 64, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) {
        const long e3 = (long)n_gens * 8, eg = (long)n_groups << (3 * c->m);
        if (c->field_id == CPB_BLS12_381_FR) {
            k_bh_table3<Bls12_381_Fr><<<(int)((e3 + 127) / 128), 128>>>(c->d_consts, d_gens, (int)n_gens, c->d_table3, 0);
            k_bh_table_group<Bls12_381_Fr><<<(int)((eg + 127) / 128), 128>>>(c->d_consts, c->d_table3, (int)n_gens, (int)n_groups, c->m, c->d_table, 0);
        } else {
            k_bh_table3<Bls12_377_Fr><<<(int)((e3 + 127) / 128), 128>>>(c->d_consts, d_gens, (int)n_gens, c->d_table3, 0);
            k_bh_table_group<Bls12_377_Fr><<<(int)((eg + 127) / 128), 128>>>(c->d_consts, c->d_table3, (int)n_gens, (int)n_groups, c->m, c->d_table, 0);
        }
        e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaDeviceSynchronize();
    }
    if (d_gens) cudaFree(d_gens);
    if (e != cudaSuccess) {
        if (c->d_consts) cudaFree(c->d_consts);
        if (c->d_table3) cudaFree(c->d_table3);
        if (c->d_table) cudaFree(c->d_table);
        if (c->stream) cudaStreamDestroy(c->stream);
        delete c;
        return fail(CPB_CUDA_ERROR, "bowe-hopwood context build failed: %s", cudaGetErrorString(e));
    }
    *out = c;
    return CPB_OK;
    });
}

void cpb_bowe_hopwood_ctx_destroy(cpb_bowe_hopwood_ctx* c) {
    if (!c) return;
    DeviceGuard g(c->device);
    if (c->stream) { cudaStreamSynchronize(c->stream); cudaStreamDestroy(c->stream); }
    if (c->d_consts) cudaFree(c->d_consts);
    if (c->d_table3) cudaFree(c->d_table3);
    if (c->d_table) cudaFree(c->d_table);
    c->s_in.release(); c->s_out.release(); c->s_aux.release();
    delete c;
}

cpb_status cpb_bowe_hopwood_crh_batch_dev(cpb_bowe_hopwood_ctx* c, const uint8_t* in, size_t len, size_t stride, uint64_t* out_x,
                                          size_t n, void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    if (!c) return fail(CPB_NULL_POINTER, "null context");
    DeviceGuard g(c->device);
    return bh_launch(c, in, len, stride, (u32*)out_x, n, (cudaStream_t)stream);
    });
}
cpb_status cpb_bowe_hopwood_two_to_one_batch_dev(cpb_bowe_hopwood_ctx* c, const uint64_t* children_x, uint64_t* out_x, size_t n,
                                                 void* scratch, void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    if (!c) return fail(CPB_NULL_POINTER, "null context");
    if (n && !scratch) return fail(CPB_NULL_POINTER, "null scratch");
    DeviceGuard g(c->device);
    return bh_two_to_one_dev(c, (const u32*)children_x, (u32*)out_x, n, (uint8_t*)scratch, (cudaStream_t)stream);
    });
}
size_t cpb_bowe_hopwood_two_to_one_scratch_bytes(const cpb_bowe_hopwood_ctx* c, size_t n) { return c ? n * bh_two_to_one_stride(c) : 0; }

cpb_status cpb_bowe_hopwood_crh_batch(cpb_bowe_hopwood_ctx* c, const uint8_t* in, size_t len, size_t stride, uint64_t* out_x, size_t n) {
    return cpb::guarded([&]() -> cpb_status {
    if (!c) return fail(CPB_NULL_POINTER, "null context");
    if (len * 8 > c->n_gens * 3)
        return fail(CPB_BAD_LENGTH, "incorrect input bitlength %zu for window params %dx%dx3", len * 8, c->window_size, c->num_windows);
    if (n == 0) return CPB_OK;
    if ((!in && len) || !out_x) return fail(CPB_NULL_POINTER, "null buffer");
    if (stride < len) return fail(CPB_BAD_PARAMS, "stride < len");
    std::lock_guard<std::mutex> lk(c->mu);
    DeviceGuard g(c->device);
    size_t in_b = (n - 1) * stride + len;
    CPB_TRY(c->s_in.reserve(in_b ? in_b : 16));
    CPB_TRY(c->s_out.reserve(n * 32));
    if (in_b) CPB_CUDA(cudaMemcpyAsync(c->s_in.ptr, in, in_b, cudaMemcpyHostToDevice, c->stream));
    CPB_TRY(bh_launch(c, (const uint8_t*)c->s_in.ptr, len, stride, (u32*)c->s_out.ptr, n, c->stream));
    CPB_CUDA(cudaMemcpyAsync(out_x, c->s_out.ptr, n * 32, cudaMemcpyDeviceToHost, c->stream));
    CPB_CUDA(cudaStreamSynchronize(c->stream));
    return CPB_OK;
    });
}
cpb_status cpb_bowe_hopwood_two_to_one_batch(cpb_bowe_hopwood_ctx* c, const uint64_t* children_x, uint64_t* out_x, size_t n) {
    return cpb::guarded([&]() -> cpb_status {
    if (!c) return fail(CPB_NULL_POINTER, "null context");
    if (n == 0) return CPB_OK;
    if (!children_x || !out_x) return fail(CPB_NULL_POINTER, "null buffer");
    std::lock_guard<std::mutex> lk(c->mu);
    DeviceGuard g(c->device);
    CPB_TRY(c->s_in.reserve(n * 64));
    CPB_TRY(c->s_aux.reserve(n * bh_two_to_one_stride(c)));
    CPB_TRY(c->s_out.reserve(n * 32));
    CPB_CUDA(cudaMemcpyAsync(c->s_in.ptr, children_x, n * 64, cudaMemcpyHostToDevice, c->stream));
    CPB_TRY(bh_two_to_one_dev(c, (const u32*)c->s_in.ptr, (u32*)c->s_out.ptr, n, (uint8_t*)c->s_aux.ptr, c->stream));
    CPB_CUDA(cudaMemcpyAsync(out_x, c->s_out.ptr, n * 32, cudaMemcpyDeviceToHost, c->stream));
    CPB_CUDA(cudaStreamSynchronize(c->stream));
    return CPB_OK;
    });
}

}  // extern "C"
