// poseidon_duplex.cuh -- batched duplex sponges: n PoseidonSponge<F> over one PoseidonConfig, states in device memory, one
// DuplexSpongeMode shared by the batch (R/sponge/poseidon/mod.rs:47-63).  Every call applies the same absorb or squeeze to all n
// sponges with per-sponge data, so the mode bookkeeping is uniform: the host runs duplex_plan to advance the mode and to form the
// launch arguments, and the kernel runs the same plan (carried in DuplexOp) to drive its loop.  A ragged call gives every sponge its
// own mode and its own span: duplex_step runs the same plan per item on the device, and pos_duplex_ragged runs pos_duplex on it.
//
// Everything here is CPB_HD so that tests/host can run the plan and the byte encoding on the CPU against the oracle.
#pragma once
#include "poseidon.cuh"

namespace cpb {

// DuplexSpongeMode: squeezing == 0 is Absorbing{next_absorb_index = index}, 1 is Squeezing{next_squeeze_index = index}.
struct DuplexMode {
    int squeezing;
    long index;
};

// What one absorb or squeeze of `count` elements does to a sponge in `mode` (absorb mod.rs:236-257 with absorb_internal :124-153;
// squeeze_native_field_elements :323-345 with squeeze_internal :156-186):
//   permute_first  permute before the first lane is touched (Absorbing{rate} before an absorb; Absorbing{_} or Squeezing{rate}
//                  before a squeeze);
//   start          the first rate lane read or written (always < rate);
//   boundaries     permutations between blocks: the op covers stream positions start .. start+count-1 of consecutive rate
//                  blocks and permutes only when another element follows a full block, never after the last one;
//   mode           the mode after the op.
// An absorb of nothing does nothing (noop).  A squeeze of nothing still takes the leading permutation and ends in Squeezing{start}.
struct DuplexPlan {
    bool noop;
    bool permute_first;
    long start;
    long boundaries;
    DuplexMode mode;
};

CPB_HD DuplexPlan duplex_plan(bool squeeze, DuplexMode mode, long rate, long count) {
    DuplexPlan p{false, false, 0, 0, mode};
    if (!squeeze && count == 0) {
        p.noop = true;
        return p;
    }
    if (squeeze) p.permute_first = !mode.squeezing || mode.index == rate;
    else p.permute_first = !mode.squeezing && mode.index == rate;
    p.start = p.permute_first || (!squeeze && mode.squeezing) ? 0 : mode.index;
    p.boundaries = count > 0 ? (p.start + count - 1) / rate : 0;
    p.mode = DuplexMode{squeeze ? 1 : 0, p.start + count - rate * p.boundaries};
    return p;
}

// A mode the reference can be in: Absorbing or Squeezing with an index in 0 ..= rate.
CPB_HD bool duplex_mode_valid(int squeezing, unsigned long long index, long rate) {
    return (squeezing == 0 || squeezing == 1) && index <= (unsigned long long)rate;
}

// ---- byte strings: the [u8] rule of Absorb (R/sponge/absorb.rs:137-141) -- an 8-byte little-endian length prefix, then the bytes,
// cut into chunks of (MODULUS_BIT_SIZE - 1) / 8 bytes, each one little-endian integer.
constexpr int kDuplexChunkBytes = 31;
static_assert((Bls12_381_Fr::BITS - 1) / 8 == kDuplexChunkBytes && (Bn254_Fr::BITS - 1) / 8 == kDuplexChunkBytes &&
                  (Jubjub_Fr::BITS - 1) / 8 == kDuplexChunkBytes && (Bls12_377_Fr::BITS - 1) / 8 == kDuplexChunkBytes,
              "every field packs 31 bytes per element");
CPB_HD long duplex_byte_elems(long len) { return (len + 8 + kDuplexChunkBytes - 1) / kDuplexChunkBytes; }

// Chunk j of the encoding of the `len` bytes at `str`, as a canonical integer in 8 little-endian limbs (below 2^248 < p).
CPB_HD void duplex_byte_chunk(u32* r, const unsigned char* str, long len, long j) {
    constexpr int chunk = kDuplexChunkBytes;
    const long lo = j * chunk, total = len + 8;
#pragma unroll
    for (int w = 0; w < 8; w++) {                 // constant limb indexes: r stays in registers
        u32 v = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int q = 4 * w + k;
            const long pos = lo + q;
            if (q >= chunk || pos >= total) continue;
            const u32 b = pos < 8 ? (u32)(((unsigned long long)len >> (8 * pos)) & 0xff) : (u32)str[pos - 8];
            v |= b << (8 * k);
        }
        r[w] = v;
    }
}

// The operation of one call, uniform over the batch.  Sponge i reads in + 8*count*i (kAbsorb), the byte string at
// bytes + stride*i (kAbsorbBytes; stride 0 broadcasts one string), or writes out + 8*count*i (kSqueeze*).  `count` is elements:
// for kAbsorbBytes it is duplex_byte_elems(len).  start, boundaries and first come from duplex_plan.
enum DuplexKind { kAbsorb = 0, kAbsorbBytes = 1, kSqueeze = 2, kSqueezeCanonical = 3 };
struct DuplexOp {
    int kind;
    int first;
    long start, boundaries, count;
    const u32* in;
    const unsigned char* bytes;
    long len, stride;
    u32* out;
};

// One sponge's whole call: the state (t elements at state) is loaded once, every permutation of the call runs on the registers,
// and the state is stored once.
template <class F, int T>
CPB_HD void pos_duplex(u32* state, const DuplexOp& op, long i, const PoseidonDev& P, const u32* cs, const u32* pm) {
    u32 s[T][8];
#pragma unroll
    for (int j = 0; j < T; j++) ld_elem(s[j], state + 8 * j);
    const int rate = P.rate, cap = P.cap;
    long done = 0;
#pragma unroll 1
    for (long b = 0; b <= op.boundaries; b++) {
        if (b > 0 || op.first) pos_permute<F, T>(s, P, cs, pm);
        const int lo = b == 0 ? (int)op.start : 0;
        const long left = op.count - done;
        const int hi = left < rate - lo ? lo + (int)left : rate;
        // a rolled walk over the T lanes with the state rotated under it (pos_rotl), so that each operation body is inlined
        // once; after T rotations every lane is back in place
#pragma unroll 1
        for (int q = 0; q < T; q++) {
            const int lane = q - cap;
            if (lane >= lo && lane < hi) {
                const long e = done + lane - lo;
                u32 x[8];
                if (op.kind == kAbsorb) {
                    ld_elem(x, op.in + 8 * (op.count * i + e));
                    fp_add<F>(s[0], s[0], x);
                } else if (op.kind == kAbsorbBytes) {
                    duplex_byte_chunk(x, op.bytes + op.stride * i, op.len, e);
                    u32 r2[8];
#pragma unroll
                    for (int k = 0; k < 8; k++) r2[k] = F::R2(k);
                    fp_mul<F>(x, x, r2, pm);                           // x < 2^248 < p: x * R mod p
                    fp_add<F>(s[0], s[0], x);
                } else if (op.kind == kSqueeze) {
                    st_elem(op.out + 8 * (op.count * i + e), s[0]);
                } else {
                    u32 one[8];
                    fp_zero(one);
                    one[0] = 1;
                    fp_mul<F>(x, s[0], one, pm);                       // out of Montgomery form
                    st_elem(op.out + 8 * (op.count * i + e), x);
                }
            }
            pos_rotl<T>(s);
        }
        done += hi - lo;
    }
#pragma unroll
    for (int j = 0; j < T; j++) st_elem(state + 8 * j, s[j]);
}

// ---- ragged calls: every sponge has its own mode and its own span (poseidon.cuh: ragged_span), so the mode bookkeeping is per item
// and runs where the item runs.  Modes are n cpb_sponge_mode in memory, two 64-bit words each: squeezing in the low 4 bytes of word
// 0 (the upper 4 are padding and are not read) and index in word 1.  A stored mode writes both words whole, the padding zeroed.
struct DuplexRagged {
    int kind;                    // DuplexKind
    u64* modes;                  // n x 2 words, read and updated
    const u64* offsets;          // n + 1; sponge i's span is [offsets[i], offsets[i+1]) in elements (kAbsorbBytes: bytes)
    u64 vbase;                   // the offset that the data pointers' first element stands for
    const u32* in;               // kAbsorb
    const unsigned char* bytes;  // kAbsorbBytes
    u32* out;                    // kSqueeze, kSqueezeCanonical
    long n;
};

// What one sponge's part of a ragged call does: `op` is rebased to the item (pos_duplex with i = 0 reads or writes its span), `mode`
// the mode after it, `perms` its permutations (permute_first + boundaries; 0 for a no-op).  A sponge whose stored mode is not one the
// reference can be in (duplex_mode_valid) is not valid: it is left untouched and its squeeze span is zeroed.
struct DuplexStep {
    bool valid, noop;
    DuplexOp op;
    DuplexMode mode;
    long perms;
};

CPB_HD DuplexStep duplex_step(int kind, int squeezing, unsigned long long index, RaggedSpan sp, const DuplexRagged& R, long rate) {
    DuplexStep s{false, true, DuplexOp{kind, 0, 0, 0, 0, nullptr, nullptr, 0, 0, nullptr}, DuplexMode{squeezing, 0}, 0};
    const long off = (long)(sp.lo - R.vbase);
    s.op.count = kind == kAbsorbBytes ? duplex_byte_elems(sp.len) : sp.len;
    if (kind == kAbsorb) s.op.in = R.in + 8 * off;
    else if (kind == kAbsorbBytes) {
        s.op.bytes = R.bytes + off;
        s.op.len = sp.len;
    } else s.op.out = R.out + 8 * off;
    if (!duplex_mode_valid(squeezing, index, rate)) return s;
    const DuplexPlan p = duplex_plan(kind >= kSqueeze, DuplexMode{squeezing, (long)index}, rate, s.op.count);
    s.valid = true;
    s.noop = p.noop;
    s.op.first = p.permute_first ? 1 : 0;
    s.op.start = p.start;
    s.op.boundaries = p.boundaries;
    s.mode = p.mode;
    s.perms = p.noop ? 0 : s.op.first + p.boundaries;
    return s;
}

// Sponge i's step as read from memory: its stored mode and its clamped span.
CPB_HD DuplexStep duplex_ragged_step(const DuplexRagged& R, long i, long rate) {
    return duplex_step(R.kind, (int)(u32)R.modes[2 * i], R.modes[2 * i + 1], ragged_span(R.offsets, i, R.n), R, rate);
}
// The ordering key of sponge i: its permutation count, clamped at kRaggedBuckets - 1.
CPB_HD int duplex_ragged_key(const DuplexRagged& R, long i, long rate) {
    const long p = duplex_ragged_step(R, i, rate).perms;
    return (int)(p < kRaggedBuckets - 1 ? p : kRaggedBuckets - 1);
}

// Sponge i's whole part of a ragged call (one thread of k_poseidon_duplex_ragged): the unchanged per-sponge body on the rebased op,
// then the new mode.
template <class F, int T>
CPB_HD void pos_duplex_ragged(u32* states, const DuplexRagged& R, long i, const PoseidonDev& P, const u32* cs, const u32* pm) {
    const DuplexStep s = duplex_ragged_step(R, i, P.rate);
    if (!s.valid) {
        if (R.kind >= kSqueeze) {
            u32 z[8];
            fp_zero(z);
            for (long e = 0; e < s.op.count; e++) st_elem(s.op.out + 8 * e, z);
        }
        return;
    }
    if (!s.noop) pos_duplex<F, T>(states + 8 * T * i, s.op, 0, P, cs, pm);
    R.modes[2 * i] = (u64)s.mode.squeezing;
    R.modes[2 * i + 1] = (u64)s.mode.index;
}

}  // namespace cpb
