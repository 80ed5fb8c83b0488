// blake2s.cuh -- Blake2s-256 (RFC 7693; unkeyed, 32-byte digest), one message per thread.
//
// The digest of the reference's Schnorr challenge (R/signature/schnorr/mod.rs:96-104, `D = Blake2s256`) and of the Blake2s
// commitment (R/commitment/blake2s/mod.rs:21-32).  A message is a byte source: any object with `byte(i)` for i < its
// length, so the Schnorr form hashes a per-thread 72-byte header followed by the message in global memory, at any byte
// offset, without copying the two together.
#pragma once
#include "ptx.cuh"

namespace cpb {

CPB_HD u32 b2s_rotr(u32 x, int n) {
#if defined(__CUDA_ARCH__)
    return __funnelshift_r(x, x, n);
#else
    return (x >> n) | (x << (32 - n));
#endif
}

CPB_HD constexpr u32 b2s_iv(int i) {
    constexpr u32 v[8] = {0x6A09E667u, 0xBB67AE85u, 0x3C6EF372u, 0xA54FF53Au, 0x510E527Fu, 0x9B05688Cu, 0x1F83D9ABu, 0x5BE0CD19u};
    return v[i];
}
CPB_HD constexpr int b2s_sigma(int r, int i) {
    constexpr unsigned char s[10][16] = {
        {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3},
        {11, 8, 12, 0, 5, 2, 15, 13, 10, 14, 3, 6, 7, 1, 9, 4}, {7, 9, 3, 1, 13, 12, 11, 14, 2, 6, 5, 10, 4, 0, 15, 8},
        {9, 0, 5, 7, 2, 4, 10, 15, 14, 1, 11, 12, 6, 8, 3, 13}, {2, 12, 6, 10, 0, 11, 8, 3, 4, 13, 7, 5, 15, 14, 1, 9},
        {12, 5, 1, 15, 14, 13, 4, 10, 0, 7, 6, 3, 9, 2, 8, 11}, {13, 11, 7, 14, 12, 1, 3, 9, 5, 0, 15, 4, 8, 6, 2, 10},
        {6, 15, 14, 9, 11, 3, 0, 8, 12, 2, 13, 7, 1, 4, 10, 5}, {10, 2, 8, 4, 7, 6, 1, 5, 15, 11, 9, 14, 3, 12, 13, 0}};
    return s[r][i];
}

CPB_HD void b2s_g(u32* v, int a, int b, int c, int d, u32 x, u32 y) {
    v[a] = v[a] + v[b] + x;
    v[d] = b2s_rotr(v[d] ^ v[a], 16);
    v[c] = v[c] + v[d];
    v[b] = b2s_rotr(v[b] ^ v[c], 12);
    v[a] = v[a] + v[b] + y;
    v[d] = b2s_rotr(v[d] ^ v[a], 8);
    v[c] = v[c] + v[d];
    v[b] = b2s_rotr(v[b] ^ v[c], 7);
}

// RFC 7693 F: h <- compress(h, m, t = bytes so far, last block flag)
CPB_HD void b2s_compress(u32* h, const u32* m, u64 t, bool last) {
    u32 v[16];
#pragma unroll
    for (int i = 0; i < 8; i++) {
        v[i] = h[i];
        v[i + 8] = b2s_iv(i);
    }
    v[12] ^= (u32)t;
    v[13] ^= (u32)(t >> 32);
    if (last) v[14] = ~v[14];
#pragma unroll
    for (int r = 0; r < 10; r++) {
        b2s_g(v, 0, 4, 8, 12, m[b2s_sigma(r, 0)], m[b2s_sigma(r, 1)]);
        b2s_g(v, 1, 5, 9, 13, m[b2s_sigma(r, 2)], m[b2s_sigma(r, 3)]);
        b2s_g(v, 2, 6, 10, 14, m[b2s_sigma(r, 4)], m[b2s_sigma(r, 5)]);
        b2s_g(v, 3, 7, 11, 15, m[b2s_sigma(r, 6)], m[b2s_sigma(r, 7)]);
        b2s_g(v, 0, 5, 10, 15, m[b2s_sigma(r, 8)], m[b2s_sigma(r, 9)]);
        b2s_g(v, 1, 6, 11, 12, m[b2s_sigma(r, 10)], m[b2s_sigma(r, 11)]);
        b2s_g(v, 2, 7, 8, 13, m[b2s_sigma(r, 12)], m[b2s_sigma(r, 13)]);
        b2s_g(v, 3, 4, 9, 14, m[b2s_sigma(r, 14)], m[b2s_sigma(r, 15)]);
    }
#pragma unroll
    for (int i = 0; i < 8; i++) h[i] ^= v[i] ^ v[i + 8];
}

// Blake2s-256 of the `len` bytes of `src` (src.byte(i), i < len); out = the digest as 8 little-endian words.
template <class Src> CPB_HD void blake2s_256(u32* out, const Src& src, u64 len) {
    u32 h[8];
#pragma unroll
    for (int i = 0; i < 8; i++) h[i] = b2s_iv(i);
    h[0] ^= 0x01010020u;                                 // depth 1, fanout 1, no key, 32-byte digest
    const u64 blocks = len ? (len + 63) / 64 : 1;
#pragma unroll 1
    for (u64 b = 0; b < blocks; b++) {
        u32 m[16];
#pragma unroll
        for (int w = 0; w < 16; w++) m[w] = src.word(64 * b + 4 * w, len);
        const bool last = b + 1 == blocks;
        b2s_compress(h, m, last ? len : 64 * (b + 1), last);
    }
#pragma unroll
    for (int i = 0; i < 8; i++) out[i] = h[i];
}

// Little-endian word of bytes p..p+3 of a byte source, zero at and beyond `len` (the padding of the last block).
template <class Src> CPB_HD u32 b2s_word_of_bytes(const Src& s, u64 p, u64 len) {
    u32 w = 0;
#pragma unroll
    for (int k = 0; k < 4; k++)
        if (p + k < len) w |= (u32)s.byte(p + k) << (8 * k);
    return w;
}

// A plain byte string.
struct B2sBytes {
    const uint8_t* p;
    CPB_HD uint8_t byte(u64 i) const { return p[i]; }
    CPB_HD u32 word(u64 q, u64 len) const { return b2s_word_of_bytes(*this, q, len); }
};

// a || b: the Blake2s commitment's input || randomness, and the Schnorr header || message.
struct B2sConcat {
    const uint8_t* a;
    u64 alen;
    const uint8_t* b;
    CPB_HD uint8_t byte(u64 i) const { return i < alen ? a[i] : b[i - alen]; }
    CPB_HD u32 word(u64 q, u64 len) const { return b2s_word_of_bytes(*this, q, len); }
};

// 72-byte Schnorr header as 18 words (salt || compressed point || u64 LE message length) || message bytes.  Words of the
// header are taken whole: block words start at multiples of 4 and the header ends on one.
struct B2sSchnorr {
    const u32* hdr;
    const uint8_t* msg;
    CPB_HD uint8_t byte(u64 i) const { return i < 72 ? (uint8_t)(hdr[i >> 2] >> (8 * (i & 3))) : msg[i - 72]; }
    CPB_HD u32 word(u64 q, u64 len) const { return q + 4 <= 72 ? hdr[q >> 2] : b2s_word_of_bytes(*this, q, len); }
};

}  // namespace cpb
