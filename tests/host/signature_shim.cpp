// CPU build of the signature device code (crypto_primitives_b200/csrc/blake2s.cuh, te_ops.cuh) for tests/test_signature_host.py:
// Blake2s over the byte sources the kernels use, point compression, from_random_bytes, and the curve operations with the
// variable-base multiplication, over Jubjub (base field BLS12-381 Fr, scalar field Jubjub Fr).  Not part of the product.
#include "../../crypto_primitives_b200/csrc/blake2s.cuh"
#include "../../crypto_primitives_b200/csrc/hostfp.hpp"
#include "../../crypto_primitives_b200/csrc/te_ops.cuh"

#include <cstring>  // field ids: 0 = BLS12-381 Fr, 2 = Jubjub Fr (include/cpb200.h)
using namespace cpb;

typedef Bls12_381_Fr Fq;
typedef Jubjub_Fr Fr;

namespace {
struct Consts {
    u32 pm[8], d2[8], sm[8];
    Consts() {
        host::Field F(host::field_modulus(0));
        host::Fe d = F.neg(F.mul(F.from_u64(10240), F.inv(F.from_u64(10241))));
        host::Fe d2 = F.add(d, d);
        memcpy(pm, F.p, 32);
        memcpy(this->d2, d2.l, 32);
        memcpy(sm, host::field_modulus(2), 32);
    }
};
const Consts& K() {
    static Consts c;
    return c;
}
void load(TePoint& p, const uint64_t* xy) {
    u32 x[8], y[8];
    memcpy(x, xy, 32);
    memcpy(y, xy + 4, 32);
    te_from_affine<Fq>(p, x, y, K().pm);
}
void store(uint64_t* xy, const TePoint& p) {
    u32 x[8], y[8];
    te_to_affine<Fq>(x, y, p, K().pm);
    memcpy(xy, x, 32);
    memcpy(xy + 4, y, 32);
}
}  // namespace

extern "C" void host_blake2s(const uint8_t* data, uint64_t len, uint8_t* out) {
    u32 h[8];
    blake2s_256(h, B2sBytes{data}, len);
    memcpy(out, h, 32);
}

extern "C" void host_blake2s_concat(const uint8_t* a, uint64_t alen, const uint8_t* b, uint64_t blen, uint8_t* out) {
    u32 h[8];
    blake2s_256(h, B2sConcat{a, alen, b}, alen + blen);
    memcpy(out, h, 32);
}

// Blake2s(salt || compress(R) || u64_le(len) || msg) as k_schnorr_sign / k_schnorr_verify build it
extern "C" void host_schnorr_digest(const uint8_t* salt, const uint64_t* r_xy, const uint8_t* msg, uint64_t len, uint8_t* out) {
    u32 hdr[18], x[8], y[8], h[8];
    memcpy(hdr, salt, 32);
    memcpy(x, r_xy, 32);
    memcpy(y, r_xy + 4, 32);
    te_compress<Fq>(hdr + 8, x, y, K().pm);
    hdr[16] = (u32)len;
    hdr[17] = (u32)(len >> 32);
    blake2s_256(h, B2sSchnorr{hdr, msg}, 72 + len);
    memcpy(out, h, 32);
}

extern "C" void host_compress(const uint64_t* xy, uint8_t* out) {
    u32 x[8], y[8], o[8];
    memcpy(x, xy, 32);
    memcpy(y, xy + 4, 32);
    te_compress<Fq>(o, x, y, K().pm);
    memcpy(out, o, 32);
}

extern "C" int host_from_random_bytes(const uint8_t* digest, uint64_t* mont) {
    u32 d[8], m[8];
    memcpy(d, digest, 32);
    fp_zero(m);
    const bool ok = fr_from_random_bytes<Fr>(m, d, K().sm);
    memcpy(mont, m, 32);
    return ok ? 1 : 0;
}

extern "C" void host_dbl(const uint64_t* xy, uint64_t* out) {
    TePoint p;
    load(p, xy);
    te_dbl<Fq>(p, K().pm);
    store(out, p);
}

extern "C" void host_add(const uint64_t* a, const uint64_t* b, uint64_t* out) {
    TePoint p, q;
    load(p, a);
    load(q, b);
    te_add<Fq>(p, q, K().d2, K().pm);
    store(out, p);
}

extern "C" void host_neg(const uint64_t* a, uint64_t* out) {
    TePoint p;
    load(p, a);
    te_neg<Fq>(p);
    store(out, p);
}

// scalar: 8 LE words (canonical integer), `nibbles` of them used
extern "C" void host_mul_words(const uint64_t* xy, const uint64_t* scalar, int nibbles, uint64_t* out) {
    u32 x[8], y[8], w[8];
    memcpy(x, xy, 32);
    memcpy(y, xy + 4, 32);
    memcpy(w, scalar, 32);
    TePoint acc;
    te_mul_var<Fq>(acc, x, y, ScalarWords{w, nibbles}, K().d2, K().pm);
    store(out, acc);
}

extern "C" void host_mul_bitrev_bytes(const uint64_t* xy, const uint8_t* bytes, uint64_t len, uint64_t* out) {
    u32 x[8], y[8];
    memcpy(x, xy, 32);
    memcpy(y, xy + 4, 32);
    TePoint acc;
    te_mul_var<Fq>(acc, x, y, ScalarBitrevBytes{bytes, len}, K().d2, K().pm);
    store(out, acc);
}
